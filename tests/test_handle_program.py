"""The seeded call program of tests/handle_program.py: every committed seed covers every transition the long-lived handle
test relies on, and where it matters the transition changes the expected answer (a transition that changes nothing would
let a missing invalidation pass)."""
import importlib

import numpy as np
import pytest

import depth_gate_model as dgm
import handle_program as hp
import match_shapes as ms
import post_nms_model as pm
import tight_frames as tf

fe = importlib.import_module("6dpose_b200.frontend")


@pytest.fixture(scope="module", params=hp.SEEDS)
def steps(request):
    return hp.program(request.param)


def calls(steps):
    return [s for s in steps if hp.is_call(s)]


def test_every_transition_is_covered(steps):
    got = hp.transitions(steps)
    missing = [k for k, v in got.items() if v == 0]
    assert not missing, missing


def test_every_call_and_state_change_occurs(steps):
    ops = {s["op"] for s in steps}
    assert ops >= {"load_bank", "select", "set_boxes", "set_template_depths", "set_depth_gate", "set_template_renders",
                   "set_pose_estimation", "set_pose_search", "set_pose_verify", "match_quantized", "bind_run", "shard_run",
                   "match_images", "match_top", "detect", "detect_batch", "track", "track_batch"}
    assert {s["estimation"] for s in steps if s["op"] == "set_pose_estimation"} >= {"point_to_point", "pso"}
    assert {s["state"]["est"] for s in calls(steps) if s["op"] in ("detect", "detect_batch", "track", "track_batch")} == set(
        hp.ESTIMATIONS)
    assert {s["verify"][0] for s in steps if s["op"] == "set_pose_verify"} == {True, False}
    assert len({s["verify"][1] for s in steps if s["op"] == "set_pose_verify" and s["verify"][0]}) == 2
    # every shard of a sharded selection is called, and the selection goes back to one shard
    sel = [s["state"]["sel"] for s in calls(steps) if s["op"] == "shard_run"]
    for layout in (0, 1):
        n = {c for _, _, c, lay in sel if lay == layout}
        assert len(n) == 1 and sorted(i for _, i, _, lay in sel if lay == layout) == list(range(n.pop()))
    assert calls(steps)[-1]["state"]["sel"] == hp.DEFAULT_STATE["sel"]


def test_program_is_deterministic_and_seeded():
    a, b = hp.program(hp.SEEDS[0]), hp.program(hp.SEEDS[0])
    assert repr(a) == repr(b)
    assert repr(a) != repr(hp.program(hp.SEEDS[1]))


def test_frame_sizes_route_as_named(steps):
    sizes = [tuple(s["size"]) for s in calls(steps)]
    spine = [sz for k, sz in enumerate(sizes) if k == 0 or sz != sizes[k - 1]]
    it = iter(spine)
    assert all(sz in it for sz in hp.SIZES), spine          # the spine's sizes in order
    for W, H in set(sizes):
        shape = ms.frame_shape(hp.T, W, H)
        assert shape["filter_ok"] == ((W, H) != hp.FILTER_OFF), (W, H)
        assert shape["bit_planes"] == ((W, H) != hp.NO_BIT_PLANES), (W, H)
    assert ms.frame_shape(hp.T, *hp.NO_BIT_PLANES)["rounds"] > ms.MAX_ROUNDS


def test_ulp_pair_changes_need(steps):
    lo = [s["thr"] for s in calls(steps) if s.get("ulp") == "lo"]
    hi = [s["thr"] for s in calls(steps) if s.get("ulp") == "hi"]
    assert len(set(lo)) == 1 and len(set(hi)) == 1 and np.float32(hi[0]) == tf.ulp_up(lo[0])
    nf = hp.filter_features("A")
    need_lo = [tf.need_of(lo[0], int(n)) for n in nf]
    need_hi = [tf.need_of(hi[0], int(n)) for n in nf]
    assert need_lo != need_hi


def test_growth_outgrows_the_buffers(steps):
    neg = {s["grows"]: s for s in calls(steps) if s.get("grows")}
    W, H = neg["candidates"]["size"]
    plane = ms.frame_shape(hp.T, W, H)["plane"]
    assert hp.n_templates(neg["candidates"]["state"]["bank"]) * plane > hp.CAND_LIST
    W, H = neg["result"]["size"]
    n = hp.n_templates(neg["result"]["state"]["bank"]) * ms.frame_shape(hp.T, W, H)["plane"]
    assert hp.RESULT_BLOCK < n <= hp.CAND_LIST


def test_wide_bank_toggles_filter_eligibility():
    nf = hp.filter_features("W")
    cb = hp.packed("W")["class_begin"]
    assert (nf > 511).any() and (nf <= 511).any()
    assert (nf[cb[1]:cb[2]] <= 511).all()   # class 02 alone: every template eligible


def test_transitions_change_the_answer(steps, oracle):
    """The thresholds, the banks, the class subset and the tolerances of the program give different answers."""
    cs = calls(steps)
    first = cs[0]
    W, H = first["size"]
    q = hp.quantized(W, H, first["fseed"], "A")
    pa = hp.packed("A")
    lists = [oracle.match(q, hp.T, pa, t) for t in (85.0, 80.0, 70.0)]
    assert len(lists[0]) < len(lists[1]) < len(lists[2])
    # two banks on the same frame
    s = next(s for s in cs if s.get("other_bank"))
    W, H = s["size"]
    q = hp.quantized(W, H, s["fseed"], s["state"]["bank"])
    a = oracle.match(q, hp.T, hp.packed(s["other_bank"]), s["thr"])
    b = oracle.match(q, hp.T, hp.packed(s["state"]["bank"]), s["thr"])
    assert len(b) > 0 and a.tobytes() != b.tobytes()
    # a class subset
    s = next(s for s in cs if s["state"]["sel"][0] is not None and s["state"]["bank"] == "A")
    W, H = s["size"]
    q = hp.quantized(W, H, s["fseed"], "A")
    full = oracle.match(q, hp.T, pa, s["thr"])
    bk = hp.bank("A")
    sub = oracle.match(q, hp.T, bk.pack([bk.class_ids()[c] for c in s["state"]["sel"][0]], hp.SLOTS), s["thr"])
    assert 0 < len(sub) < len(full)
    # the gate's tolerances and template distances
    gated = [s for s in cs if s["state"]["gate"] is not None and s["op"] == "match_images"]
    masks = set()
    for s in gated:
        W, H = s["size"]
        depth = hp.rgbd(W, H, s["fseed"])[1]
        z = hp.template_depths("A", *s["state"]["depths"])
        masks.add(dgm.gate_mask(depth, pa["tmeta"], hp.T, z, s["state"]["gate"]).tobytes())
    assert len(masks) == len(gated) == 3


def test_gate_changes_move_the_candidates(steps):
    """Each gated front-end call's candidates after the gate (lm_depth_gate_stats "after", which the GPU test compares)
    differ from the previous gated call's: the tolerance change and the distance change each move them.  The frames are
    quantized by the host front-end, which the GPU front-end equals (tests/test_gpu_frontend.py)."""
    gated = [s for s in calls(steps) if s["state"]["gate"] is not None and s["op"] == "match_images"]
    pa = hp.packed("A")
    after = []
    for s in gated:
        W, H = s["size"]
        rgb, depth = hp.rgbd(W, H, s["fseed"])
        cp = dgm.GatedOracle(fe.quantize_pyramid([rgb, depth], len(hp.T), []), hp.T, pa).coarse_pass(s["thr"])
        z = hp.template_depths("A", *s["state"]["depths"])
        after.append(dgm.gate_stats(dgm.gate_mask(depth, pa["tmeta"], hp.T, z, s["state"]["gate"]), cp, depth, hp.T, z)["after"])
    assert len(after) == 3 and after[0] != after[1] and after[1] != after[2], after


def test_renders_differ():
    r = [hp.renders("A", v)[0][0] for v in range(3)]
    assert all(not np.array_equal(r[i], r[j]) for i in range(3) for j in range(i))


def test_boxes_change_the_survivors(steps, oracle):
    """Each pair of box-NMS calls at one frame and threshold, one with the caller's boxes and one without (set_boxes(None),
    or the same bank loaded again): post_nms_model on the oracle's raw records gives different survivors."""
    cs = calls(steps)
    pairs = [(a, b) for a, b in zip(cs, cs[1:]) if a["op"] == b["op"] == "match_top" and a["fseed"] == b["fseed"]
             and a["thr"] == b["thr"] and a["state"]["bank"] == b["state"]["bank"] and a["state"]["boxes"] != b["state"]["boxes"]]
    assert len(pairs) == 2
    for a, b in pairs:
        W, H = a["size"]
        packed = hp.packed(a["state"]["bank"])
        pre = oracle.match(hp.quantized(W, H, a["fseed"], a["state"]["bank"]), hp.T, packed, a["thr"], presort=True)
        tops = []
        for s in (a, b):
            sc = s["state"]["boxes"]
            wh = packed["tmeta"].reshape(-1, hp.SLOTS, 4)[:, 0, :2] if sc is None else hp.boxes(s["state"]["bank"], sc)
            tops.append(pm.post_nms(pre, wh, packed["class_begin"], 0.5, s["top_k"])[0])
        assert len(tops[0]) > 0 and len(tops[1]) > 0 and not pm.same(tops[0], tops[1]), (len(tops[0]), len(tops[1]))
