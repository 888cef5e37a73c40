"""One long-lived handle against fresh ones, and frames in flight on several handles of one device.

The handle keeps state between calls (tests/handle_program.py): a call is only as right as the invalidations behind it,
and a fresh handle, or a repeat of the same call, cannot show a missing one.  test_long_lived_handle walks one handle
through the seeded call program and holds every call step

- to the oracle: the match list of the step's frame, selection and threshold (the union of every shard's records,
  through lm_finish, for a sharded selection; the device's own quantized images for the front-end), and for the box NMS
  tests/post_nms_model.py on the oracle's raw records with the step's boxes: survivors and record count.  Gated frames and the
  pose calls have no oracle list here; the existing suite pins them on fresh handles;
- bit for bit to a fresh handle given only the state the step depends on: lists, records, poses, residuals, counters(),
  plan(), pose_transforms(), the verification, track statuses and errors (a pose call on a bank without renders).

The lanes tests run 2, 3 and 6 handles on one device as bench.py does: every frame on the device first, then one frame
enqueued on every lane with no host synchronisation, then every lane completed, over a ring of 48 planted frames with one frame that outgrows the result
block; the lanes at different frame sizes and thresholds, and one lane's first front-end frames (its normal LUT upload)
while the other lanes run.  Measured on one H100 80GB HBM3 (700 W power limit): the whole file in 71 s, both seeds included."""
import importlib
import json
import os
import time

import numpy as np
import pytest
import torch

import handle_program as hp
import post_nms_model as pm

pytestmark = pytest.mark.gpu
lib = importlib.import_module("6dpose_b200._lib")

REPORT = {}
IOU = 0.5
MATCH_OPS = ("match_quantized", "bind_run", "shard_run", "match_images", "match_top", "detect", "detect_batch")


def same(a, b):
    if isinstance(a, dict):
        return a.keys() == b.keys() and all(same(a[k], b[k]) for k in a)
    if isinstance(a, (tuple, list)):
        return len(a) == len(b) and all(same(x, y) for x, y in zip(a, b))
    if isinstance(a, np.ndarray):
        return a.shape == b.shape and a.dtype == b.dtype and a.tobytes() == b.tobytes()
    return a == b


def first_difference(a, b, path="outputs"):
    """Name of the first field where a and b differ (None: equal)."""
    if isinstance(a, dict) and isinstance(b, dict):
        for k in list(a) + [k for k in b if k not in a]:
            if k not in a or k not in b:
                return "%s[%r] (only on one handle)" % (path, k)
            d = first_difference(a[k], b[k], "%s[%r]" % (path, k))
            if d:
                return d
        return None
    if isinstance(a, (tuple, list)) and isinstance(b, (tuple, list)):
        if len(a) != len(b):
            return "%s (length %d vs %d)" % (path, len(a), len(b))
        for i, (x, y) in enumerate(zip(a, b)):
            d = first_difference(x, y, "%s[%d]" % (path, i))
            if d:
                return d
        return None
    return None if same(a, b) else "%s: %r vs %r" % (path, a, b) if not isinstance(a, np.ndarray) else path


# ---- state changes and calls ----------------------------------------------------------------------------------------
def apply(nat, step, bank):
    op = step["op"]
    if op == "load_bank":
        nat.load_bank(hp.packed(step["bank"]), hp.SLOTS)
    elif op == "select":
        cls = step["classes"]
        nat.select(None if cls is None else list(cls), step["shard"], step["count"], step["layout"])
    elif op == "set_boxes":
        nat.set_boxes(None if step["seed"] is None else hp.boxes(bank, step["seed"]))
    elif op == "set_template_depths":
        nat.set_template_depths(0, hp.template_depths(bank, *step["range"]))
    elif op == "set_depth_gate":
        nat.set_depth_gate(step["tolerance"])
    elif op == "set_template_renders":
        nat.set_template_renders(0, *hp.renders(bank, step["variant"]))
    elif op == "set_pose_estimation":
        nat.set_pose_estimation(step["estimation"])
    elif op == "set_pose_search":
        nat.set_pose_search(*step["search"])
    elif op == "set_pose_verify":
        nat.set_pose_verify(step["verify"][0], step["verify"][1])
    else:
        raise AssertionError("unknown state change %r" % op)


def fresh_handle(state):
    """A new handle given only the state a call depends on."""
    nat = lib.NativeDetector(hp.T, 0)
    b = state["bank"]
    apply(nat, dict(op="load_bank", bank=b), b)
    cls, i, n, layout = state["sel"]
    if state["sel"] != hp.DEFAULT_STATE["sel"]:
        apply(nat, dict(op="select", classes=cls, shard=i, count=n, layout=layout), b)
    if state["boxes"] is not None:
        apply(nat, dict(op="set_boxes", seed=state["boxes"]), b)
    if state["depths"] is not None:
        apply(nat, dict(op="set_template_depths", range=state["depths"]), b)
    if state["gate"] is not None:
        apply(nat, dict(op="set_depth_gate", tolerance=state["gate"]), b)
    if state["renders"] is not None:
        apply(nat, dict(op="set_template_renders", variant=state["renders"]), b)
    for key, op, arg in (("est", "set_pose_estimation", "estimation"), ("search", "set_pose_search", "search"),
                         ("verify", "set_pose_verify", "verify")):
        if state[key] != hp.DEFAULT_STATE[key]:
            apply(nat, {"op": op, arg: state[key]}, b)
    return nat


def device_frame(q):
    ts = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for lvl in q for a in lvl]
    torch.cuda.synchronize()
    return ts, lib.NativeDetector.bind_args([t.data_ptr() for t in ts], [lvl[0].shape[0] for lvl in q], [lvl[0].shape[1] for lvl in q])


def run_call(nat, s):
    """The outputs of one call step on a handle: a dict of every field the step is compared on."""
    st, op, (W, H) = s["state"], s["op"], s["size"]
    thr = s.get("thr")
    out = {}
    sK = hp.scene_k(W, H)
    try:
        if op in ("match_quantized", "bind_run", "shard_run", "match_top"):
            q = hp.quantized(W, H, s["fseed"], st["bank"])
        if op == "match_quantized":
            out["list"] = nat.match_quantized(q, thr)
        elif op in ("bind_run", "shard_run"):
            ts, args = device_frame(q)
            nat.bind_quantized_device_args(args)
            nat.run(thr)
            recs = nat.fetch_records()
            if op == "shard_run":
                out["records"] = recs
            else:
                out["list"] = nat.finish(recs)
            del ts
        elif op == "match_top":
            out["top"] = nat.match_top(q, thr, IOU, s.get("top_k", 3))
        elif op == "match_images":
            rgb, depth = hp.rgbd(W, H, s["fseed"])
            out["list"] = nat.match_images(rgb, depth, None, thr)
            out["quantized"] = [[nat.quantized(l, m, (H >> l, W >> l)) for m in range(2)] for l in range(len(hp.T))]
            if st["gate"] is not None:
                out["gate"] = nat.depth_gate_stats()
        elif op == "detect":
            rgb, depth = hp.rgbd(W, H, s["fseed"])
            out["detect"] = nat.detect(rgb, depth, None, thr, sK, 0.5, 0, 30, False, 40.0, st["est"])
        elif op == "detect_batch":
            fr = [hp.rgbd(W, H, s["fseed"] + k) for k in range(s["frames"])]
            out["batch"] = nat.detect_batch(np.stack([f[0] for f in fr]), np.stack([f[1] for f in fr]), None, thr,
                                            np.stack([sK] * len(fr)), 0.5, 0, 30, False, True, 40.0, estimation=st["est"])
            out["batch_counts"] = nat.batch_counts
        elif op == "track":
            out["track"] = nat.track(hp.rgbd(W, H, s["fseed"])[1], sK, s["objects"], 30, 4, st["est"])
        elif op == "track_batch":
            n = len(s["objects"])
            depths = np.stack([hp.rgbd(W, H, s["fseed"] + k)[1] for k in range(n)])
            out["track"] = nat.track_batch(depths, np.stack([sK] * n), s["objects"], 30, 4, st["est"])
        else:
            raise AssertionError("unknown call %r" % op)
    except lib.LinemodLibraryError as e:
        out["error"] = str(e)
        return out
    if op in ("detect", "detect_batch", "track", "track_batch"):
        out["T"] = nat.pose_transforms()
        if st["verify"][0]:
            out["verify"] = nat.pose_verify()
    if op in MATCH_OPS:
        # a batch call leaves no completed single frame: both handles then refuse alike
        out["counters"] = or_error(nat.counters)
        out["plan"] = or_error(nat.plan)
    return out


def or_error(fn):
    try:
        return fn()
    except lib.LinemodLibraryError as e:
        return "error: %s" % e


# ---- the oracle -----------------------------------------------------------------------------------------------------
_ORACLE = {}


def oracle_list(oracle, bank, classes, q, thr, key):
    """oracle.match of the selected classes, as a MATCH_DTYPE array (class_index of the whole bank)."""
    k = (bank, classes, thr) + key
    if k not in _ORACLE:
        b = hp.bank(bank)
        ids = b.class_ids()
        order = list(range(len(ids))) if classes is None else list(classes)
        w = oracle.match(q, hp.T, b.pack([ids[c] for c in order], hp.SLOTS), thr, n_threads=os.cpu_count() or 1)
        out = np.zeros(len(w), lib.MATCH_DTYPE)
        out["x"], out["y"], out["similarity"], out["template_id"] = w["x"], w["y"], w["similarity"], w["template_id"]
        out["class_index"] = np.asarray(order, np.int32)[w["class_idx"]] if len(w) else []
        _ORACLE[k] = out
    return _ORACLE[k]


def oracle_top(oracle, st, q, thr, top_k):
    """post_nms_model on the oracle's raw kept records of the selected classes (class_index of the whole bank), with the
    state's boxes or the templates' own sizes: (survivors in pick order, counts)."""
    b = hp.bank(st["bank"])
    ids = b.class_ids()
    cls = st["sel"][0]
    order = list(range(len(ids))) if cls is None else list(cls)
    pre = oracle.match(q, hp.T, b.pack([ids[c] for c in order], hp.SLOTS), thr, n_threads=os.cpu_count() or 1, presort=True)
    recs = np.zeros(len(pre), lib.MATCH_DTYPE)
    for f in ("x", "y", "similarity", "template_id"):
        recs[f] = pre[f]
    recs["class_index"] = np.asarray(order, np.int32)[pre["class_idx"]] if len(pre) else []
    packed = hp.packed(st["bank"])
    wh = packed["tmeta"].reshape(-1, hp.SLOTS, 4)[:, 0, :2] if st["boxes"] is None else hp.boxes(st["bank"], st["boxes"])
    return pm.post_nms(recs, wh, packed["class_begin"], IOU, top_k)


def describe(i, steps, s):
    prev = steps[s["last_change"]] if s["last_change"] is not None else None
    brief = {k: v for k, v in s.items() if k not in ("state", "objects")}
    return "step %d %r state %r; previous state change: %r" % (i, brief, s["state"], prev)


@pytest.mark.parametrize("seed", hp.SEEDS)
def test_long_lived_handle(seed, oracle):
    steps = hp.program(seed)
    t0 = time.time()
    nat = lib.NativeDetector(hp.T, 0)
    bank = None
    shard_records = []
    for i, s in enumerate(steps):
        if not hp.is_call(s):
            if s["op"] == "load_bank":
                bank = s["bank"]
            apply(nat, s, bank)
            continue
        st = s["state"]
        got = run_call(nat, s)
        ref = fresh_handle(st)
        want = run_call(ref, s)
        ref.close()
        diff = first_difference(got, want)
        assert diff is None, "%s: long-lived and fresh handle differ at %s" % (describe(i, steps, s), diff)
        cls, shard, count, _ = st["sel"]
        W, H = s["size"]
        if s["op"] == "shard_run":
            shard_records = (shard_records if shard else []) + [got["records"]]
            if shard == count - 1:
                full = oracle_list(oracle, st["bank"], cls, hp.quantized(W, H, s["fseed"], st["bank"]), s["thr"], (W, H, s["fseed"]))
                union = nat.finish(np.concatenate(shard_records))
                assert same(union, full), "%s: the shards' union differs from the oracle (%d vs %d)" % (
                    describe(i, steps, s), len(union), len(full))
            continue
        if s["op"] in ("match_quantized", "bind_run", "match_top"):
            full = oracle_list(oracle, st["bank"], cls, hp.quantized(W, H, s["fseed"], st["bank"]), s["thr"], (W, H, s["fseed"]))
            lst = got["top"][0] if s["op"] == "match_top" else got["list"]
            if s["op"] == "match_top":
                top, counts = oracle_top(oracle, st, hp.quantized(W, H, s["fseed"], st["bank"]), s["thr"], s.get("top_k", 3))
                assert pm.same(lst, top) and got["top"][1] == counts[1], "%s: box NMS differs from post_nms_model (%d vs %d)" % (
                    describe(i, steps, s), len(lst), len(top))
            else:
                assert same(lst, full), "%s: list differs from the oracle (%d vs %d)" % (describe(i, steps, s), len(lst), len(full))
            if s.get("grows") == "candidates":
                assert got["counters"]["coarse_candidates"] > hp.CAND_LIST, describe(i, steps, s)
            if s.get("grows") == "result":
                assert got["counters"]["kept"] > hp.RESULT_BLOCK, describe(i, steps, s)
        if s["op"] == "match_images" and st["gate"] is None:
            full = oracle_list(oracle, st["bank"], cls, got["quantized"], s["thr"], ("images", W, H, s["fseed"]))
            assert same(got["list"], full), "%s: list differs from the oracle" % describe(i, steps, s)
        if s["op"] == "detect" and st["renders"] is None:
            assert "error" in got and "no template renders" in got["error"], describe(i, steps, s)
    nat.close()
    REPORT.setdefault("program", {})[seed] = dict(steps=len(steps), calls=sum(hp.is_call(s) for s in steps),
                                                 transitions=hp.transitions(steps), seconds=round(time.time() - t0, 1))


# ---- lanes in flight ------------------------------------------------------------------------------------------------
RING = 48


def lane_handles(n):
    nats = []
    for _ in range(n):
        nat = lib.NativeDetector(hp.T, 0)
        nat.load_bank(hp.packed("A"), hp.SLOTS)
        nats.append(nat)
    return nats


LANE_SIZES = [(640, 480), (320, 240), (512, 512)]
LANE_THRS = [75.0, 82.0, 68.0]


SPIN_CYCLES = 40_000_000   # about 20 ms at 1980 MHz
OVERFLOW = 1   # ring entry taken at a negative threshold: its records outgrow the result block


def ring_frame(variant, lanes, k):
    """(lane, quantized frame or None for an RGB-D frame, threshold, (W, H)) of ring entry k."""
    l = k % lanes
    (W, H), thr = (LANE_SIZES[l % 3], LANE_THRS[l % 3]) if variant == "sizes" else ((640, 480), 75.0)
    thr = hp.NEG if k == OVERFLOW else thr
    if variant == "frontend" and l == 0:
        return l, None, thr, (W, H)
    return l, hp.quantized(W, H, 1000 + k, "A"), thr, (W, H)


def busy(stream):
    """The handle's stream still has work queued or running (cudaStreamQuery; no synchronisation)."""
    return not torch.cuda.ExternalStream(stream).query()


@pytest.mark.parametrize("variant", ["sizes", "frontend"])
@pytest.mark.parametrize("lanes", [2, 3, 6])
def test_lanes_in_flight(lanes, variant, oracle):
    """Every round enqueues one frame on every lane with no host synchronisation in between, as bench.py's step() does
    (every ring frame is on the device before the first enqueue), then completes, fetches and finishes every lane.  Lane l
    runs at LANE_SIZES / LANE_THRS[l % 3] ("sizes"), or every lane at 640 x 480 and 75 ("frontend") except lane 0.  That
    lane's handle has not used the front-end before; it is enqueued last in every round, with lm_upload_images +
    lm_enqueue of an RGB-D frame, so that its first call uploads the normal LUT while the other lanes' frames are on the
    device: round 0's frames wait behind a bounded spin kernel, and the test checks that every other lane still has work
    queued when lane 0's first upload is issued.  Ring entry 1 (lane 1's first frame) outgrows the result block.  The
    report records how many other lanes had work queued at each of lane 0's uploads."""
    t0 = time.time()
    nats = lane_handles(lanes)
    rounds = RING // lanes
    ring = [ring_frame(variant, lanes, k) for k in range(rounds * lanes)]
    dev = [device_frame(q) if q is not None else (None, None) for _, q, _, _ in ring]   # one synchronisation, here
    order = list(range(1, lanes)) + [0] if variant == "frontend" else list(range(lanes))
    in_flight = []
    if variant == "frontend":
        # the quantized lanes have matched at their size before (so that their enqueues do no first-use work, which waits
        # for the lane's stream), and round 0's frames queue behind a bounded spin on another stream: lane 0's first
        # lm_upload_images, which uploads the normal LUT, is then issued while every other lane's frame is on the device
        for l in range(1, lanes):
            _, q, thr, _ = ring[l]
            nats[l].bind_quantized_device_args(dev[l][1])
            nats[l].run(75.0)
        side = torch.cuda.Stream()
        with torch.cuda.stream(side):
            torch.cuda._sleep(SPIN_CYCLES)
        spun = torch.cuda.Event()
        spun.record(side)
        for l in range(1, lanes):
            torch.cuda.ExternalStream(nats[l].stream()).wait_event(spun)
    for r in range(rounds):
        for l in order:
            k = r * lanes + l
            _, q, thr, (W, H) = ring[k]
            if q is None:
                in_flight.append(sum(busy(nats[j].stream()) for j in range(1, lanes)))
                rgb, depth = hp.rgbd(W, H, 500 + k)
                nats[l].upload_images(rgb, depth, None)
            else:
                nats[l].bind_quantized_device_args(dev[k][1])
            nats[l].enqueue(thr)
        got, kept = [], []
        for l in range(lanes):
            nats[l].complete()
            got.append(nats[l].finish(nats[l].fetch_records()))
            kept.append(nats[l].counters()["kept"])
        for l in range(lanes):
            k = r * lanes + l
            _, q, thr, (W, H) = ring[k]
            if q is None:
                # the same frame on a handle alone on the device: its quantized images are the oracle's input
                ref = lib.NativeDetector(hp.T, 0)
                ref.load_bank(hp.packed("A"), hp.SLOTS)
                rgb, depth = hp.rgbd(W, H, 500 + k)
                alone = ref.match_images(rgb, depth, None, thr)
                q = [[ref.quantized(lv, m, (H >> lv, W >> lv)) for m in range(2)] for lv in range(len(hp.T))]
                ref.close()
                assert same(got[l], alone), (lanes, variant, r, l)
                want = oracle_list(oracle, "A", None, q, thr, ("images", W, H, 500 + k))
            else:
                want = oracle_list(oracle, "A", None, q, thr, (W, H, 1000 + k))
            assert same(got[l], want), "lanes %d %s: round %d lane %d (ring entry %d, %dx%d, threshold %g): %d vs %d matches" % (
                lanes, variant, r, l, k, W, H, thr, len(got[l]), len(want))
            if k == OVERFLOW:
                assert kept[l] > hp.RESULT_BLOCK
    if variant == "frontend":
        assert in_flight[0] == lanes - 1, in_flight
    for nat in nats:
        nat.close()
    del dev
    REPORT.setdefault("lanes", {})["%d_%s" % (lanes, variant)] = dict(
        frames=rounds * lanes, seconds=round(time.time() - t0, 1),
        **({"lanes_busy_at_frontend_uploads": in_flight} if in_flight else {}))


def test_enqueues_without_completion(oracle):
    """Several frames enqueued on one handle with no completion in between, then one lm_complete: the last frame's list
    is the oracle's (bench.py's timed loop completes a lane only at the end).  Every frame is on the device before the
    first enqueue."""
    nat = lane_handles(1)[0]
    qs = [hp.quantized(640, 480, 2000 + k, "A") for k in range(6)]
    dev = [device_frame(q) for q in qs]
    for k, (_, args) in enumerate(dev):
        nat.bind_quantized_device_args(args)
        nat.enqueue(70.0 + k)
    nat.complete()
    got = nat.finish(nat.fetch_records())
    want = oracle_list(oracle, "A", None, qs[-1], 75.0, (640, 480, 2005))
    assert len(want) > 0 and same(got, want)
    nat.close()


def test_report():
    """Writes the program's size, transitions covered and wall times to $HANDLE_SEQUENCES_REPORT (JSON) when set."""
    path = os.environ.get("HANDLE_SEQUENCES_REPORT")
    if path:
        with open(path, "w") as f:
            json.dump(REPORT, f, indent=1, default=str)
