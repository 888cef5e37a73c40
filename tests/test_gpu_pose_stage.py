"""Pose stage on the device (lm_set_template_renders / lm_enqueue_pose / lm_complete_pose): for the NMS survivors of a
frame, R, t and residual must equal, bit for bit, lm_icp_process_batch called with each survivor's template render,
K, R and t -- NaN patterns included.  The frame is the recorded driver frame (tests/golden/driver_trace.npz) against
the allScales bank; per-template renders are the recorded render shifted by a few pixels, a handful of distinct
arrays shared by many templates."""
import importlib
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
lib = importlib.import_module("6dpose_b200._lib")
pkg = importlib.import_module("6dpose_b200")

SHIFTS = [(0, 0), (-68, -19), (-180, 57), (3, -2), (-2, 4)]  # (rows, cols): two of them put the model where survivors lie


@pytest.fixture(scope="module")
def data():
    g = np.load(os.path.join(ROOT, "tests", "golden", "driver_trace.npz"))
    b = np.load(os.path.join(ROOT, "tests", "golden", "bank_allScales_full.npz"))
    packed = dict(class_begin=b["class_begin"], tmeta=b["tmeta"].astype(np.int32), feats=b["feats"].astype(np.int32))
    G = packed["tmeta"].shape[0]
    renders = [np.ascontiguousarray(np.roll(np.roll(g["render"], dy, 0), dx, 1)) for dy, dx in SHIFTS]
    K = np.repeat(g["rf0_modelK"][None], G, 0).astype(np.float32)
    R = np.repeat(g["rf0_modelR"][None], G, 0).astype(np.float32)
    t = np.repeat(g["rf0_modelT"].reshape(1, 3), G, 0).astype(np.float32)
    t[:, 0] += (np.arange(G) % 7) - 3.0
    t[:, 2] += np.arange(G) % 11
    return dict(g=g, packed=packed, T=b["T"].tolist(), G=G, renders=renders, which=np.arange(G) % len(renders), K=K, R=R, t=t,
                sK=g["rf0_sceneK"].astype(np.float32))


def detector(data, renders=None, which=None):
    nat = lib.NativeDetector(data["T"], 0)
    nat.load_bank(data["packed"], 4)
    nat.select(None, 0, 1)
    register(nat, data, renders, which)
    return nat


def register(nat, data, renders=None, which=None, first=0, n=None):
    renders = data["renders"] if renders is None else renders
    which = data["which"] if which is None else which
    n = data["G"] - first if n is None else n
    sl = slice(first, first + n)
    nat.set_template_renders(first, [renders[k] for k in which[sl]], data["K"][sl], data["R"][sl], data["t"][sl])


def survivors(nat, data, thr, top_k, depth=None):
    g = data["g"]
    nat.upload_images(g["rgb"], g["depth"] if depth is None else depth, None)
    nat.enqueue(thr)
    nat.enqueue_post(0.5, top_k)
    return nat.complete_post()


def host_poses(data, surv, max_iterations, use_scene, renders=None, which=None, depth=None):
    renders = data["renders"] if renders is None else renders
    which = data["which"] if which is None else which
    icp = lib.NativeIcp()
    icp.set_use_scene_cloud(use_scene)
    tid = surv["template_id"].astype(np.int64)  # one class: template id == bank index
    xy = np.stack([surv["x"], surv["y"]], 1)
    scene = data["g"]["depth"] if depth is None else depth
    return icp.process_batch(scene, [renders[k] for k in which[tid]], data["sK"], data["K"][tid], data["R"][tid], data["t"][tid], xy,
                             max_iterations)


def same_poses(got, want):
    out, R, t, res, _ = got
    Rw, tw, rw = want
    assert np.array_equal(res, rw, equal_nan=True), (res, rw)
    assert np.array_equal(R, Rw, equal_nan=True)
    assert np.array_equal(t, tw, equal_nan=True)


def pose_chain(nat, data, thr, top_k, max_iterations, use_scene, depth=None):
    g = data["g"]
    return nat.match_pose(g["rgb"], g["depth"] if depth is None else depth, None, thr, data["sK"], 0.5, top_k, max_iterations, use_scene)


@pytest.mark.parametrize("max_iterations", [30, 10])
@pytest.mark.parametrize("use_scene", [False, True])
def test_real_frame_bit_identical_to_host_path(data, use_scene, max_iterations):
    nat = detector(data)
    counts = {}
    for thr, top_k in ((75.0, 1), (75.0, 3), (75.0, 0), (62.0, 0)):
        want_surv, nrec = survivors(nat, data, thr, top_k)
        got = pose_chain(nat, data, thr, top_k, max_iterations, use_scene)
        assert np.array_equal(got[0], want_surv) and got[4] == nrec
        same_poses(got, host_poses(data, want_surv, max_iterations, use_scene))
        counts[(thr, top_k)] = (len(want_surv), int(np.isfinite(got[3]).sum()), int((got[3] > 0).sum()))
    assert counts[(75.0, 1)][0] == 1 and counts[(75.0, 3)][0] == 3
    assert counts[(62.0, 0)][0] > 16, counts               # every survivor, more than one fetch window
    assert sum(c[2] for c in counts.values()) > 0, counts  # some hypotheses do find correspondences


def test_boxes_that_do_not_fit_and_no_match(data):
    g = data["g"]
    wide = np.zeros_like(g["render"])
    wide[200:260, 10:600] = 1000                               # a 598 x 68 box: fits only survivors with x < 42
    renders = data["renders"] + [wide]
    which = data["which"].copy()
    which[::2] = len(renders) - 1
    nat = detector(data, renders, which)
    got = pose_chain(nat, data, 62.0, 0, 30, False)
    tid = got[0]["template_id"]
    bw, bh = 603 - 6 + 1, 263 - 196 + 1
    early = (which[tid] == len(renders) - 1) & ((got[0]["x"] + bw >= 640) | (got[0]["y"] + bh >= 480))
    assert early.any() and (~early).any()
    assert np.all(got[3][early] == -1.0) and np.all(np.isnan(got[1][early])) and np.all(np.isnan(got[2][early]))
    same_poses(got, host_poses(data, got[0], 30, False, renders, which))
    # no match: zero survivors
    blank = pose_chain(nat, data, 100.0, 0, 30, False, depth=np.zeros_like(g["depth"]))
    assert len(blank[0]) == 0 and blank[1].shape == (0, 3, 3)


def test_anchor_zero_gives_nan_like_the_host(data):
    off = [data["renders"][2]]                                 # shifted far from the centre: render[240, 320] == 0
    assert off[0][240, 320] == 0
    which = np.zeros(data["G"], np.int64)
    nat = detector(data, off, which)
    for use_scene in (False, True):
        got = pose_chain(nat, data, 70.0, 0, 30, use_scene)
        want = host_poses(data, got[0], 30, use_scene, off, which)
        assert np.isnan(want[0]).any()
        same_poses(got, want)


def test_large_render_beyond_shared_memory(data):
    H, W = data["g"]["render"].shape
    yy, xx = np.mgrid[0:H, 0:W]
    big = np.zeros((H, W), np.uint16)
    inside = (yy >= 100) & (yy < 400) & (xx >= 150) & (xx < 450)
    big[inside] = (1050 + 25 * np.sin(xx[inside] / 11.0) * np.cos(yy[inside] / 13.0)).astype(np.uint16)
    which = np.zeros(data["G"], np.int64)
    nat = detector(data, [big], which)
    for use_scene in (False, True):
        got = pose_chain(nat, data, 75.0, 3, 10, use_scene)
        assert len(got[0]) == 3 and (got[3] != -1.0).any()     # crop 308 x 308 = 94 864 pixels
        same_poses(got, host_poses(data, got[0], 10, use_scene, [big], which))


def test_result_block_retry_reruns_the_pose_stage(data):
    probe = detector(data)
    thr = None
    for cand in (55.0, 50.0, 45.0, 40.0):
        _, nrec = survivors(probe, data, cand, 3)
        if nrec > (1 << 16):                                   # more records than the initial result block holds
            thr = cand
            break
    assert thr is not None
    nat = detector(data)                                       # fresh handle: the first frame overflows the block
    got = pose_chain(nat, data, thr, 5, 30, True)
    want_surv, nrec = survivors(probe, data, thr, 5)
    assert np.array_equal(got[0], want_surv) and got[4] == nrec
    same_poses(got, host_poses(data, want_surv, 30, True))


def test_two_ranges_equal_one(data):
    one = detector(data)
    two = lib.NativeDetector(data["T"], 0)
    two.load_bank(data["packed"], 4)
    two.select(None, 0, 1)
    half = data["G"] // 2
    register(two, data, first=half, n=data["G"] - half)
    register(two, data, first=0, n=half)
    a = pose_chain(one, data, 62.0, 0, 30, True)
    b = pose_chain(two, data, 62.0, 0, 30, True)
    assert np.array_equal(a[0], b[0]) and len(a[0]) > 16
    for x, y in zip(a[1:4], b[1:4]):
        assert np.array_equal(x, y, equal_nan=True)


def expect(rc_fn, code):
    with pytest.raises(RuntimeError) as e:
        rc_fn()
    if code == lib.LM_E_INVALID:
        assert not isinstance(e.value, lib.LinemodLibraryError), e.value
    else:
        assert ("error %d" % code) in str(e.value), e.value


def test_errors(data):
    g = data["g"]
    nat = lib.NativeDetector(data["T"], 0)
    nat.load_bank(data["packed"], 4)
    nat.select(None, 0, 1)
    K, R, t = data["K"], data["R"], data["t"]
    r0 = data["renders"][0]
    expect(lambda: nat.set_template_renders(0, [np.zeros_like(r0)], K[:1], R[:1], t[:1]), lib.LM_E_INVALID)     # empty render
    expect(lambda: nat.set_template_renders(data["G"] - 1, [r0, r0], K[:2], R[:2], t[:2]), lib.LM_E_INVALID)  # past the bank
    expect(lambda: nat.set_template_renders(-1, [r0], K[:1], R[:1], t[:1]), lib.LM_E_INVALID)
    expect(lambda: nat.set_template_renders(0, [], K[:0], R[:0], t[:0]), lib.LM_E_INVALID)                    # no render
    # no renders registered
    nat.upload_images(g["rgb"], g["depth"], None)
    nat.enqueue(75.0)
    nat.enqueue_post(0.5, 3)
    expect(lambda: nat.enqueue_pose(data["sK"]), lib.LM_E_STATE)
    nat.complete_post()
    # only part of the bank registered
    register(nat, data, first=0, n=10)
    nat.enqueue(75.0)
    nat.enqueue_post(0.5, 3)
    expect(lambda: nat.enqueue_pose(data["sK"]), lib.LM_E_STATE)
    nat.complete_post()
    register(nat, data)
    # a pose stage without enqueue_post
    nat.enqueue(75.0)
    expect(lambda: nat.enqueue_pose(data["sK"]), lib.LM_E_STATE)
    nat.complete()
    expect(lambda: nat.complete_pose(), lib.LM_E_STATE)
    # a frame without depth
    q = [[nat.quantized(l, m, (480 >> l, 640 >> l)) for m in range(2)] for l in range(2)]
    nat.upload_quantized(q)
    nat.enqueue(75.0)
    nat.enqueue_post(0.5, 3)
    expect(lambda: nat.enqueue_pose(data["sK"]), lib.LM_E_STATE)
    nat.complete_post()
    # the same handle works once the frame has depth again
    ok = pose_chain(nat, data, 75.0, 3, 30, False)
    assert len(ok[0]) == 3
    # a stale bank: loading a bank drops the renders
    nat.load_bank(data["packed"], 4)
    nat.select(None, 0, 1)
    nat.upload_images(g["rgb"], g["depth"], None)
    nat.enqueue(75.0)
    nat.enqueue_post(0.5, 3)
    expect(lambda: nat.enqueue_pose(data["sK"]), lib.LM_E_STATE)
    nat.complete_post()


def test_launches_do_not_depend_on_the_survivor_count(data):
    nat = detector(data)
    g = data["g"]
    pose_chain(nat, data, 45.0, 1, 30, True)                   # the first frame grows the result block
    deltas = {}
    for top_k in (1, 50):
        nat.upload_images(g["rgb"], g["depth"], None)
        nat.enqueue(45.0)
        nat.enqueue_post(0.5, top_k)
        before = nat.launch_count()
        nat.enqueue_pose(data["sK"], 30, True)
        out = nat.complete_pose()
        deltas[top_k] = (len(out[0]), nat.launch_count() - before)
    assert deltas[1][0] == 1 and deltas[50][0] == 50, deltas
    assert deltas[1][1] == deltas[50][1] == 5, deltas


def test_peer_exchange_gives_the_single_gpu_poses(data):
    single = detector(data)
    want = pose_chain(single, data, 62.0, 0, 30, True)
    world = 2
    dets = []
    for r in range(world):
        d = lib.NativeDetector(data["T"], 0)
        d.load_bank(data["packed"], 4)
        d.select(None, r, world)
        register(d, data)
        d.peer_export(world, 1 << 17)
        dets.append(d)
    bases = [d.peer_base() for d in dets]
    for r, d in enumerate(dets):
        d.peer_connect_local(r, world, bases)
    g = data["g"]
    for d in dets:
        d.upload_images(g["rgb"], g["depth"], None)
    for d in dets:
        d.enqueue(62.0)
    for d in dets:  # post and pose stages may synchronise (first use): every rank's match is enqueued by then
        d.enqueue_post(0.5, 0)
        d.enqueue_pose(data["sK"], 30, True)
    for d in dets:
        got = d.complete_pose()
        assert np.array_equal(got[0], want[0])
        for x, y in zip(got[1:4], want[1:4]):
            assert np.array_equal(x, y, equal_nan=True)
    for d in dets:
        d.peer_disconnect()


def test_detector_match_refine_equals_match_top_and_refine_matches(data, tmp_path):
    bk = importlib.import_module("6dpose_b200.bank")
    pr = importlib.import_module("6dpose_b200.pose_refine")
    g, packed = data["g"], data["packed"]
    bank = bk.TemplateBank()
    bank.classes["06_template"] = bk.PackedPyramids(packed["tmeta"], packed["feats"], 2)
    bank.write_packed("06_template", str(tmp_path / "06_template.lmb"), 2)
    det = pkg.Detector(int(g["num_features"]), data["T"])
    det.readClasses(["06_template"], str(tmp_path / "%s.lmb"))
    which = data["which"]
    det.setTemplateRenders({"06_template": ((data["renders"][k] for k in which), data["K"], data["R"], data["t"])})
    pairs = det.match_refine([g["rgb"], g["depth"]], 75.0, ["06_template"], data["sK"], top_k=0)
    quantized = det.quantize([g["rgb"], g["depth"]], [])
    ms, _ = det.match_top(quantized, 75.0, ["06_template"], 0.5, 0)
    assert len(pairs) == len(ms) > 0
    tid = [m.template_id for m in ms]
    want = pr.refine_matches(g["depth"], data["sK"], ms, [data["renders"][which[k]] for k in tid], data["K"][tid], data["R"][tid],
                             data["t"][tid])
    for (m, p), m2, w in zip(pairs, ms, want):
        assert (m.x, m.y, m.similarity, m.class_id, m.template_id) == (m2.x, m2.y, m2.similarity, m2.class_id, m2.template_id)
        assert p.getResidual() == w.getResidual()
        if w.getR() is None:
            assert p.getR() is None and p.getT() is None
        else:
            assert np.array_equal(p.getR(), w.getR(), equal_nan=True) and np.array_equal(p.getT(), w.getT(), equal_nan=True)
            assert p.getT().shape == (3, 1)
