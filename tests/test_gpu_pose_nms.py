"""Pose NMS on the device (lm_enqueue_pose_nms / lm_complete_detect / lm_nms_translations): the kept poses must be
exactly what lm_complete_pose returns on the same frame followed by the numpy model of tests/pose_nms_model.py --
order, lm_match, R, t and residual bit for bit, counts equal.  The frame is the recorded driver frame
(tests/golden/driver_trace.npz) against the allScales bank with per-template renders: the recorded render shifted by
a few pixels, a handful of distinct arrays shared by many templates."""
import importlib
import os

import numpy as np
import pytest

import pose_nms_model as pm

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


def detector(data, renders=None, which=None, packed=None, reversed_copy=False):
    renders = data["renders"] if renders is None else renders
    which = data["which"] if which is None else which
    nat = lib.NativeDetector(data["T"], 0)
    nat.load_bank(data["packed"] if packed is None else packed, 4)
    nat.select(None, 0, 1)
    nat.set_template_renders(0, [renders[k] for k in which], data["K"], data["R"], data["t"])
    if reversed_copy:  # class 1: the same templates in reverse order
        r = slice(None, None, -1)
        nat.set_template_renders(data["G"], [renders[k] for k in which[r]], data["K"][r], data["R"][r], data["t"][r])
    return nat


def pose_chain(nat, data, thr, top_k, use_scene, depth=None):
    g = data["g"]
    return nat.match_pose(g["rgb"], g["depth"] if depth is None else depth, None, thr, data["sK"], 0.5, top_k, 30, use_scene)


def detect_chain(nat, data, thr, top_k, use_scene, tthr, depth=None):
    g = data["g"]
    return nat.detect(g["rgb"], g["depth"] if depth is None else depth, None, thr, data["sK"], 0.5, top_k, 30, use_scene, tthr)


def expected(pose, tthr):
    surv, R, t, res, nrec = pose
    s, R2, t2, r2 = pm.detect(surv, R, t, res, tthr)
    counts = dict(survivors=len(surv), posed=int((res != np.float32(-1.0)).sum()), records=nrec)
    return (s, R2, t2, r2), counts


def same(got, want):
    (s, R, t, r, counts), (w, wc) = got, want
    assert counts == wc, (counts, wc)
    assert np.array_equal(s, w[0]), (s, w[0])
    for a, b in zip((R, t, r), w[1:]):
        assert a.dtype == b.dtype and a.shape == b.shape
        assert np.array_equal(a.view(np.uint8), b.view(np.uint8))  # bit for bit, NaN payloads included


def boundary_threshold(pose):
    """A distance between two posed survivors, computed as the model does: with it as the threshold, a real pair sits
    exactly on the boundary."""
    surv, R, t, res, _ = pose
    posed = np.flatnonzero((res != np.float32(-1.0)) & np.isfinite(t).all(1))
    if len(posed) < 2:
        return None
    first = posed[pm.order(-res[posed].astype(np.float64))[0]]
    d = pm.distances(t, first, posed[posed != first])
    d = d[d > 0]
    return float(d.min()) if d.size else None


def test_nms_translations_equals_the_model_on_every_adversarial_set():
    for name, (ts, scores, thr) in sorted(pm.adversarial_sets().items()):
        got = lib.nms_translations(ts, scores, thr)
        assert got.tolist() == pm.nms(ts, scores, thr), name


@pytest.mark.parametrize("use_scene", [False, True])
def test_real_frame_equals_complete_pose_then_the_model(data, use_scene):
    nat = detector(data)
    boundary = 0
    for thr in (62.0, 65.0, 75.0):
        for top_k in (0, 3):
            pose = pose_chain(nat, data, thr, top_k, use_scene)
            tthrs = [40.0, 0.0, np.inf]
            b = boundary_threshold(pose)
            if b is not None:
                tthrs.append(b)
            for tthr in tthrs:
                want = expected(pose, tthr)
                same(detect_chain(nat, data, thr, top_k, use_scene, tthr), want)
            if b is not None:
                with_b, without_b = pm.detect(*pose[:4], b), pm.detect(*pose[:4], np.nextafter(b, 0.0))
                boundary += len(with_b[0]) < len(without_b[0])  # the pair on the boundary is suppressed at b only
    assert boundary > 0


def test_early_returns_and_nan_translations_in_one_frame(data):
    g = data["g"]
    wide = np.zeros_like(g["render"])
    wide[200:260, 10:600] = 1000                                      # a 598 x 68 box: fits only survivors with x < 42
    off = data["renders"][2]                                          # render[240, 320] == 0: zero anchor, NaN translation
    assert off[240, 320] == 0
    renders = data["renders"] + [wide]
    which = data["which"].copy()
    which[::3] = len(renders) - 1
    which[1::3] = 2
    nat = detector(data, renders, which)
    pose = pose_chain(nat, data, 62.0, 0, False)
    early = pose[3] == np.float32(-1.0)
    nan_t = ~early & np.isnan(pose[2]).any(1)
    assert early.any() and nan_t.any() and (~early & ~nan_t).any()
    for tthr in (40.0, 0.0, np.inf):
        want = expected(pose, tthr)
        got = detect_chain(nat, data, 62.0, 0, False, tthr)
        same(got, want)
        kept = set(map(tuple, got[0][["x", "y", "template_id"]].tolist()))
        assert not kept & set(map(tuple, pose[0][early][["x", "y", "template_id"]].tolist()))
        # once a NaN translation is kept, nothing after it is
        bad = np.flatnonzero(np.isnan(got[2]).any(1))
        if bad.size:
            assert bad[0] == len(got[0]) - 1


def test_two_classes(data):
    p = data["packed"]
    G, nf = data["G"], p["feats"].shape[0]
    tm2 = p["tmeta"][::-1].copy()  # reversed: where the classes tie, the lower template id wins the box NMS
    tm2[..., 2] += nf
    packed = dict(class_begin=np.array([0, G, 2 * G], np.int32), tmeta=np.concatenate([p["tmeta"], tm2]),
                  feats=np.concatenate([p["feats"], p["feats"]]))
    nat = detector(data, packed=packed, reversed_copy=True)
    pose = pose_chain(nat, data, 65.0, 0, False)
    assert set(pose[0]["class_index"].tolist()) == {0, 1}
    for tthr in (40.0, 0.0):
        same(detect_chain(nat, data, 65.0, 0, False, tthr), expected(pose, tthr))


def test_result_block_retry(data):
    probe = detector(data)
    thr = None
    for cand in (55.0, 50.0, 45.0, 40.0):
        pose = pose_chain(probe, data, cand, 0, True)
        if pose[4] > (1 << 16):                                       # more records than the initial result block holds
            thr = cand
            break
    assert thr is not None
    nat = detector(data)                                              # fresh handle: the first frame overflows the block
    same(detect_chain(nat, data, thr, 0, True, 40.0), expected(pose, 40.0))


def test_one_launch_per_frame(data):
    nat = detector(data)
    g = data["g"]
    pose_chain(nat, data, 62.0, 0, False)
    for top_k in (3, 0):
        nat.upload_images(g["rgb"], g["depth"], None)
        nat.enqueue(62.0)
        nat.enqueue_post(0.5, top_k)
        nat.enqueue_pose(data["sK"], 30, False)
        before = nat.launch_count()
        nat.enqueue_pose_nms(40.0)
        out = nat.complete_detect()
        assert nat.launch_count() - before == 1
        a = nat.launch_count()
        pose_chain(nat, data, 62.0, top_k, False)
        b = nat.launch_count()
        detect_chain(nat, data, 62.0, top_k, False, 40.0)
        assert nat.launch_count() - b == b - a + 1
        assert out[4]["survivors"] == 3 if top_k else out[4]["survivors"] > 3


def expect(fn, code):
    with pytest.raises(RuntimeError) as e:
        fn()
    if code == lib.LM_E_INVALID:
        assert not isinstance(e.value, lib.LinemodLibraryError), e.value
    else:
        assert ("error %d" % code) in str(e.value), e.value


def test_errors(data):
    g = data["g"]
    nat = detector(data)
    want = pose_chain(nat, data, 75.0, 3, False)
    # no pose stage enqueued
    expect(lambda: nat.enqueue_pose_nms(40.0), lib.LM_E_STATE)
    expect(lambda: nat.complete_detect(), lib.LM_E_STATE)
    nat.upload_images(g["rgb"], g["depth"], None)
    nat.enqueue(75.0)
    nat.enqueue_post(0.5, 3)
    expect(lambda: nat.enqueue_pose_nms(40.0), lib.LM_E_STATE)
    nat.enqueue_pose(data["sK"], 30, False)
    expect(lambda: nat.enqueue_pose_nms(float("nan")), lib.LM_E_INVALID)
    expect(lambda: nat.enqueue_pose_nms(-1.0), lib.LM_E_INVALID)
    nat.enqueue_pose_nms(40.0)
    expect(lambda: nat.enqueue_pose_nms(40.0), lib.LM_E_STATE)        # once per frame
    expect(lambda: nat.complete_pose(), lib.LM_E_STATE)               # the frame completes through complete_detect
    same(nat.complete_detect(), expected(want, 40.0))
    expect(lambda: nat.complete_detect(), lib.LM_E_STATE)
    # without the pose NMS, lm_complete_pose returns what it did
    again = pose_chain(nat, data, 75.0, 3, False)
    assert np.array_equal(again[0], want[0]) and again[4] == want[4]
    for a, b in zip(again[1:4], want[1:4]):
        assert np.array_equal(a, b, equal_nan=True)
    # the standalone entry point
    expect(lambda: lib.nms_translations(np.zeros((1025, 3)), np.zeros(1025), 40.0), lib.LM_E_CAPACITY)
    expect(lambda: lib.nms_translations(np.zeros((3, 3)), np.zeros(3), float("nan")), lib.LM_E_INVALID)
    expect(lambda: lib.nms_translations(np.zeros((3, 3)), np.zeros(3), -0.5), lib.LM_E_INVALID)
    assert lib.nms_translations(np.zeros((0, 3)), np.zeros(0), 40.0).tolist() == []


def test_detector_detect_equals_match_refine_and_nms_translations(data, tmp_path):
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
    for thr in (65.0, 75.0):
        got = det.detect([g["rgb"], g["depth"]], thr, ["06_template"], data["sK"])
        pairs = det.match_refine([g["rgb"], g["depth"]], thr, ["06_template"], data["sK"], top_k=0)
        posed = [(m, p) for m, p in pairs if p.getResidual() != -1.0]
        ts = np.array([p.getT().reshape(3) for _, p in posed]).reshape(-1, 3)
        keep = pr.nms_translations(ts, [-p.getResidual() for _, p in posed], 40.0)
        assert len(got) == len(keep) > 0
        for (m, p), k in zip(got, keep):
            m2, p2 = posed[k]
            assert (m.x, m.y, m.similarity, m.class_id, m.template_id) == (m2.x, m2.y, m2.similarity, m2.class_id, m2.template_id)
            assert p.getResidual() == p2.getResidual()
            assert np.array_equal(p.getR(), p2.getR(), equal_nan=True) and np.array_equal(p.getT(), p2.getT(), equal_nan=True)
            assert p.getT().shape == (3, 1)
