"""A batch of RGB-D frames through one pose stage (lm_detect_batch, Detector.match_refine_batch / detect_batch): every
frame's entries must equal, bit for bit, what the single-frame chain (match_pose / detect) returns for that frame alone
on a handle that never ran a batch -- match records, R, t and residual (NaN patterns included) and all four counts.
The data are those of tests/test_gpu_pose_stage.py: the recorded driver frame against the allScales bank, per-template
renders that are the recorded render shifted by a few pixels."""
import ctypes
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
    rgb, depth = g["rgb"], g["depth"]
    H, W = depth.shape
    mask = np.zeros((H, W), np.uint8)
    mask[:, W // 3:] = 255
    frames = dict(
        recorded=(rgb, depth, None),
        rolled=(np.roll(rgb, (17, -23), (0, 1)), np.roll(depth, (17, -23), (0, 1)), None),
        mirrored=(np.ascontiguousarray(rgb[:, ::-1]), np.ascontiguousarray(depth[:, ::-1]), None),
        blank=(np.zeros_like(rgb), np.zeros_like(depth), None),
        masked=(rgb, depth, (mask, mask)),
    )
    return dict(g=g, packed=packed, T=b["T"].tolist(), G=G, renders=renders, which=np.arange(G) % len(renders), K=K, R=R, t=t,
                sK=g["rf0_sceneK"].astype(np.float32), frames=frames)


def detector(data, renders=None, which=None):
    renders = data["renders"] if renders is None else renders
    which = data["which"] if which is None else which
    nat = lib.NativeDetector(data["T"], 0)
    nat.load_bank(data["packed"], 4)
    nat.select(None, 0, 1)
    nat.set_template_renders(0, [renders[k] for k in which], data["K"], data["R"], data["t"])
    return nat


def scene_ks(data, n):
    # a different focal length and principal point per frame: the scene clouds and centroids depend on them
    K = np.repeat(data["sK"][None], n, 0).copy()
    K[:, 0, 0] *= 1.0 + 0.01 * np.arange(n)
    K[:, 1, 2] += np.arange(n)
    return K


def single(nat, frame, K, thr, top_k, iters, use_scene, pose_nms, tthr=40.0):
    rgb, depth, masks = frame
    mk = list(masks) if masks else None
    if pose_nms:
        return nat.detect(rgb, depth, mk, thr, K, 0.5, top_k, iters, use_scene, tthr)
    return nat.match_pose(rgb, depth, mk, thr, K, 0.5, top_k, iters, use_scene)


def batch(nat, frames, K, thr, top_k, iters, use_scene, pose_nms, tthr=40.0, cap=None):
    masks = [list(f[2]) if f[2] else [None, None] for f in frames]
    return nat.detect_batch(np.stack([f[0] for f in frames]), np.stack([f[1] for f in frames]), masks, thr, K, 0.5, top_k, iters,
                            use_scene, pose_nms, tthr, cap)


def same(got, want, counts, pose_nms):
    out, R, t, res, extra = got
    assert np.array_equal(out, want[0])
    assert np.array_equal(res, want[3], equal_nan=True), (res, want[3])
    assert np.array_equal(R, want[1], equal_nan=True)
    assert np.array_equal(t, want[2], equal_nan=True)
    assert extra == want[4]
    if pose_nms:
        assert counts.tolist() == [len(want[0]), want[4]["survivors"], want[4]["posed"], want[4]["records"]]
    else:
        assert counts.tolist() == [len(want[0]), len(want[0]), int((want[3] != -1.0).sum()), want[4]]


@pytest.fixture(scope="module")
def handles(data):
    return dict(single=detector(data), batch=detector(data))


@pytest.mark.parametrize("iters", [30, 10])
@pytest.mark.parametrize("use_scene", [False, True])
@pytest.mark.parametrize("pose_nms", [False, True])
@pytest.mark.parametrize("top_k", [1, 3, 0])
def test_batch_equals_single_frames(data, handles, top_k, pose_nms, use_scene, iters):
    fr = data["frames"]
    frames = [fr["recorded"], fr["rolled"], fr["mirrored"], fr["recorded"], fr["blank"], fr["masked"]]
    K = scene_ks(data, len(frames))
    K[3] = K[0]                                                       # the same frame twice, intrinsics included
    got = batch(handles["batch"], frames, K, 75.0, top_k, iters, use_scene, pose_nms)
    assert len(got) == len(frames)
    for f, frame in enumerate(frames):
        want = single(handles["single"], frame, K[f], 75.0, top_k, iters, use_scene, pose_nms)
        same(got[f], want, handles["batch"].batch_counts[f], pose_nms)
    n = [len(g[0]) for g in got]
    assert n[4] == 0 and min(n[0], n[1], n[2], n[5]) > 0, n           # the blank frame has no match, the others do
    assert np.array_equal(got[0][0], got[3][0])
    for x, y in zip(got[0][1:4], got[3][1:4]):
        assert np.array_equal(x, y, equal_nan=True)


def test_one_frame_and_shared_scene_matrix(data, handles):
    frame = data["frames"]["recorded"]
    for pose_nms in (False, True):
        got = batch(handles["batch"], [frame], data["sK"][None], 75.0, 0, 30, True, pose_nms)
        same(got[0], single(handles["single"], frame, data["sK"], 75.0, 0, 30, True, pose_nms), handles["batch"].batch_counts[0],
             pose_nms)


def test_survivors_beyond_one_chunk(data, handles):
    fr = data["frames"]
    frames = [fr["recorded"], fr["rolled"], fr["recorded"], fr["mirrored"]]
    K = scene_ks(data, len(frames))
    for pose_nms in (True, False):
        got = batch(handles["batch"], frames, K, 65.0, 0, 30, False, pose_nms)
        survivors = handles["batch"].batch_counts[:, 1]
        assert survivors.sum() > 1024 and survivors.max() <= 1024, survivors  # two chunks
        for f, frame in enumerate(frames):
            same(got[f], single(handles["single"], frame, K[f], 65.0, 0, 30, False, pose_nms), handles["batch"].batch_counts[f], pose_nms)


def test_early_returns_and_nan_anchors(data):
    g = data["g"]
    wide = np.zeros_like(g["render"])
    wide[200:260, 10:600] = 1000                               # a 598 x 68 box: fits only survivors with x < 42
    off = data["renders"][2]                                   # render[240, 320] == 0: the scene centroid is NaN
    assert off[240, 320] == 0
    renders = [wide, off]
    which = np.arange(data["G"]) % 2
    ref, nat = detector(data, renders, which), detector(data, renders, which)
    fr = data["frames"]
    frames = [fr["recorded"], fr["mirrored"], fr["rolled"]]
    K = scene_ks(data, 3)
    for pose_nms in (False, True):
        for use_scene in (False, True):
            got = batch(nat, frames, K, 62.0, 0, 30, use_scene, pose_nms)
            for f, frame in enumerate(frames):
                same(got[f], single(ref, frame, K[f], 62.0, 0, 30, use_scene, pose_nms), nat.batch_counts[f], pose_nms)
            if not pose_nms:
                res = np.concatenate([x[3] for x in got])
                R = np.concatenate([x[1] for x in got])
                assert (res == -1.0).any() and (res != -1.0).any()
                assert np.isnan(R[res != -1.0]).any()


def test_result_block_retry_inside_a_batch(data):
    probe = detector(data)
    g = data["g"]
    thr = None
    for cand in (55.0, 50.0, 45.0, 40.0):
        probe.upload_images(g["rgb"], g["depth"], None)
        probe.enqueue(cand)
        probe.enqueue_post(0.5, 5)
        if probe.complete_post()[1] > (1 << 16):               # more records than the initial result block holds
            thr = cand
            break
    assert thr is not None
    fr = data["frames"]
    frames = [fr["blank"], fr["recorded"], fr["mirrored"]]
    K = scene_ks(data, 3)
    for pose_nms in (False, True):
        nat = detector(data)                                   # fresh handle: the second frame overflows the block
        got = batch(nat, frames, K, thr, 5, 30, True, pose_nms)
        ref = detector(data)
        for f, frame in enumerate(frames):
            same(got[f], single(ref, frame, K[f], thr, 5, 30, True, pose_nms), nat.batch_counts[f], pose_nms)
        assert nat.batch_counts[1, 3] > (1 << 16)


def match_launches(nat, frame, thr, top_k):
    rgb, depth, _ = frame
    before = nat.launch_count()
    nat.upload_images(rgb, depth, None)
    nat.enqueue(thr)
    nat.enqueue_post(0.5, top_k)
    nat.complete_post()
    return nat.launch_count() - before


def test_pose_launches_per_chunk(data):
    nat = detector(data)
    frame = data["frames"]["recorded"]
    for thr, n_frames in ((75.0, 1), (75.0, 8), (65.0, 3)):
        match_launches(nat, frame, thr, 0)                     # first use of this threshold
        per_frame = match_launches(nat, frame, thr, 0)
        for pose_nms in (False, True):
            K = scene_ks(data, n_frames)
            batch(nat, [frame] * n_frames, K, thr, 0, 30, False, pose_nms)  # warm: buffers sized
            before = nat.launch_count()
            batch(nat, [frame] * n_frames, K, thr, 0, 30, False, pose_nms)
            S = int(nat.batch_counts[:, 1].sum())
            chunks = (S + 1023) // 1024
            assert chunks == (2 if thr == 65.0 else 1), S
            assert nat.launch_count() - before == n_frames * per_frame + 5 * chunks + (1 if pose_nms else 0)


def test_single_frame_after_a_batch(data, handles):
    fr = data["frames"]
    nat = detector(data)
    batch(nat, [fr["rolled"], fr["recorded"]], scene_ks(data, 2), 65.0, 0, 10, True, True)
    for pose_nms in (True, False):
        got = single(nat, fr["recorded"], data["sK"], 75.0, 3, 30, False, pose_nms)
        want = single(handles["single"], fr["recorded"], data["sK"], 75.0, 3, 30, False, pose_nms)
        assert np.array_equal(got[0], want[0])
        for x, y in zip(got[1:4], want[1:4]):
            assert np.array_equal(x, y, equal_nan=True)
        assert got[4] == want[4]


def expect(fn, code):
    with pytest.raises(RuntimeError) as e:
        fn()
    if code == lib.LM_E_INVALID:
        assert not isinstance(e.value, lib.LinemodLibraryError), e.value
    else:
        assert ("error %d" % code) in str(e.value), e.value


def test_capacity(data, handles):
    fr = data["frames"]
    frames = [fr["recorded"], fr["mirrored"]]
    K = scene_ks(data, 2)
    nat = handles["batch"]
    for pose_nms in (False, True):
        full = batch(nat, frames, K, 75.0, 0, 30, False, pose_nms)
        total = sum(len(x[0]) for x in full)
        assert total > 1
        grown = batch(nat, frames, K, 75.0, 0, 30, False, pose_nms, cap=1)  # too small: the binding grows it and calls again
        for x, y in zip(full, grown):
            assert np.array_equal(x[0], y[0])
            for a, b in zip(x[1:4], y[1:4]):
                assert np.array_equal(a, b, equal_nan=True)
        # the C-ABI itself: LM_E_CAPACITY with the needed total and the frame counts
        L = lib.load()
        rgb = np.ascontiguousarray(np.stack([f[0] for f in frames]))
        depth = np.ascontiguousarray(np.stack([f[1] for f in frames]))
        n, counts = ctypes.c_int64(), np.zeros((2, 4), np.int64)
        rc = L.lm_detect_batch(nat._h, 2, rgb.ctypes.data_as(ctypes.POINTER(ctypes.c_uint8)),
                               depth.ctypes.data_as(ctypes.POINTER(ctypes.c_uint16)), 480, 640, None, ctypes.c_float(75.0),
                               np.ascontiguousarray(K).ctypes.data_as(ctypes.POINTER(ctypes.c_float)), 0.5, 0, 30, 0,
                               1 if pose_nms else 0, 40.0, None, None, None, None, 0, ctypes.byref(n),
                               counts.ctypes.data_as(ctypes.POINTER(ctypes.c_int64)))
        assert rc == lib.LM_E_CAPACITY and n.value == total
        assert counts[:, 0].tolist() == [len(x[0]) for x in full]


def test_errors(data):
    fr = data["frames"]
    frames = [fr["recorded"]]
    K = scene_ks(data, 1)
    nat = detector(data)
    empty = (np.zeros((0, 480, 640, 3), np.uint8), np.zeros((0, 480, 640), np.uint16))
    expect(lambda: nat.detect_batch(*empty, None, 75.0, np.zeros((0, 3, 3), np.float32)), lib.LM_E_INVALID)  # n_frames 0
    expect(lambda: batch(nat, frames, K, 75.0, 0, 30, False, True, tthr=float("nan")), lib.LM_E_INVALID)
    expect(lambda: batch(nat, frames, K, 75.0, 0, 30, False, True, tthr=-1.0), lib.LM_E_INVALID)
    bare = lib.NativeDetector(data["T"], 0)                    # no renders registered
    bare.load_bank(data["packed"], 4)
    bare.select(None, 0, 1)
    expect(lambda: batch(bare, frames, K, 75.0, 0, 30, False, True), lib.LM_E_STATE)
    # a connected exchange: the batch is single-GPU only
    world = 2
    dets = []
    for r in range(world):
        d = detector(data)
        d.select(None, r, world)
        d.peer_export(world, 1 << 17)
        dets.append(d)
    bases = [d.peer_base() for d in dets]
    for r, d in enumerate(dets):
        d.peer_connect_local(r, world, bases)
    expect(lambda: batch(dets[0], frames, K, 75.0, 0, 30, False, False), lib.LM_E_STATE)
    for d in dets:
        d.peer_disconnect()
    # the handle still works
    got = batch(nat, frames, K, 75.0, 3, 30, False, False)
    assert len(got[0][0]) == 3


def test_detector_batch_methods(data, tmp_path):
    bk = importlib.import_module("6dpose_b200.bank")
    g, packed = data["g"], data["packed"]
    bank = bk.TemplateBank()
    bank.classes["06_template"] = bk.PackedPyramids(packed["tmeta"], packed["feats"], 2)
    bank.write_packed("06_template", str(tmp_path / "06_template.lmb"), 2)
    det = pkg.Detector(int(g["num_features"]), data["T"])
    det.readClasses(["06_template"], str(tmp_path / "%s.lmb"))
    which = data["which"]
    det.setTemplateRenders({"06_template": ((data["renders"][k] for k in which), data["K"], data["R"], data["t"])})
    fr = data["frames"]
    frames = [[fr["recorded"][0], fr["recorded"][1]], [fr["mirrored"][0], fr["mirrored"][1]], [fr["masked"][0], fr["masked"][1]]]
    masks = [[], [], list(fr["masked"][2])]
    K = scene_ks(data, 3)

    def same_pairs(a, b):
        assert len(a) == len(b)
        for (m, p), (m2, p2) in zip(a, b):
            assert (m.x, m.y, m.similarity, m.class_id, m.template_id) == (m2.x, m2.y, m2.similarity, m2.class_id, m2.template_id)
            assert p.getResidual() == p2.getResidual()
            if p2.getR() is None:
                assert p.getR() is None and p.getT() is None
            else:
                assert np.array_equal(p.getR(), p2.getR(), equal_nan=True) and np.array_equal(p.getT(), p2.getT(), equal_nan=True)

    got = det.match_refine_batch(frames, 75.0, ["06_template"], K, top_k=3, masks=masks)
    for f in range(3):
        same_pairs(got[f], det.match_refine(frames[f], 75.0, ["06_template"], K[f], top_k=3, masks=masks[f]))
    got = det.detect_batch(frames, 75.0, ["06_template"], list(K), masks=masks)
    for f in range(3):
        same_pairs(got[f], det.detect(frames[f], 75.0, ["06_template"], K[f], masks=masks[f]))
    # one frame, one shared 3x3 sceneK
    got = det.detect_batch(frames[:1], 75.0, ["06_template"], data["sK"])
    assert len(got) == 1 and len(got[0]) > 0
    same_pairs(got[0], det.detect(frames[0], 75.0, ["06_template"], data["sK"]))
