"""RGB-D frames already in device memory (lm_bind_images_device, lm_detect_batch_device, the Detector methods with CUDA
tensors): every result must equal, bit for bit, the host-frame path on the same frame -- label images, depth, matches,
R, t, residual and counts.  Frames: the recorded driver frame (tests/golden/driver_trace.npz) and its patched copy
(frame_half_case1.npz), against the allScales bank with the shifted renders of tests/test_gpu_detect_batch.py."""
import ctypes
import importlib
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
lib = importlib.import_module("6dpose_b200._lib")
pkg = importlib.import_module("6dpose_b200")

SHIFTS = [(0, 0), (-68, -19), (-180, 57), (3, -2), (-2, 4)]


@pytest.fixture(scope="module")
def data():
    g = np.load(os.path.join(GOLD, "driver_trace.npz"))
    b = np.load(os.path.join(GOLD, "bank_allScales_full.npz"))
    h = np.load(os.path.join(GOLD, "frame_half_case1.npz"))
    packed = dict(class_begin=b["class_begin"], tmeta=b["tmeta"].astype(np.int32), feats=b["feats"].astype(np.int32))
    G = packed["tmeta"].shape[0]
    renders = [np.ascontiguousarray(np.roll(np.roll(g["render"], dy, 0), dx, 1)) for dy, dx in SHIFTS]
    K = np.repeat(g["rf0_modelK"][None], G, 0).astype(np.float32)
    R = np.repeat(g["rf0_modelR"][None], G, 0).astype(np.float32)
    t = np.repeat(g["rf0_modelT"].reshape(1, 3), G, 0).astype(np.float32)
    t[:, 0] += (np.arange(G) % 7) - 3.0
    t[:, 2] += np.arange(G) % 11
    rgb, depth = g["rgb"], g["depth"]
    rgb_h, depth_h = rgb[..., ::-1].copy(), depth.copy()
    rgb_h.reshape(-1, 3)[h["index"]] = h["bgr"]
    depth_h.reshape(-1)[h["index"]] = h["depth"]
    rgb_h = np.ascontiguousarray(rgb_h[..., ::-1])
    H, W = depth.shape
    mask = np.zeros((H, W), np.uint8)
    mask[:, W // 3:] = 255
    mask2 = np.zeros((H, W), np.uint8)
    mask2[H // 5:, :W - W // 4] = 255
    frames = dict(recorded=(rgb, depth), half=(rgb_h, depth_h), rolled=(np.roll(rgb, (17, -23), (0, 1)), np.roll(depth, (17, -23), (0, 1))),
                  mirrored=(np.ascontiguousarray(rgb[:, ::-1]), np.ascontiguousarray(depth[:, ::-1])),
                  blank=(np.zeros_like(rgb), np.zeros_like(depth)))
    return dict(g=g, packed=packed, T=b["T"].tolist(), G=G, renders=renders, which=np.arange(G) % len(renders), K=K, R=R, t=t,
                sK=g["rf0_sceneK"].astype(np.float32), frames=frames, masks=(mask, mask2),
                z=np.load(os.path.join(GOLD, "allScales_depths.npz"))["z_mm"])


def detector(data, shard=(0, 1)):
    nat = lib.NativeDetector(data["T"], 0)
    nat.load_bank(data["packed"], 4)
    nat.select(None, shard[0], shard[1])
    nat.set_template_renders(0, [data["renders"][k] for k in data["which"]], data["K"], data["R"], data["t"])
    nat.set_template_depths(0, data["z"])
    return nat


@pytest.fixture(scope="module")
def handles(data):
    return dict(host=detector(data), dev=detector(data))


def cuda(a, crop=False):
    """A CUDA tensor holding numpy image a; crop: a view into a larger tensor whose row pitch is no multiple of 16 bytes."""
    a = np.ascontiguousarray(a)
    src = torch.from_numpy(a.view(np.int16) if a.dtype == np.uint16 else a).cuda()
    if a.dtype == np.uint16:
        src = src.view(torch.uint16)
    if not crop:
        return src
    H, W = a.shape[:2]
    big = torch.zeros((H + 3, W + 5) + a.shape[2:], dtype=src.dtype, device=src.device)
    view = big[1:H + 1, 2:W + 2]
    view.copy_(src)
    return view


def bind(nat, rgb, depth, masks=None, depth_scale=1.0, stream=None):
    nat.bind_frame(lib.frame_inputs(rgb, depth, masks, depth_scale, stream, 0))


def host_depth(d, scale):
    """The driver's conversion (linemod_and_levelup_test.py:315-317) where it is defined, 0 (no depth) elsewhere."""
    v = np.asarray(d, np.float32) * np.float32(scale)
    ok = (v >= 0) & (v < 65536)
    return np.where(ok, np.where(ok, v, 0).astype(np.uint16), 0).astype(np.uint16)


def same_labels(a, b, T, shape):
    for l in range(len(T)):
        s = (shape[0] >> l, shape[1] >> l)
        for m in range(2):
            assert np.array_equal(a.quantized(l, m, s), b.quantized(l, m, s)), (l, m)
    assert np.array_equal(a.depth_image(shape), b.depth_image(shape))


@pytest.mark.parametrize("crop", [False, True])
@pytest.mark.parametrize("with_masks", [False, True])
def test_labels_equal_the_host_upload(data, handles, crop, with_masks):
    for rgb, depth in (data["frames"]["recorded"], data["frames"]["half"]):
        masks = list(data["masks"]) if with_masks else None
        handles["host"].upload_images(rgb, depth, masks)
        dm = [cuda(m, crop) for m in masks] if masks else None
        r, d = cuda(rgb, crop), cuda(depth, crop)
        if crop:
            assert r.stride(0) % 16 and (d.stride(0) * 2) % 16 and (not dm or dm[0].stride(0) % 16)
        bind(handles["dev"], r, d, dm)
        same_labels(handles["dev"], handles["host"], data["T"], depth.shape)


def test_only_one_mask(data, handles):
    rgb, depth = data["frames"]["half"]
    for m in (0, 1):
        masks = [None, None]
        masks[m] = data["masks"][m]
        handles["host"].upload_images(rgb, depth, masks)
        bind(handles["dev"], cuda(rgb), cuda(depth, True), [cuda(x, True) if x is not None else None for x in masks])
        same_labels(handles["dev"], handles["host"], data["T"], depth.shape)


@pytest.mark.parametrize("scale", [1.0, 0.1])
def test_float_depth_equals_the_converted_host_frame(data, handles, scale):
    rng = np.random.default_rng(7)
    rgb, depth = data["frames"]["recorded"]
    d = (depth.astype(np.float32) + rng.uniform(0, 0.999, depth.shape).astype(np.float32)) / np.float32(scale)
    u16 = host_depth(d, scale)
    assert np.abs(u16.astype(np.int64) - depth).max() <= 1
    handles["host"].upload_images(rgb, u16, None)
    bind(handles["dev"], cuda(rgb), cuda(d, True), None, depth_scale=scale)
    same_labels(handles["dev"], handles["host"], data["T"], depth.shape)
    want = handles["host"].match_images(rgb, u16, None, 75.0)
    got = handles["dev"].match_images(cuda(rgb), cuda(d), None, 75.0, depth_scale=scale)
    assert len(want) > 0 and np.array_equal(got, want)
    # salted: NaN, negative, infinite, >= 65536 and x.9999 values
    s = d.copy().reshape(-1)
    n = s.size
    idx = rng.permutation(n)[:6000].reshape(6, -1)
    s[idx[0]] = np.nan
    s[idx[1]] = -rng.uniform(0.001, 5000, idx.shape[1]).astype(np.float32)
    s[idx[2]] = np.float32(np.inf) * np.where(rng.random(idx.shape[1]) < 0.5, 1, -1).astype(np.float32)
    s[idx[3]] = (np.float32(65536.0) + rng.uniform(0, 1e6, idx.shape[1]).astype(np.float32)) / np.float32(scale)
    s[idx[4]] = (rng.integers(0, 65535, idx.shape[1]).astype(np.float32) + np.float32(0.9999)) / np.float32(scale)
    s[idx[5]] = np.nextafter(np.float32(65536.0) / np.float32(scale), np.float32(0))
    s = s.reshape(depth.shape)
    bind(handles["dev"], cuda(rgb), cuda(s, True), None, depth_scale=scale)
    got = handles["dev"].depth_image(depth.shape)
    want = host_depth(s, scale)
    assert np.array_equal(got, want)
    assert (want.reshape(-1)[idx[:4].reshape(-1)] == 0).all() and (want.reshape(-1)[idx[4]] > 0).mean() > 0.99
    with np.errstate(invalid="ignore"):
        ok = np.isfinite(s) & (s * np.float32(scale) >= 0) & (s * np.float32(scale) < 65536)
        assert np.array_equal(want[ok], (s[ok] * np.float32(scale)).astype(np.uint16))


def same_pose(got, want):
    assert np.array_equal(got[0], want[0])
    for x, y in zip(got[1:4], want[1:4]):
        assert np.array_equal(x, y, equal_nan=True)
    assert got[4] == want[4]


@pytest.mark.parametrize("gate", [None, 0.2])
@pytest.mark.parametrize("estimation", ["point_to_plane", "point_to_point"])
@pytest.mark.parametrize("thr", [75.0, 65.0])
def test_match_refine_and_detect_equal_the_host_frame(data, handles, thr, estimation, gate):
    host, dev = handles["host"], handles["dev"]
    for nat in (host, dev):
        nat.set_depth_gate(gate)
    try:
        for name in ("recorded", "half"):
            rgb, depth = data["frames"][name]
            r, d = cuda(rgb, True), cuda(depth)
            want = host.match_images(rgb, depth, None, thr)
            assert len(want) > 0
            assert np.array_equal(dev.match_images(r, d, None, thr), want)
            want = host.match_pose(rgb, depth, None, thr, data["sK"], 0.5, 3, 30, False, estimation)
            same_pose(dev.match_pose(r, d, None, thr, data["sK"], 0.5, 3, 30, False, estimation), want)
            want = host.detect(rgb, depth, None, thr, data["sK"], 0.5, 0, 30, False, 40.0, estimation)
            assert len(want[0]) > 0
            same_pose(dev.detect(r, d, None, thr, data["sK"], 0.5, 0, 30, False, 40.0, estimation), want)
    finally:
        for nat in (host, dev):
            nat.set_depth_gate(None)


def host_batch(nat, frames, masks, K, thr, pose_nms):
    return nat.detect_batch(np.stack([f[0] for f in frames]), np.stack([f[1] for f in frames]), masks, thr, K, 0.5, 0, 30, False,
                            pose_nms, 40.0)


def device_batch(nat, frames, masks, K, thr, pose_nms, crop=False, depth_scale=1.0, stream=None):
    batch = lib.DeviceBatch([lib.DeviceFrame(cuda(f[0], crop), cuda(f[1], crop),
                                             [cuda(x, crop) if x is not None else None for x in m] if m else None, depth_scale, stream, 0)
                             for f, m in zip(frames, masks or [None] * len(frames))])
    return nat.detect_batch_device(batch, thr, K, 0.5, 0, 30, False, pose_nms, 40.0)


@pytest.mark.parametrize("pose_nms", [True, False])
def test_batch_equals_the_host_batch(data, handles, pose_nms):
    fr = data["frames"]
    frames = [fr["recorded"], fr["rolled"], fr["mirrored"], fr["half"], fr["blank"], fr["recorded"]]
    masks = [[None, None]] * 5 + [list(data["masks"])]
    K = np.repeat(data["sK"][None], len(frames), 0)
    K[:, 0, 0] *= 1.0 + 0.01 * np.arange(len(frames))
    want = host_batch(handles["host"], frames, masks, K, 75.0, pose_nms)
    want_counts = handles["host"].batch_counts.copy()
    for crop in (False, True):
        got = device_batch(handles["dev"], frames, masks, K, 75.0, pose_nms, crop)
        assert np.array_equal(handles["dev"].batch_counts, want_counts)
        for g, w in zip(got, want):
            same_pose(g, w)
    # more than 1024 survivors: the pose stage runs in two chunks
    frames = [fr["recorded"], fr["rolled"], fr["recorded"], fr["mirrored"]]
    K = K[:4]
    want = host_batch(handles["host"], frames, None, K, 65.0, pose_nms)
    want_counts = handles["host"].batch_counts.copy()
    assert want_counts[:, 1].sum() > 1024
    got = device_batch(handles["dev"], frames, None, K, 65.0, pose_nms)
    assert np.array_equal(handles["dev"].batch_counts, want_counts)
    for g, w in zip(got, want):
        same_pose(g, w)


def test_detector_methods_take_tensors(data, tmp_path):
    bk = importlib.import_module("6dpose_b200.bank")
    packed = data["packed"]
    bank = bk.TemplateBank()
    bank.classes["06_template"] = bk.PackedPyramids(packed["tmeta"], packed["feats"], 2)
    bank.write_packed("06_template", str(tmp_path / "06_template.lmb"), 2)
    det = pkg.Detector(int(data["g"]["num_features"]), data["T"])
    det.device = 0
    det.readClasses(["06_template"], str(tmp_path / "%s.lmb"))
    det.setTemplateRenders({"06_template": ((data["renders"][k] for k in data["which"]), data["K"], data["R"], data["t"])})
    fr = data["frames"]
    host = [list(fr["recorded"]), list(fr["half"])]
    d_f32 = fr["half"][1].astype(np.float32) * np.float32(10.0) + np.float32(3.0)   # 0.1 mm units; truncates to the mm
    dev = [[cuda(fr["recorded"][0]), cuda(fr["recorded"][1], True)], [cuda(fr["half"][0], True), cuda(d_f32)]]
    flat = lambda pairs: [((m.x, m.y, m.similarity, m.class_id, m.template_id), p.getResidual(),
                           None if p.getR() is None else (p.getR().tobytes(), p.getT().tobytes())) for m, p in pairs]
    ms = lambda ms_: [(m.x, m.y, m.similarity, m.class_id, m.template_id) for m in ms_]
    for f in range(2):
        kw = dict(depth_scale=0.1) if f == 1 else {}
        assert ms(det.match(dev[f], 75.0, ["06_template"], [], **kw)) == ms(det.match(host[f], 75.0, ["06_template"], []))
        assert flat(det.match_refine(dev[f], 75.0, ["06_template"], data["sK"], **kw)) == flat(
            det.match_refine(host[f], 75.0, ["06_template"], data["sK"]))
        assert flat(det.detect(dev[f], 75.0, ["06_template"], data["sK"], **kw)) == flat(det.detect(host[f], 75.0, ["06_template"], data["sK"]))
    det.frontend = "cv2"                                        # not for tensors: match still takes the GPU front-end
    assert len(det.match(dev[0], 75.0, ["06_template"], [])) > 0
    det.frontend = "gpu"
    K = np.repeat(data["sK"][None], 2, 0)
    with pytest.raises(ValueError, match="row pitch"):               # a contiguous and a cropped frame in one batch
        det.detect_batch([dev[0], [cuda(fr["half"][0], True), cuda(fr["half"][1], True)]], 75.0, ["06_template"], K)
    dev_b = [[cuda(fr["recorded"][0], True), cuda(fr["recorded"][1], True)], [cuda(fr["half"][0], True), cuda(fr["half"][1], True)]]
    got = det.detect_batch(dev_b, 75.0, ["06_template"], K)
    want = det.detect_batch(host, 75.0, ["06_template"], K)
    assert [flat(x) for x in got] == [flat(x) for x in want] and len(want[0]) > 0
    got = det.match_refine_batch(dev_b, 75.0, ["06_template"], K, masks=[[], [cuda(data["masks"][0]), None]])
    want = det.match_refine_batch(host, 75.0, ["06_template"], K, masks=[[], [data["masks"][0], None]])
    assert [flat(x) for x in got] == [flat(x) for x in want]
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        r, d = cuda(fr["rolled"][0]), cuda(fr["rolled"][1])
    got = det.detect([r, d], 75.0, ["06_template"], data["sK"], stream=side)
    assert flat(got) == flat(det.detect(list(fr["rolled"]), 75.0, ["06_template"], data["sK"]))


def test_ordering_across_streams(data, handles):
    """A frame written on a side stream and bound on it, with no host synchronise in between, in two phases run once each.
    1. Only the side stream is held back (a sleep kernel before its write of frame A); the handle's stream is idle.  The
       ingest must wait for the write (the first event): without it, it would read the zero-filled buffer.
    2. Only the handle's stream is held back (a sleep kernel ahead of the ingest); right after the call the side stream
       overwrites the buffer with frame B.  That write must wait for the ingest (the second event): without it, the
       ingest would read B.  The next call on the side stream then returns B's matches."""
    host, dev = handles["host"], handles["dev"]
    fa, fb = data["frames"]["recorded"], data["frames"]["rolled"]
    want_a = host.match_images(fa[0], fa[1], None, 75.0)
    want_b = host.match_images(fb[0], fb[1], None, 75.0)
    blank = data["frames"]["blank"]
    want_blank = host.match_images(blank[0], blank[1], None, 75.0)
    assert len(want_a) > 0 and not np.array_equal(want_a, want_b) and not np.array_equal(want_a, want_blank)
    a = (cuda(fa[0]), cuda(fa[1]))
    b = (cuda(fb[0]), cuda(fb[1]))
    buf = (torch.zeros_like(a[0]), torch.zeros_like(a[1]))
    side = torch.cuda.Stream()
    # every kernel of the phases launched once: with lazy module loading the first launch of a kernel may synchronise the
    # device, which would order the streams by itself
    assert np.array_equal(dev.match_images(a[0], a[1], None, 75.0, stream=side), want_a)
    torch.cuda._sleep(1)
    torch.cuda.synchronize()
    # phase 1: the write is late, the ingest is not
    with torch.cuda.stream(side):
        torch.cuda._sleep(100_000_000)
        buf[0].copy_(a[0])
        buf[1].copy_(a[1])
    bind(dev, buf[0], buf[1], None, stream=side)
    dev.run(75.0)
    assert np.array_equal(dev.finish(dev.fetch_records()), want_a)
    torch.cuda.synchronize()
    # phase 2: the ingest is late, the next write is not
    with torch.cuda.stream(torch.cuda.ExternalStream(dev.stream())):
        torch.cuda._sleep(100_000_000)
    bind(dev, buf[0], buf[1], None, stream=side)
    with torch.cuda.stream(side):
        buf[0].copy_(b[0])
        buf[1].copy_(b[1])
    dev.run(75.0)
    assert np.array_equal(dev.finish(dev.fetch_records()), want_a)
    assert np.array_equal(dev.match_images(buf[0], buf[1], None, 75.0, stream=side), want_b)
    torch.cuda.synchronize()


def test_errors_before_any_device_work(data, handles):
    dev = handles["dev"]
    L = lib.load()
    rgb, depth = data["frames"]["recorded"]
    H, W = depth.shape
    r, d, f = cuda(rgb), cuda(depth), cuda(depth.astype(np.float32))
    m = cuda(data["masks"][0])

    def call(rgb_p=r.data_ptr(), rgb_pitch=3 * W, depth_p=d.data_ptr(), depth_pitch=2 * W, fmt=lib.DEPTH_U16_MM, scale=1.0, rows=H,
             cols=W, m0=None, m1=None, mask_pitch=W, stream=None):
        before = dev.launch_count()
        rc = L.lm_bind_images_device(dev._h, rgb_p, rgb_pitch, depth_p, depth_pitch, fmt, ctypes.c_float(scale), rows, cols, m0, m1,
                                     mask_pitch, stream)
        assert dev.launch_count() == before
        return rc, L.lm_last_error().decode()

    host_rgb = np.ascontiguousarray(rgb)
    pinned = torch.zeros((H, W), dtype=torch.uint8).pin_memory()
    cases = [
        dict(rgb_p=None), dict(depth_p=None),
        dict(rgb_p=host_rgb.ctypes.data), dict(depth_p=depth.ctypes.data), dict(m0=pinned.data_ptr()),
        dict(rgb_pitch=3 * W - 1), dict(depth_pitch=2 * W - 2), dict(m1=m.data_ptr(), mask_pitch=W - 1),
        dict(depth_p=d.data_ptr() + 1), dict(depth_pitch=2 * W + 1),
        dict(depth_p=f.data_ptr() + 2, depth_pitch=4 * W, fmt=lib.DEPTH_F32),
        dict(depth_p=f.data_ptr(), depth_pitch=4 * W, fmt=lib.DEPTH_F32, scale=0.0),
        dict(depth_p=f.data_ptr(), depth_pitch=4 * W, fmt=lib.DEPTH_F32, scale=float("nan")),
        dict(depth_p=f.data_ptr(), depth_pitch=4 * W, fmt=lib.DEPTH_F32, scale=-0.1),
        dict(fmt=2), dict(fmt=-1),
        dict(rows=H - 1), dict(cols=W - 3),
    ]
    if torch.cuda.device_count() >= 2:
        other = torch.zeros((H, W, 3), dtype=torch.uint8, device="cuda:1")
        other_stream = torch.cuda.Stream(device=1)
        cases += [dict(rgb_p=other.data_ptr()), dict(stream=other_stream.cuda_stream)]
        with pytest.raises(ValueError, match="cuda:0"):
            dev.match_images(other, cuda(depth), None, 75.0)
    for kw in cases:
        rc, msg = call(**kw)
        assert rc == lib.LM_E_INVALID, (kw, rc, msg)
    # the batch checks every frame first
    vp = ctypes.c_void_p
    rgbs, depths = (vp * 2)(r.data_ptr(), r.data_ptr()), (vp * 2)(d.data_ptr(), depth.ctypes.data)
    n, counts = ctypes.c_int64(), np.zeros((2, 4), np.int64)
    before = dev.launch_count()
    rc = L.lm_detect_batch_device(dev._h, 2, rgbs, 3 * W, depths, 2 * W, lib.DEPTH_U16_MM, ctypes.c_float(1.0), H, W, None, W, None,
                                  ctypes.c_float(75.0), np.ascontiguousarray(np.repeat(data["sK"][None], 2, 0)).ctypes.data_as(
                                      ctypes.POINTER(ctypes.c_float)), 0.5, 0, 30, 0, 1, 40.0, None, None, None, None, 0,
                                  ctypes.byref(n), counts.ctypes.data_as(ctypes.POINTER(ctypes.c_int64)))
    assert rc == lib.LM_E_INVALID and "frame 1" in L.lm_last_error().decode()
    assert dev.launch_count() == before
    # and the handle still works
    assert np.array_equal(dev.match_images(r, d, None, 75.0), handles["host"].match_images(rgb, depth, None, 75.0))


def test_connected_detect_from_device_frames(data):
    """A single-frame detect with the pose stage shared over two ranks (handles of one process on one device) from
    device frames equals the unconnected result."""
    single = detector(data)
    dets = [detector(data, (r, 2)) for r in range(2)]
    for d in dets:
        d.peer_export(2, 1 << 17)
    bases = [d.peer_base() for d in dets]
    for r, d in enumerate(dets):
        d.peer_connect_local(r, 2, bases)
    rgb, depth = data["frames"]["recorded"]
    r, dd = cuda(rgb), cuda(depth)

    def frame(nats, thr, top_k, on_device):
        for d in nats:
            if on_device:
                bind(d, r, dd)
            else:
                d.upload_images(rgb, depth, None)
        for d in nats:
            d.enqueue(thr)
        for d in nats:
            d.enqueue_post(0.5, top_k)
            d.enqueue_pose(data["sK"], 30, False)
            d.enqueue_pose_nms(40.0)
        return [d.complete_detect() for d in nats]

    try:
        frame(dets, 75.0, 0, False)                            # grows every pose stage's buffers before sharing
        for d in dets:
            d.peer_share_pose(True)
        for thr, top_k in ((75.0, 0), (65.0, 3)):
            want = frame([single], thr, top_k, False)[0]
            assert len(want[0]) > 0
            for got in frame(dets, thr, top_k, True):
                same_pose(got, want)
            assert all(d.pose_stats()[3] == 1 for d in dets)
    finally:
        for d in dets:
            d.peer_disconnect()
        for d in dets:
            d.close()
