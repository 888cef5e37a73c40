"""poseRefine on depths already in device memory (lm_icp_process_batch_device, NativeIcp.process_batch_device, and
poseRefine.process / refine_matches with CUDA tensors): R, t and residual must equal, bit for bit (NaNs as bits),
lm_icp_process_batch on the converted uint16 numpy images.  Every case runs under both estimations and with the scene
cloud on and off.  Inputs: the seeded cases of tests/icp_clouds.py, the recorded driver frame
(tests/golden/driver_trace.npz) with the shifted renders of tests/test_gpu_pose_stage.py and its box-NMS survivors, and
edge renders (early returns on both sides of the frame edge, clipped boxes, empty renders, a zero anchor, odd sizes)."""
import importlib
import os

import numpy as np
import pytest
import torch

import icp_clouds

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
lib = importlib.import_module("6dpose_b200._lib")
pr = importlib.import_module("6dpose_b200.pose_refine")

SHIFTS = [(0, 0), (-68, -19), (-180, 57), (3, -2), (-2, 4)]
MODES = [(e, s) for e in ("point_to_plane", "point_to_point") for s in (False, True)]


@pytest.fixture(scope="module")
def data():
    g = np.load(os.path.join(GOLD, "driver_trace.npz"))
    b = np.load(os.path.join(GOLD, "bank_allScales_full.npz"))
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


@pytest.fixture(scope="module")
def icp():
    return lib.NativeIcp(0)


def cuda(a, crop=False):
    """A CUDA tensor holding numpy depth a (uint16 or float32); crop: a view into a larger tensor whose row pitch is no
    multiple of 16 bytes."""
    a = np.ascontiguousarray(a)
    src = torch.from_numpy(a.view(np.int16) if a.dtype == np.uint16 else a).cuda()
    if a.dtype == np.uint16:
        src = src.view(torch.uint16)
    if not crop:
        return src
    H, W = a.shape
    big = torch.zeros((H + 3, W + 5), dtype=src.dtype, device=src.device)
    view = big[1:H + 1, 2:W + 2]
    view.copy_(src)
    return view


def to_mm(d, scale):
    """lm_depth_mm: one float32 product, truncated into [0, 65536), else 0."""
    v = np.asarray(d, np.float32) * np.float32(scale)
    ok = (v >= 0) & (v < 65536)
    return np.where(ok, np.trunc(np.where(ok, v, 0)), 0).astype(np.uint16)


def set_mode(icp, mode):
    icp.set_estimation(mode[0])
    icp.set_use_scene_cloud(mode[1])


def bits(out):
    return tuple(np.ascontiguousarray(a).tobytes() for a in out)


def compare(icp, mode, scene, renders, K, Ks, Rs, ts, xy, scene_t=None, renders_t=None, depth_scale=1.0, render_scale=1.0,
            stream=None, it=30):
    """Host path on the u16 scene / renders against the device path on the tensors (default: their u16 copies)."""
    set_mode(icp, mode)
    n = len(renders)
    want = icp.process_batch(scene, renders, K, Ks, Rs, ts, xy, it)
    scene_t = cuda(scene) if scene_t is None else scene_t
    renders_t = [cuda(r) for r in renders] if renders_t is None else renders_t
    dev = lib.DeviceDepths(scene_t, renders_t, depth_scale, render_scale, stream, 0)
    got = icp.process_batch_device(dev, K, Ks, Rs, ts, xy, it)
    assert bits(got) == bits(want), (mode, np.asarray(got[2][:8]), np.asarray(want[2][:8]), n)
    return want


def rep(a, n):
    return np.repeat(np.asarray(a, np.float32)[None], n, 0)


@pytest.mark.parametrize("mode", MODES)
def test_icp_clouds_cases(icp, mode):
    for c in icp_clouds.all_cases():
        compare(icp, mode, c.scene, [c.model], c.K, c.K[None], c.R[None], c.t.reshape(1, 3), [c.xy])


def survivors(data, thr, top_k):
    nat = lib.NativeDetector(data["T"], 0)
    nat.load_bank(data["packed"], 4)
    nat.select(None, 0, 1)
    g = data["g"]
    nat.upload_images(g["rgb"], g["depth"], None)
    nat.enqueue(thr)
    nat.enqueue_post(0.5, top_k)
    return nat.complete_post()[0]


@pytest.mark.parametrize("mode", MODES)
def test_driver_frame(data, icp, mode):
    g = data["g"]
    # the three recorded refinements of the driver
    rf = ["rf%d_" % k for k in range(3)]
    want = compare(icp, mode, g["depth"], [g[p + "modelDepth"] for p in rf], g["rf0_sceneK"].astype(np.float32),
                   np.stack([g[p + "modelK"] for p in rf]).astype(np.float32), np.stack([g[p + "modelR"] for p in rf]).astype(np.float32),
                   np.stack([g[p + "modelT"].reshape(3) for p in rf]).astype(np.float32), [g[p + "xy"] for p in rf])
    assert (want[2] != -1).all()
    # every box-NMS survivor at 75 and 65 with the shifted renders (a handful of tensors, shared)
    shared = [cuda(r) for r in data["renders"]]
    for thr in (75.0, 65.0):
        surv = survivors(data, thr, 0)
        tid = surv["template_id"].astype(np.int64)
        which = data["which"][tid]
        want = compare(icp, mode, g["depth"], [data["renders"][k] for k in which], data["sK"], data["K"][tid], data["R"][tid],
                       data["t"][tid], np.stack([surv["x"], surv["y"]], 1), renders_t=[shared[k] for k in which])
        assert len(surv) >= 3 and (want[2] != -1).any()


def blob(shape, seed=0):
    """A curved blob of depth (mm) filling the middle of an image of `shape`."""
    H, W = shape
    yy, xx = np.mgrid[0:H, 0:W].astype(np.float64)
    rng = np.random.default_rng(seed)
    cy, cx = H / 2 + rng.uniform(-2, 2), W / 2 + rng.uniform(-2, 2)
    r2 = ((yy - cy) / (0.35 * H)) ** 2 + ((xx - cx) / (0.35 * W)) ** 2
    return np.where(r2 < 1, 900 + 30 * r2 + 4 * np.sin(xx / 5.0), 0).astype(np.uint16)


@pytest.mark.parametrize("mode", MODES)
def test_edges(data, icp, mode):
    g = data["g"]
    scene, sK = g["depth"], data["sK"]
    S_H, S_W = scene.shape
    r0 = g["render"]
    bw, bh = 353 + 4 - 292 + 1, 269 + 4 - 221 + 1           # the recorded render's box (296..353 x 225..269, grown by 4)
    tl = np.zeros_like(r0)
    tl[0:30, 0:40] = scene[200:230, 300:340]                  # box clipped at the top and left edges
    br = np.zeros_like(r0)
    br[-30:, -40:] = scene[200:230, 300:340]                  # clipped at the bottom and right edges
    empty = np.zeros_like(r0)
    off = data["renders"][2]                                  # render[240, 320] == 0: a zero anchor
    assert off[240, 320] == 0
    cases = [(r0, (S_W - 1 - bw, 200)), (r0, (S_W - bw, 200)), (r0, (300, S_H - 1 - bh)), (r0, (300, S_H - bh)),
             (r0, (-5, -7)), (r0, (-100, 10)), (r0, (20, -300)), (tl, (10, 10)), (tl, (S_W - 40, 5)), (br, (0, 0)), (br, (5, 3)),
             (empty, (100, 100)), (empty, (S_W, 0)), (off, (300, 150)), (off, (273, 153))]
    renders = [c[0] for c in cases]
    xy = np.array([c[1] for c in cases], np.int32)
    n = len(cases)
    want = compare(icp, mode, scene, renders, sK, rep(g["rf0_modelK"], n), rep(g["rf0_modelR"], n), rep(g["rf0_modelT"].reshape(3), n), xy)
    early = want[2] == -1
    assert early[1] and early[3] and not early[0] and not early[2] and early[12] and not early[11]
    assert np.isnan(want[1][11]).all() and np.isnan(want[1][13]).any()   # empty render, zero anchor: NaN like the host
    # odd and non-multiple-of-32 render sizes, and renders larger than the scene
    for shape in ((37, 53), (101, 77), (480, 641)):
        r = blob(shape, shape[0])
        K = np.array([[500, 0, shape[1] / 2], [0, 500, shape[0] / 2], [0, 0, 1]], np.float32)
        xy = np.array([[200, 150], [0, 0], [S_W - 60, S_H - 40], [-3, 400]], np.int32)
        compare(icp, mode, scene, [r] * 4, sK, rep(K, 4), rep(np.eye(3), 4), rep([0, 0, 900], 4), xy)
    small = np.ascontiguousarray(scene[150:390, 200:520])     # 240 x 320 scene, 480 x 640 renders
    compare(icp, mode, small, [r0, data["renders"][3]], sK, rep(g["rf0_modelK"], 2), rep(g["rf0_modelR"], 2),
            rep(g["rf0_modelT"].reshape(3), 2), [[60, 80], [200, 150]], scene_t=cuda(small, True))


def driver_batch(data, n, seed=1):
    g = data["g"]
    rng = np.random.default_rng(seed)
    k = rng.integers(0, len(data["renders"]), n)
    xy = np.stack([rng.integers(-20, 640, n), rng.integers(-20, 480, n)], 1).astype(np.int32)
    near = max(1, n // 2)                                     # these lie where the scene has the object
    xy[:near] = np.array(g["rf0_xy"]) + rng.integers(-6, 7, (near, 2))
    return k, xy


@pytest.mark.parametrize("mode", MODES)
def test_layouts_and_float_depth(data, icp, mode):
    g = data["g"]
    k, xy = driver_batch(data, 12)
    renders = [data["renders"][i] for i in k]
    args = (data["sK"], data["K"][:12], data["R"][:12], data["t"][:12], xy)
    want = compare(icp, mode, g["depth"], renders, *args, scene_t=cuda(g["depth"], True), renders_t=[cuda(r, True) for r in renders])
    stack = torch.stack([cuda(r) for r in renders])
    set_mode(icp, mode)
    got = icp.process_batch_device(lib.DeviceDepths(cuda(g["depth"]), stack, 1.0, 1.0, None, 0), *args)
    assert bits(got) == bits(want)                            # one [n, H, W] tensor == a list of tensors
    one = cuda(data["renders"][0])
    compare(icp, mode, g["depth"], [data["renders"][0]] * 12, *args, renders_t=[one] * 12)
    # float32 planes: fractions, negatives, NaN, infinities and products >= 65536 convert as lm_depth_mm does
    rng = np.random.default_rng(5)
    sf = g["depth"].astype(np.float32) * np.float32(10.0) + rng.uniform(0, 9.99, g["depth"].shape).astype(np.float32)
    for val in (np.nan, -7.0, np.inf, -np.inf, 1e6, 655360.0):
        idx = rng.integers(0, sf.size, 400)
        sf.reshape(-1)[idx] = val
    rf = [r.astype(np.float32) * np.float32(2.0) + np.float32(0.75) for r in renders]
    for i, r in enumerate(rf):
        r[r > 1] -= rng.uniform(0, 1.5, int((r > 1).sum())).astype(np.float32)
        r[240 + i, 290:300] = [np.nan, -1.0, np.inf, 131072.0, 131071.9, -np.inf, 1.5, 0.5, -0.0, np.nan]
    compare(icp, mode, to_mm(sf, 0.1), [to_mm(r, 0.5) for r in rf], *args, scene_t=cuda(sf, True), renders_t=[cuda(r) for r in rf],
            depth_scale=0.1, render_scale=0.5)


@pytest.mark.parametrize("mode", MODES)
def test_batch_sizes_and_launches(data, icp, mode):
    g = data["g"]
    set_mode(icp, mode)
    zero = icp.process_batch_device(lib.DeviceDepths(cuda(g["depth"]), [], 1.0, 1.0, None, 0), data["sK"], np.zeros((0, 3, 3)),
                                    np.zeros((0, 3, 3)), np.zeros((0, 3)), np.zeros((0, 2)))
    assert [a.shape for a in zero] == [(0, 3, 3), (0, 3), (0,)]
    shared = [cuda(r) for r in data["renders"]]
    per_chunk = 5 if mode[0] == "point_to_plane" else 4
    for n in (1, 50, 1025):
        k, xy = driver_batch(data, n, n)
        sel = np.arange(n) % data["G"]
        args = (data["sK"], data["K"][sel], data["R"][sel], data["t"][sel], xy)
        want = compare(icp, mode, g["depth"], [data["renders"][i] for i in k], *args, renders_t=[shared[i] for i in k])
        assert (want[2] != -1).any() and (n == 1 or (want[2] == -1).any())
        before = icp.launch_count()
        icp.process_batch_device(lib.DeviceDepths(cuda(g["depth"]), [shared[i] for i in k], 1.0, 1.0, None, 0), *args)
        assert icp.launch_count() - before == 3 + per_chunk * ((n + 1023) // 1024), n


def test_ordering_across_streams(data, icp):
    """A scene written on a side stream and refined on it, with no host synchronise in between, in two phases run once
    each.  1. The side stream is held back (a sleep kernel before its write of scene A): the reads must wait for the write
    (the first event); without it they would see the zero-filled buffer.  2. Right after the call the side stream
    overwrites the buffer with scene B: the call has read A (its outputs are A's), and the next call on the side stream
    reads B."""
    g = data["g"]
    set_mode(icp, MODES[0])
    a, b = g["depth"], np.ascontiguousarray(np.roll(g["depth"], (3, -5), (0, 1)))
    renders = [g["rf%d_modelDepth" % k] for k in range(3)]
    args = (data["sK"], rep(g["rf0_modelK"], 3), np.stack([g["rf%d_modelR" % k] for k in range(3)]).astype(np.float32),
            np.stack([g["rf%d_modelT" % k].reshape(3) for k in range(3)]).astype(np.float32), [g["rf%d_xy" % k] for k in range(3)])
    want_a, want_b = bits(icp.process_batch(a, renders, *args)), bits(icp.process_batch(b, renders, *args))
    want_0 = bits(icp.process_batch(np.zeros_like(a), renders, *args))
    assert want_a != want_b and want_a != want_0
    ta, tb, rt = cuda(a), cuda(b), [cuda(r) for r in renders]
    buf = torch.zeros_like(ta)
    side = torch.cuda.Stream()
    run = lambda: bits(icp.process_batch_device(lib.DeviceDepths(buf, rt, 1.0, 1.0, side, 0), *args))
    # every kernel launched once first: a first launch may synchronise the device, which would order the streams by itself
    with torch.cuda.stream(side):
        buf.copy_(ta)
    assert run() == want_a
    torch.cuda._sleep(1)
    torch.cuda.synchronize()
    buf.zero_()
    torch.cuda.synchronize()
    # phase 1: the write is late
    with torch.cuda.stream(side):
        torch.cuda._sleep(100_000_000)
        buf.copy_(ta)
    assert run() == want_a
    # phase 2: the next write follows the call at once
    with torch.cuda.stream(side):
        buf.copy_(tb)
    assert run() == want_b
    torch.cuda.synchronize()


@pytest.mark.parametrize("estimation", ["point_to_plane", "point_to_point"])
@pytest.mark.parametrize("use_scene", [False, True])
def test_pose_refine_surface_takes_tensors(data, estimation, use_scene):
    g = data["g"]
    native = pr._native(pr._default_device())
    native.set_use_scene_cloud(use_scene)
    try:
        K = g["rf0_sceneK"].astype(np.float32)
        host, dev = pr.poseRefine(estimation), pr.poseRefine(estimation)
        scene_t = cuda(g["depth"], True)
        for k in range(3):
            p = "rf%d_" % k
            a = (K, g[p + "modelK"], g[p + "modelR"], g[p + "modelT"], int(g[p + "xy"][0]), int(g[p + "xy"][1]))
            host.process(g["depth"], g[p + "modelDepth"], *a)
            dev.process(scene_t, cuda(g[p + "modelDepth"]), *a)
            assert dev.getResidual() == host.getResidual() != -1
            assert dev.getR().tobytes() == host.getR().tobytes() and dev.getT().tobytes() == host.getT().tobytes()
        # an early return keeps the previous pose
        host.process(g["depth"], g["render"], K, K, np.eye(3, dtype=np.float32), np.zeros(3, np.float32), 639, 0)
        dev.process(scene_t, cuda(g["render"]).float(), K, K, np.eye(3, dtype=np.float32), np.zeros(3, np.float32), 639, 0)
        assert dev.getResidual() == host.getResidual() == -1 and dev.getR().tobytes() == host.getR().tobytes()
        # refine_matches: numpy against one [n, H, W] tensor, and float32 depth with its scale
        surv = survivors(data, 70.0, 0)
        tid = surv["template_id"].astype(np.int64)
        ms = [type("Match", (), dict(x=int(m["x"]), y=int(m["y"])))() for m in surv]
        renders = [data["renders"][i] for i in data["which"][tid]]
        args = (data["K"][tid], data["R"][tid], data["t"][tid])
        want = pr.refine_matches(g["depth"], data["sK"], ms, renders, *args, estimation=estimation)
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())           # the tensors were made on the current stream
        got = pr.refine_matches(cuda(g["depth"]).float() * 4.0, data["sK"], ms, torch.stack([cuda(r) for r in renders]), *args,
                                estimation=estimation, depth_scale=0.25, stream=side)
        flat = lambda ps: [(p.getResidual(), None if p.getR() is None else (p.getR().tobytes(), p.getT().tobytes())) for p in ps]
        assert flat(got) == flat(want) and len(want) > 3
    finally:
        native.set_use_scene_cloud(False)


def test_device_call_captures_what_a_host_call_captures(data, icp):
    """Capture keeps every item of a device call (point-to-plane), each bitwise the host-buffer call's on the same input."""
    g = data["g"]
    set_mode(icp, MODES[0])
    args = (data["sK"], data["K"][:1], data["R"][:1], data["t"][:1], [[300, 200]])
    icp.set_capture(True)
    try:
        icp.process_batch(g["depth"], [g["render"]], *args)
        want = icp.capture(0)
        icp.process_batch_device(lib.DeviceDepths(cuda(g["depth"]), [cuda(g["render"])], 1.0, 1.0, None, 0), *args)
        buf = np.zeros(1 << 20, np.uint8)
        L = lib.load()
        for what in ("counts", "source", "target", "normals", "init", "result", "knn", "corr_first", "corr_last"):
            assert L.lm_icp_capture(icp._h, 0, lib.CAPTURE_ITEMS[what], buf.ctypes.data, buf.nbytes) == lib.LM_OK, what
        got = icp.capture(0)
        for what in ("source", "target", "normals", "init", "T", "knn", "corr_first", "corr_last"):
            assert got[what] is not None and got[what].tobytes() == want[what].tobytes(), what
        assert (got["fitness"], got["rmse"], got["iterations"]) == (want["fitness"], want["rmse"], want["iterations"])
    finally:
        icp.set_capture(False)


def test_argument_refusals(data, icp):
    g = data["g"]
    scene = cuda(g["depth"])
    r = cuda(g["render"])
    args = (data["sK"], data["K"][:1], data["R"][:1], data["t"][:1], [[300, 200]])
    wide = np.zeros((2100, 1100), np.uint16)
    wide[1:2099, 1:1099] = 1000                                # a 1100 x 2100 box: 2^21 pixels or more
    with pytest.raises(RuntimeError, match="too large"):
        icp.process_batch_device(lib.DeviceDepths(scene, [cuda(wide)], 1.0, 1.0, None, 0), *args)
    L = lib.load()
    Ro, to, res = np.zeros(9), np.zeros(3), np.zeros(1, np.float32)
    import ctypes
    f32p, f64p, vp = ctypes.POINTER(ctypes.c_float), ctypes.POINTER(ctypes.c_double), ctypes.c_void_p
    K = np.ascontiguousarray(data["sK"])
    xy = np.int32([300, 200])

    def call(scene_ptr=scene.data_ptr(), pitch=1280, fmt=0, scale=1.0, mfmt=0, mscale=1.0, mptr=r.data_ptr(), mpitch=1280, stream=None):
        return L.lm_icp_process_batch_device(icp._h, 1, scene_ptr, pitch, fmt, ctypes.c_float(scale), 480, 640, (vp * 1)(mptr),
                                             (ctypes.c_int64 * 1)(mpitch), mfmt, ctypes.c_float(mscale), 480, 640,
                                             K.ctypes.data_as(f32p), K.ctypes.data_as(f32p), K.ctypes.data_as(f32p),
                                             K.ctypes.data_as(f32p), xy.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)), 30,
                                             Ro.ctypes.data_as(f64p), to.ctypes.data_as(f64p), res.ctypes.data_as(f32p), stream)
    assert call() == lib.LM_OK
    host = np.zeros(480 * 640, np.uint16)
    for kw in (dict(fmt=2), dict(mfmt=-1), dict(fmt=1, scale=float("nan"), pitch=2560), dict(mfmt=1, mscale=-1.0, mpitch=2560),
               dict(pitch=1278), dict(mpitch=1000), dict(mptr=r.data_ptr() + 1), dict(scene_ptr=host.ctypes.data),
               dict(mptr=host.ctypes.data), dict(fmt=1, pitch=1280)):
        assert call(**kw) == lib.LM_E_INVALID, kw
