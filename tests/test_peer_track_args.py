"""Arguments of tracking over the peer exchange, refused before any device work: the declarations of lm_peer_track_batch /
lm_peer_track_batch_device against their ctypes bindings; every refusal on a host-only handle (device -1), which can never
be connected, so that a call whose arguments are all fine ends at "needs a connected peer exchange"; and
dist.track_batch_sharded's refusals before the native handle exists."""
import ctypes
import importlib
import math
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
lib = importlib.import_module("6dpose_b200._lib")
pkg = importlib.import_module("6dpose_b200")
dist = importlib.import_module("6dpose_b200.dist")
synth = importlib.import_module("6dpose_b200.synth")
pr = importlib.import_module("6dpose_b200.pose_refine")

DECLS = {"lm_peer_track_batch": 16, "lm_peer_track_batch_device": 20}
RENDER = np.zeros((48, 64), np.uint16)
RENDER[10:30, 20:40] = 500
OK = (0, 0, np.eye(4))
UNCONNECTED = "lm_peer_track_batch needs a connected peer exchange"


def test_header_and_binding():
    h = open(os.path.join(ROOT, "include", "linemod_b200.h")).read()
    L = lib.load()
    for name, n in DECLS.items():
        decl = re.search(r"int %s\(([^)]*)\);" % name, h)
        assert decl, name
        assert len([p for p in decl.group(1).split(",") if p.strip()]) == n, name
        assert getattr(L, name).argtypes == getattr(L, name.replace("peer_", "")).argtypes, name
        assert name in lib.SYMBOLS


@pytest.fixture()
def host():
    bank = synth.synth_bank(3, num_features=30, seed=1, variants=2)
    nat = lib.NativeDetector([4, 8], device=-1)
    nat.load_bank(bank.pack(bank.class_ids(), 4), 4)
    G = bank.num_templates(bank.class_ids()[0])
    eye = np.repeat(np.eye(3, dtype=np.float32)[None], G, 0)
    nat.set_template_renders(0, [RENDER] * (G - 1), eye[:G - 1], eye[:G - 1], np.zeros((G - 1, 3), np.float32))  # the last has none
    return nat, G


def call(nat, frames, counts=None, n_frames=None, margin=4, iters=30, shape=RENDER.shape, device=None, estimation="point_to_plane",
         null=None):
    """lm_peer_track_batch (device: (format, scale) of lm_peer_track_batch_device on null-ish planes) with raw arguments;
    frames is one list of objects per frame.  null names an argument passed as NULL."""
    objects = [o for f in frames for o in f]
    arr = lib.NativeDetector.track_objects(objects)
    counts = np.array([len(f) for f in frames] if counts is None else counts, np.int32)
    n_frames = len(frames) if n_frames is None else n_frames
    m = max(len(objects), 1)
    T, R, t = np.zeros((m, 16)), np.zeros((m, 9)), np.zeros((m, 3))
    res, st, box = np.zeros(m, np.float32), np.zeros(m, np.int32), np.zeros((m, 4), np.int32)
    f32p, f64p, i32p = ctypes.POINTER(ctypes.c_float), ctypes.POINTER(ctypes.c_double), ctypes.POINTER(ctypes.c_int32)
    sK = np.repeat(np.eye(3, dtype=np.float32)[None], max(n_frames, 1), 0)
    depth = np.zeros((max(n_frames, 1),) + tuple(shape), np.uint16)
    nat._L.lm_set_pose_estimation(nat._h, lib.estimation_code(estimation))
    args = dict(sK=sK.ctypes.data_as(f32p), objects=ctypes.cast(arr, ctypes.c_void_p), counts=counts.ctypes.data_as(i32p),
                T=T.ctypes.data_as(f64p))
    if null:
        args[null] = None
    tail = (args["sK"], args["objects"], args["counts"], iters, margin, args["T"], R.ctypes.data_as(f64p), t.ctypes.data_as(f64p),
            res.ctypes.data_as(f32p), st.ctypes.data_as(i32p), box.ctypes.data_as(i32p))
    if device is None:
        rc = nat._L.lm_peer_track_batch(nat._h, n_frames, depth.ctypes.data_as(ctypes.POINTER(ctypes.c_uint16)), shape[0], shape[1], *tail)
    else:
        planes = (ctypes.c_void_p * max(n_frames, 1))(*([16] * max(n_frames, 1)))
        rc = nat._L.lm_peer_track_batch_device(nat._h, n_frames, planes, 128, device[0], ctypes.c_float(device[1]), shape[0], shape[1],
                                               *tail, None)
    return rc, nat._L.lm_last_error().decode()


def test_c_abi_refusals(host):
    nat, G = host
    ok = [[OK], [], [OK, OK]]
    for dev in (None, (lib.DEPTH_F32, 1000.0), (lib.DEPTH_U16_MM, 1.0)):
        rc, err = call(nat, ok, device=dev)
        assert rc == lib.LM_E_STATE and UNCONNECTED in err, (dev, err)  # every argument was fine
    assert call(nat, [[], []]) == (lib.LM_E_STATE, UNCONNECTED)  # no objects at all is fine up to the exchange
    assert call(nat, [[], []], null="T") == (lib.LM_E_STATE, UNCONNECTED)  # no outputs are needed without objects
    bad_class, bad_tpl = (1, 0, np.eye(4)), (0, G, np.eye(4))
    cases = [
        (dict(frames=[[OK], [bad_class]]), lib.LM_E_INVALID, "frame 1: object 0: class"),
        (dict(frames=[[OK, OK], [], [OK, (-1, 0, np.eye(4))]]), lib.LM_E_INVALID, "frame 2: object 1: class"),
        (dict(frames=[[bad_tpl]]), lib.LM_E_INVALID, "frame 0: object 0: template"),
        (dict(frames=[[OK], [(0, -1, np.eye(4))]]), lib.LM_E_INVALID, "frame 1: object 0: template"),
        (dict(frames=[[], [OK, (0, 0, np.full((4, 4), np.nan))]]), lib.LM_E_INVALID, "frame 1: object 1: T[0] is not finite"),
        (dict(frames=[[(0, 0, np.diag([1.0, 1.0, math.inf, 1.0]))]]), lib.LM_E_INVALID, "not finite"),
        (dict(frames=[[OK], [(0, G - 1, np.eye(4))]]), lib.LM_E_STATE, "frame 1: object 0: no template render"),
        (dict(frames=ok, margin=-1), lib.LM_E_INVALID, "margin"),
        (dict(frames=ok, iters=-1), lib.LM_E_INVALID, "max_iterations"),
        (dict(frames=ok, n_frames=0), lib.LM_E_INVALID, "n_frames 0 < 1"),
        (dict(frames=[[OK], [OK]], counts=[1, 1025]), lib.LM_E_INVALID, "frame 1: 1025 objects"),
        (dict(frames=[[OK], [OK]], counts=[-1, 2]), lib.LM_E_INVALID, "frame 0: -1 objects"),
        (dict(frames=ok, shape=(0, 4)), lib.LM_E_INVALID, "empty"),
        (dict(frames=ok, null="sK"), lib.LM_E_INVALID, "null argument"),
        (dict(frames=ok, null="counts"), lib.LM_E_INVALID, "null argument"),
        (dict(frames=ok, null="objects"), lib.LM_E_INVALID, "null argument"),
        (dict(frames=ok, null="T"), lib.LM_E_INVALID, "null argument"),
        (dict(frames=ok, device=(7, 1.0)), lib.LM_E_INVALID, "format"),
        (dict(frames=ok, device=(lib.DEPTH_F32, 0.0)), lib.LM_E_INVALID, "scale"),
        (dict(frames=ok, device=(lib.DEPTH_F32, math.nan)), lib.LM_E_INVALID, "scale"),
        (dict(frames=ok, estimation="pso"), lib.LM_E_STATE, "LM_POSE_PSO"),
        (dict(frames=ok, estimation="pso", device=(lib.DEPTH_U16_MM, 1.0)), lib.LM_E_STATE, "LM_POSE_PSO"),
    ]
    for kw, code, msg in cases:
        rc, err = call(nat, **kw)
        assert rc == code and msg in err, (kw, rc, err)
    assert nat._L.lm_peer_track_batch(None, 1, None, 1, 1, None, None, None, 0, 0, None, None, None, None, None, None) == lib.LM_E_INVALID
    assert nat._L.lm_peer_track_batch_device(None, 1, None, 0, 0, 1.0, 1, 1, None, None, None, 0, 0, None, None, None, None, None, None,
                                             None) == lib.LM_E_INVALID


def test_native_binding_refusals(host):
    nat, _ = host
    with pytest.raises(ValueError, match="2 frames"):
        nat.peer_track_batch(np.zeros((2, 48, 64), np.uint16), np.zeros((3, 3, 3), np.float32), [[OK], []])
    with pytest.raises(TypeError):
        nat.peer_track_batch(np.zeros((48, 64), np.uint16), np.eye(3, dtype=np.float32), [[OK]])
    with pytest.raises(lib.LinemodLibraryError, match="needs a connected peer exchange"):
        nat.peer_track_batch(np.zeros((2, 48, 64), np.uint16), np.zeros((2, 3, 3), np.float32), [[OK], []])


@pytest.fixture()
def group():
    """A one-rank gloo process group."""
    tdist = pytest.importorskip("torch.distributed")
    import socket
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    tdist.init_process_group("gloo", init_method="tcp://127.0.0.1:%d" % port, rank=0, world_size=1)
    try:
        yield None
    finally:
        tdist.destroy_process_group()


def detector():
    det = pkg.Detector([4, 8])
    det.bank = synth.synth_bank(3, num_features=30, seed=1, variants=2)
    det._bank_dirty = True
    cid = det.bank.class_ids()[0]
    return det, cid, det.bank.num_templates(cid)


def test_track_batch_sharded_refusals_touch_no_device(group):
    det, cid, n = detector()
    K = np.eye(3, dtype=np.float32)
    q = pr.poseRefine()
    q._T = np.eye(4)
    good = (pkg.Match(0, 0, 1.0, cid, 0), q)
    d = RENDER
    with pytest.raises(RuntimeError, match="track_batch_sharded\\(\\) needs a detector connected to the peer exchange of rank 0 of 1"):
        dist.track_batch_sharded(det, [d], K, [[good]])
    assert det._native is None
    det._peers = (0, 1)  # as dist.connect_peers leaves it: the Python checks that follow come before any native call
    p = pr.poseRefine()
    p._R, p._t = np.eye(3), np.zeros((3, 1))
    cases = [
        (TypeError, "frame 1: object 0's poseRefine has no transformation", ([d, d], K, [[good], [(pkg.Match(0, 0, 1.0, cid, 0), p)]]), {}),
        (ValueError, "frame 0: object 0: class 'nope' is not in the bank",
         ([d], K, [[dict(class_id="nope", template_id=0, R=np.eye(3), t=np.zeros(3))]]), {}),
        (ValueError, "frame 2: object 1: template", ([d, d, d], K, [[], [good], [good, (pkg.Match(0, 0, 1.0, cid, n), q)]]), {}),
        (ValueError, "frame 1: 1025 objects", ([d, d], K, [[good], [good] * 1025]), {}),
        (ValueError, "track_batch_sharded: no frames", ([], K, []), {}),
        (ValueError, "2 object lists for 3 frames", ([d, d, d], K, [[good], [good]]), {}),
        (ValueError, "sceneK", ([d, d], np.zeros((3, 3, 3), np.float32), [[good], [good]]), {}),
        (ValueError, "depths\\[1\\] is", ([d, d[:, :10]], K, [[good], [good]]), {}),
        (TypeError, "depths\\[0\\] must be a uint16", ([d.astype(np.float32)], K, [[good]]), {}),
        (ValueError, "estimation", ([d], K, [[good]]), dict(estimation="swarm")),
        (TypeError, "stream", ([d], K, [[good]]), dict(stream=object())),
        (ValueError, "depth_scale", ([d], K, [[good]]), dict(depth_scale=1000.0)),
    ]
    for exc, msg, args, kw in cases:
        with pytest.raises(exc, match=msg):
            dist.track_batch_sharded(det, *args, **kw)
    assert det._native is None
