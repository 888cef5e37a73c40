"""Arguments of tracking, refused before any device work: Detector.track's TypeError / ValueError, and every refusal of
lm_track / lm_track_device / lm_pose_transforms on a host-only handle (device -1), whose last check is that handle
itself; and the C declarations against their ctypes bindings."""
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
synth = importlib.import_module("6dpose_b200.synth")
pr = importlib.import_module("6dpose_b200.pose_refine")

DECLS = {"lm_track": 15, "lm_track_device": 19, "lm_pose_transforms": 4}
RENDER = np.zeros((48, 64), np.uint16)
RENDER[10:30, 20:40] = 500


def test_header_and_binding():
    h = open(os.path.join(ROOT, "include", "linemod_b200.h")).read()
    L = lib.load()
    for name, n in DECLS.items():
        decl = re.search(r"int %s\(([^)]*)\);" % name, h)
        assert decl, name
        assert len([p for p in decl.group(1).split(",") if p.strip()]) == n, name
        assert len(getattr(L, name).argtypes) == n, name
        assert name in lib.SYMBOLS
    for k, v in enumerate(("TRACKED", "OUTSIDE", "WINDOW", "NO_DEPTH")):
        assert "#define LM_TRACK_%s %d" % (v, k) in h and lib.TRACK_STATUS[k] == v.lower()
    assert "#define LM_POSE_CAPTURE_WINDOW 14" in h and lib.CAPTURE_ITEMS["window"] == 14
    assert ctypes.sizeof(lib.TrackObject) == 136


@pytest.fixture()
def host():
    bank = synth.synth_bank(3, num_features=30, seed=1, variants=2)
    nat = lib.NativeDetector([4, 8], device=-1)
    nat.load_bank(bank.pack(bank.class_ids(), 4), 4)
    G = bank.num_templates(bank.class_ids()[0])
    eye = np.repeat(np.eye(3, dtype=np.float32)[None], G, 0)
    nat.set_template_renders(0, [RENDER] * (G - 1), eye[:G - 1], eye[:G - 1], np.zeros((G - 1, 3), np.float32))  # the last has none
    return nat, G


def call(nat, objects, n=None, margin=4, iters=30, depth=RENDER, device=None, estimation="point_to_plane"):
    """lm_track (device: (format, scale) of lm_track_device on a null plane) with raw arguments."""
    arr = lib.NativeDetector.track_objects(objects)
    n = len(objects) if n is None else n
    m = max(n, 1)
    T, R, t = np.zeros((m, 16)), np.zeros((m, 9)), np.zeros((m, 3))
    res, st, box = np.zeros(m, np.float32), np.zeros(m, np.int32), np.zeros((m, 4), np.int32)
    f32p, f64p, i32p = ctypes.POINTER(ctypes.c_float), ctypes.POINTER(ctypes.c_double), ctypes.POINTER(ctypes.c_int32)
    sK = np.eye(3, dtype=np.float32)
    nat._L.lm_set_pose_estimation(nat._h, lib.estimation_code(estimation))
    tail = (sK.ctypes.data_as(f32p), ctypes.cast(arr, ctypes.c_void_p), n, iters, margin, T.ctypes.data_as(f64p), R.ctypes.data_as(f64p),
            t.ctypes.data_as(f64p), res.ctypes.data_as(f32p), st.ctypes.data_as(i32p), box.ctypes.data_as(i32p))
    if device is None:
        rc = nat._L.lm_track(nat._h, depth.ctypes.data_as(ctypes.POINTER(ctypes.c_uint16)), depth.shape[0], depth.shape[1], *tail)
    else:
        rc = nat._L.lm_track_device(nat._h, ctypes.c_void_p(16), 128, device[0], ctypes.c_float(device[1]), depth.shape[0], depth.shape[1],
                                    *tail, None)
    return rc, nat._L.lm_last_error().decode()


def test_c_abi_refusals(host):
    nat, G = host
    ok = [(0, 0, np.eye(4))]
    assert call(nat, ok)[0] == lib.LM_E_STATE and "host-only" in call(nat, ok)[1]  # every argument was fine
    assert call(nat, ok, device=(lib.DEPTH_F32, 1000.0))[0] == lib.LM_E_STATE
    cases = [
        (dict(objects=[(1, 0, np.eye(4))]), lib.LM_E_INVALID, "class"),
        (dict(objects=[(-1, 0, np.eye(4))]), lib.LM_E_INVALID, "class"),
        (dict(objects=[(0, G, np.eye(4))]), lib.LM_E_INVALID, "template"),
        (dict(objects=[(0, -1, np.eye(4))]), lib.LM_E_INVALID, "template"),
        (dict(objects=ok + [(0, 0, np.full((4, 4), np.nan))]), lib.LM_E_INVALID, "not finite"),
        (dict(objects=[(0, 0, np.diag([1.0, 1.0, math.inf, 1.0]))]), lib.LM_E_INVALID, "not finite"),
        (dict(objects=ok, margin=-1), lib.LM_E_INVALID, "margin"),
        (dict(objects=ok, iters=-1), lib.LM_E_INVALID, "max_iterations"),
        (dict(objects=ok, n=1025), lib.LM_E_INVALID, "1024"),
        (dict(objects=ok, n=-1), lib.LM_E_INVALID, "n < 0"),
        (dict(objects=ok, depth=np.zeros((0, 4), np.uint16)), lib.LM_E_INVALID, "empty"),
        (dict(objects=ok, device=(7, 1.0)), lib.LM_E_INVALID, "format"),
        (dict(objects=ok, device=(lib.DEPTH_F32, 0.0)), lib.LM_E_INVALID, "scale"),
        (dict(objects=ok, device=(lib.DEPTH_F32, math.nan)), lib.LM_E_INVALID, "scale"),
        (dict(objects=ok, estimation="pso"), lib.LM_E_STATE, "LM_POSE_PSO"),
        (dict(objects=[(0, G - 1, np.eye(4))]), lib.LM_E_STATE, "no template render"),
    ]
    for kw, code, msg in cases:
        rc, err = call(nat, **kw)
        assert rc == code and msg in err, (kw, rc, err)
    n = ctypes.c_int64()
    assert nat._L.lm_pose_transforms(nat._h, None, 0, ctypes.byref(n)) == lib.LM_E_STATE
    assert nat._L.lm_pose_transforms(nat._h, None, 0, None) == lib.LM_E_INVALID
    assert nat._L.lm_track(None, None, 1, 1, None, None, 0, 0, 0, None, None, None, None, None, None) == lib.LM_E_INVALID


def test_detector_track_refusals_touch_no_device():
    det = pkg.Detector([4, 8])
    det.bank = synth.synth_bank(3, num_features=30, seed=1, variants=2)
    det._bank_dirty = True
    cid = det.bank.class_ids()[0]
    n = det.bank.num_templates(cid)
    depth = RENDER
    K = np.eye(3, dtype=np.float32)
    p = pr.poseRefine()  # as refine_matches / process leave it: no transformation
    p._R, p._t = np.eye(3), np.zeros((3, 1))
    with pytest.raises(TypeError, match="no transformation"):
        det.track(depth, K, [(pkg.Match(0, 0, 1.0, cid, 0), p)])
    with pytest.raises(ValueError, match="not in the bank"):
        det.track(depth, K, [dict(class_id="nope", template_id=0, R=np.eye(3), t=np.zeros(3))])
    with pytest.raises(ValueError, match="outside class"):
        det.track(depth, K, [dict(class_id=cid, template_id=n, R=np.eye(3), t=np.zeros(3))])
    q = pr.poseRefine()
    q._T = np.eye(4)
    with pytest.raises(ValueError, match="outside class"):
        det.track(depth, K, [(pkg.Match(0, 0, 1.0, cid, -1), q)])
    with pytest.raises(ValueError):
        det.track(depth, K, [(pkg.Match(0, 0, 1.0, cid, 0), q)] * 1025)
    with pytest.raises(ValueError, match="estimation"):
        det.track(depth, K, [], estimation="swarm")
    with pytest.raises(TypeError):
        det.track(depth, K, [(pkg.Match(0, 0, 1.0, cid, 0), p)], stream=object())
    assert det._native is None


def test_accessors_default_to_none():
    p = pr.poseRefine()
    assert p.getTransformation() is None and p.getTrackStatus() is None
