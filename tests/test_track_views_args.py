"""Arguments of view following, refused before any device work: lm_set_track_views, lm_track_templates and
lm_track_views_points on a host-only handle (device -1) or without a device, Detector.setTrackViews's TypeError /
ValueError, and the C declarations against their ctypes bindings."""
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

DECLS = {"lm_set_track_views": 3, "lm_track_templates": 4, "lm_track_views_points": 9}
BAD_TURNS = [math.nan, -1e-300, -1.0, 180.0, 360.0, math.inf, -math.inf]


def test_header_and_binding():
    h = open(os.path.join(ROOT, "include", "linemod_b200.h")).read()
    L = lib.load()
    for name, n in DECLS.items():
        decl = re.search(r"int %s\(([^)]*)\);" % name, h)
        assert decl, name
        assert len([p for p in decl.group(1).split(",") if p.strip()]) == n, name
        assert len(getattr(L, name).argtypes) == n, name
        assert name in lib.SYMBOLS


@pytest.fixture()
def host():
    bank = synth.synth_bank(3, num_features=30, seed=1, variants=2)
    nat = lib.NativeDetector([4, 8], device=-1)
    nat.load_bank(bank.pack(bank.class_ids(), 4), 4)
    return nat, bank


def test_set_track_views(host):
    nat, bank = host
    L = nat._L
    for turn in (0.0, 1e-300, 30.0, 179.99999999999997):
        assert L.lm_set_track_views(nat._h, 1, turn) == lib.LM_OK, turn
    for turn in BAD_TURNS:
        assert L.lm_set_track_views(nat._h, 1, turn) == lib.LM_E_INVALID, turn
        assert "turn_deg" in L.lm_last_error().decode()
        assert L.lm_set_track_views(nat._h, 0, turn) == lib.LM_OK, turn  # off ignores the angle
    assert L.lm_set_track_views(None, 0, 0.0) == lib.LM_E_INVALID
    nat.set_track_views(True, 25.0)
    nat.load_bank(bank.pack(bank.class_ids(), 4), 4)  # another bank keeps it (nothing to observe without a device: no error)


def test_track_templates_before_any_track_run(host):
    nat, _ = host
    L = nat._L
    n = ctypes.c_int64(-5)
    assert L.lm_track_templates(nat._h, None, 0, ctypes.byref(n)) == lib.LM_E_STATE
    assert L.lm_track_templates(nat._h, None, 0, None) == lib.LM_E_INVALID
    assert L.lm_track_templates(None, None, 0, ctypes.byref(n)) == lib.LM_E_INVALID
    G = host[1].num_templates(host[1].class_ids()[0])
    eye = np.repeat(np.eye(3, dtype=np.float32)[None], G, 0)
    render = np.zeros((16, 16), np.uint16)
    render[4:8, 4:8] = 500
    nat.set_template_renders(0, [render] * G, eye, eye, np.zeros((G, 3), np.float32))
    assert L.lm_track_templates(nat._h, None, 0, ctypes.byref(n)) == lib.LM_E_STATE
    assert "no track run" in L.lm_last_error().decode()
    with pytest.raises(RuntimeError):
        nat.track_templates()


def points(n=3, k=0, T=None, turn=30.0, null=None):
    m = min(max(n, 1), 4)  # n beyond the arrays is refused before they are read
    Rb = np.repeat(np.eye(3, dtype=np.float32)[None], m, 0)
    tb = np.zeros((m, 3), np.float32)
    T = np.eye(4) if T is None else np.asarray(T, np.float64)
    out = np.zeros(16)
    ch = ctypes.c_int64()
    f32p, f64p = ctypes.POINTER(ctypes.c_float), ctypes.POINTER(ctypes.c_double)
    args = [0, n, Rb.ctypes.data_as(f32p), tb.ctypes.data_as(f32p), k, T.ctypes.data_as(f64p), turn, ctypes.byref(ch), out.ctypes.data_as(f64p)]
    if null is not None:
        args[null] = None
    L = lib.load()
    return L.lm_track_views_points(*args), L.lm_last_error().decode()


def test_points_refusals():
    for null in (2, 3, 5, 7, 8):
        rc, err = points(null=null)
        assert rc == lib.LM_E_INVALID and "null" in err, null
    cases = [(dict(n=0), "templates"), (dict(n=-1), "templates"), (dict(n=1 << 31), "templates"), (dict(k=3), "outside"),
             (dict(k=-1), "outside"), (dict(T=np.full((4, 4), np.nan)), "not finite"), (dict(T=np.diag([1, 1, math.inf, 1])), "not finite")]
    cases += [(dict(turn=t), "turn_deg") for t in BAD_TURNS]
    for kw, msg in cases:
        rc, err = points(**kw)
        assert rc == lib.LM_E_INVALID and msg in err, (kw, rc, err)
    for kw in (dict(n=3, k=2), dict(turn=0.0)):  # every argument fine: only the device is missing (or the call runs)
        assert points(**kw)[0] in (lib.LM_OK, lib.LM_E_CUDA)
    with pytest.raises(ValueError):
        lib.track_views_points(np.zeros((2, 3, 3)), np.zeros((3, 3)), 0, np.eye(4), 30.0)


def test_detector_set_track_views_touches_no_device():
    det = pkg.Detector([4, 8])
    for turn in (None, 0, 0.0, 45, 179.5, np.float32(10.0), np.int64(3)):
        det.setTrackViews(turn)
    assert det._views == (1, 3.0)
    det.setTrackViews()
    assert det._views == (0, 0.0)
    for bad in (math.nan, -1.0, 180.0, 200, math.inf):
        with pytest.raises(ValueError, match="turn_deg"):
            det.setTrackViews(bad)
    for bad in ("30", True, [30.0], object()):
        with pytest.raises(TypeError, match="turn_deg"):
            det.setTrackViews(bad)
    assert det._views == (0, 0.0)
    assert det._native is None
