"""Arguments of the particle-swarm estimation, checked before any device work: the "pso" estimation string,
Detector.setPoseSearch, the pose_search keyword of poseRefine.process / refine_matches, the C-ABI's refusals on a
host-only handle, and the C declarations against their ctypes bindings."""
import importlib
import math
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
lib = importlib.import_module("6dpose_b200._lib")
pkg = importlib.import_module("6dpose_b200")
pr = importlib.import_module("6dpose_b200.pose_refine")
dist = importlib.import_module("6dpose_b200.dist")

DECLS = {"lm_set_pose_search": 7, "lm_icp_set_pose_search": 7, "lm_pose_search_points": 18}
BAD = [dict(particles=0), dict(particles=257), dict(iterations=-1), dict(iterations=1001), dict(dt_mm=-1.0), dict(dt_mm=math.nan),
       dict(dt_mm=math.inf), dict(dr_deg=45.5), dict(dr_deg=-0.1), dict(clamp_mm=math.nan), dict(clamp_mm=2e6)]


def test_header_and_binding():
    h = open(os.path.join(ROOT, "include", "linemod_b200.h")).read()
    L = lib.load()
    for name, n in DECLS.items():
        decl = re.search(r"int %s\(([^)]*)\);" % name, h)
        assert decl, name
        assert len([p for p in decl.group(1).split(",") if p.strip()]) == n, name
        assert len(getattr(L, name).argtypes) == n, name
        assert name in lib.SYMBOLS
    assert "#define LM_POSE_PSO 3" in h and "#define LM_ICP_CAPTURE_SEARCH 13" in h
    assert lib.ESTIMATIONS["pso"] == 3 and lib.CAPTURE_ITEMS["search"] == 13
    # the earlier names and values stay as they were
    assert lib.ESTIMATIONS["point_to_plane"] == 0 and lib.ESTIMATIONS["point_to_point"] == 1


def test_estimation_strings():
    assert lib.estimation_code("pso") == 3
    for bad in ("PSO", "swarm", 3, None):
        with pytest.raises(ValueError, match="estimation must be one of"):
            lib.estimation_code(bad)
    assert pr.poseRefine("pso").estimation == "pso"


def test_search_options():
    assert lib.pose_search_options() == (64, 40, 40.0, 30.0, 20.0, 0)
    assert lib.pose_search_options(1, 0, 0, 0, 0, 2 ** 64 - 1) == (1, 0, 0.0, 0.0, 0.0, 2 ** 64 - 1)
    assert lib.pose_search_options(np.int32(256), np.int64(1000), np.float32(1e4), 45, 1e6) == (256, 1000, 1e4, 45.0, 1e6, 0)
    for bad in BAD + [dict(seed=-1), dict(seed=2 ** 64)]:
        with pytest.raises(ValueError):
            lib.pose_search_options(**bad)
    for bad in (dict(particles=2.0), dict(iterations=True), dict(dt_mm="1"), dict(seed=1.5)):
        with pytest.raises(TypeError):
            lib.pose_search_options(**bad)


def test_settings_need_no_device():
    det = pkg.Detector()
    assert det._search == (64, 40, 40.0, 30.0, 20.0, 0)
    det.setPoseSearch(particles=8, iterations=3, seed=5)
    assert det._search == (8, 3, 40.0, 30.0, 20.0, 5) and det._native is None
    with pytest.raises(ValueError):
        det.setPoseSearch(particles=0)
    assert det._search == (8, 3, 40.0, 30.0, 20.0, 5)  # a refused setting leaves the last one
    rgb, depth = np.zeros((8, 8, 3), np.uint8), np.zeros((8, 8), np.uint16)
    K = np.eye(3, dtype=np.float32)
    with pytest.raises(ValueError):
        det.match_refine([rgb, depth], 80.0, [], K, estimation="swarm")
    with pytest.raises(ValueError):
        dist.detect_batch_sharded(det, [[rgb, depth]], 80.0, [], K, estimation="swarm")
    assert det._native is None


def test_pose_refine_keywords():
    p = pr.poseRefine("pso")
    K = np.eye(3, dtype=np.float32)
    d = np.zeros((8, 8), np.uint16)
    pr._icp.clear()
    for bad in (dict(particles=0), dict(dr_deg=90.0), dict(unknown=1)):
        with pytest.raises((ValueError, TypeError)):
            p.process(d, d, K, K, K, np.zeros(3, np.float32), 0, 0, pose_search=bad)
        with pytest.raises((ValueError, TypeError)):
            pr.refine_matches(d, K, [], [], [], [], [], estimation="pso", pose_search=bad)
    assert not pr._icp  # refused before any library call


def test_c_abi_refusals_without_a_device():
    L = lib.load()
    nat = lib.NativeDetector([4, 8], device=-1)
    nat.set_pose_estimation("pso")
    nat.set_pose_search(1, 0, 0.0, 0.0, 0.0, 0)
    nat.set_pose_search(256, 1000, 1e4, 45.0, 1e6, 2 ** 64 - 1)
    for bad in BAD:
        args = dict(lib.POSE_SEARCH_DEFAULTS, **bad)
        with pytest.raises(RuntimeError, match="pose search"):
            nat.set_pose_search(**args)
        assert L.lm_icp_set_pose_search(None, *[args[k] for k in lib.POSE_SEARCH_DEFAULTS]) == lib.LM_E_INVALID
    for bad in (2, -1, 4):
        assert L.lm_set_pose_estimation(nat._h, bad) == lib.LM_E_INVALID
    assert L.lm_set_pose_search(None, 64, 40, 40.0, 10.0, 20.0, 0) == lib.LM_E_INVALID
    # lm_pose_search_points checks its arguments before it looks for a device
    pts, scene = np.zeros((2, 3)), np.zeros((4, 4), np.uint16)
    for bad in BAD:
        with pytest.raises(RuntimeError, match="pose search"):
            check_points(L, pts, scene, **{**lib.POSE_SEARCH_DEFAULTS, **bad})
    with pytest.raises(RuntimeError, match="points"):
        check_points(L, np.zeros((0, 3)), scene, **lib.POSE_SEARCH_DEFAULTS)
    with pytest.raises(RuntimeError, match="job"):
        check_points(L, pts, scene, job=1 << 40, **lib.POSE_SEARCH_DEFAULTS)
    with pytest.raises(RuntimeError, match="needs"):
        check_points(L, pts, scene, cap=8, **lib.POSE_SEARCH_DEFAULTS)
    with pytest.raises(TypeError):
        lib.pose_search_points(pts, np.zeros(3), scene.astype(np.int32), np.eye(3))


def check_points(L, pts, scene, job=0, cap=None, **opts):
    """lm_pose_search_points with the raw settings (the Python checks bypassed)."""
    ct = lib.ctypes
    f64p = ct.POINTER(ct.c_double)
    P, I = opts["particles"], opts["iterations"]
    words = np.zeros(max(6 + I + 19 * P, 1), np.int64)
    T = np.zeros(16)
    sK = np.eye(3, dtype=np.float32)
    st = np.zeros(3)
    lib.check(L.lm_pose_search_points(0, pts.ctypes.data_as(f64p), pts.shape[0], st.ctypes.data_as(f64p),
                                      scene.ctypes.data_as(ct.POINTER(ct.c_uint16)), scene.shape[0], scene.shape[1],
                                      sK.ctypes.data_as(ct.POINTER(ct.c_float)), *[opts[k] for k in lib.POSE_SEARCH_DEFAULTS], job,
                                      T.ctypes.data_as(f64p), words.ctypes.data_as(ct.c_void_p), words.nbytes if cap is None else cap))
