"""Arguments of the pose verification, checked before any device work: Detector.setPoseVerification, the verify_mm
keyword of poseRefine.process / refine_matches, the C-ABI's refusals on a host-only handle, and the C declarations
against their ctypes bindings."""
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

DECLS = {"lm_set_pose_verify": 5, "lm_pose_verify": 5, "lm_pose_verify_points": 11, "lm_icp_set_verify": 3, "lm_icp_verify": 5}


def test_header_and_binding():
    h = open(os.path.join(ROOT, "include", "linemod_b200.h")).read()
    L = lib.load()
    for name, n in DECLS.items():
        decl = re.search(r"int %s\(([^)]*)\);" % name, h)
        assert decl, name
        assert len([p for p in decl.group(1).split(",") if p.strip()]) == n, name
        assert len(getattr(L, name).argtypes) == n, name
        assert name in lib.SYMBOLS
    assert re.search(r"#define LM_VERIFY_RANK_FITNESS 0", h) and re.search(r"#define LM_VERIFY_RANK_SCORE 1", h)
    assert lib.VERIFY_RANKS == {"fitness": 0, "score": 1}


def test_verify_options():
    assert lib.verify_options(None) == (0, 10.0, 0, -math.inf)
    assert lib.verify_options(10.0) == (1, 10.0, 0, -math.inf)
    assert lib.verify_options(0, "score", 0.5) == (1, 0.0, 1, 0.5)
    assert lib.verify_options(np.float32(2.5), min_score=-1) == (1, 2.5, 0, -1.0)
    for bad in (math.nan, -1.0, math.inf, -0.5):
        with pytest.raises(ValueError):
            lib.verify_options(bad)
    for bad in ("10", True, None.__class__):
        with pytest.raises(TypeError):
            lib.verify_options(bad)
    with pytest.raises(ValueError, match="rank_by"):
        lib.verify_options(10.0, "residual")
    with pytest.raises(ValueError, match="NaN"):
        lib.verify_options(10.0, min_score=math.nan)
    with pytest.raises(TypeError):
        lib.verify_options(10.0, min_score="0.5")
    with pytest.raises(ValueError, match="need pose verification"):
        lib.verify_options(None, "score")
    with pytest.raises(ValueError, match="need pose verification"):
        lib.verify_options(None, min_score=0.5)


def test_detector_setting_needs_no_device():
    det = pkg.Detector()
    assert det._verify[0] == 0
    det.setPoseVerification(5.0, "score", 0.25)
    assert det._verify == (1, 5.0, 1, 0.25) and det._native is None
    with pytest.raises(ValueError):
        det.setPoseVerification(-1.0)
    assert det._verify == (1, 5.0, 1, 0.25)  # a refused setting leaves the last one
    det.setPoseVerification(None)
    assert det._verify[0] == 0


def test_pose_refine_surface():
    p = pr.poseRefine()
    assert p.getScore() is None and p.getVerification() is None
    K = np.eye(3, dtype=np.float32)
    d = np.zeros((8, 8), np.uint16)
    pr._icp.clear()
    for bad in (math.nan, -1.0):
        with pytest.raises(ValueError):
            p.process(d, d, K, K, K, np.zeros(3, np.float32), 0, 0, verify_mm=bad)
        with pytest.raises(ValueError):
            pr.refine_matches(d, K, [], [], [], [], [], verify_mm=bad)
    assert not pr._icp  # refused before any library call


def test_c_abi_refusals_without_a_device():
    L = lib.load()
    nat = lib.NativeDetector([4, 8], device=-1)
    nat.set_pose_verify(True, 10.0, 1, 0.5)
    nat.set_pose_verify(False)
    for args in ((1, math.nan, 0, -math.inf), (1, -1.0, 0, -math.inf), (1, math.inf, 0, -math.inf), (1, 10.0, 2, -math.inf),
                 (1, 10.0, 0, math.nan), (0, 10.0, 1, -math.inf), (0, 10.0, 0, 0.5)):
        with pytest.raises(RuntimeError):
            nat.set_pose_verify(*args)
    with pytest.raises(lib.LinemodLibraryError, match="error -3"):  # LM_E_STATE: nothing verified yet
        nat.pose_verify()
    assert L.lm_set_pose_verify(None, 1, 10.0, 0, -math.inf) == lib.LM_E_INVALID
    assert L.lm_icp_set_verify(None, 1, 10.0) == lib.LM_E_INVALID
    assert L.lm_icp_verify(None, None, None, 0, None) == lib.LM_E_INVALID
    # lm_pose_verify_points checks its arguments before it looks for a device
    scene = np.zeros((4, 4), np.uint16)
    for delta in (math.nan, -1.0):
        with pytest.raises(RuntimeError, match="inlier"):
            lib.pose_verify_points(np.zeros((1, 3)), np.eye(4), scene, np.eye(3), delta)
    with pytest.raises(TypeError):
        lib.pose_verify_points(np.zeros((1, 3)), np.eye(4), scene.astype(np.int32), np.eye(3))
