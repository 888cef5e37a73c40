"""The point-to-point estimation (TransformationEstimationPointToPoint, Eigen's umeyama without scaling) without a device:
the oracle's Umeyama and ICP loop, the header's declarations, and the Python surface's argument check."""
import importlib
import os

import numpy as np
import pytest
from scipy.spatial.transform import Rotation

import icp_p2p_oracle as p2p
from oracle import icp_oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def rigid(seed):
    rng = np.random.default_rng(seed)
    return Rotation.random(random_state=seed).as_matrix(), rng.normal(size=3) * 0.05


@pytest.mark.parametrize("seed", range(8))
def test_umeyama_recovers_rigid_transforms(seed):
    rng = np.random.default_rng(100 + seed)
    p = rng.normal(size=(int(rng.integers(3, 400)), 3)) * 0.05 + [0.0, 0.0, 1.0]  # a cloud about 1 m away
    R, t = rigid(seed)
    T = p2p.umeyama(p, p @ R.T + t)
    assert np.abs(T[:3, :3] - R).max() <= 1e-12 and np.abs(T[:3, 3] - t).max() <= 1e-12
    assert np.array_equal(T[3], [0, 0, 0, 1])


@pytest.mark.parametrize("seed", range(6))
def test_umeyama_agrees_with_scipy_align_vectors(seed):
    rng = np.random.default_rng(seed)
    p = rng.normal(size=(60, 3)) * [0.06, 0.04, 0.02]
    R, t = rigid(seed)
    q = p @ R.T + t + rng.normal(size=p.shape) * 1e-3  # noisy: the least-squares rotation
    T = p2p.umeyama(p, q)
    want, _ = Rotation.align_vectors(q - q.mean(0), p - p.mean(0))
    assert np.abs(T[:3, :3] - want.as_matrix()).max() <= 1e-9
    assert np.abs(T[:3, 3] - (q.mean(0) - T[:3, :3] @ p.mean(0))).max() <= 1e-12


def test_umeyama_reflection_rule_gives_a_proper_rotation():
    rng = np.random.default_rng(3)
    p = rng.normal(size=(40, 3)) * [0.05, 0.03, 0.01]
    q = p * [1.0, 1.0, -1.0]  # a mirror image: the best orthogonal fit is the reflection, det -1
    U, _, Vt = np.linalg.svd((q - q.mean(0)).T @ (p - p.mean(0)))
    assert np.linalg.det(U) * np.linalg.det(Vt) < 0  # the rule fires
    R = p2p.umeyama(p, q)[:3, :3]
    assert abs(np.linalg.det(R) - 1.0) <= 1e-12 and np.abs(R @ R.T - np.eye(3)).max() <= 1e-12


def test_umeyama_empty_and_one_pair():
    assert np.array_equal(p2p.umeyama(np.zeros((0, 3)), np.zeros((0, 3))), np.eye(4))
    p, q = np.array([[0.01, -0.02, 0.9]]), np.array([[0.015, -0.01, 0.93]])
    T = p2p.umeyama(p, q)
    assert np.array_equal(T[:3, :3], np.eye(3)) and np.allclose(T[:3, 3], (q - p)[0], rtol=0, atol=1e-15)


def blob(n=900, z=0.9):
    rng = np.random.default_rng(1)
    xy = rng.uniform(-0.04, 0.04, (n, 2))
    zz = z + 0.02 * np.sin(xy[:, 0] / 0.013) * np.cos(xy[:, 1] / 0.017) + 0.3 * (xy ** 2).sum(1)
    return icp_oracle.voxel_down_sample(np.concatenate([xy, zz[:, None]], 1))


@pytest.mark.parametrize("target", ["model", "scene"])
def test_oracle_point_to_point_icp_converges(target):
    src = blob()
    R, _ = rigid(4)
    R = Rotation.from_rotvec(Rotation.from_matrix(R).as_rotvec() * 0.03).as_matrix()  # about 1.5 degrees
    t = np.array([0.002, -0.0015, 0.001])
    if target == "model":  # the reference's target: the source cloud itself, from a perturbed start
        tgt, init = src, np.eye(4)
        init[:3, :3], init[:3, 3] = R, t
        want = np.eye(4)
    else:                  # a scene cloud moved by (R, t), from the identity
        c = src.mean(0)
        tgt, init = (src - c) @ R.T + c + t, np.eye(4)
        want = np.eye(4)
        want[:3, :3], want[:3, 3] = R, c + t - R @ c
    T, fit, rmse, it = p2p.registration_icp_p2p(src, tgt, icp_oracle.MAX_DIST, init, max_iter=200)
    assert 1 <= it < 200 and fit == 1.0 and rmse <= 1e-6, (it, fit, rmse)
    assert np.abs(T - want).max() <= 1e-6, T


def test_header_declares_the_estimation_api():
    with open(os.path.join(ROOT, "include", "linemod_b200.h")) as f:
        h = f.read()
    for decl in ("#define LM_ICP_POINT_TO_PLANE 0", "#define LM_ICP_POINT_TO_POINT 1",
                 "int lm_icp_set_estimation(lm_icp* h, int estimation);", "int lm_set_pose_estimation(lm_detector* d, int estimation);"):
        assert decl in h, decl
    lib = importlib.import_module("6dpose_b200._lib")
    assert "lm_icp_set_estimation" in lib.SYMBOLS and "lm_set_pose_estimation" in lib.SYMBOLS


def test_unknown_estimation_raises_before_any_device_work():
    pkg = importlib.import_module("6dpose_b200")
    lib = importlib.import_module("6dpose_b200._lib")
    pr = importlib.import_module("6dpose_b200.pose_refine")
    dist = importlib.import_module("6dpose_b200.dist")
    assert lib.estimation_code("point_to_plane") == 0 and lib.estimation_code("point_to_point") == 1
    for bad in ("point_to_planes", "P2P", None, 1):
        with pytest.raises(ValueError):
            lib.estimation_code(bad)
    with pytest.raises(ValueError):
        pr.poseRefine(estimation="plane")
    assert pr.poseRefine().estimation == "point_to_plane"
    with pytest.raises(ValueError):
        pr.refine_matches(np.zeros((4, 4), np.uint16), np.eye(3, dtype=np.float32), [object()], [], [], [], [], estimation="x")
    det = pkg.Detector()
    rgb, depth = np.zeros((8, 8, 3), np.uint8), np.zeros((8, 8), np.uint16)
    K = np.eye(3, dtype=np.float32)
    with pytest.raises(ValueError):
        det.match_refine([rgb, depth], 80.0, [], K, estimation="x")
    with pytest.raises(ValueError):
        det.detect([rgb, depth], 80.0, [], K, estimation="x")
    with pytest.raises(ValueError):
        det.match_refine_batch([[rgb, depth]], 80.0, [], K, estimation="x")
    with pytest.raises(ValueError):
        det.detect_batch([[rgb, depth]], 80.0, [], K, estimation="x")
    with pytest.raises(ValueError):
        dist.match_refine_batch_sharded(det, [[rgb, depth]], 80.0, [], K, estimation="x")
    with pytest.raises(ValueError):
        dist.detect_batch_sharded(det, [[rgb, depth]], 80.0, [], K, estimation="x")
    assert det._native is None  # nothing reached the device
