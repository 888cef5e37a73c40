"""poseRefine on the GPU (lm_icp_process through the C-ABI) against the ICP oracle.

Tolerance (BASELINE.json north_star): refined poses within 1e-4 relative of the reference -- here
||R - R_ref||_F / ||R_ref||_F and ||t - t_ref|| / ||t_ref||.  Parity of the ICP arithmetic itself is
UNPINNED (Open3D is external to the reference, see oracle/icp_oracle.py)."""
import importlib
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "icp_case1.npz")
TOL = 1e-4


def rel(a, b):
    return float(np.linalg.norm(np.asarray(a, np.float64).ravel() - np.asarray(b, np.float64).ravel()) /
                 max(np.linalg.norm(np.asarray(b, np.float64).ravel()), 1e-300))


@pytest.fixture(scope="module")
def gold():
    return np.load(GOLD)


def test_pose_refine_surface_and_golden(gold):
    mod = importlib.import_module("linemodLevelup_pybind")
    for name in ("shift_0", "shift_1", "shift_2", "shift_3", "scene_a", "scene_b"):
        scene = gold["scene"] if name.startswith("scene") else gold["scene_" + name]
        p = mod.poseRefine()
        assert p.getResidual() == -1 and p.getR() is None
        x, y = [int(v) for v in gold["xy_" + name]]
        p.process(scene, gold["model"], gold["K"], gold["K"], gold["R"], gold["t"].reshape(3, 1), x, y)
        assert p.getR().shape == (3, 3) and p.getR().dtype == np.float64
        assert p.getT().shape == (3, 1) and p.getT().dtype == np.float64
        assert rel(p.getR(), gold["R_" + name]) <= TOL, name
        assert rel(p.getT(), gold["t_" + name]) <= TOL, name
        assert abs(p.getResidual() - float(gold["res_" + name])) <= 1e-6, name
    # early return when the model box does not fit at the match position (LL.cpp:52-55)
    p = mod.poseRefine()
    x, y = [int(v) for v in gold["xy_scene_edge"]]
    p.process(gold["scene"], gold["model"], gold["K"], gold["K"], gold["R"], gold["t"], x, y)
    assert p.getResidual() == -1 and p.getR() is None and p.getT() is None
    with pytest.raises(TypeError):
        p.process(gold["scene"].astype(np.float32), gold["model"], gold["K"], gold["K"], gold["R"], gold["t"], 0, 0)


def blob_depth(rng, H=240, W=320, cx=160, cy=120, r=45, z0=900.0):
    yy, xx = np.mgrid[0:H, 0:W]
    d2 = ((xx - cx) / r) ** 2 + ((yy - cy) / (0.8 * r)) ** 2
    bump = 60.0 * np.sqrt(np.clip(1 - d2, 0, None)) + 6 * np.sin(xx / 7.0) * np.cos(yy / 9.0)
    depth = np.where(d2 < 1, z0 - bump, 0)
    return depth.astype(np.uint16)


@pytest.mark.parametrize("use_scene", [False, True])
def test_icp_against_oracle_on_perturbed_blobs(use_scene):
    from oracle import icp_oracle
    lib = importlib.import_module("6dpose_b200._lib")
    icp = lib.NativeIcp()
    icp.set_use_scene_cloud(use_scene)
    K = np.array([[570, 0, 160], [0, 570, 120], [0, 0, 1]], np.float32)
    rng = np.random.default_rng(0)
    model = blob_depth(rng)
    ys, xs = np.nonzero(model)
    worst = 0.0
    for seed in range(6):
        rng = np.random.default_rng(seed)
        sx, sy, dz = int(rng.integers(-2, 3)), int(rng.integers(-2, 3)), int(rng.integers(-7, 8))
        scene = np.roll(np.roll(model, sy, 0), sx, 1).astype(np.int32)
        scene = np.where(scene > 0, scene + dz + rng.integers(-1, 2, scene.shape), 0).astype(np.uint16)
        ang = rng.uniform(-0.5, 0.5, 3)
        Rm = (icp_oracle.vec6_to_mat4(np.concatenate([ang, [0, 0, 0]]))[:3, :3]).astype(np.float32)
        t = np.array([rng.uniform(-30, 30), rng.uniform(-30, 30), 900.0], np.float32)
        xy = [int(xs.min()), int(ys.min())]
        want = icp_oracle.pose_refine(scene, model, K, K, Rm, t, xy[0], xy[1], use_scene_cloud=use_scene)
        Ro, to, res = icp.process_batch(scene, [model], K, K[None], Rm[None], t[None], [xy])
        st = icp.last_stats()
        assert st["points"] == want["n_points"]
        assert st["iterations"] == want["iterations"], (seed, st, want["iterations"])
        assert abs(float(res[0]) - want["residual"]) <= 1e-6
        # the KD-tree and the kernel's (d^2, index) rule pick different 30th neighbours where neighbours 30 and 31
        # are nearly tied; tests/test_gpu_icp_stages.py checks that those are the only normals that differ, among the
        # normals its model can compare (an eigenvalue gap large enough against the covariance's rounding)
        assert abs(st["rmse"] - want["rmse"]) <= 1e-9 + TOL * want["rmse"]
        worst = max(worst, rel(Ro[0], want["R"]), rel(to[0], want["t"]))
    assert worst <= TOL, worst


def test_icp_batch_equals_single_calls_and_iteration_cap():
    from oracle import icp_oracle
    lib = importlib.import_module("6dpose_b200._lib")
    icp = lib.NativeIcp()
    icp.set_use_scene_cloud(True)
    K = np.array([[570, 0, 160], [0, 570, 120], [0, 0, 1]], np.float32)
    rng = np.random.default_rng(3)
    models = [blob_depth(rng, r=r) for r in (30, 45, 38)]
    scene = np.where(models[1] > 0, models[1] + 5, 0).astype(np.uint16)
    Rs = np.stack([np.eye(3, dtype=np.float32)] * 3)
    ts = np.array([[0, 0, 900]] * 3, np.float32)
    xy = [[int(np.nonzero(m)[1].min()), int(np.nonzero(m)[0].min())] for m in models]
    Rb, tb, rb = icp.process_batch(scene, models, K, np.stack([K] * 3), Rs, ts, xy, max_iterations=10)
    for i in range(3):
        R1, t1, r1 = icp.process_batch(scene, [models[i]], K, K[None], Rs[i:i + 1], ts[i:i + 1], [xy[i]], max_iterations=10)
        assert np.array_equal(R1[0], Rb[i]) and np.array_equal(t1[0], tb[i]) and r1[0] == rb[i]
        want = icp_oracle.pose_refine(scene, models[i], K, K, Rs[i], ts[i], xy[i][0], xy[i][1], max_iter=10, use_scene_cloud=True)
        assert rel(Rb[i], want["R"]) <= TOL and rel(tb[i], want["t"]) <= TOL
    # max_iterations = 0: no update at all, the initial guess comes back
    R0, t0, r0 = icp.process_batch(scene, [models[1]], K, K[None], Rs[:1], ts[:1], [xy[1]], max_iterations=0)
    want = icp_oracle.pose_refine(scene, models[1], K, K, Rs[0], ts[0], xy[1][0], xy[1][1], max_iter=0, use_scene_cloud=True)
    assert rel(t0[0], want["t"]) <= TOL


def test_refine_matches_batch_equals_single_calls(gold):
    """The NMS-survivor hand-off (SURVEY.md 8f-3): one batched call == the drivers' per-match loop."""
    mod = importlib.import_module("linemodLevelup_pybind")
    pr = importlib.import_module("6dpose_b200.pose_refine")
    det = importlib.import_module("6dpose_b200.detector")
    names = ("scene_a", "scene_b", "scene_edge")
    ms = []
    for nme in names:
        m = det.Match()
        m.x, m.y = [int(v) for v in gold["xy_" + nme]]
        ms.append(m)
    n = len(ms)
    got = pr.refine_matches(gold["scene"], gold["K"], ms, [gold["model"]] * n, [gold["K"]] * n, [gold["R"]] * n,
                            [gold["t"]] * n)
    for m, g in zip(ms, got):
        p = mod.poseRefine()
        p.process(gold["scene"], gold["model"], gold["K"], gold["K"], gold["R"], gold["t"], m.x, m.y)
        assert g.getResidual() == p.getResidual()
        if p.getR() is None:
            assert g.getR() is None and g.getT() is None
        else:
            assert np.array_equal(g.getR(), p.getR()) and np.array_equal(g.getT(), p.getT())
    assert pr.refine_matches(gold["scene"], gold["K"], [], [], [], [], []) == []
