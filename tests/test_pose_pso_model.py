"""The particle-swarm model (tests/pose_pso_model.py) on the CPU: its generator, Rodrigues' formula, T(x), the integer
cost and the swarm's invariants."""
import math

import numpy as np
import pytest
from scipy.spatial.transform import Rotation

import pose_pso_model as pm
from pose_verify_model import SK, _pt

MASK = (1 << 64) - 1


def _splitmix_int(seed, number):
    z = (seed + (number + 1) * pm.GOLDEN) & MASK
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & MASK
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & MASK
    return z ^ (z >> 31)


def test_generator_known_answers():
    # splitmix64 seeded with 0: its published first outputs
    assert [int(pm.splitmix64(0, k)) for k in range(3)] == [0xE220A8397B1DCDAF, 0x6E789E6AA1B965F4, 0x06C45D188009454F]
    for seed in (0, 1, 12345, MASK):
        for number in (0, 1, 2 ** 40 + 7, MASK - 1):
            assert int(pm.splitmix64(seed, number)) == _splitmix_int(seed, number)
    # the draw's counter packs (job, iteration, particle, draw) without overlap
    r = pm.draw(7, 3, 5, 9, 11)
    assert r == (_splitmix_int(7, ((3 * 1024 + 5) * 1024 + 9) * 16 + 11) >> 11) * 2.0 ** -53
    rs = pm.draw(0, 0, 0, np.arange(256), np.arange(16)[:, None]).ravel()
    assert np.all((rs >= 0.0) & (rs < 1.0)) and np.unique(rs).size == rs.size


def test_rotation():
    assert np.array_equal(pm.rotation([0.0, 0.0, 0.0]), np.eye(3))
    rng = np.random.default_rng(3)
    for _ in range(200):
        w = rng.uniform(-1.0, 1.0, 3) * (45 * pm.DEG)
        R = pm.rotation(w)
        assert np.abs(R - Rotation.from_rotvec(w).as_matrix()).max() < 4e-16
    tiny = pm.rotation([1e-200, 0.0, 0.0])  # y underflows to 0
    assert np.array_equal(tiny, np.eye(3))


def test_pose_is_a_rotation_about_the_centroid():
    c, s = np.array([0.01, -0.02, 0.6]), np.array([0.003, 0.001, 0.002])
    assert np.array_equal(pm.pose(np.zeros(6), c, s), np.block([[np.eye(3), s[:, None]], [np.zeros((1, 3)), np.ones((1, 1))]]))
    x = np.array([0.05, -0.1, 0.02, 0.004, -0.003, 0.01])
    T = pm.pose(x, c, s)
    # the centroid under S goes to c + t
    q = T[:3, :3] @ (c - s) + T[:3, 3]
    assert np.abs(q - (c + x[3:])).max() < 1e-15


def _scene(rows=48, cols=64, z=500):
    return np.full((rows, cols), z, np.uint16)


def _cloud(n, seed=0):
    rng = np.random.default_rng(seed)
    return np.stack([rng.uniform(-0.05, 0.05, n), rng.uniform(-0.05, 0.05, n), rng.uniform(0.45, 0.55, n)], 1)


def test_cost_is_order_independent_and_clamped():
    sK = np.array([[80.0, 0, 32], [0, 80.0, 24], [0, 0, 1]], np.float32)
    pts = _cloud(500, 1)
    T = pm.pose([0.01, 0.02, -0.01, 0.001, 0.0, -0.002], pts.mean(0), np.zeros(3))
    scene = _scene()
    scene[10:20, 10:30] = 0
    c = pm.point_costs(pts, T, scene, sK, 20.0)
    assert c.min() >= 0 and c.max() <= 20000
    perm = np.random.default_rng(2).permutation(len(pts))
    assert pm.cost(pts[perm], T, scene, sK, 20.0) == pm.cost(pts, T, scene, sK, 20.0) == int(c.sum())
    # at |d| = clamp exactly and one ulp either side (z_q = 500 mm exactly)
    for zs, want in ((520, 20000), (480, 20000), (510, 10000)):
        assert pm.point_costs([_pt(3, 2)], np.eye(4), _scene(6, 8, zs), SK, 20.0)[0] == want
    assert pm.point_costs([_pt(3, 2)], np.eye(4), _scene(6, 8, 520), SK, np.nextafter(20.0, 0.0))[0] == 19999
    assert pm.point_costs([_pt(-1, 2)], np.eye(4), _scene(6, 8), SK, 20.0)[0] == 20000  # outside


def _case(n=300, seed=0):
    sK = np.array([[80.0, 0, 32], [0, 80.0, 24], [0, 0, 1]], np.float32)
    pts = _cloud(n, seed)
    scene = _scene()
    scene[:, 40:] = 520
    return pts, np.array([0.004, -0.002, 0.003]), scene, sK


@pytest.mark.parametrize("opts", [dict(particles=1, iterations=10), dict(particles=16, iterations=0)])
def test_one_particle_or_no_iteration_returns_the_start(opts):
    pts, s, scene, sK = _case()
    T, rec = pm.search(pts, s, scene, sK, job=3, **opts)
    S = np.eye(4)
    S[:3, 3] = s
    assert np.array_equal(T, S) and rec["best"] == -1 and rec["cost"] == rec["cost_start"]


def test_trajectory_is_monotone_and_never_worse_than_the_start():
    pts, s, scene, sK = _case(400, 4)
    for seed in (0, 9):
        T, rec = pm.search(pts, s, scene, sK, job=1, particles=12, iterations=15, seed=seed)
        tr = rec["trace"]
        assert tr.size == 15 and np.all(np.diff(tr) <= 0) and tr[0] <= rec["cost_start"]
        assert rec["cost"] == tr[-1] == pm.cost(pts, T, scene, sK, 20.0)
        assert rec["cost"] <= rec["cost_start"]
        D = np.array([30 * pm.DEG] * 3 + [0.04] * 3)
        assert np.all(np.abs(rec["x"]) <= D) and np.all(np.abs(rec["v"]) <= D)
        for i in range(12):
            assert rec["cost_best"][i] == pm.cost(pts, pm.pose(rec["p"][i], rec["c"], s), scene, sK, 20.0)


def test_zero_bounds_keep_every_particle_at_the_start():
    pts, s, scene, sK = _case(50, 5)
    T, rec = pm.search(pts, s, scene, sK, particles=5, iterations=4, dt_mm=0.0, dr_deg=0.0)
    assert not rec["x"].any() and rec["best"] == -1 and np.array_equal(T[:3, 3], s)


def test_settings_conversion():
    P, I, dt, dr, clamp, seed = pm.settings(**pm.DEFAULTS)
    assert (P, I, clamp, seed) == (64, 40, 20.0, 0) and dt == 0.04 and dr == 30.0 * 0.017453292519943295
    assert math.isclose(dr, math.radians(30.0), rel_tol=1e-15)
