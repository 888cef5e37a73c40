"""The pass checks of tests/icp_clouds.py (stop_pass, check_plane_step, check_point_step, corr_check, step_from_T), which
tests/test_gpu_icp_passes.py holds the kernel to, fed a float64 restatement of the ICP loop: icp_oracle's
registration_icp_p2pl and icp_p2p_oracle's registration_icp_p2p stepped one pass at a time.  No GPU needed.

  stop rule    stop_pass on the restatement's fitness and rmse gives the oracles' own iteration counts, on every case
               of icp_clouds.all_cases() with both targets and both estimations
  recovery     step_from_T inverts TransformVector6dToMatrix4d(x) @ T0 for rotated T0, up to principal_angles
  floor        the oracle moves its points in place, pass after pass; the model steps from transform(T_k, src).  The
               two float64 evaluations of every pass's update agree within the checks' bounds with the margin
               FLOOR_MARGIN, where the bound without the floor does not hold"""
import numpy as np
import pytest
from scipy.spatial import cKDTree

import icp_clouds as ic
import icp_p2p_oracle
from oracle import icp_oracle

P2PL, P2P = "point_to_plane", "point_to_point"
FLOOR_MARGIN = 1.0   # K of both checks here: 80 times the worst point-to-plane ratio, 5 times point-to-point's
CASES = {c.name: c for c in ic.all_cases()}
_CLOUDS = {}


def clouds(name, use_scene):
    if (name, use_scene) not in _CLOUDS:
        src, tgt, init, _ = ic.host_clouds(CASES[name], use_scene)
        _CLOUDS[name, use_scene] = src, tgt, init, icp_oracle.estimate_normals(tgt)
    return _CLOUDS[name, use_scene]


def stepped(src, tgt, normals, init, est, max_iter=icp_oracle.MAX_ITER):
    """The oracles' loop, pass by pass, with their arithmetic: points moved in place by every update.  Returns per pass
    k = 0 ... (the stop pass) dicts of T (T_k), p (the points of pass k), corr (target index or -1), fitness, rmse."""
    T = np.array(init, np.float64)
    tree = cKDTree(tgt)
    p = src @ T[:3, :3].T + T[:3, 3]
    out = []
    for k in range(max_iter + 1):
        d, j = tree.query(p, k=1)
        ok = d * d < icp_oracle.MAX_DIST * icp_oracle.MAX_DIST
        cnt = int(ok.sum())
        out.append(dict(T=T.copy(), p=p.copy(), corr=np.where(ok, j, -1), fitness=cnt / p.shape[0],
                        rmse=float(np.sqrt((d[ok] ** 2).sum() / cnt)) if cnt else 0.0))
        if k >= 1 and abs(out[-2]["fitness"] - out[-1]["fitness"]) < icp_oracle.REL_FITNESS and \
                abs(out[-2]["rmse"] - out[-1]["rmse"]) < icp_oracle.REL_RMSE:
            break
        if k == max_iter:
            break
        si, tj = np.nonzero(ok)[0], j[ok]
        if est == P2P:
            upd = icp_p2p_oracle.umeyama(p[si], tgt[tj])
        else:
            vs, vt, nt = p[si], tgt[tj], normals[tj]
            J = np.concatenate([np.cross(vs, nt), nt], 1)
            try:
                upd = icp_oracle.vec6_to_mat4(np.linalg.solve(J.T @ J, -(J.T @ ((vs - vt) * nt).sum(1))))
                if not np.all(np.isfinite(upd)):
                    upd = np.eye(4)
            except np.linalg.LinAlgError:
                upd = np.eye(4)
        T = upd @ T
        p = p @ upd[:3, :3].T + upd[:3, 3]
    return out


KEYS = [(name, s, est) for name in sorted(CASES) for s in (False, True) for est in (P2PL, P2P)]


@pytest.mark.parametrize("name,use_scene,est", KEYS)
def test_stop_rule_reproduces_the_oracles(name, use_scene, est):
    src, tgt, init, nrm = clouds(name, use_scene)
    if est == P2PL:
        T, fit, rmse, it = icp_oracle.registration_icp_p2pl(src, tgt, nrm, icp_oracle.MAX_DIST, init)
    else:
        T, fit, rmse, it = icp_p2p_oracle.registration_icp_p2p(src, tgt, icp_oracle.MAX_DIST, init)
    passes = stepped(src, tgt, nrm, init, est)
    assert np.array_equal(passes[-1]["T"], T) and (passes[-1]["fitness"], passes[-1]["rmse"]) == (fit, rmse)
    got = ic.stop_pass([q["fitness"] for q in passes], [q["rmse"] for q in passes], icp_oracle.MAX_ITER)
    assert got == it == len(passes) - 1, (got, it, len(passes))
    # a shorter cap stops there, and the evaluator needs every pass up to the stop
    fits, rmses = [q["fitness"] for q in passes], [q["rmse"] for q in passes]
    for cap in (0, 1, 2, 7):
        assert ic.stop_pass(fits, rmses, cap) == min(cap, it)
    assert ic.stop_pass(fits[:it], rmses[:it], icp_oracle.MAX_ITER) is None


def test_stop_rule_is_strict_and_needs_both():
    f, r = [0.5, 0.5 + 1e-6, 0.5 + 1e-6], [0.002, 0.002, 0.002 + 2e-6]
    assert ic.stop_pass(f, r, 30) is None  # |df| == 1e-6 exactly does not stop; then |dr| = 2e-6 does not either
    assert ic.stop_pass([0.0, 0.0], [0.0, 0.0], 30) == 1  # no pairs twice: pass 1 stops, never pass 0
    assert ic.stop_pass([0.3, 0.3], [0.004, 0.004], 0) == 0
    assert ic.stop_pass([0.3, 0.4, 0.4], [0.004, 0.004, 0.003], 30) is None


def test_step_from_T_inverts_for_rotated_poses():
    rng = np.random.default_rng(11)
    for _ in range(50):
        T0 = icp_oracle.vec6_to_mat4(np.concatenate([rng.uniform(-0.6, 0.6, 3), rng.uniform(-0.1, 0.1, 2), [0.3]]))
        x = np.concatenate([rng.uniform(-0.2, 0.2, 3), rng.uniform(-0.02, 0.02, 3)])
        T1 = icp_oracle.vec6_to_mat4(x) @ T0
        assert np.abs(ic.step_from_T(T1, T0) - x).max() <= 1e-14
        U = ic.update_of(T1, T0)
        assert np.abs(U @ T0 - T1).max() <= 1e-15
    # a diverging step's angles: step_from_T recovers the same rotation on its own branch, principal_angles maps x there
    for _ in range(50):
        x = np.concatenate([rng.uniform(-9, 9, 3), rng.uniform(-1, 1, 3)])
        T0 = icp_oracle.vec6_to_mat4(np.concatenate([rng.uniform(-0.6, 0.6, 3), [0, 0, 0.3]]))
        xp = ic.principal_angles(x)
        assert np.abs(icp_oracle.vec6_to_mat4(xp) - icp_oracle.vec6_to_mat4(x)).max() <= 1e-14
        assert np.abs(ic.step_from_T(icp_oracle.vec6_to_mat4(x) @ T0, T0) - xp).max() <= 1e-12
    x = np.array([0.1, -0.2, 0.3, 1e-3, 2e-3, 3e-3])
    assert np.array_equal(ic.principal_angles(x), x)


@pytest.mark.parametrize("est,least", [(P2PL, 250), (P2P, 90)])
def test_floor_bounds_two_float64_evaluations(est, least):
    """Every pass of every case: the oracle's T_{k+1} (its update from points moved in place) against the model's step
    from transform(T_k, src), through the same check the kernel gets, at K = FLOOR_MARGIN; the pairs of the first
    passes pass corr_check at T_k.  Without the floor the bound fails: where a pass has converged, |x| is down to the
    rounding of the residuals themselves (measured: worst ratio 0.012 with the floor and 1.2e6 without for
    point-to-plane; 0.20 and 12 for point-to-point)."""
    worst, worst_nofloor, compared = 0.0, 0.0, 0
    for name in sorted(CASES):
        for use_scene in (False, True):
            src, tgt, init, nrm = clouds(name, use_scene)
            passes = stepped(src, tgt, nrm, init, est)
            for k in range(len(passes) - 1):
                key = "%s/%s pass %d" % (name, "scene" if use_scene else "model", k)
                T0, T1, corr = passes[k]["T"], passes[k + 1]["T"], passes[k]["corr"]
                if k < 3 and src.shape[0] <= 2100:
                    ok, _ = ic.corr_check(ic.transform(T0, src), tgt, corr)
                    assert ok.all(), key
                if est == P2PL:
                    check = lambda K, floor: ic.check_plane_step(key, src, tgt, nrm, T0, T1, corr, K, floor)
                else:
                    check = lambda K, floor: ic.check_point_step(key, src, tgt, T0, T1, corr, K, floor)
                outcome, ratio, _ = check(FLOOR_MARGIN, True)
                if outcome == "compared":
                    compared += 1
                    worst = max(worst, ratio)
                    worst_nofloor = max(worst_nofloor, check(np.inf, False)[1])
    print("%s: %d passes compared, worst ratio %.3g (%.3g without the floor)" % (est, compared, worst, worst_nofloor))
    assert compared >= least
    assert worst_nofloor > 10 * FLOOR_MARGIN
