"""The ICP kernels stage by stage (lm_icp_set_capture / lm_icp_capture) against the brute-force model of
tests/icp_clouds.py, on every case there, with the reference's target (the model cloud) and with the scene cloud.

  1 clouds and init    the uploaded clouds equal the host's cloud building, restated with sequential sums: bitwise
  2 neighbour sets     k_icp_normals keeps the 30 smallest (d^2, index): valid within BAND, equal to the model's outside it
  3 normals            the model's normal from the captured neighbour list, at 1e-9 (up to sign) where comparable
  4 correspondences    every captured index is a nearest target within the strict radius; fitness and rmse follow
  5 one step           the update k_icp_point_to_plane applied equals the model's Gauss-Newton step within
                       STEP_K * cond(J^T J) * eps relative
  6 capture            changes no output; a batch equals its single-hypothesis calls
A failure names the stage, the case and the point."""
import importlib
import json
import os

import numpy as np
import pytest

import icp_clouds as ic
from oracle import icp_oracle

pytestmark = pytest.mark.gpu

CASES = {c.name: c for c in ic.all_cases()}
STEP_K = 8           # worst measured on an H100: 0.66 (step error / (cond * eps * |x|)); see test_report
REPORT = {}


@pytest.fixture(scope="module")
def icp():
    lib = importlib.import_module("6dpose_b200._lib")
    return lib.NativeIcp()


def run(icp, c, use_scene, max_iter, capture=True):
    icp.set_use_scene_cloud(use_scene)
    icp.set_capture(capture)
    R, t, res = icp.process_batch(c.scene, [c.model], c.K, c.K[None], c.R[None], c.t[None], [c.xy], max_iter)
    st = icp.last_stats()
    st.pop("kernel_us")
    return (R, t, res, st), (icp.capture(0) if capture else None)


def check_clouds(c, use_scene, cap):
    src, tgt, init, init_np = ic.host_clouds(c, use_scene)
    for what, want in (("source", src), ("target", tgt)):
        got = cap[what]
        assert got.shape == want.shape, "stage 1 (clouds) %s: %s points, host %s" % (what, got.shape, want.shape)
        bad = np.nonzero((got != want).any(1))[0]
        assert bad.size == 0, "stage 1 (clouds) %s point %d: %r != %r" % (what, bad[0], got[bad[0]], want[bad[0]])
    assert np.array_equal(cap["init"], init), "stage 1 (init): %r != %r" % (cap["init"][:3, 3], init[:3, 3])
    assert np.max(np.abs(cap["init"] - init_np)) <= 1e-12, "stage 1 (init) against icp_oracle.build_clouds"
    if not use_scene:
        assert np.array_equal(cap["source"], cap["target"])
    return src, tgt


def check_knn(c, tgt, kept):
    n = tgt.shape[0]
    have = min(ic.KNN, n)
    assert kept.shape == (n, ic.KNN)
    assert np.all(kept[:, have:] == -1), "stage 2 (neighbours): padding"
    k = kept[:, :have]
    bad = np.nonzero(((k < 0) | (k >= n)).any(1))[0]
    assert bad.size == 0, "stage 2 (neighbours) point %d keeps %r of %d" % (bad[0], k[bad[0]], n)
    srt = np.sort(k, 1)
    bad = np.nonzero((srt[:, 1:] == srt[:, :-1]).any(1))[0]
    assert bad.size == 0, "stage 2 (neighbours) point %d keeps an index twice: %r" % (bad[0], k[bad[0]])
    bad = np.nonzero(k[:, 0] != np.arange(n))[0]
    assert bad.size == 0, "stage 2 (neighbours) point %d: the self point is not first (%r)" % (bad[0], k[bad[0]])
    kd2, out_min = ic.knn_check(tgt, kept)
    bad = np.nonzero(~ic.knn_valid(kd2, out_min))[0]
    assert bad.size == 0, "stage 2 (neighbours) point %d: kept d2 up to %.17g, left out %.17g" % (
        bad[0], np.nanmax(kd2[bad[0]]), out_min[bad[0]])
    # kept order: ascending d^2 within the band
    d = kd2[:, :have]
    bad = np.nonzero((d[:, 1:] < d[:, :-1] - ic.BAND * d[:, 1:]).any(1))[0] if have > 1 else []
    assert len(bad) == 0, "stage 2 (neighbours) point %d: kept out of d2 order" % bad[0]
    idx, d2, nxt = ic.knn_model(tgt)
    if c.exact_ties:  # exact arithmetic: the (d^2, index) order is the whole answer
        bad = np.nonzero((k != idx).any(1))[0]
        assert bad.size == 0, "stage 2 (neighbours) point %d: %r, model %r" % (bad[0], k[bad[0]], idx[bad[0]])
    clear = nxt - d2[:, -1] > 4 * ic.BAND * d2[:, -1]
    bad = np.nonzero(clear & (srt != np.sort(idx, 1)).any(1))[0]
    assert bad.size == 0, "stage 2 (neighbours) point %d: %r, model %r" % (bad[0], k[bad[0]], idx[bad[0]])
    return have, d2, nxt


def check_normals(c, tgt, kept, have, d2, nxt, nrm):
    n = tgt.shape[0]
    hv = np.full(n, have)
    want, comparable, degenerate, vmax = ic.normal_model(tgt, kept.astype(np.int64), hv)
    if have < 3:
        bad = np.nonzero((nrm != (0.0, 0.0, 1.0)).any(1))[0]
        assert bad.size == 0, "stage 3 (normals) point %d of %d: %r, want (0, 0, 1)" % (bad[0], n, nrm[bad[0]])
        return
    diff = np.minimum(np.abs(nrm - want).max(1), np.abs(nrm + want).max(1))
    bad = np.nonzero(comparable & (diff > ic.NORMAL_TOL))[0]
    assert bad.size == 0, "stage 3 (normals) point %d: %r, model %r" % (bad[0], nrm[bad[0]], want[bad[0]])
    unit = np.abs(np.linalg.norm(nrm, axis=1) - 1) <= 1e-12
    orth = np.abs((nrm * vmax).sum(1)) <= ic.NORMAL_TOL
    bad = np.nonzero(degenerate & ~(unit & orth))[0]
    assert bad.size == 0, "stage 3 (normals) degenerate point %d: %r" % (bad[0], nrm[bad[0]])
    if not c.planar and n >= 100:
        assert comparable.mean() >= 0.5, "stage 3 (normals): only %.2f comparable" % comparable.mean()
    # against the oracle's cKDTree neighbours: every normal that moves by more than 1e-9 has a near-tie at 30 / 31
    ora = icp_oracle.estimate_normals(tgt)
    dora = np.minimum(np.abs(nrm - ora).max(1), np.abs(nrm + ora).max(1))
    near_tie = ~(nxt - d2[:, -1] > 1e3 * ic.BAND * d2[:, -1])
    bad = np.nonzero(comparable & (dora > ic.NORMAL_TOL) & ~near_tie)[0]
    assert bad.size == 0, "stage 3 (normals) point %d differs from icp_oracle.estimate_normals without a tie" % bad[0]
    REPORT.setdefault("oracle_normals_moved", {})[c.name] = int((comparable & (dora > ic.NORMAL_TOL)).sum())


def check_corr(label, src, tgt, T, corr, fitness, rmse):
    n = src.shape[0]
    Ps = ic.transform(T, src)
    ok, d2 = ic.corr_check(Ps, tgt, corr)
    bad = np.nonzero(~ok)[0]
    assert bad.size == 0, "stage 4 (correspondences, %s) source point %d -> %d" % (label, bad[0], corr[bad[0]])
    cnt = int((corr >= 0).sum())
    assert fitness == (cnt / n if n else 0.0), "stage 4 (%s): fitness %r, %d of %d pairs" % (label, fitness, cnt, n)
    want = float(np.sqrt(np.nansum(d2) / cnt)) if cnt else 0.0
    # 1e-12 relative, plus the few ulps of |p| by which the kernel's transformed points may differ from these: every
    # distance, and so the rmse, moves by at most that much (it matters where the pose converged onto its own cloud)
    dp = 8 * ic.EPS * float(np.abs(Ps).max()) if n else 0.0
    assert abs(rmse - want) <= 1e-12 * want + dp, "stage 4 (%s): rmse %r, pairs give %r" % (label, rmse, want)


def check_step(c, use_scene, src, tgt, cap1):
    key = "%s/%s" % (c.name, "scene" if use_scene else "model")
    # pass 0 from init = [I | c]: the step relative to |x| alone (no rounding floor), which is far from zero here
    outcome, ratio, cond = ic.check_plane_step("stage 5 " + key, src, tgt, cap1["normals"], cap1["init"], cap1["T"],
                                               cap1["corr_first"], STEP_K, floor=False)
    # With 30 points or fewer every point keeps the same neighbour set, so every normal is the same and J^T J has rank 4
    # at most; a plane gives (nearly) equal normals too.  Every other case must reach the comparison.
    must_compare = src.shape[0] > ic.KNN and not c.flat
    assert not (must_compare and outcome != "compared"), \
        "stage 5 (step): %s has cond(J^T J) %.3g, the step is not compared" % (key, cond)
    if outcome == "singular" or cond == np.inf:  # the model's solve found J^T J singular: so does the kernel's, at pass 0
        assert np.array_equal(cap1["T"], cap1["init"]), "stage 5 (step): singular J^T J must give the identity update"
        REPORT.setdefault("step_singular", []).append(key)
    elif outcome == "cond":
        REPORT.setdefault("step_skipped_cond", {})[key] = cond
    else:
        REPORT.setdefault("step_ratio", {})[key] = [ratio, cond]


@pytest.mark.parametrize("use_scene", [False, True], ids=["model_target", "scene_target"])
@pytest.mark.parametrize("name", sorted(CASES))
def test_icp_stages(icp, name, use_scene):
    c = CASES[name]
    full, cap = run(icp, c, use_scene, 30)
    src, tgt = check_clouds(c, use_scene, cap)
    have, d2, nxt = check_knn(c, tgt, cap["knn"])
    check_normals(c, tgt, cap["knn"], have, d2, nxt, cap["normals"])
    # the last pass of a full run, then pass 0 alone
    check_corr("last pass", src, tgt, cap["T"], cap["corr_last"], cap["fitness"], cap["rmse"])
    out0, cap0 = run(icp, c, use_scene, 0)
    assert np.array_equal(cap0["T"], cap0["init"]) and cap0["iterations"] == 0
    assert np.array_equal(cap0["corr_first"], cap0["corr_last"]) and np.array_equal(cap0["corr_first"], cap["corr_first"])
    check_corr("pass 0", src, tgt, cap0["init"], cap0["corr_first"], cap0["fitness"], cap0["rmse"])
    if use_scene and c.info.get("straddle"):
        # the radius itself: correspondences just inside 1 cm, and points whose nearest target is just outside it
        near = np.sqrt(ic.pair_d2(ic.transform(cap0["init"], src), tgt).min(1))
        inside, outside = cap0["corr_first"] >= 0, cap0["corr_first"] < 0
        assert cap0["fitness"] < 1 and np.any(outside & (near < 0.0106)) and np.any(inside & (near > 0.0098)), \
            "stage 4 (pass 0): the radius is not exercised (fitness %r)" % cap0["fitness"]
    out1, cap1 = run(icp, c, use_scene, 1)
    assert np.array_equal(cap1["normals"], cap["normals"]) and np.array_equal(cap1["knn"], cap["knn"])
    check_step(c, use_scene, src, tgt, cap1)
    # stage 6: capture changes nothing
    for it, with_capture in ((30, full), (0, out0), (1, out1)):
        without, _ = run(icp, c, use_scene, it, capture=False)
        for a, b in zip(with_capture[:3], without[:3]):
            assert np.array_equal(a, b, equal_nan=True), "stage 6 (capture) changed an output at %d iterations" % it
        assert with_capture[3] == without[3]


@pytest.mark.parametrize("use_scene", [False, True], ids=["model_target", "scene_target"])
def test_batch_equals_single_calls(icp, use_scene):
    """One batch mixing sizes 1 to 6000 (k_icp_normals' grid is sized for the largest job) against one scene."""
    big = CASES["size_6000"]
    depth = ic.blob_depth(6000)
    models = [np.where(ic.disk_mask(n), np.rint(depth), 0).astype(np.uint16) for n in (6000, 1, 3, 30, 129, 257, 513, 1025, 2)]
    xy = [(icp_oracle.model_bbox(m)[0] + 5, icp_oracle.model_bbox(m)[1] + 5) for m in models]
    nb = len(models)
    Rs, ts, Ks = np.stack([big.R] * nb), np.stack([big.t] * nb), np.stack([big.K] * nb)
    icp.set_use_scene_cloud(use_scene)
    icp.set_capture(True)
    Rb, tb, rb = icp.process_batch(big.scene, models, big.K, Ks, Rs, ts, xy, 30)
    caps = [icp.capture(i) for i in range(nb)]
    for i in range(nb):
        R1, t1, r1 = icp.process_batch(big.scene, models[i:i + 1], big.K, Ks[:1], Rs[:1], ts[:1], xy[i:i + 1], 30)
        assert np.array_equal(R1[0], Rb[i]) and np.array_equal(t1[0], tb[i]) and r1[0] == rb[i], "stage 6 (batch) hypothesis %d" % i
        one = icp.capture(0)
        for k, v in one.items():
            assert np.array_equal(np.asarray(v), np.asarray(caps[i][k])), "stage 6 (batch) hypothesis %d: %s" % (i, k)


def test_capture_errors(icp):
    """An early return has nothing to capture; a short buffer is refused."""
    import ctypes
    lib = importlib.import_module("6dpose_b200._lib")
    c = CASES["size_129"]
    icp.set_use_scene_cloud(False)
    icp.set_capture(True)
    far = (c.scene.shape[1] - 3, c.xy[1])
    _, _, res = icp.process_batch(c.scene, [c.model, c.model], c.K, np.stack([c.K] * 2), np.stack([c.R] * 2), np.stack([c.t] * 2),
                                  [c.xy, far], 30)
    assert res[1] == -1 and res[0] >= 0
    assert icp.capture(0)["source"].shape == (129, 3)
    L = lib.load()
    buf = np.zeros(129 * 3, np.float64)
    assert L.lm_icp_capture(icp._h, 1, 1, buf.ctypes.data_as(ctypes.c_void_p), buf.nbytes) == lib.LM_E_STATE
    assert L.lm_icp_capture(icp._h, 0, 1, buf.ctypes.data_as(ctypes.c_void_p), buf.nbytes - 8) == lib.LM_E_CAPACITY
    assert L.lm_icp_capture(icp._h, 2, 1, buf.ctypes.data_as(ctypes.c_void_p), buf.nbytes) == lib.LM_E_INVALID
    icp.set_capture(False)
    assert L.lm_icp_capture(icp._h, 0, 1, buf.ctypes.data_as(ctypes.c_void_p), buf.nbytes) == lib.LM_E_INVALID


def test_report():
    """Writes what the stage checks measured (step error over cond * eps * |x| per case, normals that move against the
    oracle) to $ICP_STAGES_REPORT when set.  It checks nothing: the per-case tests hold the tolerances."""
    path = os.environ.get("ICP_STAGES_REPORT")
    if path and REPORT:
        if REPORT.get("step_ratio"):
            REPORT["step_ratio_worst"] = max(v[0] for v in REPORT["step_ratio"].values())
        with open(path, "w") as f:
            json.dump(REPORT, f, indent=1, sort_keys=True)
