"""The ICP test cases and the brute-force model of tests/icp_clouds.py, on the CPU: each generator builds what it says,
and the model's normals equal the oracle's (cKDTree) wherever the 30th and 31st neighbours are not nearly tied."""
import numpy as np
import pytest

import icp_clouds as ic
from oracle import icp_oracle

CASES = {c.name: c for c in ic.all_cases()}


@pytest.mark.parametrize("name", sorted(CASES))
def test_generator_premise(name):
    c = CASES[name]
    bx, by, bw, bh = icp_oracle.model_bbox(c.model)
    assert c.xy[0] + bw < c.scene.shape[1] and c.xy[1] + bh < c.scene.shape[0], "the box must fit: no early return"
    for use_scene in (False, True):
        src, tgt, init, init_np = ic.host_clouds(c, use_scene)
        assert np.all(np.isfinite(init)), "the scene centroid must have points"
        assert np.max(np.abs(init - init_np)) <= 1e-12
        n_px = int((c.model > 0).sum())
        if c.n_model is not None:
            assert src.shape[0] == c.n_model == n_px, (src.shape, c.n_model)
            assert tgt.shape[0] == (c.n_scene if use_scene else c.n_model)
        # the clouds come out sorted by voxel column (x major): the kernels' pruning relies on it
        vox = np.floor((tgt[:, 0] - (tgt[:, 0].min() - icp_oracle.VOXEL / 2)) / icp_oracle.VOXEL)
        assert np.all(np.diff(vox) >= 0)
    if name.startswith("strip_x"):
        assert np.ptp(src[:, 0]) > 1.0 and np.ptp(src[:, 1]) < 0.01   # 1 m long: a 256-point tile is a 25 cm slab
    if name.startswith("strip_y"):
        assert np.ptp(src[:, 0]) < 0.01 and len(np.unique(vox)) == 3   # three voxel columns: tiles are not pruned
    if name.startswith("clusters"):
        L, S = c.info["large"], c.info["small"]
        assert S < ic.KNN and L % 256 == 0 and src.shape[0] == L + S
        gap = src[L:, 0].min() - src[:L, 0].max()
        assert gap > (c.info["gap_px"] + 0.5) * 0.0025          # a gap of empty voxel columns
        nb, _, _ = ic.knn_model(src)
        assert np.all((nb[L:] < L).sum(1) == ic.KNN - S)                # the small cluster's sets cross it
    if c.info.get("straddle"):
        # with the scene cloud as the target, pass 0 has nearest targets just inside and just outside the 1 cm radius
        src, tgt, init, _ = ic.host_clouds(c, True)
        near = np.sqrt(ic.pair_d2(ic.transform(init, src), tgt).min(1))
        assert np.any((near > 0.0098) & (near < 0.01)) and np.any((near > 0.01) & (near < 0.0106)) and near.max() > 0.015
    if name == "lo_gap":
        # A's last voxel column holds two points, the one sorted last (the tile's last point) with 2 mm less x; B's
        # corner keeps the other among its 30 neighbours, yet every point of B's first block is farther in x from the
        # tile's last point than its own 30th neighbour: only the one-voxel slack of the lo-side bound keeps tile 0
        assert src.shape[0] == 256 + 192
        col = np.floor((src[:, 0] - (src[:, 0].min() - icp_oracle.VOXEL / 2)) / icp_oracle.VOXEL)
        assert col[254] == col[255] != col[253] and src[254, 0] - src[255, 0] > 0.0019
        nb, d2, _ = ic.knn_model(src)
        blk = np.arange(256, 384)
        assert np.all(src[blk, 0] - src[255, 0] > np.sqrt(d2[blk, -1]))
        assert np.any(nb[blk] == 254)
    if name == "pitch_1.25mm":
        assert src.shape[0] < 0.6 * (c.model > 0).sum()                 # several pixels per voxel
        raw, _, _, _ = icp_oracle.build_clouds(c.scene, c.model, c.K, c.K, c.xy[0], c.xy[1], (bx, by, bw, bh))
        u = (raw[:, 0] - (raw[:, 0].min() - icp_oracle.VOXEL / 2)) / icp_oracle.VOXEL
        # (c - cx) / f is rounded to float32: a pixel within that rounding of a column boundary lands on either side
        on_edge = np.abs(u - np.rint(u)) < 1e-5
        assert on_edge.mean() > 0.3                                     # a third of the pixels sit on a column boundary
    if c.exact_ties:
        _, d2, nxt = ic.knn_model(src)
        assert np.mean(d2[:, -1] == nxt) > 0.5                           # the 30th and 31st neighbours tie exactly
        # exactness: every squared distance is a multiple of a power of two far above the rounding unit
        q = src / 2.0 ** -12
        assert np.array_equal(q, np.rint(q))
    if c.planar:
        assert np.all(src[:, 2] == 0.25)


@pytest.mark.parametrize("name", ["size_3", "size_31", "size_257", "size_1025", "strip_x", "strip_y", "clusters_512_12_gap20",
                                  "pitch_1.25mm", "tie_grid"])
def test_model_normals_equal_the_oracle(name):
    """Away from a near-tie at neighbour 30 / 31 the model picks the oracle's neighbour set, and its normals agree at
    1e-12 (up to sign)."""
    c = CASES[name]
    src, _, _, _ = ic.host_clouds(c, False)
    want = icp_oracle.estimate_normals(src)
    got, idx = ic.model_normals(src)
    _, d2, nxt = ic.knn_model(src)
    clear = nxt - d2[:, -1] > 1e3 * ic.BAND * d2[:, -1]
    diff = np.minimum(np.abs(got - want).max(1), np.abs(got + want).max(1))
    assert clear.mean() > 0.5 or c.exact_ties
    bad = np.nonzero(clear & (diff > 1e-12))[0]
    assert bad.size == 0, (name, bad[:10], diff[bad[:10]])


def test_model_step_recovery_roundtrip():
    """step_from_T inverts TransformVector6dToMatrix4d(x) @ init."""
    rng = np.random.default_rng(5)
    for _ in range(20):
        x = np.concatenate([rng.uniform(-0.3, 0.3, 3), rng.uniform(-0.05, 0.05, 3)])
        init = np.eye(4)
        init[:3, 3] = rng.uniform(-0.1, 0.1, 3)
        T1 = icp_oracle.vec6_to_mat4(x) @ init
        assert np.allclose(ic.step_from_T(T1, init), x, rtol=0, atol=1e-14)


def test_knn_valid_and_corr_check_reject_wrong_answers():
    """The checks the GPU test relies on fail on a neighbour set or a correspondence that is wrong by one point."""
    c = CASES["size_513"]
    src, _, _, _ = ic.host_clouds(c, False)
    idx, _, _ = ic.knn_model(src)
    kept = idx.astype(np.int32)
    kd2, out_min = ic.knn_check(src, kept)
    assert ic.knn_valid(kd2, out_min).all()
    bad = kept.copy()
    far = np.argmax(ic.pair_d2(src[:1], src)[0])
    bad[0, -1] = far
    kd2, out_min = ic.knn_check(src, bad)
    assert not ic.knn_valid(kd2, out_min)[0]
    Ps = src + np.array([0.004, 0.0, 0.0])
    D = ic.pair_d2(Ps, src)
    corr = np.where(D.min(1) < ic.MAX_D2, D.argmin(1), -1).astype(np.int32)
    ok, _ = ic.corr_check(Ps, src, corr)
    assert ok.all()
    second = np.argsort(D[0])[1]
    corr[0] = second
    corr[1] = -1
    ok, _ = ic.corr_check(Ps, src, corr)
    assert not ok[0] and not ok[1]
