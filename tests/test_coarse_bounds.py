"""The coarse-bound constructions of tests/coarse_frames.py reach the bounds they are built for, on the oracle alone: raw
scores at exactly raw_min and raw_min - 1 of every threshold of the sweep, CH = 255 and CN = 255, the label wrap's
neighbour response, P at every residue mod 32, P = 1 and P <= 0, features outside the level, the byte kernel's
raw 32 764.  The model's candidate count equals the oracle's coarse_candidates stat.  No device needed."""
import numpy as np
import pytest

import coarse_frames as cf
import match_shapes as ms


def _model(oracle, bank, q, T):
    packed = bank.pack(bank.class_ids(), M_SLOTS * len(T))
    assert ms.reference_overreads(T, q[0][0].shape[1], q[0][0].shape[0], packed) == []
    return packed, cf.CoarseModel(oracle, q, T, packed)


M_SLOTS = cf.M


def _candidates_match_oracle(oracle, q, T, packed, model, thresholds):
    for thr in thresholds:
        _, st = oracle.match(q, T, packed, thr, want_stats=True)
        assert int(model.passes(thr).sum()) == int(st["coarse_candidates"]), thr


@pytest.mark.parametrize("nf", cf.SWEEP_NF)
def test_sweep_bank_attains_every_raw(oracle, nf):
    """One template per attainable raw, constant over its P cells and zero beyond; every strict threshold of the sweep
    puts raw_min where it is meant to be, with a template at raw_min and one at raw_min - 1 wherever both exist."""
    T, W, H = cf.SWEEP_SHAPE
    bank, q = cf.sweep_bank(nf)
    packed, mdl = _model(oracle, bank, q, T)
    want = sorted(cf.attainable(nf))
    assert mdl.G == len(want) and (mdl.nf == nf).all()
    P = int(mdl.P[0, 0])
    assert P == 55 and (mdl.P == P).all()
    assert (mdl.raw[:, P:] == 0).all()
    assert (mdl.raw[:, :P] == np.asarray(want)[:, None]).all()
    have = set(want)
    for r in range(0, 4 * nf + 2):
        assert cf.min_passing_raw(cf.score(r - 1, nf), nf) == r
        assert cf.min_passing_raw(cf.score(r, nf), nf) == min(r + 1, 4 * nf + 1)
        if r in have and r - 1 in have:
            thr = cf.score(r - 1, nf)
            p = mdl.passes(thr)
            assert p[want.index(r), :P].all() and not p[want.index(r - 1)].any()
    assert cf.min_passing_raw(-1.0, nf) == 0
    thrs = cf.sweep_thresholds(nf)
    assert len(thrs) >= 4 * nf + 3
    _candidates_match_oracle(oracle, q, T, packed, mdl, [thrs[0], thrs[len(thrs) // 2], thrs[-1]])


def test_saturation_patterns_fill_their_counters(oracle):
    """CH = 255 (raw 1020), CN = 255 (raw 255) and the 127 -> 128 / 254 -> 255 mixes score 4a + b at every cell; every
    template has one full round and one remainder word of positions."""
    T, W, H = cf.SAT_SHAPE
    q = cf.onehot_frame(W, H, 1, cf.SAT_LABEL)
    packed, mdl = _model(oracle, cf.saturation_bank(fillers=3), q, T)
    assert mdl.plane == 1056 and mdl.nwords == 33 and (mdl.P == mdl.plane).all()
    want = [4 * a + b for _, a, b in cf.PATTERNS] + [0] * 3
    assert (mdl.raw == np.asarray(want)[:, None]).all()
    assert 1020 in want and 255 in [b for _, _, b in cf.PATTERNS]
    assert list(mdl.nf[:len(cf.PATTERNS)]) == [nf for nf, _, _ in cf.PATTERNS]
    _candidates_match_oracle(oracle, q, T, packed, mdl, cf.ladder()[:3] + [-1.0])


def _response(lab, o):
    return 4 if lab == o else (1 if (lab - o) % 8 in (1, 7) else 0)


@pytest.mark.parametrize("o", [0, 7])
def test_label_wrap_responds_through_the_wrap(oracle, o):
    """A label-0 feature on a label-7 frame (and 7 on 0) responds 1: the neighbour label lies across the wrap."""
    T, W, H = cf.WRAP_SHAPE
    q = cf.onehot_frame(W, H, 1, o)
    bank = cf.wrap_bank(o)
    packed, mdl = _model(oracle, bank, q, T)
    feats = np.asarray(packed["feats"]).reshape(-1, 3)
    tm = np.asarray(packed["tmeta"]).reshape(mdl.G, 2, 4)
    for g in range(mdl.G):
        f = np.concatenate([feats[b:b + n] for b, n in tm[g, :, 2:4]])
        want = sum(_response(int(lab), o) for lab in f[:, 2])
        assert (mdl.raw[g, :mdl.plane] == want).all(), g
    assert mdl.raw[0, 0] == 40          # 40 features across the wrap, response 1 each
    assert mdl.nf.max() > 255           # one template on the byte kernel
    _candidates_match_oracle(oracle, q, T, packed, mdl, [0.0, 20.0, -1.0])


@pytest.mark.parametrize("shape", [cf.EDGE_SHAPE, cf.TINY_SHAPE], ids=["33x31", "5x3"])
def test_position_edges(oracle, shape):
    """P takes every residue mod 32 the level allows, and 1, and <= 0 (the map stays zero); the plane is not a multiple
    of 32."""
    T, W, H = shape
    q = cf.random_frame(W, H, 1, seed=11)
    bank, sizes = cf.edge_bank(W, H, T[0])
    packed, mdl = _model(oracle, bank, q, T)
    P = mdl.P[:, 0]
    assert (mdl.P[:, 0] == mdl.P[:, 1]).all() and mdl.plane % 32 != 0
    if mdl.plane >= 32 * 32:
        assert set((P[P > 0] % 32).tolist()) == set(range(32))
    assert 1 in P.tolist() and (P <= 0).sum() == 2
    for g in range(mdl.G):
        assert (mdl.raw[g, max(int(P[g]), 0):] == 0).all()
        if P[g] > 0:
            assert mdl.raw[g, :P[g]].any()
    assert cf.min_passing_raw(-0.5, 24) == 0
    _candidates_match_oracle(oracle, q, T, packed, mdl, [-0.5, 0.0, 30.0])


def test_features_outside_the_level_add_nothing(oracle):
    """Features beyond cols or rows count in nf and add nothing: the map equals that of the template without them."""
    T, W, H = cf.EDGE_SHAPE
    q = cf.random_frame(W, H, 1, seed=12)
    bank = cf.outside_bank(W, H)
    packed, mdl = _model(oracle, bank, q, T)
    feats = np.asarray(packed["feats"]).reshape(-1, 3)
    tm = np.asarray(packed["tmeta"]).reshape(mdl.G, 2, 4)
    n_out = 0
    for g in range(mdl.G):
        inside = []
        for b, n in tm[g, :, 2:4]:
            f = feats[b:b + n]
            keep = (f[:, 0] < W) & (f[:, 1] < H)
            n_out += int((~keep).sum())
            inside.append(f[keep])
        ft = np.concatenate(inside)
        tl = tm[g].copy()
        tl[0, 2:] = (0, len(inside[0]))
        tl[1, 2:] = (len(inside[0]), len(inside[1]))
        cmap, _ = oracle.coarse_map(q[0], T[0], tl, ft)
        assert np.array_equal(mdl.raw[g], cmap.astype(np.int64).ravel())
    assert n_out == 2 * (5 + 20 + 9 + 30) and list(mdl.nf) == [40, 255, 300, 700]   # per modality
    _candidates_match_oracle(oracle, q, T, packed, mdl, [10.0, 25.0])


def test_byte_bank_reaches_its_limits(oracle):
    """Every feature a hit: raw = sum of 4 * count over the modalities whose P covers the cell, 32 764 at 8191
    features; per-modality counts around the 63-feature flush and the 512-feature tile; unequal P."""
    T, W, H = cf.EDGE_SHAPE
    q = cf.onehot_frame(W, H, 1, cf.BYTE_LABEL)
    packed, mdl = _model(oracle, cf.byte_bank(), q, T)
    j = np.arange(mdl.plane)
    for g, (counts, _) in enumerate(cf.BYTE_SPECS):
        want = sum(4 * c * (j < mdl.P[g, m]) for m, c in enumerate(counts))
        assert np.array_equal(mdl.raw[g], want), g
    assert mdl.raw.max() == 32764
    counts = {c for cs, _ in cf.BYTE_SPECS for c in cs}
    assert {62, 63, 64, 126, 127, 189, 511, 512, 513} <= counts
    assert {256, 257} <= set(mdl.nf.tolist())
    assert any(mdl.P[g, 0] != mdl.P[g, 1] for g in range(mdl.G))
    _candidates_match_oracle(oracle, q, T, packed, mdl, [50.0, 99.99])


@pytest.mark.parametrize("name", list(cf.STAGING))
def test_staging_frames(oracle, name):
    """The two-level frames around the bit-planes' shared-memory limit carry the saturation patterns."""
    T, W, H = cf.STAGING[name]
    q = cf.onehot_frame(W, H, 2, cf.SAT_LABEL)
    packed, mdl = _model(oracle, cf.saturation_bank(levels=2), q, T)
    assert (mdl.raw[:, :mdl.plane] == np.asarray([4 * a + b for _, a, b in cf.PATTERNS])[:, None]).all()
    assert ms.frame_shape(T, W, H)["k2_smem"] == (name == "k2_shared")
    _candidates_match_oracle(oracle, q, T, packed, mdl, [0.0, cf.ladder()[-2]])
