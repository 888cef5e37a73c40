"""Premises of the tight-bound frames (tests/tight_frames.py) and the numpy model of the refinement filter, on CPU.

tests/test_gpu_refine_bounds.py runs these frames through the CUDA pipeline; the checks here make sure that the frames
really put the filter and the arg-max on their bounds, and that the model which predicts the filter's counter agrees
with the oracle.  No GPU."""
import numpy as np
import pytest

import tight_frames as tf


@pytest.mark.parametrize("T,W,H", [([4, 8], 640, 480), ([5, 8], 640, 480), ([2, 4, 8], 640, 480), ([4, 4], 648, 480),
                                   ([4, 8], 640, 2064)])
def test_mosaic_responses_are_one_or_four(oracle, T, W, H):
    """Every T x T window (T >= 3) of a mosaic level holds a whole 2x2 tile: no label responds 0 outside the last T rows
    and columns, so raw = 3*CH + nf holds at every cell a clamped patch reaches."""
    q = tf.mosaic_frame(W, H, len(T), seed=0)
    resp = tf.response_maps(oracle, q, T)
    checked = 0
    for l, t in enumerate(T):
        if t < 3:
            continue
        for m in range(2):
            assert set(np.unique(tf.reachable_responses(resp[l][m], t)).tolist()) == {1, 4}, (l, m)
            checked += 1
    assert checked >= 4


@pytest.mark.parametrize("kind,T,W,H,ok", [
    ("mosaic", [4, 8], 640, 480, True), ("mosaic", [4, 8], 640, 464, True), ("mosaic", [5, 8], 640, 480, True),
    ("mosaic", [4, 4], 648, 480, False),   # Wd = 162
    ("mosaic", [4, 8], 640, 2064, False),  # Hd = 516
    ("zero", [4, 8], 320, 256, True),
    ("zero", [4, 4], 328, 256, False),     # Wd = 82
    ("zero", [4, 8], 320, 2064, False),    # Hd = 516
])
def test_filter_takes_the_frames_it_should(oracle, kind, T, W, H, ok):
    """The filtered level's Wd must be a multiple of 4, with at most 512 cell rows (prepare_bank): the GPU tests reach
    k_refine<false> through the frames that fail this (the staircase frames have the mosaic frames' sizes)."""
    if kind == "mosaic":
        bank, q = tf.mosaic_case(T, W, H)
        packed = bank.pack(bank.class_ids(), len(T) * 2)
    else:
        T, _, q, packed = tf.zero_case(False, T, W, H)
    assert tf.Model(oracle, q, T, packed).filter_ok() == ok


def _stair_packed(nf, k, unsafe=False):
    bank = tf.stair_bank(nf, k, unsafe)
    return bank.pack(bank.class_ids(), 4)


@pytest.mark.parametrize("T,pct", [([4, 8], (50, 90, 99)), ([2, 4, 8], (50,))])
def test_mixed_banks_have_unsafe_and_safe_templates(oracle, T, pct):
    """With every third template unsafe, the safe ones stay eligible for the filter and some unsafe template has coarse
    candidates at every tight threshold: the filter hands them to k_refine<true> next to the filtered ones.  The
    staircase bank's unsafe copy is its last template."""
    s = tf.mosaic_setup(oracle, T, 640, 480, percentiles=pct, unsafe=True)
    mdl = s["model"]
    unsafe = [g for g in range(mdl.G) if not mdl.t[g]["safe"]]
    assert unsafe == list(range(0, mdl.G, 3))
    assert all(mdl.eligible(g) for g in range(mdl.G) if g not in unsafe)
    for thr in s["thresholds"]:
        for t in (thr, tf.ulp_up(thr)):
            assert any(len(mdl.candidates(g, t)) > 0 for g in unsafe), t
    mdl = tf.Model(oracle, tf.uniform_frame(640, 480, 2), [4, 8], _stair_packed(65, 2, unsafe=True))
    assert mdl.eligible(0) and not mdl.t[mdl.G - 1]["safe"]


@pytest.mark.parametrize("T,pct", [([4, 8], (50, 90, 99)), ([2, 4, 8], (50,))])
def test_mosaic_thresholds_put_kept_candidates_on_the_bound(oracle, T, pct):
    """At each tight threshold at least 100 candidates the filtered level keeps have max CH == need (zero filter slack),
    raw = 3*CH + nf holds with equality at every cell (claim 2 of test_refine_bitslice_model.py), and one ulp higher none
    of them is kept."""
    s = tf.mosaic_setup(oracle, T, 640, 480, percentiles=pct)
    mdl = s["model"]
    assert len(set(s["thresholds"])) == len(pct)
    for thr in s["thresholds"]:
        up = tf.ulp_up(thr)
        tight = 0
        for g in range(mdl.G):
            nf = mdl.t[g]["nf"]
            d = mdl.decisions(g, thr)
            assert np.array_equal(d["raw"], 3 * d["ch"] + nf)
            assert tf.min_kept_raw(thr, nf) == 3 * d["need"] + nf  # a similarity the frame attains: no rounding slack
            kept = ~(tf.score(d["best"], nf) < thr)
            on_bound = kept & (d["max_ch"] == d["need"])
            tight += int(on_bound.sum())
            du = mdl.decisions(g, up)
            assert du["need"] == d["need"] + 1
            assert np.array_equal(du["cells"], d["cells"])  # the coarse scan does not move by one ulp here
            assert not np.any(~(tf.score(du["best"], nf) < up) & on_bound)
        assert tight >= 100, (thr, tight)


def test_staircase_ties_every_cell_at_the_bound(oracle):
    """Uniform frame, staircase templates: every cell of every patch has CH = k and raw = 3k + nf, the first maximum is
    cell (0, 0), need = k keeps every candidate and need = k + 1 (one ulp higher) keeps none."""
    T = [4, 8]
    q = tf.uniform_frame(640, 480, 2)
    cases = tf.stair_cases()
    assert {nf for nf, *_ in cases} == set(tf.STAIR_NF)
    seen_full = False
    for nf, k, thr, need in cases:
        bank = tf.stair_bank(nf, k)
        packed = bank.pack(bank.class_ids(), 4)
        mdl = tf.Model(oracle, q, T, packed)
        assert mdl.eligible(0) and mdl.t[0]["nf"] == nf
        d = mdl.decisions(0, thr)
        assert d["need"] == need and len(d["cells"]) > 900
        assert np.all(d["ch"] == k) and np.all(d["raw"] == 3 * k + nf) and np.all(d["first"] == 0)
        want = oracle.match(q, T, packed, thr, presort=True)
        mine = want[want["template_id"] == 0]
        assert len(mine) == (len(d["cells"]) if need == k else 0)
        if nf == 511:
            assert not mdl.eligible(1) and mdl.t[1]["nf"] == 512  # the byte-wise path's template, always kept
            assert int((want["template_id"] == 1).sum()) == len(mdl.candidates(1, thr)) > 0
            seen_full |= k == 511 and int(d["best"].max()) == 2044
    assert seen_full


@pytest.mark.parametrize("thr", [0.0, -1.0])
def test_zero_score_patches_exist(oracle, thr):
    """Level 0 blanked over the left half: at least 50 kept matches score 0 at every cell, and the reference leaves their
    best cell at (-1, -1), one cell up and left of the patch origin: (x / T - 9) * T + offset."""
    T, _, q, packed = tf.zero_case()
    mdl = tf.Model(oracle, q, T, packed)
    want = oracle.match(q, T, packed, thr, presort=True)
    zero = want[want["similarity"] == 0]
    assert len(zero) >= 50
    n0 = 0
    for g in range(mdl.G):
        d = mdl.decisions(g, thr)
        z = d["best"] == 0
        n0 += int(z.sum())
        assert np.all(d["first"][z] == -1)
        zx = (d["x"][z] // 4 - 9) * 4 + 1
        zy = (d["y"][z] // 4 - 9) * 4 + 1
        got = sorted(zip(zero["x"][zero["template_id"] == g].tolist(), zero["y"][zero["template_id"] == g].tolist()))
        assert got == sorted(zip(zx.tolist(), zy.tolist()))
    assert n0 == len(zero)


def _model_vs_oracle(oracle, q, T, packed, thr, mdl=None):
    mdl = mdl or tf.Model(oracle, q, T, packed)
    want, st = oracle.match(q, T, packed, thr, want_stats=True, presort=True)
    assert sum(len(mdl.candidates(g, thr)) for g in range(mdl.G)) == int(st["coarse_candidates"])
    assert tf.records(want) == sorted(mdl.kept(thr))
    return len(want)


def test_model_matches_the_oracle_on_mosaic_frames(oracle):
    """The model's kept records equal the oracle's (as a multiset) and its coarse candidate count equals the oracle's, at
    the tight thresholds, one ulp above them and on three more frame shapes."""
    s = tf.mosaic_setup(oracle, [4, 8], 640, 480)
    for thr in s["thresholds"]:
        for t in (thr, tf.ulp_up(thr)):
            assert _model_vs_oracle(oracle, s["q"], [4, 8], s["packed"], t, s["model"]) > 0
    for T, W, H in (([4, 8], 640, 512), ([4, 8], 640, 464), ([5, 8], 640, 480)):
        s = tf.mosaic_setup(oracle, T, W, H, percentiles=(90,))
        assert _model_vs_oracle(oracle, s["q"], T, s["packed"], s["thresholds"][0], s["model"]) > 0


def test_model_matches_the_oracle_on_staircase_and_zero_frames(oracle):
    T = [4, 8]
    q = tf.uniform_frame(640, 480, 2)
    for nf, k in ((65, 2), (256, 64), (511, 511)):
        bank = tf.stair_bank(nf, k)
        packed = bank.pack(bank.class_ids(), 4)
        for _, _, thr, _ in [c for c in tf.stair_cases() if c[0] == nf and c[1] == k]:
            _model_vs_oracle(oracle, q, T, packed, thr)
    for thr in (0.0, -1.0):
        T, _, qz, packed = tf.zero_case()
        assert _model_vs_oracle(oracle, qz, T, packed, thr) > 0


def test_model_counts_the_drops_the_filter_must_make(oracle):
    """The expected filter_dropped_bytes: 256 * nf per candidate of an eligible template with need > nf, or with need > 0
    and no cell at CH >= need.  Candidates the model drops are never kept by the oracle, and the ones on the bound
    (max CH == need) are not dropped."""
    s = tf.mosaic_setup(oracle, [4, 8], 640, 480)
    mdl = s["model"]
    thr = s["thresholds"][0]
    total = 0
    for g in range(mdl.G):
        assert mdl.eligible(g)
        d = mdl.decisions(g, thr)
        nf = mdl.t[g]["nf"]
        drop = d["max_ch"] < d["need"]
        kept = ~(tf.score(d["best"], nf) < thr)
        assert not np.any(drop & kept)
        total += 256 * nf * int(drop.sum())
    assert total == mdl.dropped_bytes(thr) > 0
    assert mdl.dropped_bytes(np.float32(-1.0)) == 0
    assert mdl.dropped_bytes(np.float32(101.0)) == 0  # no coarse candidate above 100 %
