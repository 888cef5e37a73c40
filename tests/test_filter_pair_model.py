"""CPU checks of the paired refinement filter's model (tests/filter_pair_model.py): it agrees with tight_frames.Model and
the oracle on what is kept and dropped, its plane-word count is right on a hand-worked case, and the frames
tests/test_gpu_filter_pairs.py runs give the filter's warps every kind of pair."""
import numpy as np
import pytest

import filter_pair_model as fpm
import tight_frames as tf


def _agrees(oracle, q, T, packed, thr, mdl=None):
    """Per template: the model's drops are the candidates with max CH < need, none of them is kept by the reference, and
    its dropped bytes equal tight_frames.Model's; the kept records of the frame equal the oracle's (before std::unique)."""
    mdl = mdl or tf.Model(oracle, q, T, packed)
    fm = fpm.FilterModel(mdl, thr)
    at = 0
    for g in range(mdl.G):
        d = mdl.decisions(g, thr)
        n = len(d["cells"])
        dead = fm.c["dead"][at:at + n] if n else np.zeros(0, bool)
        assert fm.n == 0 or np.all(fm.c["cell"][at:at + n] == d["cells"])
        at += n
        if fm.n and n and fm.c["kind"][at - 1] == fpm.COUNTED:
            assert np.array_equal(dead, d["max_ch"] < d["need"]), g
            assert not np.any(dead & ~(tf.score(d["best"], mdl.t[g]["nf"]) < np.float32(thr))), g
        else:
            assert not dead.any()
    assert at == fm.n
    assert fm.dropped_bytes() == mdl.dropped_bytes(thr)
    if mdl.L == 2 and all(mdl.t[g]["safe"] for g in range(mdl.G)):
        assert tf.records(oracle.match(q, T, packed, thr, presort=True)) == sorted(mdl.kept(thr))
    return fm


def test_triage_one_and_need_zero_are_all_or_nothing():
    """need > nf only above threshold 100 (no coarse candidate: the filter's triage 1 is unreachable) and need <= 0 for
    every nf at threshold <= 25 and for none above: a counted candidate never shares a warp with a need <= 0 one."""
    hi, lo = fpm.need_facts()
    assert (hi, lo) == (np.float32(100.0), np.float32(25.0))


def test_agrees_with_the_bound_model_on_mosaic_staircase_and_zero_frames(oracle):
    s = tf.mosaic_setup(oracle, [4, 8], 640, 480)
    for thr in s["thresholds"]:
        for t in (thr, tf.ulp_up(thr)):
            assert _agrees(oracle, s["q"], [4, 8], s["packed"], t, s["model"]).dropped_bytes() > 0
    q = tf.uniform_frame(640, 480, 2)
    for nf, k, thr, need in tf.stair_cases():
        if nf in (65, 256, 511):
            bank = tf.stair_bank(nf, k)
            fm = _agrees(oracle, q, [4, 8], bank.pack(bank.class_ids(), 4), thr)
            # every cell ties: need = k keeps every candidate, k + 1 drops every one of the staircase template
            assert (fm.c["dead"][fm.c["item"] == 0].all() if need > k else not fm.c["dead"].any()), (nf, k, need)
    for unsafe in (False, True):
        T, _, qz, packed = tf.zero_case(unsafe)
        for thr in (0.0, -1.0):
            fm = _agrees(oracle, qz, T, packed, thr)
            assert fm.n > 0 and fm.words() == 0 and set(fm.c["kind"].tolist()) <= {fpm.NEED0, fpm.SURV2}


def test_words_on_a_hand_worked_case(oracle):
    """One staircase template (nf = 160, the last 60 features odd) on the uniform odd frame: every cell has CH = 0 for
    the first 100 features, then + 1 per feature.  Checks at 64, 128 and 160 (the end: 160 is no multiple of 64).
    need 60 (threshold = score(3 * 60 + 160)): thr at 64 = 60 - 96 <= 0, no check; at 128: thr = 28 and CH = 28, every
    column lives; at 160: thr = 60 = CH.  Five steps of 16 live columns: 5 * 32 * 16 words per candidate, kept.
    need 61: at 128 thr = 29 > 28, every column dies: four steps, 4 * 32 * 16 words, dropped at step 128."""
    q = tf.uniform_frame(320, 256, 2)
    bank = tf.make_bank([tf.staircase_template(160, 60, seed=4)])
    packed = bank.pack(bank.class_ids(), 4)
    mdl = tf.Model(oracle, q, [4, 8], packed)
    assert fpm.check_points(160) == [64, 128, 160]
    thr = tf.score(3 * 60 + 160, 160)
    for t, need, steps, dead in ((thr, 60, 5, False), (tf.ulp_up(thr), 61, 4, True)):
        assert tf.need_of(t, 160) == need
        fm = fpm.FilterModel(mdl, t)
        assert fm.n > 0
        assert np.all(fm.c["words"] == steps * 32 * 16) and np.all(fm.c["dead"] == dead)
        assert np.all(fm.c["end"] == (128 if dead else 160)) and not fm.c["partial"].any()
        # k_refine_bits then reads an H and an N window per feature of each survivor: 32 * 160 words
        assert fm.bytes_read() == 4 * fm.n * (steps * 32 * 16 + (0 if dead else 32 * 160))
        assert fm.dropped_bytes() == (256 * 160 * fm.n if dead else 0)
        assert fm.plan() == [fm.n, 0 if dead else fm.n, -1]


def test_partial_column_deaths_count_only_live_columns():
    """run_counted on a synthetic prefix-CH map: columns 0..3 reach the threshold, the others do not."""
    snaps = {}
    base = np.zeros((20, 20), np.int32)
    base[:, :4] = 40
    for done in (64, 96):
        snaps[done] = base
    r = fpm.run_counted(snaps, 96, 40, np.array([0]), np.array([0]))
    # step 32: 16 columns, step 64: 16 (check at 64: thr = 40 - 32 = 8, columns 0..3 live), step 96: 4; alive at the end
    assert r["words"].tolist() == [32 * (16 + 16 + 4)] and not r["dead"][0] and r["partial"][0]
    r = fpm.run_counted(snaps, 96, 41, np.array([3]), np.array([0]))   # columns 0 only (cx = 3): dies at 96
    assert r["words"].tolist() == [32 * (16 + 16 + 1)] and r["dead"][0] and r["end"][0] == 96 and r["last"][0]


@pytest.fixture(scope="module")
def coverage(oracle):
    cases = fpm.coverage_cases(oracle)
    counts = {}
    for c in cases.values():
        mdl = tf.Model(oracle, c["q"], fpm.PAIR_T, c["packed"])
        for thr in c["thresholds"]:
            for k, v in fpm.FilterModel(mdl, thr).pair_classes().items():
                counts[k] = counts.get(k, 0) + v
    return cases, counts


def test_coverage_frames_give_every_pair_class(coverage):
    """Every pair class the paired loop has a branch for occurs in the frames the GPU test runs; the cheap ones several
    times."""
    _, counts = coverage
    missing = [(k, n, counts.get(k, 0)) for k, n in fpm.REQUIRED if counts.get(k, 0) < n]
    assert not missing, missing


def test_coverage_frames_agree_with_the_oracle(oracle, coverage):
    cases, _ = coverage
    for name, c in cases.items():
        for thr in c["thresholds"]:
            _agrees(oracle, c["q"], fpm.PAIR_T, c["packed"], thr)
