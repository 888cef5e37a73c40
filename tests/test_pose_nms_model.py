"""CPU checks of the pose NMS model (tests/pose_nms_model.py): it agrees with a plain restatement of
linemod_ros/detect.py's nms_norms where any argsort agrees, its distance is np.linalg.norm bit for bit, and each
adversarial set the GPU tests run has the property it is there for."""
import numpy as np
import pytest

import pose_nms_model as pm

SETS = pm.adversarial_sets()


@pytest.mark.parametrize("k", range(40))
def test_model_equals_restated_nms_norms(k):
    ts, scores, thr = pm.plain_sets()[k]
    assert pm.nms(ts, scores, thr) == pm.nms_norms_restated(ts, scores, thr)


def _bits_equal(a, b):
    nan = np.isnan(a)
    return np.array_equal(nan, np.isnan(b)) and np.array_equal(a[~nan].view(np.uint64), b[~nan].view(np.uint64))


@pytest.mark.parametrize("name", sorted(SETS))
def test_model_distance_is_numpy_norm(name):
    ts, _, _ = SETS[name]
    allj = np.arange(len(ts))
    for i in range(0, len(ts), max(1, len(ts) // 64)):
        assert _bits_equal(pm.distances(ts, i, allj), np.linalg.norm(ts[i] - ts[allj], axis=1))


def test_plain_sets_have_no_ties():
    for ts, scores, _ in pm.plain_sets():
        assert len(np.unique(scores)) == len(scores) and not np.isnan(scores).any() and not np.isnan(ts).any()


def test_exact_threshold_pairs():
    ts, scores, thr = SETS["exact_40"]
    d = pm.distances(ts, 0, np.arange(4))
    assert d[1] == 40.0 and d[2] == 40.0 and d[3] > 40.0
    assert pm.distances(ts, 1, np.array([3]))[0] == 40.0 and pm.distances(ts, 2, np.array([3]))[0] == 40.0
    assert pm.nms(ts, scores, 40.0) == [0, 3]                              # equal to thr suppresses
    assert pm.nms(*SETS["exact_40_ulp_below"]) == [0, 1, 2, 3]             # one ulp under: every distance is beyond it
    assert pm.nms(*SETS["exact_40_ulp_above"]) == [0, 3]
    assert SETS["exact_40_ulp_below"][2] < 40.0 < SETS["exact_40_ulp_above"][2]


def test_score_ties_go_in_index_order():
    ts, scores, thr = SETS["all_equal"]
    assert pm.order(scores) == list(range(len(scores)))
    ts, scores, thr = SETS["signed_zero"]
    assert (np.signbit(scores) != np.signbit(scores[0])).any() and pm.order(scores) == list(range(len(scores)))
    keep = pm.nms(ts, scores, thr)
    assert keep == sorted(keep) and len(keep) > 1


def test_nan_scores_come_first():
    ts, scores, thr = SETS["nan_scores"]
    nan = np.flatnonzero(np.isnan(scores))
    assert len(nan) == 4
    o = pm.order(scores)
    assert o[:4] == sorted(nan.tolist())
    rest = np.array(o[4:])
    assert np.all(np.diff(scores[rest]) <= 0)
    # where argsort()[::-1] puts NaN too
    assert set(np.argsort(scores)[::-1][:4].tolist()) == set(nan.tolist())


def test_nan_translations():
    ts, scores, thr = SETS["nan_t_first"]
    best = int(np.argmax(scores))
    assert np.isnan(ts[best]).all()
    assert pm.nms(ts, scores, thr) == [best]                              # a kept NaN suppresses every pose after it
    ts, scores, thr = SETS["nan_t_later"]
    keep = pm.nms(ts, scores, thr)
    bad = np.flatnonzero(np.isnan(ts[:, 0]))
    assert len(bad) == 2 and not set(bad.tolist()) & set(keep)            # NaN distance to the first kept: suppressed
    assert len(keep) > 2


def test_suppression_chain():
    ts, scores, thr = SETS["chain"]
    assert pm.distances(ts, 1, np.array([2]))[0] <= thr                    # B would have dropped C
    assert pm.nms(ts, scores, thr) == [0, 2, 4]                            # A drops B, so C stays


def test_sizes():
    for n in pm.SIZES:
        ts, scores, thr = SETS["n%d" % n]
        assert len(ts) == len(scores) == n
        keep = pm.nms(ts, scores, thr)
        assert (len(keep) > 0) == (n > 0) and len(set(keep)) == len(keep)
        if n >= 31:
            assert len(np.unique(scores)) < n and len(keep) < n           # ties and duplicates present


def test_thresholds_zero_and_infinity():
    ts, scores, _ = SETS["thr_0"]
    keep = pm.nms(ts, scores, 0.0)
    assert len(keep) == len(np.unique(ts, axis=0)) == len(ts) - 10        # only exact duplicates go
    assert pm.nms(ts, scores, np.inf) == [int(np.argmax(scores))]          # every distance is within +inf


def test_detect_model_drops_early_returns_and_keeps_the_sign():
    surv = np.arange(5)
    R = np.arange(45, dtype=np.float64).reshape(5, 3, 3)
    t = np.array([[0, 0, 500], [100, 0, 500], [200, 0, 500], [300, 0, 500], [400, 0, 500.0]])
    res = np.array([0.9, -1.0, 0.1, 0.5, 0.1], np.float32)
    s, R2, t2, r2 = pm.detect(surv, R, t, res, 40.0)
    assert s.tolist() == [2, 4, 3, 0]                                      # lowest fitness first, ties in pick order
    assert np.array_equal(R2, R[s]) and np.array_equal(t2, t[s]) and np.array_equal(r2, res[s])
