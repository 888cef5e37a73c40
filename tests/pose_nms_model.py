"""numpy model of the pose NMS (include/linemod_b200.h, lm_enqueue_pose_nms / lm_nms_translations) and the
adversarial inputs its tests run on.

Semantics: candidates are the box-NMS survivors with a pose (residual != -1); score -(double)residual; order by score
descending, -0.0 == +0.0, ties by ascending index, NaN scores first (ascending index); greedy pass keeping the first
remaining pose and dropping every remaining j with not (d_ij > thr), d_ij = sqrt((dx*dx + dy*dy) + dz*dz) in float64."""
import numpy as np


def distances(ts, i, js):
    """d(i, j) for every j of js: each operation a float64 numpy ufunc, so correctly rounded and never fused."""
    d = ts[i] - ts[js]
    return np.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2])


def order(scores):
    scores = np.asarray(scores, np.float64)
    nan = np.isnan(scores)
    return sorted(range(len(scores)), key=lambda i: (0, 0.0, i) if nan[i] else (1, -scores[i], i))


def nms(ts, scores, thr):
    """Steps 3-4: keep indices in keep order."""
    ts = np.asarray(ts, np.float64).reshape(-1, 3)
    rest = np.asarray(order(scores), np.int64)
    keep = []
    while rest.size:
        i, rest = rest[0], rest[1:]
        keep.append(int(i))
        if rest.size:
            rest = rest[distances(ts, i, rest) > thr]
    return keep


def detect(surv, R, t, residual, thr):
    """Steps 1-5 on lm_complete_pose's output (survivors in pick order, R [n,3,3], t [n,3] mm, residual [n] f32):
    (kept survivors, R, t, residual) in keep order."""
    posed = np.flatnonzero(residual != np.float32(-1.0))
    keep = posed[np.asarray(nms(t[posed], -residual[posed].astype(np.float64), thr), np.int64)] if posed.size else posed
    return surv[keep], R[keep], t[keep], residual[keep]


def nms_norms_restated(ts, scores, thresh):
    """linemod_ros/detect.py:41-50, restated: argsort()[::-1] order, then drop every remaining translation within
    `thresh` (not strictly beyond it) of the one kept."""
    remaining = np.argsort(scores)[::-1]
    kept = []
    while len(remaining):
        head, tail = remaining[0], remaining[1:]
        kept.append(int(head))
        far = np.linalg.norm(ts[head] - ts[tail], axis=1) > thresh
        remaining = tail[far]
    return kept


# ---- adversarial sets: name -> (ts [n,3] f64 mm, scores [n] f64, thr) ----
def _cloud(rng, n, spread=120.0):
    return rng.uniform(-spread, spread, (n, 3)) + np.array([0.0, 0.0, 800.0])


def exact_threshold_sets():
    ts = np.array([[0, 0, 0], [24, 32, 0], [0, 0, 40], [24, 32, 40.0]], np.float64)  # 40 from the first, the last 40 from 2 and 3
    scores = np.array([4.0, 3.0, 2.0, 1.0])
    below, above = np.nextafter(40.0, 0.0), np.nextafter(40.0, np.inf)
    return {"exact_40": (ts, scores, 40.0), "exact_40_ulp_below": (ts, scores, below), "exact_40_ulp_above": (ts, scores, above)}


def score_tie_sets(rng):
    n = 64
    ts = _cloud(rng, n, 60.0)
    zero = np.where(np.arange(n) % 2 == 0, 0.0, -0.0)
    nan = -rng.uniform(0, 1, n)
    nan[[3, 10, 11, 40]] = np.nan
    return {"all_equal": (ts, np.full(n, -0.5), 40.0), "signed_zero": (ts, zero, 40.0), "nan_scores": (ts, nan, 40.0)}


def nan_translation_sets(rng):
    n = 40
    ts = _cloud(rng, n)
    scores = -rng.uniform(0, 1, n)
    first = ts.copy()
    first[int(np.argmax(scores))] = np.nan                   # the best pose has a NaN translation
    later = ts.copy()
    later[np.argsort(scores)[::-1][[5, 17]]] = np.nan        # two later in the order
    return {"nan_t_first": (first, scores, 40.0), "nan_t_later": (later, scores, 40.0)}


def chain_sets():
    ts = np.array([[0, 0, 500], [30, 0, 500], [60, 0, 500], [90, 0, 500], [120, 0, 500.0]], np.float64)
    return {"chain": (ts, np.array([-0.1, -0.2, -0.3, -0.4, -0.5]), 40.0)}


SIZES = (0, 1, 31, 32, 33, 1023, 1024)


def size_sets(rng):
    out = {}
    for n in SIZES:
        ts = _cloud(rng, n, 400.0)
        ts[1::7] = ts[0::7][:len(ts[1::7])]                 # exact duplicates: distance 0
        scores = -np.round(rng.uniform(0, 1, n), 2)          # ties
        out["n%d" % n] = (ts, scores, 40.0)
    return out


def threshold_sets(rng):
    n = 200
    ts = _cloud(rng, n)
    ts[50:60] = ts[0:10]
    scores = -rng.uniform(0, 1, n)
    return {"thr_0": (ts, scores, 0.0), "thr_inf": (ts, scores, np.inf)}


def adversarial_sets(seed=5):
    rng = np.random.default_rng(seed)
    sets = {}
    for part in (exact_threshold_sets(), score_tie_sets(rng), nan_translation_sets(rng), chain_sets(), size_sets(rng),
                 threshold_sets(rng)):
        sets.update(part)
    return sets


def plain_sets(seed=9, count=40):
    """Sets without score ties or NaN, where any argsort agrees."""
    rng = np.random.default_rng(seed)
    out = []
    for k in range(count):
        n = int(rng.integers(0, 300))
        ts = _cloud(rng, n, float(rng.uniform(20, 400)))
        scores = -rng.permutation(n).astype(np.float64) / max(n, 1)  # distinct
        out.append((ts, scores, float(rng.choice([0.0, 10.0, 40.0, 75.0, 1e3]))))
    return out
