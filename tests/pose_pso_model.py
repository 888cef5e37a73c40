"""numpy float64 model of the particle-swarm pose estimation (include/linemod_b200.h, LM_POSE_PSO): the generator, the
pose T(x), the integer cost and the swarm, one IEEE operation per step of the header.  numpy's float64 ufuncs are
correctly rounded and never fused, and uint64 arithmetic wraps modulo 2^64, so every value restates the device's bit
for bit.  The projection is pose verification's (tests/pose_verify_model.classify)."""
import math

import numpy as np

from pose_verify_model import INLIER, classify

GOLDEN = 0x9E3779B97F4A7C15
W, C1, C2 = 0.7298, 1.49618, 1.49618
DEG = 0.017453292519943295
# sin(s)/s and (1 - cos(s))/s^2 as series in y = s^2: (-1)^k/(2k+1)! and (-1)^k/(2k+2)! rounded to double
SA = [(-1) ** k / math.factorial(2 * k + 1) for k in range(11)]
SB = [(-1) ** k / math.factorial(2 * k + 2) for k in range(11)]
INT64_MAX = np.iinfo(np.int64).max
DEFAULTS = dict(particles=64, iterations=40, dt_mm=40.0, dr_deg=30.0, clamp_mm=20.0, seed=0)


def splitmix64(seed, number):
    """Output `number` (0-based) of splitmix64 seeded with seed; number may be an array."""
    with np.errstate(over="ignore"):
        z = np.uint64(seed) + (np.asarray(number, np.uint64) + np.uint64(1)) * np.uint64(GOLDEN)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        return z ^ (z >> np.uint64(31))


def draw(seed, job, k, i, q):
    """Draw (i, k, q) of job J: r in [0, 1), the top 53 bits of its splitmix64 output."""
    number = ((np.uint64(job) * np.uint64(1024) + np.uint64(k)) * np.uint64(1024) + np.asarray(i, np.uint64)) * np.uint64(16) + \
        np.asarray(q, np.uint64)
    return (splitmix64(seed, number) >> np.uint64(11)).astype(np.float64) * 2.0 ** -53


def rotation(w):
    """Rot(w) by Rodrigues' formula with the header's series; exactly I at w = 0."""
    w0, w1, w2 = (np.float64(v) for v in w)
    y = (w0 * w0 + w1 * w1) + w2 * w2
    R = np.eye(3)
    if y == 0.0:
        return R
    A, B = np.float64(SA[10]), np.float64(SB[10])
    for k in range(9, -1, -1):
        A = np.float64(SA[k]) + y * A
        B = np.float64(SB[k]) + y * B
    ww = (w0, w1, w2)
    K = np.array([[0.0, -w2, w1], [w2, 0.0, -w0], [-w1, w0, 0.0]])
    for r in range(3):
        for c in range(3):
            k2 = ww[r] * ww[r] - y if r == c else ww[r] * ww[c]
            R[r, c] = (np.float64(1.0 if r == c else 0.0) + A * K[r, c]) + B * k2
    return R


def pose(x, c, s):
    """T(x) = Trans(c + t) Rot(w) Trans(-c) S as a 4x4, S = [I | s]."""
    x = np.asarray(x, np.float64)
    R = rotation(x[:3])
    a = [np.float64(s[r]) - np.float64(c[r]) for r in range(3)]
    T = np.eye(4)
    T[:3, :3] = R
    for r in range(3):
        m = (R[r, 0] * a[0] + R[r, 1] * a[1]) + R[r, 2] * a[2]
        T[r, 3] = (np.float64(s[r]) + (m - a[r])) + x[3 + r]
    return T


def centroid(pts, s):
    """c: the points under S, summed from 0.0 in index order, over n."""
    pts = np.asarray(pts, np.float64).reshape(-1, 3)
    c = np.zeros(3)
    for r in range(3):
        acc = np.float64(0.0)
        col = pts[:, r] + np.float64(s[r])
        for v in col:
            acc = acc + v
        c[r] = acc / np.float64(pts.shape[0])
    return c


def point_costs(pts, T, scene, sK, clamp_mm):
    """Per point (int64): (int32)floor(e * 1000), e = clamp outside / on missing depth, else min(|d|, clamp)."""
    pts = np.asarray(pts, np.float64).reshape(-1, 3)
    T = np.asarray(T, np.float64).reshape(4, 4)
    sK = np.asarray(sK, np.float32).reshape(3, 3)
    cls = classify(pts, T, scene, sK, math.inf)
    out = np.full(pts.shape[0], int(math.floor(np.float64(clamp_mm) * 1000.0)), np.int64)
    ok = cls == INLIER
    if ok.any():
        p = pts[ok]
        with np.errstate(all="ignore"):
            q = [((T[r, 0] * p[:, 0] + T[r, 1] * p[:, 1]) + T[r, 2] * p[:, 2]) + T[r, 3] for r in range(3)]
            u = np.float64(sK[0, 0]) * (q[0] / q[2]) + np.float64(sK[0, 2])
            v = np.float64(sK[1, 1]) * (q[1] / q[2]) + np.float64(sK[1, 2])
        zs = scene[np.floor(v + 0.5).astype(np.int64), np.floor(u + 0.5).astype(np.int64)].astype(np.float64)
        d = zs - q[2] * 1000.0
        e = np.minimum(np.abs(d), np.float64(clamp_mm))
        out[ok] = np.floor(e * 1000.0).astype(np.int64)
    return out


def cost(pts, T, scene, sK, clamp_mm):
    """A pose's cost: the point costs summed in int64 (exact in any order)."""
    return int(point_costs(pts, T, scene, sK, clamp_mm).sum())


def settings(particles=64, iterations=40, dt_mm=40.0, dr_deg=30.0, clamp_mm=20.0, seed=0):
    """lm_set_pose_search's conversion: (P, I, dt (m), dr (rad), clamp (mm), seed)."""
    return int(particles), int(iterations), np.float64(dt_mm) / 1000.0, np.float64(dr_deg) * DEG, float(clamp_mm), int(seed)


def search(pts, s, scene, sK, job=0, **opts):
    """The swarm of one job: (T [4,4], record dict as _lib.search_record gives it)."""
    P, I, dt, dr, clamp, seed = settings(**{**DEFAULTS, **opts})
    pts = np.asarray(pts, np.float64).reshape(-1, 3)
    s = np.asarray(s, np.float64).reshape(3)
    n = pts.shape[0]
    S = np.eye(4)
    S[:3, 3] = s
    c = centroid(pts, s)
    D = np.array([dr, dr, dr, dt, dt, dt])
    q = np.arange(6)
    x = np.zeros((P, 6))
    v = np.zeros((P, 6))
    p = np.zeros((P, 6))
    fp = np.full(P, INT64_MAX, np.int64)
    g = np.zeros(6)
    gi = -1
    trace = []
    np_ = P if I > 0 else 1
    fs = fg = None
    for k in range(max(I, 1)):
        for i in range(np_):
            if k == 0:
                if i > 0:
                    x[i] = (2.0 * D) * draw(seed, job, 0, i, q) - D
                p[i] = x[i]
            else:
                r1, r2 = draw(seed, job, k, i, q), draw(seed, job, k, i, 6 + q)
                nv = (W * v[i] + (C1 * r1) * (p[i] - x[i])) + (C2 * r2) * ((g if gi >= 0 else np.zeros(6)) - x[i])
                nv = np.where(nv > D, D, np.where(nv < -D, -D, nv))
                nx = x[i] + nv
                hi, lo = nx > D, nx < -D
                nx = np.where(hi, D, np.where(lo, -D, nx))
                nv = np.where(hi | lo, 0.0, nv)
                x[i], v[i] = nx, nv
        f = np.array([cost(pts, pose(x[i], c, s), scene, sK, clamp) for i in range(np_)], np.int64)
        if k == 0:
            fs = fg = int(f[0])
        if I > 0:
            better = f < fp
            fp[better] = f[better]
            p[better] = x[better]
            for i in range(P):
                if fp[i] < fg:
                    fg, gi = int(fp[i]), i
            if gi >= 0:
                g = p[gi].copy()
            trace.append(fg)
    T = S.copy() if gi < 0 else pose(g, c, s)
    if I == 0:
        x[:], v[:], p[:] = 0.0, 0.0, 0.0
    rec = dict(cost_start=fs, cost=fg, best=gi, c=c, trace=np.array(trace, np.int64), x=x, v=v, p=p,
               cost_best=fp if I > 0 else np.full(P, INT64_MAX, np.int64))
    rec["fitness"] = np.float64(fg) / np.float64(n) / 1000.0
    rec["rmse"] = np.float64(fs) / np.float64(n) / 1000.0
    return T, rec
