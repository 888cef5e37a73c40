"""numpy float64 model of view following (include/linemod_b200.h, lm_set_track_views / k_track_views): the threshold, the
object's rotation, every template's score, the decision and the re-expression of T, operation for operation.  Every
step is one correctly rounded IEEE operation in the order the header writes it (numpy float64 scalars never fuse), so
the comparison with the device is bit for bit."""
import math

import numpy as np


def tau(turn_deg):
    """Step 1 with Python's math.cos (libm, as the host's cos; np.cos may take a SIMD path)."""
    return 1.0 + 2.0 * math.cos(float(turn_deg) * 0.017453292519943295)


def dot3(a0, b0, a1, b1, a2, b2):
    return (a0 * b0 + a1 * b1) + a2 * b2


def rotation(T, Rk):
    """Step 2: Ro = T[:3, :3] Rk, each entry summed left to right."""
    T = np.asarray(T, np.float64).reshape(4, 4)
    Rk = np.asarray(Rk, np.float32).reshape(3, 3).astype(np.float64)
    Ro = np.zeros((3, 3))
    for r in range(3):
        for c in range(3):
            Ro[r, c] = dot3(T[r, 0], Rk[0, c], T[r, 1], Rk[1, c], T[r, 2], Rk[2, c])
    return Ro


def score(Ro, Rj):
    """Step 3: trace(Ro^T Rj) accumulated from 0.0, r outer, c inner."""
    Rj = np.asarray(Rj, np.float32).reshape(3, 3).astype(np.float64)
    s = np.float64(0.0)
    for r in range(3):
        for c in range(3):
            s = s + np.float64(Ro[r, c]) * Rj[r, c]
    return s


def scores(Ro, R_b):
    """Step 3 vectorised over templates R_b [n,3,3]: the same nine products and sums in the same order."""
    Rb = np.asarray(R_b, np.float32).reshape(-1, 9).astype(np.float64)
    s = np.zeros(Rb.shape[0])
    Rf = Ro.reshape(9)
    for q in range(9):
        s = s + Rf[q] * Rb[:, q]
    return s


def reexpress(T, Rk, tk, Rj, tj):
    """Step 5: T' = T [Q_R | Q_t], Q_R = Rk Rj^T, Q_t = b_k - Q_R b_j, b = t_b / 1000 on every axis."""
    T = np.asarray(T, np.float64).reshape(4, 4)
    Rk = np.asarray(Rk, np.float32).reshape(3, 3).astype(np.float64)
    Rj = np.asarray(Rj, np.float32).reshape(3, 3).astype(np.float64)
    bk = np.asarray(tk, np.float32).reshape(3).astype(np.float64) / 1000.0
    bj = np.asarray(tj, np.float32).reshape(3).astype(np.float64) / 1000.0
    QR = np.zeros((3, 3))
    for r in range(3):
        for c in range(3):
            QR[r, c] = dot3(Rk[r, 0], Rj[c, 0], Rk[r, 1], Rj[c, 1], Rk[r, 2], Rj[c, 2])
    Qt = np.array([bk[r] - dot3(QR[r, 0], bj[0], QR[r, 1], bj[1], QR[r, 2], bj[2]) for r in range(3)])
    out = np.eye(4)
    for r in range(3):
        for c in range(3):
            out[r, c] = dot3(T[r, 0], QR[0, c], T[r, 1], QR[1, c], T[r, 2], QR[2, c])
        out[r, 3] = dot3(T[r, 0], Qt[0], T[r, 1], Qt[1], T[r, 2], Qt[2]) + T[r, 3]
    return out


def choose(R_b, t_b, k, T, turn_deg, has=None):
    """Steps 2-5 for one object at template k of a class whose templates are R_b [n,3,3], t_b [n,3] (has [n]: which
    carry a render; None: all).  Returns (chosen template, T' [4,4], the scores, s_k, tau)."""
    R_b = np.asarray(R_b, np.float32).reshape(-1, 3, 3)
    t_b = np.asarray(t_b, np.float32).reshape(-1, 3)
    T = np.asarray(T, np.float64).reshape(4, 4)
    th = tau(turn_deg)
    with np.errstate(invalid="ignore", over="ignore"):  # a non-finite R_b gives a NaN score, which is no candidate
        Ro = rotation(T, R_b[k])
        s = scores(Ro, R_b)
    sk = s[k]
    if not (sk < th):
        return k, T.copy(), s, sk, th
    ok = ~np.isnan(s) if has is None else (~np.isnan(s) & np.asarray(has, bool))
    if not ok.any():
        return k, T.copy(), s, sk, th
    best = np.max(s[ok])
    j = int(np.nonzero(ok & (s == best))[0][0])
    if j == k or not (s[j] > sk):
        return k, T.copy(), s, sk, th
    with np.errstate(invalid="ignore", over="ignore"):  # an infinite R_b can win and give NaN entries, as on the device
        return j, reexpress(T, R_b[k], t_b[k], R_b[j], t_b[j]), s, sk, th
