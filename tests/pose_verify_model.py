"""numpy model of the pose verification (include/linemod_b200.h, lm_set_pose_verify) and the boundary cases its tests
run on.

Steps 1-6 of the header, one IEEE operation per step: float64 numpy ufuncs are correctly rounded and never fused, and
the score is one float32 division.  The model cloud is the oracle's restatement of the cloud building
(oracle/icp_oracle.build_clouds), before voxel down-sampling."""
import numpy as np

from oracle import icp_oracle

OUTSIDE, MISSING, INLIER, OCCLUDED, VIOLATION = range(5)
NAMES = ("outside", "missing", "inlier", "occluded", "violation")


def model_cloud(model, K):
    """Step 1: every crop pixel of render `model` (u16 mm) with depth > 0, back-projected with K (metres, row-major)."""
    bbox = icp_oracle.model_bbox(model)
    zero = np.zeros_like(model)
    return icp_oracle.build_clouds(zero, model, K, K, bbox[0] + 4, bbox[1] + 4, bbox)[0]


def classify(pts, T, scene, sK, delta):
    """Steps 3-4: one class per point of pts [n,3] under T (4x4) against scene (u16 mm) with intrinsics sK."""
    pts = np.asarray(pts, np.float64).reshape(-1, 3)
    T = np.asarray(T, np.float64).reshape(4, 4)
    sK = np.asarray(sK, np.float32).reshape(3, 3)
    rows, cols = scene.shape
    px, py, pz = pts[:, 0], pts[:, 1], pts[:, 2]
    cls = np.full(pts.shape[0], OUTSIDE, np.int64)
    with np.errstate(all="ignore"):
        q = [((T[r, 0] * px + T[r, 1] * py) + T[r, 2] * pz) + T[r, 3] for r in range(3)]
        front = q[2] > 0
        u = np.float64(sK[0, 0]) * (q[0] / q[2]) + np.float64(sK[0, 2])
        v = np.float64(sK[1, 1]) * (q[1] / q[2]) + np.float64(sK[1, 2])
        c = np.floor(u + 0.5)
        r = np.floor(v + 0.5)
        ok = front & np.isfinite(u) & np.isfinite(v) & (c >= 0) & (c < cols) & (r >= 0) & (r < rows)
        zs = scene[r[ok].astype(np.int64), c[ok].astype(np.int64)]
        d = zs.astype(np.float64) - q[2][ok] * 1000.0
    cls[ok] = np.where(zs == 0, MISSING, np.where(np.abs(d) <= delta, INLIER, np.where(d < 0, OCCLUDED, VIOLATION)))
    return cls


def verify(pts, T, scene, sK, delta):
    """Steps 3-5: (score float32, counts [6] int32 = n_model, outside, missing, inlier, occluded, violation)."""
    cls = classify(pts, T, scene, sK, delta)
    counts = np.array([cls.size] + [int((cls == k).sum()) for k in range(5)], np.int32)
    den = int(counts[1 + INLIER] + counts[1 + OCCLUDED] + counts[1 + VIOLATION])
    score = np.float32(counts[1 + INLIER]) / np.float32(den) if den else np.float32(0.0)
    return np.float32(score), counts


def no_pose():
    """What a survivor without a pose gets."""
    return np.float32(-1.0), np.zeros(6, np.int32)


# ---- boundary cases: name -> (pts [n,3], T [4,4], scene, sK, delta, expected classes) ----
ROWS, COLS = 6, 8
SK = np.array([[64.0, 0.0, 0.5], [0.0, 64.0, 0.5], [0.0, 0.0, 1.0]], np.float32)  # exact in binary: u = 64 x / z + 0.5


def _scene(z=500):
    return np.full((ROWS, COLS), z, np.uint16)


def _pt(col, row, z=0.5):
    """The point that projects (identity T, SK) exactly to u = col, v = row at depth z (m): x = (col - 0.5) z / 64."""
    return [(col - 0.5) * z / 64.0, (row - 0.5) * z / 64.0, z]


def boundary_cases():
    I = np.eye(4)
    cases = {}
    up, down = np.nextafter(10.0, np.inf), np.nextafter(10.0, 0.0)
    # |d| = delta exactly (z_q = 500 mm is exact), and delta one ulp either side of it
    for zs, name in ((510, "behind"), (490, "front")):
        sc = _scene(zs)
        far = VIOLATION if zs > 500 else OCCLUDED
        cases["d_eq_delta_%s" % name] = ([_pt(3, 2)], I, sc, SK, 10.0, [INLIER])
        cases["d_eq_delta_%s_delta_ulp_below" % name] = ([_pt(3, 2)], I, sc, SK, down, [far])
        cases["d_eq_delta_%s_delta_ulp_above" % name] = ([_pt(3, 2)], I, sc, SK, up, [INLIER])
    cases["delta_zero_exact"] = ([_pt(3, 2)], I, _scene(500), SK, 0.0, [INLIER])
    # u and v at x.5: floor(u + 0.5) rounds half up; -0.5 lands on column 0, one ulp less on -1
    cases["u_half"] = ([_pt(2.5, 1), _pt(3.5, 1), _pt(-0.5, 1), _pt(COLS - 0.5, 1)], I, _scene(500), SK, 10.0,
                       [INLIER, INLIER, INLIER, OUTSIDE])
    cases["v_half"] = ([_pt(1, 2.5), _pt(1, -0.5), _pt(1, ROWS - 0.5)], I, _scene(500), SK, 10.0, [INLIER, INLIER, OUTSIDE])
    below = _pt(-0.5, 1)
    below[0] = np.nextafter(below[0], -np.inf)
    cases["u_below_minus_half"] = ([below], I, _scene(500), SK, 10.0, [OUTSIDE])
    # q_z == 0, -0 and negative
    Tneg0 = np.eye(4)
    Tneg0[2, 3] = -0.0
    cases["qz_zero"] = ([[0.01, 0.01, 0.0]], I, _scene(), SK, 10.0, [OUTSIDE])
    cases["qz_negative_zero"] = ([[-0.01, -0.01, -0.0]], Tneg0, _scene(), SK, 10.0, [OUTSIDE])
    cases["qz_negative"] = ([[0.0, 0.0, -0.5]], I, _scene(), SK, 10.0, [OUTSIDE])
    cases["qz_tiny_u_infinite"] = ([[1e10, 0.0, 1e-300]], I, _scene(), SK, 10.0, [OUTSIDE])
    # each edge of the frame, from both sides
    cases["edges"] = ([_pt(0, 2), _pt(-1, 2), _pt(COLS - 1, 2), _pt(COLS, 2), _pt(3, 0), _pt(3, -1), _pt(3, ROWS - 1), _pt(3, ROWS)],
                      I, _scene(500), SK, 10.0, [INLIER, OUTSIDE, INLIER, OUTSIDE, INLIER, OUTSIDE, INLIER, OUTSIDE])
    # z_s == 0
    sc = _scene(500)
    sc[2, 3] = 0
    cases["scene_zero"] = ([_pt(3, 2), _pt(4, 2)], I, sc, SK, 10.0, [MISSING, INLIER])
    # a NaN pose (zero anchor depth) and an empty cloud
    Tnan = np.eye(4)
    Tnan[:3, 3] = np.nan
    cases["nan_pose"] = ([_pt(3, 2), _pt(4, 2)], Tnan, _scene(500), SK, 10.0, [OUTSIDE, OUTSIDE])
    cases["empty"] = (np.zeros((0, 3)), I, _scene(500), SK, 10.0, [])
    # a translation and a rotation: every class at once
    Tm = np.eye(4)
    Tm[:3, :3] = [[0.0, -1.0, 0.0], [1.0, 0.0, 0.0], [0.0, 0.0, 1.0]]
    Tm[2, 3] = 0.25
    sc = _scene(750)
    sc[0, 0] = 0
    sc[1, 1] = 700
    sc[2, 2] = 800
    p = lambda col, row: [(row - 0.5) * 0.75 / 64.0, -(col - 0.5) * 0.75 / 64.0, 0.5]  # R^T of the point at (col, row)
    cases["every_class"] = ([p(0, 0), p(1, 1), p(2, 2), p(3, 3), p(20, 3)], Tm, sc, SK, 10.0,
                            [MISSING, OCCLUDED, VIOLATION, INLIER, OUTSIDE])
    return {k: (np.asarray(v[0], np.float64).reshape(-1, 3), np.asarray(v[1], np.float64), v[2], v[3], float(v[4]),
                np.asarray(v[5], np.int64)) for k, v in cases.items()}
