"""Seeded depth-image cases for the ICP kernels and a brute-force float64 model of each of their stages.

Every case is a (scene, model render) pair that goes through the real cloud building (poseRefine's mask, box and
back-projection, then voxel down-sampling).  Most use a pixel pitch of about 3 mm, wider than the 2.5 mm voxel, so every
pixel is its own voxel and the down-sampled cloud has exactly as many points as the render has non-zero pixels.  The
scene is the render moved by (sx, sy) pixels and dz mm, and the match position puts it under the render, so the scene
cloud has the same count.

The model restates what k_icp_normals and k_icp_point_to_plane compute, by brute force over all pairs:
  knn_model / knn_valid   the 30 smallest (d^2, index) pairs of every target point
  normal_model            the smallest eigenvector of E[x x^T] - E[x] E[x]^T, summed in a given neighbour order
  corr_check              nearest target within the strict radius d^2 < 1e-4
  gn_step                 one Gauss-Newton step from given correspondences and normals
and checks one pass of the ICP loop from any pose T_k the kernel had (T_{k+1} = U T_k):
  check_plane_step        U against gn_step, relative to cond * eps * |x| plus the residuals' rounding (step_floor)
  check_point_step        U against a float64 Umeyama of the pass's pairs, relative to kappa * eps plus the points' rounding
  stop_pass               the pass the stop rule ends on, from the fitness and rmse of every pass
The kernels' squared distances and sums may be FMA-contracted, so where a decision compares two of them the model
accepts either answer inside a band of a few ulps (BAND).
"""
from dataclasses import dataclass, field

import numpy as np

from oracle import icp_oracle
import pose_cloud_model
from pose_cloud_model import seq_sum, voxel_down_sample_seq  # noqa: F401 (the model's, re-exported)

KNN = 30
MAX_D2 = icp_oracle.MAX_DIST ** 2
EPS = np.finfo(np.float64).eps
BAND = 8 * EPS          # relative band on a squared distance computed with or without FMA
H, W = 480, 640         # render and scene size


@dataclass
class Case:
    name: str
    scene: np.ndarray
    model: np.ndarray
    K: np.ndarray
    R: np.ndarray
    t: np.ndarray
    xy: tuple
    n_model: int = None       # intended down-sampled model cloud size (None: decided by rounding)
    n_scene: int = None       # the same for the scene cloud
    exact_ties: bool = False  # squared distances are exact in float64: equal ones tie exactly
    planar: bool = False      # every normal is exactly (0, 0, +-1): J^T J is exactly singular
    flat: bool = False        # a plane: J^T J is singular or nearly so, one step is not comparable
    info: dict = field(default_factory=dict)


def _K(f, cx=W / 2, cy=H / 2):
    return np.array([[f, 0, cx], [0, f, cy], [0, 0, 1]], np.float32)


def _case(name, mask, depth_mm, f, shift=(1, 1), dz=2, unique=True, **kw):
    """mask: HxW bool, depth_mm: HxW array (rounded to u16 mm).  The scene is the render moved by shift=(sx, sy)
    pixels and dz mm; the match position puts the moved render under the box."""
    model = np.where(mask, np.rint(depth_mm), 0).astype(np.uint16)
    sx, sy = shift
    scene = np.roll(np.roll(model, sy, 0), sx, 1).astype(np.int32)
    scene = np.where(scene > 0, scene + dz, 0).astype(np.uint16)
    bx, by, bw, bh = icp_oracle.model_bbox(model)
    xy = (bx + 4 + sx, by + 4 + sy)
    n = int(mask.sum())
    c = Case(name, scene, model, _K(f), np.eye(3, dtype=np.float32), np.array([0, 0, float(depth_mm[H // 2, W // 2])], np.float32),
             xy, n if unique else None, n if unique else None, **kw)
    return c


def _yx():
    return np.mgrid[0:H, 0:W].astype(np.float64)


def disk_mask(n, cx=W // 2, cy=H // 2, aspect=1.0):
    """The n pixels nearest to (cx, cy) (elliptical distance, ties by row then column)."""
    yy, xx = _yx()
    d = ((xx - cx) / aspect) ** 2 + (yy - cy) ** 2
    order = np.lexsort((xx.ravel(), yy.ravel(), d.ravel()))[:n]
    m = np.zeros(H * W, bool)
    m[order] = True
    return m.reshape(H, W)


def blob_depth(seed, z0=300.0, cx=W // 2, cy=H // 2, R=45.0):
    """A bowl of radius R pixels, 5 to 11 mm deep, with a ripple.  Its slope times the distance from the principal point
    stays small, so neighbouring pixels stay more than 2.5 mm apart at 3 mm pitch (test_icp_model checks the counts)."""
    rng = np.random.default_rng(seed)
    yy, xx = _yx()
    a, b, p = rng.uniform(0.6, 1.4), rng.uniform(0.6, 1.4), rng.uniform(0, 6)
    rho2 = ((xx - cx) / R) ** 2 + ((yy - cy) / R) ** 2
    return z0 + 8.0 * a * rho2 + 2.5 * b * np.sin((xx - cx) / 11.0 + p) * np.cos((yy - cy) / 13.0)


SIZES = (1, 2, 3, 29, 30, 31, 127, 128, 129, 255, 256, 257, 511, 512, 513, 1025, 6000)


def size_case(n):
    """A disk of n pixels on a bowl of the disk's own radius, so that even small disks stay curved after the depth is
    rounded to whole millimetres."""
    return _case("size_%d" % n, disk_mask(n), blob_depth(n, R=np.sqrt(n / np.pi) + 1), 100.0)


def strip_x_case(length=400):
    """3 pixels high, long in x: a 256-point tile covers 85 columns, so most tiles are pruned.  Depth is constant along x
    (it varies from row to row), which keeps neighbouring columns 3 mm apart at either end of the strip."""
    m = np.zeros((H, W), bool)
    m[H // 2 - 1:H // 2 + 2, W // 2 - length // 2:W // 2 + length // 2] = True
    yy, _ = _yx()
    return _case("strip_x", m, 300.0 + 2.0 * ((yy - H // 2) % 3) ** 2, 100.0)


def strip_y_case(length=400):
    """3 pixels wide, long in y: three voxel columns of 400 points each, so almost nothing is pruned.  Depth varies from
    column to column only."""
    m = np.zeros((H, W), bool)
    m[H // 2 - length // 2:H // 2 + length // 2, W // 2 - 1:W // 2 + 2] = True
    _, xx = _yx()
    return _case("strip_y", m, 300.0 + 2.0 * ((xx - W // 2) % 3) ** 2, 100.0)


def clusters_case(small=12, large=512, gap_px=20, width=4, scene_move=0, scene_ramp=False):
    """A large blob of exactly `large` points (a multiple of 256), and `gap_px` empty columns to its right a 3 x 4 cluster
    of `small` < 30 points.  The small cluster sorts last, alone in the last 256-point tile: its points start with
    `small` neighbours and have to cross the gap for the other 30 - small.  scene_move moves the small cluster by that many
    columns in the scene only: with the scene cloud as the target, its correspondences are then 3 * scene_move mm away,
    in a tile of their own; scene_ramp puts row k of the moved cluster k mm deeper."""
    big = disk_mask(large)
    cols = np.nonzero(big.any(0))[0]
    c0 = cols.max() + 1 + gap_px
    m = big.copy()
    hs = small // width
    m[H // 2 - hs // 2:H // 2 - hs // 2 + hs, c0:c0 + width] = True
    assert m.sum() == large + small
    name = "clusters_%d_%d_gap%d" % (large, small, gap_px) + ("_move%+d" % scene_move if scene_move else "") + ("_ramp" if scene_ramp else "")
    c = _case(name, m, blob_depth(7), 100.0)
    if scene_move:
        cols = slice(c0 + 1, c0 + 1 + width)  # the scene is the render moved by (1, 1)
        rows = slice(H // 2 - hs // 2 + 1, H // 2 - hs // 2 + hs + 1)
        part = c.scene[rows, cols].copy()
        if scene_ramp:  # row k of the moved cluster k mm deeper: its distances straddle the 1 cm radius
            part = np.where(part > 0, part + np.arange(hs)[:, None], 0).astype(np.uint16)
        c.scene[rows, cols] = 0
        c.scene[rows, cols.start + scene_move:cols.stop + scene_move] = part
    c.info.update(large=large, small=small, gap_px=gap_px, straddle=scene_ramp)
    return c


def lo_gap_case(gap_px=6, step_rows=3, arows=20, brows=16, bcols=12, ca=W // 2 + 100):
    """The lo-side pruning bound of k_icp_normals: a point of voxel column a has x in [lo_a, lo_a + 2.5 mm), so the last
    point of a tile may have up to one voxel less x than points before it.  Cluster A is exactly 256 points (tile 0); its
    last voxel column holds two pixels of image column ca, 100 pixels right of the principal point, where x = z: the
    upper one 2 mm deeper, so 2 mm further right, and sorted first.  Cluster B (tile 1) starts gap_px columns to the right
    with its top-left corner on the row of the deeper pixel, which is among the 30 nearest neighbours of that corner,
    while every point of B's first block is farther in x from the tile's last point than its 30th neighbour."""
    m = np.zeros((H, W), bool)
    d = np.full((H, W), 300.0)
    r1 = H // 2 - 40
    acols = -(-254 // arows)  # A's rectangle, filled from column ca - 1 leftwards
    pix = [(r, c) for c in range(ca - 1, ca - 1 - acols, -1) for r in range(r1 - arows // 2, r1 - arows // 2 + arows)][:254]
    m[tuple(np.array(pix).T)] = True
    m[r1, ca] = m[r1 + step_rows, ca] = True
    d[r1, ca] = 302.0
    m[r1:r1 + brows, ca + gap_px:ca + gap_px + bcols] = True
    c = _case("lo_gap", m, d, 100.0, flat=True)
    c.info.update(acols=acols)
    return c


def pitch_plane_case():
    """A plane at z = 0.25 m with a 1.25 mm pixel pitch: two to three pixels per voxel column, many of them on a voxel
    boundary, where the rounding of (x - origin) / 0.0025 decides the column."""
    m = disk_mask(1600, aspect=1.3)
    return _case("pitch_1.25mm", m, np.full((H, W), 250.0), 200.0, unique=False, flat=True)


def tie_grid_case():
    """A plane at z = 0.25 m with f = 64: x = (c - cx) / 64 * 0.25 and y are exact, so every squared distance is exact
    and a regular grid has many exactly equidistant neighbours; the normals are exactly (0, 0, 1)."""
    m = disk_mask(700)
    c = _case("tie_grid", m, np.full((H, W), 250.0), 64.0, dz=0, exact_ties=True, planar=True, flat=True)
    return c


def shape_cases():
    return [strip_x_case(), strip_y_case(), clusters_case(), clusters_case(small=20, large=256, gap_px=6),
            clusters_case(small=12, large=512, gap_px=2), clusters_case(small=12, large=2048, gap_px=20, width=1, scene_move=2, scene_ramp=True),
            lo_gap_case(), pitch_plane_case(), tie_grid_case()]


def all_cases():
    return [size_case(n) for n in SIZES] + shape_cases()


# ------------------------------------------------------------------------------------------------------------------
# clouds as poseRefine builds them, with sequential sums (the host's order): tests/pose_cloud_model.py
# ------------------------------------------------------------------------------------------------------------------
def host_clouds(c, use_scene):
    """(source, target, init 4x4, oracle init) of case c: the clouds and initial guess lm_icp_process_batch builds."""
    m = pose_cloud_model.clouds(c.scene, c.model, c.K, c.K, c.xy[0], c.xy[1], use_scene)
    _, cm_np, cs_np, _ = icp_oracle.build_clouds(c.scene, c.model, c.K, c.K, c.xy[0], c.xy[1], m["box"])
    init_np = np.eye(4)
    init_np[:3, 3] = cs_np - cm_np
    return m["source"], m["target"], m["init"], init_np


# ------------------------------------------------------------------------------------------------------------------
# neighbour sets and normals
# ------------------------------------------------------------------------------------------------------------------
def pair_d2(A, B):
    """Squared distances, (dx*dx + dy*dy) + dz*dz in float64 without contraction."""
    d = A[:, None, :] - B[None, :, :]
    return (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]


def knn_model(P, k=KNN, chunk=512):
    """For every point of P: the min(k, n) smallest (d^2, index) pairs (indices, d^2), and the (k+1)-th d^2 (inf if none)."""
    n = P.shape[0]
    kk = min(k, n)
    idx = np.zeros((n, kk), np.int64)
    d2k = np.zeros((n, kk))
    nxt = np.full(n, np.inf)
    ar = np.arange(n)
    for s in range(0, n, chunk):
        D = pair_d2(P[s:s + chunk], P)
        o = np.lexsort((np.broadcast_to(ar, D.shape), D), axis=1)
        idx[s:s + chunk] = o[:, :kk]
        d2k[s:s + chunk] = np.take_along_axis(D, o[:, :kk], 1)
        if n > kk:
            nxt[s:s + chunk] = np.take_along_axis(D, o[:, kk:kk + 1], 1)[:, 0]
    return idx, d2k, nxt


def knn_check(P, kept, chunk=512):
    """For captured neighbour lists kept (n x 30, -1 padded): per point, (the model d^2 of the kept list, the smallest d^2
    left out).  knn_valid is max(kept) <= min(left out) within BAND."""
    n = P.shape[0]
    kk = min(KNN, n)
    kd2 = np.full(kept.shape, np.nan)
    out_min = np.full(n, np.inf)
    for s in range(0, n, chunk):
        D = pair_d2(P[s:s + chunk], P)
        ks = kept[s:s + chunk, :kk]
        kd2[s:s + chunk, :kk] = np.take_along_axis(D, np.clip(ks, 0, n - 1), 1)
        Dm = D.copy()
        np.put_along_axis(Dm, np.clip(ks, 0, n - 1), np.inf, 1)
        out_min[s:s + chunk] = Dm.min(1) if n > kk else np.inf
    return kd2, out_min


def knn_valid(kd2, out_min):
    mx = np.nanmax(kd2, 1)
    return mx <= out_min + BAND * mx


def covariance(P, idx, have):
    """Per point: E[x x^T] - E[x] E[x]^T of P[idx[i, :have[i]]], summed in list order exactly as k_icp_normals does."""
    n = idx.shape[0]
    c = np.zeros((n, 9))
    for k in range(idx.shape[1]):
        live = have > k
        q = P[np.where(live, idx[:, k], 0)]
        x, y, z = q[:, 0], q[:, 1], q[:, 2]
        add = np.stack([x, y, z, x * x, x * y, x * z, y * y, y * z, z * z], 1)
        c[live] += add[live]
    c /= np.maximum(have, 1)[:, None]
    C = np.empty((n, 3, 3))
    C[:, 0, 0] = c[:, 3] - c[:, 0] * c[:, 0]
    C[:, 0, 1] = C[:, 1, 0] = c[:, 4] - c[:, 0] * c[:, 1]
    C[:, 0, 2] = C[:, 2, 0] = c[:, 5] - c[:, 0] * c[:, 2]
    C[:, 1, 1] = c[:, 6] - c[:, 1] * c[:, 1]
    C[:, 1, 2] = C[:, 2, 1] = c[:, 7] - c[:, 1] * c[:, 2]
    C[:, 2, 2] = c[:, 8] - c[:, 2] * c[:, 2]
    return C, np.abs(c[:, 3:]).max(1)


NORMAL_TOL = 1e-9


def normal_model(P, idx, have):
    """(normals, comparable, degenerate, v_max).  The normal is the eigenvector of the smallest eigenvalue.  A normal is
    comparable when the bound have * u * max|E[x x^T]| on the covariance's rounding, over the gap between the two
    smallest eigenvalues, is at most NORMAL_TOL / 10.  Degenerate neighbourhoods (a zero second eigenvalue: collinear
    points) only fix the normal's plane: v_max is the eigenvector it has to be orthogonal to."""
    C, scale = covariance(P, idx, have)
    w, v = np.linalg.eigh(C)
    nrm = v[:, :, 0].copy()
    gap = w[:, 1] - w[:, 0]
    pert = have * (EPS / 2) * scale
    comparable = (have >= 3) & (pert <= 0.1 * NORMAL_TOL * gap)
    degenerate = (have >= 3) & ~comparable & (pert <= 0.1 * NORMAL_TOL * (w[:, 2] - w[:, 1]))
    nrm[have < 3] = (0.0, 0.0, 1.0)
    return nrm, comparable, degenerate, v[:, :, 2]


def model_normals(P):
    """Normals of P from the model's own neighbour sets (30 smallest (d^2, index), in that order)."""
    idx, _, _ = knn_model(P)
    have = np.full(P.shape[0], idx.shape[1])
    return normal_model(P, idx, have)[0], idx


# ------------------------------------------------------------------------------------------------------------------
# correspondences and one Gauss-Newton step
# ------------------------------------------------------------------------------------------------------------------
def transform(T, S):
    return S @ T[:3, :3].T + T[:3, 3]


def corr_check(Ps, Q, corr, chunk=1024):
    """Ps: the source transformed by the pass's T; corr: captured target index per source point (-1: none).  Returns a
    dict of boolean arrays: ok (the captured index is a nearest target within the radius, or -1 is allowed), and the
    recomputed squared distance of every pair."""
    n = Ps.shape[0]
    ok = np.zeros(n, bool)
    d2 = np.full(n, np.nan)
    # the kernel's transformed points may differ from these by a few ulps of |p|: a band on d^2 of 2 |d| dp + BAND d^2
    dp = 8 * EPS * np.abs(Ps).max() if n else 0.0
    for s in range(0, n, chunk):
        D = pair_d2(Ps[s:s + chunk], Q)
        dmin = D.min(1)
        c = corr[s:s + chunk]
        dc = np.where(c >= 0, np.take_along_axis(D, np.clip(c, 0, None)[:, None], 1)[:, 0], np.inf)
        band = lambda x: BAND * x + 4 * np.sqrt(x) * dp
        near = dc <= dmin + band(dmin)
        inside = dc < MAX_D2 + band(MAX_D2)
        none_ok = dmin >= MAX_D2 - band(MAX_D2)
        ok[s:s + chunk] = np.where(c >= 0, near & inside, none_ok)
        d2[s:s + chunk] = np.where(c >= 0, dc, np.nan)
    return ok, d2


def gn_step(Ps, Q, Nq, corr, full=False):
    """One Gauss-Newton step of point-to-plane ICP from given correspondences (float64).  Returns (x or None when J^T J
    is exactly singular, cond(J^T J)), and with full=True also the step's rounding floor (step_floor) and whether J^T J
    has an exactly zero row (no pair, or a column of J zero in every pair: singular in any elimination order)."""
    si = np.nonzero(corr >= 0)[0]
    vs, vt, nt = Ps[si], Q[corr[si]], Nq[corr[si]]
    r = ((vs - vt) * nt).sum(1)
    J = np.concatenate([np.cross(vs, nt), nt], 1)
    JTJ, JTr = J.T @ J, J.T @ r
    zero_row = bool((JTJ == 0).all(1).any())
    try:
        x = np.linalg.solve(JTJ, -JTr)
    except np.linalg.LinAlgError:
        return (None, np.inf, np.inf, zero_row) if full else (None, np.inf)
    cond = float(np.linalg.cond(JTJ))
    if not full:
        return x, cond
    return x, cond, step_floor(JTJ, J, vs, vt), zero_row


def step_floor(JTJ, J, vs, vt):
    """||(J^T J)^-1||_2 * sum_i ||J_i|| * eps * (|p_i|_inf + |q_i|_inf): how far the rounding of the residuals
    r_i = (p_i - q_i) . n_i alone moves the solution.  A step relative to |x| cannot bound a converged pass, where |x|
    is down to the residuals' own rounding; this term does."""
    inv = 1.0 / float(np.linalg.svd(JTJ, compute_uv=False)[-1])
    mag = np.abs(vs).max(1) + np.abs(vt).max(1)
    return inv * float((np.linalg.norm(J, axis=1) * EPS * mag).sum())


def update_of(T1, T0):
    """The update U with T1 = U @ T0, for rigid T0 (its rotation block transposed, not inverted)."""
    U = np.eye(4)
    U[:3, :3] = T1[:3, :3] @ T0[:3, :3].T
    U[:3, 3] = T1[:3, 3] - U[:3, :3] @ T0[:3, 3]
    return U


def principal_angles(x):
    """x with the angles step_from_T recovers from TransformVector6dToMatrix4d(x): x1 in [-pi/2, pi/2], x0 and x2 in
    [-pi, pi].  A diverging step (an ill-conditioned J^T J) can leave that branch; (x0 + pi, pi - x1, x2 + pi) is the
    same rotation.  x is returned unchanged, without rounding, when it is inside."""
    a = np.array(x[:3], np.float64)
    if np.all(np.abs(a) <= [np.pi, np.pi / 2, np.pi]):
        return np.asarray(x, np.float64)
    wrap = lambda v: (v + np.pi) % (2 * np.pi) - np.pi
    a = wrap(a)
    if abs(a[1]) > np.pi / 2:
        a = wrap(np.array([a[0] + np.pi, np.pi - a[1], a[2] + np.pi]))
    return np.concatenate([a, np.asarray(x[3:], np.float64)])


def step_from_T(T1, T0):
    """The 6-vector x with T1 = TransformVector6dToMatrix4d(x) @ T0, for any rigid T0 (for T0 = [I | c] the rotation
    is T1's own, exactly)."""
    U = update_of(T1, T0)
    t = U[:3, 3]
    return np.array([np.arctan2(U[2, 1], U[2, 2]), np.arcsin(-U[2, 0]), np.arctan2(U[1, 0], U[0, 0]), t[0], t[1], t[2]])


# ------------------------------------------------------------------------------------------------------------------
# the update of pass k: T_{k+1} = U T_k from the pairs of pass k
# ------------------------------------------------------------------------------------------------------------------
STEP_COND_MAX = 1e10  # point-to-plane steps of a J^T J above this condition number are not compared
STOP_TOL = 1e-6      # the stop rule's thresholds (ICPConvergenceCriteria's relative_fitness and relative_rmse)


def proper_rotation(R, tol=1e-12):
    return bool(np.all(np.isfinite(R)) and abs(np.linalg.det(R) - 1) <= tol and np.abs(R @ R.T - np.eye(3)).max() <= tol)


def check_plane_step(key, src, tgt, normals, T0, T1, corr, K, floor=True):
    """The point-to-plane update of one pass, T1 = U T0, against gn_step from the pass's pairs corr at T0.  Returns
    (outcome, ratio, cond): "singular" (J^T J has an exactly zero row: T1 == T0 bit for bit), "cond" (singular to
    rounding, or cond(J^T J) above STEP_COND_MAX: U need only be a proper rotation) or "compared", where
        |x_kernel - x_model|_inf <= K (cond eps |x|_inf + floor) + recover
    (floor: step_floor, or none with floor=False; recover: the rounding of step_from_T) and ratio is the error over the
    bracket."""
    x_m, cond, fl, zero_row = gn_step(transform(T0, src), tgt, normals, corr, full=True)
    if zero_row:
        assert np.array_equal(T1, T0), "step %s: singular J^T J must give the identity update" % key
        return "singular", None, cond
    U = update_of(T1, T0)
    assert np.all(np.isfinite(U)) and proper_rotation(U[:3, :3]), "step %s: the update is not a proper rotation" % key
    if x_m is None or cond > STEP_COND_MAX:  # singular to rounding only: the kernel's elimination may not see it
        return "cond", None, cond
    x_k, x_m = step_from_T(T1, T0), principal_angles(x_m)
    err = float(np.abs(x_k - x_m).max())
    scale = cond * EPS * float(np.abs(x_m).max()) + (fl if floor else 0.0)
    recover = 16 * EPS * (1 + float(np.abs(T0).max()))
    ratio = err / max(scale, 1e-300)
    assert err <= K * scale + recover, "step %s: %r, model %r (cond %.3g, ratio %.3g)" % (key, x_k, x_m, cond, ratio)
    return "compared", ratio, cond


def umeyama_model(p, q):
    """Two-pass float64 Umeyama: (R, t, singular values d, s = det U det V sign, pbar)."""
    pb, qb = p.mean(0), q.mean(0)
    sig = (q - qb).T @ (p - pb) / p.shape[0]
    U, d, Vt = np.linalg.svd(sig)
    s = -1.0 if np.linalg.det(U) * np.linalg.det(Vt) < 0 else 1.0
    R = (U * [1.0, 1.0, s]) @ Vt
    return R, qb - R @ pb, d, s, pb


def p2p_cost(R, t, p, q):
    return float(((p @ R.T + t - q) ** 2).sum())


def check_point_step(key, src, tgt, T0, T1, corr, K, floor=True):
    """The point-to-point update of one pass, T1 = U T0, against umeyama_model of the pass's pairs at T0.  Returns
    (outcome, ratio, kappa): "empty" (no pair: T1 == T0 bit for bit), "degenerate" (one or two pairs, or collinear ones:
    any proper rotation at the model's minimum cost; one pair keeps R exactly) or "compared", where with
    kappa = d1 / (d2 + s d3) of the pairs' covariance
        |R_kernel - R_model|_inf <= K (kappa eps + floor),   |t_kernel - t_model|_inf <= K (1 + |pbar|_inf)(kappa eps + floor)
    floor = eps sum_i (|p_i - pbar| + |q_i - qbar|)(|p_i|_inf + |q_i|_inf) / (n (d2 + s d3)): the rounding of the points
    themselves through the covariance (none with floor=False), and ratio is the larger error over its bracket."""
    si = np.nonzero(corr >= 0)[0]
    if si.size == 0:
        assert np.array_equal(T1, T0), "step %s: no pair must give the identity update" % key
        return "empty", None, None
    p, q = transform(T0, src)[si], tgt[corr[si]]
    upd = update_of(T1, T0)
    Rk, tk = upd[:3, :3], upd[:3, 3]
    assert np.all(np.isfinite(upd)), "step %s: %r" % (key, upd)
    Rm, tm, d, s, pb = umeyama_model(p, q)
    if si.size == 1:
        assert np.array_equal(T1[:3, :3], T0[:3, :3]), "step %s: one pair must give R = I exactly" % key
    gap = d[1] + s * d[2]
    if si.size < 3 or not gap > 1e-9 * d[0]:
        assert proper_rotation(Rk), "step %s: %r is not a proper rotation" % (key, Rk)
        cm, ck = p2p_cost(Rm, tm, p, q), p2p_cost(Rk, tk, p, q)
        scale = float(((p - p.mean(0)) ** 2).sum() + ((q - q.mean(0)) ** 2).sum())
        assert ck <= cm + 1e-12 * scale + 1e-24, "step %s: cost %r, minimum %r" % (key, ck, cm)
        return "degenerate", None, None
    kappa = d[0] / gap
    fl = 0.0
    if floor:
        spread = np.linalg.norm(p - pb, axis=1) + np.linalg.norm(q - q.mean(0), axis=1)
        fl = EPS * float((spread * (np.abs(p).max(1) + np.abs(q).max(1))).sum()) / (p.shape[0] * gap)
    bracket = kappa * EPS + fl
    eR = float(np.abs(Rk - Rm).max()) / bracket
    et = float(np.abs(tk - tm).max()) / ((1 + float(np.abs(pb).max())) * bracket)
    assert eR <= K and et <= K, "step %s: R ratio %.3g, t ratio %.3g (kappa %.3g)" % (key, eR, et, kappa)
    return "compared", max(eR, et), kappa


def stop_pass(fits, rmses, max_iter):
    """The pass RegistrationICP stops at, from the fitness and rmse of passes 0, 1, ...: the first k >= 1 with
    |f_{k-1} - f_k| < 1e-6 and |r_{k-1} - r_k| < 1e-6 (strict, float64), capped at max_iter.  None when the passes
    given end before either."""
    for k in range(0, len(fits)):
        if k >= 1 and abs(fits[k - 1] - fits[k]) < STOP_TOL and abs(rmses[k - 1] - rmses[k]) < STOP_TOL:
            return k
        if k >= max_iter:
            return k
    return None
