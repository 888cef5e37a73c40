"""numpy float64 model of tracking's steps 1-3 (include/linemod_b200.h, lm_track): the pose -> T conversion, the window
the model cloud projects to under T, the statuses, and the window's scene cloud.  Every step is the same IEEE operation
as the device's (float64 numpy ufuncs are correctly rounded and never fused), so the comparison is bit for bit.  The
projection is pose verification's (tests/pose_verify_model.py), the back-projection and the voxel down-sampling the pose
stage's (tests/pose_cloud_model.py)."""
import numpy as np

import pose_cloud_model as pcm

TRACKED, OUTSIDE, WINDOW, NO_DEPTH = range(4)
NAMES = ("tracked", "outside", "window", "no_depth")


def pose_to_transform(R, t, R_b, t_b):
    """T of a pose (R [3,3], t [3] mm) of a template rendered at (R_b, t_b) (f32): T_R = R R_b^T, T_t = t / 1000 - T_R b,
    b = (t_b.x, t_b.y, float32(t_b.z / 1000)), summed left to right."""
    R = np.asarray(R, np.float64).reshape(3, 3)
    t = np.asarray(t, np.float64).reshape(3)
    Rb = np.asarray(R_b, np.float32).reshape(3, 3).astype(np.float64)
    tb = np.asarray(t_b, np.float32).reshape(3)
    b = np.array([tb[0], tb[1], tb[2] / np.float32(1000.0)], np.float64)
    TR = (R[:, 0:1] * Rb[:, 0][None]) + R[:, 1:2] * Rb[:, 1][None]
    TR = TR + R[:, 2:3] * Rb[:, 2][None]
    Tt = t / 1000.0 - (((TR[:, 0] * b[0]) + TR[:, 1] * b[1]) + TR[:, 2] * b[2])
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = TR, Tt
    return T


def init_base(R_b, t_b):
    """LL.cpp:34-38's init_base as float32 entries (only t.z in metres), widened."""
    base = np.eye(4, dtype=np.float32)
    base[:3, :3] = np.asarray(R_b, np.float32).reshape(3, 3)
    tb = np.asarray(t_b, np.float32).reshape(3)
    base[:3, 3] = [tb[0], tb[1], tb[2] / np.float32(1000.0)]
    return base.astype(np.float64)


def compose(T, R_b, t_b):
    """(R, t mm) of T * init_base, summed as lm_complete_pose sums them: s = 0.0, then + T[r][k] base[k][c], k = 0..3."""
    base = init_base(R_b, t_b)
    T = np.asarray(T, np.float64).reshape(4, 4)
    res = np.zeros((4, 4))
    for k in range(4):
        res = res + T[:, k:k + 1] * base[k][None]
    return res[:3, :3], res[:3, 3] * 1000.0


def model_cloud(render, mK):
    """Step 1: the pose stage's raw model cloud of the template (every crop pixel with depth > 0, row-major)."""
    from oracle import icp_oracle
    render = np.asarray(render, np.uint16)
    bx, by, bw, bh = icp_oracle.model_bbox(render)
    mK = np.asarray(mK, np.float32).reshape(3, 3)
    rr, cc = np.mgrid[0:bh, 0:bw]
    mr, mc = rr + by, cc + bx
    md = render[mr, mc]
    sel = md > 0
    z = md[sel].astype(np.float64) / 1000.0
    return np.stack([pcm.backproject(mc[sel], mK[0, 2], mK[0, 0], z), pcm.backproject(mr[sel], mK[1, 2], mK[1, 1], z), z], 1)


def project(pts, T, rows, cols, sK):
    """Verification's step 3: (in-frame mask, column, row) of every point under T."""
    T = np.asarray(T, np.float64).reshape(4, 4)
    sK = np.asarray(sK, np.float32).reshape(3, 3)
    px, py, pz = pts[:, 0], pts[:, 1], pts[:, 2]
    with np.errstate(all="ignore"):
        q = [((T[r, 0] * px + T[r, 1] * py) + T[r, 2] * pz) + T[r, 3] for r in range(3)]
        u = np.float64(sK[0, 0]) * (q[0] / q[2]) + np.float64(sK[0, 2])
        v = np.float64(sK[1, 1]) * (q[1] / q[2]) + np.float64(sK[1, 2])
        c = np.floor(u + 0.5)
        r = np.floor(v + 0.5)
        ok = (q[2] > 0) & np.isfinite(u) & np.isfinite(v) & (c >= 0) & (c < cols) & (r >= 0) & (r < rows)
    return ok, c, r


def window(pts, T, rows, cols, sK, margin, cap):
    """Step 2: (status, window (x, y, w, h), box (x, y, w, h)); OUTSIDE gives zeros, WINDOW a window of more than cap
    pixels (4 x the largest registered crop on the device)."""
    ok, c, r = project(pts, T, rows, cols, sK)
    if not ok.any():
        return OUTSIDE, (0, 0, 0, 0), (0, 0, 0, 0)
    x0, x1, y0, y1 = int(c[ok].min()), int(c[ok].max()), int(r[ok].min()), int(r[ok].max())
    box = (x0, y0, x1 - x0 + 1, y1 - y0 + 1)
    wx0, wy0 = max(x0 - margin, 0), max(y0 - margin, 0)
    wx1, wy1 = min(x1 + margin, cols - 1), min(y1 + margin, rows - 1)
    win = (wx0, wy0, wx1 - wx0 + 1, wy1 - wy0 + 1)
    return (WINDOW if win[2] * win[3] > cap else TRACKED), win, box


def scene_cloud(scene, sK, win):
    """Step 3: every window pixel with depth > 0, row-major, back-projected with sK (metres)."""
    sK = np.asarray(sK, np.float32).reshape(3, 3)
    x, y, w, h = win
    rr, cc = np.mgrid[y:y + h, x:x + w]
    d = scene[rr, cc]
    sel = d > 0
    z = d[sel].astype(np.float64) / 1000.0
    return np.stack([pcm.backproject(cc[sel], sK[0, 2], sK[0, 0], z), pcm.backproject(rr[sel], sK[1, 2], sK[1, 1], z), z], 1)


def track(scene, sK, render, mK, T, margin, cap):
    """Steps 1-3 for one object: a dict of status, window, box and, where TRACKED, raw_model / raw_scene and the
    down-sampled source / target with the ICP's start init = T."""
    scene = np.asarray(scene, np.uint16)
    rows, cols = scene.shape
    raw_model = model_cloud(render, mK)
    status, win, box = window(raw_model, T, rows, cols, sK, margin, cap)
    out = dict(status=status, window=win, box=box, raw_model=raw_model)
    if status != TRACKED:
        return out
    raw_scene = scene_cloud(scene, sK, win)
    if raw_scene.shape[0] == 0:
        out["status"] = NO_DEPTH
        return out
    out.update(raw_scene=raw_scene, source=pcm.voxel_down_sample_seq(raw_model), target=pcm.voxel_down_sample_seq(raw_scene),
               init=np.asarray(T, np.float64).reshape(4, 4))
    return out
