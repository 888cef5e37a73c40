"""A float64 model of the clouds poseRefine::process builds (LL.cpp:43-109), which the pose stage's k_pose_cloud,
segmented sort and k_pose_voxel compute for the detector and for lm_icp_process_batch(_device).

Every arithmetic step is the same IEEE operation as theirs, so the comparison is bit for bit:
  back-projection   f32 (c - cx) / f  (int -> f32, f32 subtract, f32 divide), widened, times the f64 z = d / 1000.0
  centroids         sequential f64 sums in row-major pixel order, divided by the count (0 / 0 -> NaN)
  voxel keys        floor((p - (min - 0.00125)) / 0.0025), sorted stably (x, y, z major to minor)
  voxel means       each voxel's points summed sequentially in sorted order, divided by the count
Scene and render may differ in size and intrinsics; the render's anchor is render[rows // 2][cols // 2].
"""
import numpy as np

from oracle import icp_oracle

HALF = 4                   # the 9 x 9 dilation (LL.cpp:43-50)
VOXEL = icp_oracle.VOXEL   # 0.0025 m
WINDOW = 0.4               # |z - anchor| < 0.4 m enters the scene centroid (LL.cpp:97)


def seq_sum(a):
    """Sum along axis 0 one term after another (np.cumsum is sequential; np.sum is pairwise)."""
    a = np.asarray(a, np.float64)
    return np.cumsum(a, 0)[-1] if a.shape[0] else np.zeros(a.shape[1:])


def voxel_keys(pts, voxel=VOXEL):
    """Per point its voxel index (int64 [n,3]) of PointCloud::VoxelDownSample."""
    origin = pts.min(0) - voxel * 0.5
    return np.floor((pts - origin) / voxel).astype(np.int64)


def voxel_runs(pts, voxel=VOXEL):
    """(order, starts, counts): the stable sort of the points by voxel key, and each occupied voxel's run in it."""
    idx = voxel_keys(pts, voxel)
    order = np.lexsort((idx[:, 2], idx[:, 1], idx[:, 0]))  # stable
    idx = idx[order]
    new = np.ones(len(idx), bool)
    new[1:] = np.any(idx[1:] != idx[:-1], 1)
    starts = np.nonzero(new)[0]
    return order, starts, np.diff(np.append(starts, len(idx)))


def voxel_down_sample_seq(pts, voxel=VOXEL):
    """icp_oracle.voxel_down_sample with every voxel summed sequentially in stable-sort order."""
    if pts.shape[0] == 0:
        return pts
    order, starts, counts = voxel_runs(pts, voxel)
    p = pts[order]
    acc = np.zeros((len(starts), 3))
    for k in range(int(counts.max())):
        sel = counts > k
        acc[sel] += p[starts[sel] + k]
    return acc / counts[:, None]


def backproject(pix, c, f, z):
    """(pix - c) / f in float32, widened and multiplied by the float64 z."""
    return ((np.asarray(pix).astype(np.float32) - np.float32(c)) / np.float32(f)).astype(np.float64) * z


def fits(box, x, y, srows, scols):
    """LL.cpp:52-55: the box placed at the match lies inside the frame (else the early return)."""
    return not (x + box[2] >= scols or y + box[3] >= srows)


def dilated(render):
    """dilate(render > 0, 9 x 9 ones)."""
    rows, cols = render.shape
    pad = np.pad(render > 0, HALF)
    out = np.zeros(render.shape, bool)
    for dy in range(2 * HALF + 1):
        for dx in range(2 * HALF + 1):
            out |= pad[dy:dy + rows, dx:dx + cols]
    return out


def clouds(scene, render, sK, mK, x, y, use_scene):
    """What the pose stage builds for a survivor at (x, y) whose template renders `render` with intrinsics mK, on a scene
    depth with intrinsics sK (both u16 mm).  Returns a dict: posed, box, and where posed raw_model / raw_scene [n,3]
    (row-major; raw_scene empty without use_scene), centroid_points (the scene points of the scene centroid), init 4x4,
    source / target (down-sampled; target is the source without use_scene) and counts (len(source), len(target))."""
    scene = np.asarray(scene, np.uint16)
    render = np.asarray(render, np.uint16)
    sK = np.asarray(sK, np.float32).reshape(3, 3)
    mK = np.asarray(mK, np.float32).reshape(3, 3)
    srows, scols = scene.shape
    box = icp_oracle.model_bbox(render)
    out = dict(posed=fits(box, x, y, srows, scols), box=box)
    if not out["posed"]:
        return out
    bx, by, bw, bh = box
    rr, cc = np.mgrid[0:bh, 0:bw]
    mr, mc = rr + by, cc + bx
    sr, sc = np.maximum(rr + y - HALF, 0), np.maximum(cc + x - HALF, 0)
    inmask = dilated(render)[mr, mc]
    md = render[mr, mc]
    sd = scene[sr, sc]
    m_sel = inmask & (md > 0)
    zm = md[m_sel].astype(np.float64) / 1000.0
    raw_model = np.stack([backproject(mc[m_sel], mK[0, 2], mK[0, 0], zm), backproject(mr[m_sel], mK[1, 2], mK[1, 1], zm), zm], 1)
    s_sel = inmask & (sd > 0)
    zs = sd.astype(np.float64) / 1000.0
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        xs, ys = backproject(sc, sK[0, 2], sK[0, 0], zs), backproject(sr, sK[1, 2], sK[1, 1], zs)
    scene_pts = np.stack([xs[s_sel], ys[s_sel], zs[s_sel]], 1)
    anchor = float(render[render.shape[0] // 2, render.shape[1] // 2]) / 1000.0
    c_sel = s_sel & (md > 0) & (np.abs(zs - anchor) < WINDOW)
    cpts = np.stack([xs[c_sel], ys[c_sel], zs[c_sel]], 1)
    with np.errstate(divide="ignore", invalid="ignore"):
        cm = seq_sum(raw_model) / np.float64(raw_model.shape[0])
        cs = seq_sum(cpts) / np.float64(cpts.shape[0])
    init = np.eye(4)
    init[:3, 3] = cs - cm
    src = voxel_down_sample_seq(raw_model)
    tgt = voxel_down_sample_seq(scene_pts) if use_scene else src
    out.update(raw_model=raw_model, raw_scene=scene_pts if use_scene else np.zeros((0, 3)), centroid_points=cpts, init=init,
               source=src, target=tgt, counts=(src.shape[0], tgt.shape[0]), anchor=anchor)
    return out
