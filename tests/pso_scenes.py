"""Synthetic scenes with a known pose for the particle-swarm estimation (tests/test_gpu_pose_pso.py, tools/pso_probe.py):
the recorded render's cloud (tests/golden/driver_trace.npz) supersampled 2x, moved by a seeded perturbation U{a, a}
(every rotation axis uniform in [-a, a] degrees about the cloud's centroid, every translation axis uniform in [-a, a] mm)
and z-buffer splatted, with a scene K unlike the render's, in front of a tilted table plane.  Each estimator refines the
unmoved render at the moved object's match position through lm_icp_process_batch.  Errors: the rotation angle of
R_est R_true^T (degrees) and the distance between where the estimated and the true motion put the render's centroid
(mm)."""
import numpy as np

ESTIMATIONS = ("pso", "point_to_plane", "point_to_point")
LEVELS = (10, 20, 30, 40)


def rodrigues(w):
    th = np.linalg.norm(w)
    if th == 0:
        return np.eye(3)
    k = w / th
    K = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + np.sin(th) * K + (1 - np.cos(th)) * K @ K


def render_cloud(render, K):
    """The render's pixels supersampled 2x (four sub-pixel samples at the pixel's depth), metres, camera frame."""
    r, c = np.nonzero(render)
    z = render[r, c].astype(np.float64) / 1000.0
    pts = []
    for dy in (-0.25, 0.25):
        for dx in (-0.25, 0.25):
            pts.append(np.stack([(c + dx - K[0, 2]) / K[0, 0] * z, (r + dy - K[1, 2]) / K[1, 1] * z, z], 1))
    return np.concatenate(pts)


def splat(pts, K, rows, cols, table):
    """Nearest-depth z-buffer of pts (m) in mm, over a tilted table plane (mm at each pixel)."""
    u = np.floor(K[0, 0] * pts[:, 0] / pts[:, 2] + K[0, 2] + 0.5).astype(np.int64)
    v = np.floor(K[1, 1] * pts[:, 1] / pts[:, 2] + K[1, 2] + 0.5).astype(np.int64)
    ok = (u >= 0) & (u < cols) & (v >= 0) & (v < rows) & (pts[:, 2] > 0)
    z = np.full(rows * cols, np.inf)
    np.minimum.at(z, v[ok] * cols + u[ok], pts[ok, 2] * 1000.0)
    z = np.minimum(z.reshape(rows, cols), table)
    return np.round(z).astype(np.uint16)


class Scenes:
    """The render, its K, R, t, its supersampled cloud M and centroid, the scene K and the table of the recorded frame."""

    def __init__(self, g):
        self.render, self.mK = g["render"], g["rf0_modelK"].astype(np.float64)
        self.R0, self.t0 = g["rf0_modelR"].astype(np.float32), g["rf0_modelT"].astype(np.float32).reshape(3)
        self.rows, self.cols = self.render.shape
        sK = self.mK.copy()
        sK[0, 0] *= 1.04
        sK[1, 1] *= 1.04
        sK[0, 2] += 6.0
        sK[1, 2] -= 4.0
        self.sK = sK
        self.M = render_cloud(self.render, self.mK)
        self.cM = self.M.mean(0)
        yy, xx = np.mgrid[0:self.rows, 0:self.cols]
        self.table = (self.cM[2] * 1000.0 + 60.0) + 0.08 * (yy - self.rows / 2) + 0.03 * (xx - self.cols / 2)
        r, c = np.nonzero(self.render)
        self.x0, self.y0 = int(c.min()), int(r.min())

    def case(self, a, rng):
        """One perturbation U{a, a}: (scene u16, match position [[x, y]], true motion T_true 4x4 of the camera-frame cloud)."""
        Rt = rodrigues(np.radians(rng.uniform(-a, a, 3)))
        tt = self.cM + rng.uniform(-a, a, 3) / 1000.0 - Rt @ self.cM
        scene = splat(self.M @ Rt.T + tt, self.sK, self.rows, self.cols, self.table)
        cs, cm, sK, mK = Rt @ self.cM + tt, self.cM, self.sK, self.mK
        du = sK[0, 0] * cs[0] / cs[2] + sK[0, 2] - (mK[0, 0] * cm[0] / cm[2] + mK[0, 2])
        dv = sK[1, 1] * cs[1] / cs[2] + sK[1, 2] - (mK[1, 1] * cm[1] / cm[2] + mK[1, 2])
        T = np.eye(4)
        T[:3, :3], T[:3, 3] = Rt, tt
        return scene, [[int(round(self.x0 + du)), int(round(self.y0 + dv))]], T

    def refine(self, icp, scene, xy):
        return icp.process_batch(scene, [self.render], self.sK.astype(np.float32), self.mK[None].astype(np.float32), self.R0[None],
                                 self.t0[None], xy, 30)

    def errors(self, T_true, Ro, to, res):
        """(rotation error in degrees, centroid error in mm) of lm_icp's output for one hypothesis; inf without a pose."""
        if res[0] == -1.0 or not np.isfinite(Ro[0]).all() or not np.isfinite(to[0]).all():
            return np.inf, np.inf
        # lm_icp returns T_est * init_base, init_base = [R0 | t0] with only t0.z in metres (LL.cpp:34-38)
        base = np.eye(4)
        base[:3, :3], base[:3, 3] = self.R0, self.t0
        base[2, 3] /= 1000.0
        got = np.eye(4)
        got[:3, :3], got[:3, 3] = Ro[0], to[0] / 1000.0
        T_est = got @ np.linalg.inv(base)
        dR = T_est[:3, :3] @ T_true[:3, :3].T
        ang = np.degrees(np.arccos(np.clip((np.trace(dR) - 1) / 2, -1, 1)))
        dc = np.linalg.norm((T_est[:3, :3] @ self.cM + T_est[:3, 3]) - (T_true[:3, :3] @ self.cM + T_true[:3, 3])) * 1000.0
        return float(ang), float(dc)


def accuracy(lib, g, cases, search, levels=LEVELS, estimations=ESTIMATIONS):
    """Per level and estimator: median, 90th percentile and maximum of both errors over `cases` seeded perturbations."""
    sc = Scenes(g)
    icps = {e: lib.NativeIcp() for e in estimations}
    for e, icp in icps.items():
        icp.set_estimation(e)
        icp.set_use_scene_cloud(e != "pso")
        icp.set_pose_search(*search)
    out = {}
    for a in levels:
        rng = np.random.default_rng(1000 + a)
        errs = {e: [] for e in estimations}
        for _ in range(cases):
            scene, xy, T = sc.case(a, rng)
            for e, icp in icps.items():
                errs[e].append(sc.errors(T, *sc.refine(icp, scene, xy)))
        out["U{%d,%d}" % (a, a)] = {}
        for e in estimations:
            rot, cen = np.array([v[0] for v in errs[e]]), np.array([v[1] for v in errs[e]])
            out["U{%d,%d}" % (a, a)][e] = dict(rot_deg_median=round(float(np.median(rot)), 3), rot_deg_p90=round(float(np.percentile(rot, 90)), 3),
                                               rot_deg_max=round(float(rot.max()), 3), centroid_mm_median=round(float(np.median(cen)), 3),
                                               centroid_mm_p90=round(float(np.percentile(cen, 90)), 3),
                                               centroid_mm_max=round(float(cen.max()), 3))
    return out
