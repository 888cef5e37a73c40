"""CPU restatement of poseRefine::process's point-to-point branch (LL.cpp:131-135, compiled without USE_OPEN3D_P2PL):
RegistrationICP with TransformationEstimationPointToPoint and no normals -- TEST INFRASTRUCTURE ONLY, the counterpart of
oracle/icp_oracle.py's point-to-plane restatement, whose cloud building, voxel down-sampling and constants it reuses.

PARITY UNPINNED, as the rest of the ICP oracle: Open3D and Eigen are not in the reference.  The estimation step is
restated [3p, from memory] of Open3D 0.8/0.9 (TransformationEstimationPointToPoint::ComputeTransformation with
with_scaling = false) and Eigen 3.3 (umeyama(source, target, false)):
  no correspondences: the identity;
  pbar, qbar = the means of the corresponding source / target points;
  sig = (1/n) sum (q - qbar)(p - pbar)^T  (two passes here: no cancellation);
  sig = U diag(d) V^T by a 3x3 SVD, d descending;  S = diag(1, 1, -1) if det U * det V < 0, else I;
  R = U S V^T, t = qbar - R pbar.
"""
import numpy as np
from scipy.spatial import cKDTree

from oracle import icp_oracle


def umeyama(p, q):
    """The update of one pass: p, q [n, 3] f64 (the source points already transformed by the current T, and their
    targets).  Returns the 4x4 update."""
    T = np.eye(4)
    p = np.asarray(p, np.float64).reshape(-1, 3)
    q = np.asarray(q, np.float64).reshape(-1, 3)
    if p.shape[0] == 0:
        return T
    pb, qb = p.mean(0), q.mean(0)
    sig = (q - qb).T @ (p - pb) / p.shape[0]
    U, d, Vt = np.linalg.svd(sig)
    S = np.ones(3)
    if np.linalg.det(U) * np.linalg.det(Vt) < 0:
        S[2] = -1.0
    R = (U * S) @ Vt
    T[:3, :3] = R
    T[:3, 3] = qb - R @ pb
    return T


def registration_icp_p2p(src, tgt, max_d, init, max_iter=icp_oracle.MAX_ITER, rel_fitness=icp_oracle.REL_FITNESS,
                         rel_rmse=icp_oracle.REL_RMSE):
    """RegistrationICP(..., TransformationEstimationPointToPoint(false)): the loop of icp_oracle.registration_icp_p2pl with
    umeyama as the update.  Returns (T 4x4, fitness, rmse, iterations)."""
    T = np.array(init, np.float64)
    if src.shape[0] == 0 or tgt.shape[0] == 0:
        return T, 0.0, 0.0, 0
    tree = cKDTree(tgt)
    p = src @ T[:3, :3].T + T[:3, 3]

    def correspond(p):
        d, j = tree.query(p, k=1)
        ok = d * d < max_d * max_d  # radius search is strict in FLANN
        n = int(ok.sum())
        rmse = float(np.sqrt((d[ok] ** 2).sum() / n)) if n else 0.0
        return np.nonzero(ok)[0], j[ok], n / p.shape[0], rmse

    si, tj, fit, rmse = correspond(p)
    it = 0
    for it in range(1, max_iter + 1):
        upd = umeyama(p[si], tgt[tj])
        T = upd @ T
        p = p @ upd[:3, :3].T + upd[:3, 3]
        fit0, rmse0 = fit, rmse
        si, tj, fit, rmse = correspond(p)
        if abs(fit0 - fit) < rel_fitness and abs(rmse0 - rmse) < rel_rmse:
            break
    return T, fit, rmse, it


def pose_refine(scene_depth, model_depth, sceneK, modelK, modelR, modelT, detectX, detectY, max_iter=icp_oracle.MAX_ITER,
                use_scene_cloud=False):
    """icp_oracle.pose_refine with the point-to-point branch: the same clouds and initial guess, no EstimateNormals, and
    registration_icp_p2p.  Returns what icp_oracle.pose_refine returns."""
    scene_depth = np.asarray(scene_depth)
    model_depth = np.asarray(model_depth)
    init_base = np.zeros((4, 4), np.float32)
    init_base[:3, :3] = np.asarray(modelR, np.float32).reshape(3, 3)
    init_base[:3, 3] = np.asarray(modelT, np.float32).reshape(3)
    init_base[2, 3] = init_base[2, 3] / np.float32(1000.0)  # only the z component (LL.cpp:37)
    init_base[3, 3] = 1
    bbox = icp_oracle.model_bbox(model_depth)
    if detectX + bbox[2] >= scene_depth.shape[1] or detectY + bbox[3] >= scene_depth.shape[0]:
        return dict(R=None, t=None, residual=-1.0, iterations=0)
    model_pts, c_model, c_scene, scene_pts = icp_oracle.build_clouds(scene_depth, model_depth, sceneK, modelK, detectX, detectY, bbox)
    init_guess = np.eye(4)
    init_guess[:3, 3] = c_scene - c_model
    down = icp_oracle.voxel_down_sample(model_pts)
    target = icp_oracle.voxel_down_sample(scene_pts) if use_scene_cloud else down  # the reference: model cloud again (LL.cpp:109)
    T, fit, rmse, it = registration_icp_p2p(down, target, icp_oracle.MAX_DIST, init_guess, max_iter)
    result = T @ init_base.astype(np.float64)
    return dict(R=result[:3, :3].copy(), t=(result[:3, 3] * 1000.0).reshape(3, 1), residual=float(np.float32(fit)), iterations=it,
                n_points=int(down.shape[0]), rmse=rmse)
