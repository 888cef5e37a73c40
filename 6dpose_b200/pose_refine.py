"""poseRefine -- host mirror of the reference class (linemodLevelup/linemodLevelup.h:8-19, bound at
linemodLevelup/pybind11.cpp:9-14).  process() runs the ICP on the GPU through the C-ABI
(lm_icp_process); getR/getT/getResidual keep the reference's conventions: None before the first
successful call (an empty cv::Mat converts to None), residual = ICP fitness, -1 initially and after
the early return of LL.cpp:52-55.

process() and refine_matches() also take depths already in device memory: the scene and the renders as CUDA tensors
(uint16 mm, or float32 scaled by depth_scale / render_scale), read in order on `stream` (lm_icp_process_batch_device).
Numpy images are copied to the device and run the same kernels (lm_icp_process_batch), so the results are bit for bit
those of the same call on the converted uint16 numpy images."""
import numpy as np

from . import _lib
from .detector import _default_device

_icp = {}


def _native(device):
    if device not in _icp:
        _icp[device] = _lib.NativeIcp(device)
    return _icp[device]


class poseRefine:
    max_iterations = 30  # Open3D ICPConvergenceCriteria default used by the reference (LL.cpp:128-130)

    def __init__(self, estimation="point_to_plane"):
        """estimation (not in the reference's surface, which takes no argument): the ICP's estimation step,
        "point_to_plane" (TransformationEstimationPointToPlane, the reference's active branch), "point_to_point"
        (TransformationEstimationPointToPoint, its other branch at LL.cpp:131-135: no normals, Umeyama's rigid fit) or
        "pso" (a particle swarm against the scene depth, include/linemod_b200.h LM_POSE_PSO; see process's pose_search)."""
        _lib.estimation_code(estimation)
        self.estimation = estimation
        self._residual = -1.0
        self._R = None
        self._t = None
        self._score = None         # pose verification (verify_mm, Detector.setPoseVerification): score, counts
        self._verification = None
        self._T = None             # the ICP's 4x4 transformation (Detector's pose calls and track)
        self._track_status = None  # Detector.track's status
        self.device = _default_device()

    @staticmethod
    def _mat(a, dtype, shape, name):
        a = np.asarray(a)
        if a.dtype != dtype:
            raise TypeError("%s must be %s (the reference reads it with .at<%s>)" % (name, np.dtype(dtype).name, np.dtype(dtype).name))
        if a.size != int(np.prod(shape)):
            raise RuntimeError("%s must have %s elements" % (name, "x".join(map(str, shape))))
        return np.ascontiguousarray(a).reshape(shape)

    @staticmethod
    def _depth(a, name):
        a = np.asarray(a)
        if a.dtype != np.uint16 or a.ndim != 2:
            raise TypeError("%s must be a uint16 HxW depth image (mm)" % name)
        return a

    def process(self, sceneDepth, modelDepth, sceneK, modelK, modelR, modelT, detectX, detectY, depth_scale=1.0, render_scale=1.0,
                stream=None, verify_mm=None, pose_search=None):
        """sceneDepth / modelDepth: uint16 HxW numpy images (mm), or CUDA tensors on this object's device: uint16 (mm) or
        float32 [H, W], pixels packed within a row.  depth_scale / render_scale convert float32 depth to mm (the driver's
        depth_ren.astype(np.uint16) is render_scale 1.0); stream: the torch stream the tensors are ordered on (None: the
        current stream).  verify_mm (not in the reference's surface): verify the refined pose against the scene depth with
        this inlier distance in mm (include/linemod_b200.h, lm_set_pose_verify); getScore / getVerification then return
        the result.  None: no verification.  pose_search (estimation "pso" only): a dict of the swarm's settings
        (Detector.setPoseSearch's keywords); None: the defaults."""
        if verify_mm is not None:
            _lib.inlier_mm(verify_mm)
        search = _lib.pose_search_options(**(pose_search or {}))
        dev = _lib.depth_inputs(sceneDepth, [modelDepth], depth_scale, render_scale, stream, self.device,
                                host=dict(sceneK=sceneK, modelK=modelK, modelR=modelR, modelT=modelT))
        if dev is None:
            scene = np.asarray(sceneDepth)
            model = np.asarray(modelDepth)
            if scene.dtype != np.uint16 or scene.ndim != 2 or model.dtype != np.uint16 or model.ndim != 2:
                raise TypeError("sceneDepth / modelDepth must be uint16 HxW depth images (mm)")
        sK = self._mat(sceneK, np.float32, (3, 3), "sceneK")
        mK = self._mat(modelK, np.float32, (3, 3), "modelK")
        R = self._mat(modelR, np.float32, (3, 3), "modelR")
        t = self._mat(modelT, np.float32, (3,), "modelT")
        args = (sK, mK[None], R[None], t[None], [[int(detectX), int(detectY)]], self.max_iterations, self.estimation)
        icp = _native(self.device)
        icp.set_verify(verify_mm)
        icp.set_pose_search(*search)
        if dev is None:
            Ro, to, res = icp.process_batch(scene, [model], *args)
        else:
            Ro, to, res = icp.process_batch_device(dev, *args)
        self._residual = float(res[0])
        self._score, self._verification = _lib.verify_arrays(*icp.verify())[0] if verify_mm is not None else (None, None)
        if res[0] == -1.0:  # early return: R_refined / t_refiend keep their previous value (LL.cpp:52-55)
            return
        self._R = Ro[0].copy()
        self._t = to[0].reshape(3, 1).copy()

    def getResidual(self):
        return self._residual

    def getR(self):
        return self._R

    def getT(self):
        return self._t

    def getScore(self):
        """The pose verification's depth-consistency score: inlier / (inlier + occluded + violation), 0 when that sum is 0,
        -1 without a pose; None when the call did not verify."""
        return self._score

    def getTransformation(self):
        """The ICP's 4x4 transformation T (f64, row-major), which maps the template's render cloud into the scene camera
        (include/linemod_b200.h, lm_track): what Detector.track starts the next frame from.  None when the pose did not
        come from Detector's match_refine, detect, batch calls or track, or has none."""
        return self._T

    def getTrackStatus(self):
        """Detector.track's status of this pose: "tracked", "outside" (no model point lands in the frame), "window" (the
        window exceeds the scene slot) or "no_depth" (no scene depth in the window); None when it did not come from
        track."""
        return self._track_status

    def getVerification(self):
        """The pose verification's counts, a dict of n_model, outside, missing, inlier, occluded and violation (the last five
        sum to n_model); None when the call did not verify."""
        return self._verification


def refine_matches(sceneDepth, sceneK, matches, modelDepths, modelKs, modelRs, modelTs, device=None, estimation="point_to_plane",
                   depth_scale=1.0, render_scale=1.0, stream=None, verify_mm=None, pose_search=None):
    """The drivers' loop over the NMS survivors (linemod_and_levelup_test.py:348-367: one poseRefine per
    match, fed with the render of the matched template's pose) as ONE batched GPU call: hypothesis i is
    matches[i] (its x, y) with modelDepths[i] / modelKs[i] / modelRs[i] / modelTs[i].  Returns a list of
    poseRefine objects in the state process() would have left them in.  estimation as poseRefine().
    Depths in device memory: sceneDepth a CUDA tensor and modelDepths a list of [H, W] CUDA tensors or one [n, H, W]
    tensor, with depth_scale, render_scale and stream as poseRefine.process.  verify_mm as poseRefine.process: every
    survivor comes back with its score, none is dropped.  pose_search as poseRefine.process; match i draws the swarm's
    random numbers as job i."""
    _lib.estimation_code(estimation)
    if verify_mm is not None:
        _lib.inlier_mm(verify_mm)
    search = _lib.pose_search_options(**(pose_search or {}))
    n = len(matches)
    dev = _default_device() if device is None else int(device)
    renders = modelDepths if _lib.is_tensor(modelDepths) else list(modelDepths)
    inputs = _lib.depth_inputs(sceneDepth, renders, depth_scale, render_scale, stream, dev, n,
                               dict(sceneK=sceneK, modelKs=modelKs, modelRs=modelRs, modelTs=modelTs))
    out = [poseRefine(estimation) for _ in range(n)]
    if n == 0:
        return out
    if inputs is None:
        scene = np.asarray(sceneDepth)
        if scene.dtype != np.uint16 or scene.ndim != 2:
            raise TypeError("sceneDepth must be a uint16 HxW depth image (mm)")
        models = [np.asarray(m) for m in renders]
        if len(models) != n or any(m.dtype != np.uint16 or m.ndim != 2 for m in models):
            raise TypeError("modelDepths: one uint16 HxW render per match")
    sK = poseRefine._mat(sceneK, np.float32, (3, 3), "sceneK")
    mK = np.stack([poseRefine._mat(k, np.float32, (3, 3), "modelK") for k in modelKs])
    R = np.stack([poseRefine._mat(r, np.float32, (3, 3), "modelR") for r in modelRs])
    t = np.stack([poseRefine._mat(v, np.float32, (3,), "modelT") for v in modelTs])
    xy = [[int(m.x), int(m.y)] for m in matches]
    icp = _native(dev)
    icp.set_verify(verify_mm)
    icp.set_pose_search(*search)
    if inputs is None:
        Ro, to, res = icp.process_batch(scene, models, sK, mK, R, t, xy, poseRefine.max_iterations, estimation)
    else:
        Ro, to, res = icp.process_batch_device(inputs, sK, mK, R, t, xy, poseRefine.max_iterations, estimation)
    ver = _lib.verify_arrays(*icp.verify()) if verify_mm is not None else [(None, None)] * n
    for i, p in enumerate(out):
        p._residual = float(res[i])
        p._score, p._verification = ver[i]
        if res[i] != -1.0:
            p._R = Ro[i].copy()
            p._t = to[i].reshape(3, 1).copy()
    return out


def pose_to_transform(R, t, R_b, t_b):
    """The transformation T (4x4 f64) of a pose (R [3,3], t [3] mm, as getR / getT return it) of a template whose render
    was made at (R_b, t_b) (f32, t_b mm), in the order include/linemod_b200.h states (lm_track): T_R = R R_b^T, T_t = t /
    1000 - T_R b with b = (t_b.x, t_b.y, t_b.z / 1000 in float32).  Every operation is one correctly rounded float64
    operation."""
    R = np.asarray(R, np.float64).reshape(3, 3)
    t = np.asarray(t, np.float64).reshape(3)
    Rb = np.asarray(R_b, np.float32).reshape(3, 3).astype(np.float64)
    tb = np.asarray(t_b, np.float32).reshape(3)
    b = [float(tb[0]), float(tb[1]), float(tb[2] / np.float32(1000.0))]
    T = np.eye(4)
    for r in range(3):
        for c in range(3):
            T[r, c] = ((float(R[r, 0]) * float(Rb[c, 0])) + float(R[r, 1]) * float(Rb[c, 1])) + float(R[r, 2]) * float(Rb[c, 2])
        T[r, 3] = float(t[r]) / 1000.0 - (((T[r, 0] * b[0]) + T[r, 1] * b[1]) + T[r, 2] * b[2])
    return T


def nms_translations(ts, scores, thr, device=None):
    """linemod_ros/detect.py's nms_norms(ts, scores, thr) (:41-50) for the poses of refine_matches, on the GPU
    (lm_nms_translations, the routine behind Detector.detect): ts [n,3] mm, scores [n] (detect.py passes -residual),
    n <= 1024.  Returns the kept indices in keep order.  Equal scores go in index order, NaN scores first; a distance
    equal to thr, or NaN, suppresses."""
    dev = _default_device() if device is None else int(device)
    return _lib.nms_translations(ts, scores, thr, dev)
