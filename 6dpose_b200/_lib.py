"""ctypes binding of the C-ABI shared library (include/linemod_b200.h).

Fails loudly when the library is missing or cannot be loaded: there is no CPU / PyTorch fallback
for the hot path.
"""
import ctypes
import math
import os
import re
import sys

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
# LINEMOD_B200_LIB: another build of the same library (A/B runs of compile-time variants); never a different backend
LIB_PATH = os.environ.get("LINEMOD_B200_LIB") or os.path.join(_HERE, "csrc", "liblinemod_b200.so")

LM_OK, LM_E_INVALID, LM_E_CUDA, LM_E_STATE, LM_E_CAPACITY = 0, -1, -2, -3, -4
# capture items of lm_icp_capture and lm_debug_pose_clouds (include/linemod_b200.h)
CAPTURE_ITEMS = dict(counts=0, source=1, target=2, normals=3, init=4, result=5, knn=6, corr_first=7, corr_last=8, slots=9, posed=10,
                     raw_model=11, raw_scene=12, search=13, window=14)
# lm_track's statuses (LM_TRACK_* of include/linemod_b200.h) by the name poseRefine.getTrackStatus returns
TRACK_STATUS = ("tracked", "outside", "window", "no_depth")
TRACK_MAX = 1024  # objects per lm_track call
SHARD_CONTIGUOUS, SHARD_INTERLEAVED = 0, 1

MATCH_DTYPE = np.dtype([("x", "<i4"), ("y", "<i4"), ("similarity", "<f4"), ("class_index", "<i4"), ("template_id", "<i4")])
RECORD_DTYPE = np.dtype([("x", "<i2"), ("y", "<i2"), ("similarity", "<f4"), ("work", "<i4"), ("seq", "<i4")])
HEADER_DTYPE = np.dtype([("count", "<i4"), ("coarse_candidates", "<i4"), ("capacity", "<i4"), ("shard", "<i4")])

# every symbol include/linemod_b200.h declares (tests check the .so exports all of them)
PEER_HANDLE_BYTES = 64

SYMBOLS = [
    "lm_last_error", "lm_create", "lm_destroy", "lm_load_bank", "lm_select", "lm_select_layout", "lm_shard_range", "lm_prepare", "lm_coarse_tasks", "lm_coarse_descriptors",
    "lm_upload_quantized", "lm_upload_images", "lm_match_images", "lm_debug_quantized", "lm_bind_quantized_device",
    "lm_bind_images_device", "lm_detect_batch_device", "lm_debug_depth", "lm_debug_plan", "lm_debug_coarse", "lm_debug_pose_clouds", "lm_run", "lm_enqueue", "lm_complete", "lm_set_result_buffer", "lm_device_result", "lm_fetch_records",
    "lm_finish", "lm_match_quantized", "lm_debug_linear_memories", "lm_debug_time_k1", "lm_debug_bit_planes", "lm_counters", "lm_set_timing",
    "lm_stage_times", "lm_stream", "lm_launch_count",
    "lm_set_boxes", "lm_enqueue_post", "lm_complete_post", "lm_match_top",
    "lm_set_template_renders", "lm_enqueue_pose", "lm_complete_pose",
    "lm_enqueue_pose_nms", "lm_complete_detect", "lm_nms_translations", "lm_detect_batch", "lm_peer_detect_batch",
    "lm_peer_export", "lm_peer_base", "lm_peer_connect", "lm_peer_connect_local", "lm_peer_disconnect", "lm_peer_share_pose",
    "lm_pose_stats", "lm_set_pose_estimation", "lm_set_template_depths", "lm_set_depth_gate", "lm_depth_gate_stats",
    "lm_icp_create", "lm_icp_destroy", "lm_icp_process", "lm_icp_process_batch", "lm_icp_last_stats", "lm_icp_launch_count", "lm_icp_set_use_scene_cloud",
    "lm_icp_set_estimation", "lm_icp_set_capture", "lm_icp_capture", "lm_icp_process_batch_device",
    "lm_set_pose_verify", "lm_pose_verify", "lm_pose_verify_points", "lm_icp_set_verify", "lm_icp_verify",
    "lm_set_pose_search", "lm_icp_set_pose_search", "lm_pose_search_points",
    "lm_track", "lm_track_device", "lm_track_batch", "lm_track_batch_device", "lm_pose_transforms",
    "lm_peer_track_batch", "lm_peer_track_batch_device", "lm_set_track_views", "lm_track_templates", "lm_track_views_points",
]

# The pose stage's estimation (LM_ICP_POINT_TO_PLANE / LM_ICP_POINT_TO_POINT / LM_POSE_PSO of include/linemod_b200.h) by
# the name the Python surface takes
ESTIMATIONS = {"point_to_plane": 0, "point_to_point": 1, "pso": 3}


def estimation_code(estimation):
    """The C-ABI value of estimation="point_to_plane" | "point_to_point" | "pso"; ValueError for anything else (no device
    work)."""
    if not isinstance(estimation, str) or estimation not in ESTIMATIONS:
        raise ValueError("estimation must be one of %s, got %r" % (", ".join(repr(k) for k in ESTIMATIONS), estimation))
    return ESTIMATIONS[estimation]


# Pose verification (lm_set_pose_verify): the pose NMS's ranking by the name the Python surface takes, and the names of
# the six counts
VERIFY_RANKS = {"fitness": 0, "score": 1}
VERIFY_COUNTS = ("n_model", "outside", "missing", "inlier", "occluded", "violation")


def _real(v, what):
    if isinstance(v, (bool, np.bool_)) or not isinstance(v, (int, float, np.integer, np.floating)):
        raise TypeError("%s must be a number, got %s" % (what, type(v).__name__))
    return float(v)


def inlier_mm(v):
    """The verification's inlier distance delta (mm) as a float: finite and >= 0, else ValueError (no device work)."""
    d = _real(v, "inlier_mm")
    if not (math.isfinite(d) and d >= 0.0):
        raise ValueError("inlier_mm must be finite and >= 0, got %r" % v)
    return d


def verify_options(inlier, rank_by="fitness", min_score=None):
    """lm_set_pose_verify's (on, inlier_mm, rank_by, min_score) for Detector.setPoseVerification; inlier None turns
    verification off, which takes neither rank_by="score" nor a min_score.  ValueError / TypeError before any device work."""
    if not isinstance(rank_by, str) or rank_by not in VERIFY_RANKS:
        raise ValueError("rank_by must be one of %s, got %r" % (", ".join(repr(k) for k in VERIFY_RANKS), rank_by))
    lo = -math.inf
    if min_score is not None:
        lo = _real(min_score, "min_score")
        if math.isnan(lo):
            raise ValueError("min_score is NaN")
    if inlier is None:
        if rank_by != "fitness" or min_score is not None:
            raise ValueError("rank_by=\"score\" and min_score need pose verification on (inlier_mm not None)")
        return 0, 10.0, 0, -math.inf
    return 1, inlier_mm(inlier), VERIFY_RANKS[rank_by], lo


def track_views_option(turn_deg):
    """lm_set_track_views's (on, turn_deg) for Detector.setTrackViews: None turns view following off; otherwise a number
    in [0, 180) degrees.  TypeError / ValueError before any device work."""
    if turn_deg is None:
        return 0, 0.0
    d = _real(turn_deg, "turn_deg")
    if not 0.0 <= d < 180.0:
        raise ValueError("turn_deg must lie in [0, 180) degrees, got %r" % turn_deg)
    return 1, d


# The particle swarm of estimation="pso" (lm_set_pose_search): its settings by name, with their defaults and limits
POSE_SEARCH_DEFAULTS = dict(particles=64, iterations=40, dt_mm=40.0, dr_deg=30.0, clamp_mm=20.0, seed=0)
POSE_SEARCH_LIMITS = dict(particles=(1, 256), iterations=(0, 1000), dt_mm=(0.0, 10000.0), dr_deg=(0.0, 45.0), clamp_mm=(0.0, 1e6))


def pose_search_options(particles=64, iterations=40, dt_mm=40.0, dr_deg=30.0, clamp_mm=20.0, seed=0):
    """lm_set_pose_search's (particles, iterations, dt_mm, dr_deg, clamp_mm, seed) for Detector.setPoseSearch and the
    pose_search keyword of poseRefine.process / refine_matches.  TypeError / ValueError before any device work."""
    out = []
    for name, v in (("particles", particles), ("iterations", iterations)):
        if isinstance(v, (bool, np.bool_)) or not isinstance(v, (int, np.integer)):
            raise TypeError("%s must be an int, got %s" % (name, type(v).__name__))
        lo, hi = POSE_SEARCH_LIMITS[name]
        if not lo <= int(v) <= hi:
            raise ValueError("%s must lie in [%d, %d], got %r" % (name, lo, hi, v))
        out.append(int(v))
    for name, v in (("dt_mm", dt_mm), ("dr_deg", dr_deg), ("clamp_mm", clamp_mm)):
        x = _real(v, name)
        lo, hi = POSE_SEARCH_LIMITS[name]
        if not (math.isfinite(x) and lo <= x <= hi):
            raise ValueError("%s must be finite and in [%g, %g], got %r" % (name, lo, hi, v))
        out.append(x)
    if isinstance(seed, (bool, np.bool_)) or not isinstance(seed, (int, np.integer)):
        raise TypeError("seed must be an int, got %s" % type(seed).__name__)
    if not 0 <= int(seed) < 1 << 64:
        raise ValueError("seed must lie in [0, 2^64), got %r" % seed)
    out.append(int(seed))
    return tuple(out)


def search_record(words, particles, iterations):
    """A swarm record (LM_ICP_CAPTURE_SEARCH, lm_pose_search_points) as a dict: cost_start, cost and best (int), c [3]
    f64, trace [I] int64 (the global-best cost after each iteration), x, v, p [P,6] f64 and cost_best [P] int64."""
    w = np.ascontiguousarray(words, np.int64)
    P, I = int(particles), int(iterations)
    sw = w[6 + I:]
    return dict(cost_start=int(w[0]), cost=int(w[1]), best=int(w[2]), c=w[3:6].view(np.float64).copy(), trace=w[6:6 + I].copy(),
                x=sw[:6 * P].view(np.float64).reshape(P, 6).copy(), v=sw[6 * P:12 * P].view(np.float64).reshape(P, 6).copy(),
                p=sw[12 * P:18 * P].view(np.float64).reshape(P, 6).copy(), cost_best=sw[18 * P:19 * P].copy())


def verify_arrays(score, counts):
    """[(score, {count name: value})] of lm_pose_verify's / lm_icp_verify's outputs."""
    return [(float(s), dict(zip(VERIFY_COUNTS, (int(v) for v in c)))) for s, c in zip(score.tolist(), counts)]


def depth_gate_tolerance(tolerance):
    """The depth gate's tolerance as a float in [0, 1); ValueError otherwise (no device work)."""
    if isinstance(tolerance, (bool, np.bool_)) or not isinstance(tolerance, (int, float, np.integer, np.floating)):
        raise TypeError("depth gate tolerance must be a number, got %s" % type(tolerance).__name__)
    t = float(tolerance)
    if not (0.0 <= t < 1.0):
        raise ValueError("depth gate tolerance must lie in [0, 1), got %r" % tolerance)
    return t


# Depth formats of lm_bind_images_device (include/linemod_b200.h)
DEPTH_U16_MM, DEPTH_F32 = 0, 1


def is_tensor(a):
    """True for a torch.Tensor.  torch is not imported for this: a caller holding a tensor has imported it already."""
    torch = sys.modules.get("torch")
    return torch is not None and isinstance(a, torch.Tensor)


def depth_scale_value(depth_scale, name="depth_scale"):
    """depth_scale as a float, finite and > 0; TypeError / ValueError otherwise (no device work)."""
    if isinstance(depth_scale, (bool, np.bool_)) or not isinstance(depth_scale, (int, float, np.integer, np.floating)):
        raise TypeError("%s must be a number, got %s" % (name, type(depth_scale).__name__))
    s = float(depth_scale)
    if not (math.isfinite(s) and s > 0.0):
        raise ValueError("%s must be finite and > 0, got %r" % (name, depth_scale))
    return s


class DeviceFrame:
    """An RGB-D frame already on the GPU, checked for lm_bind_images_device without any library call: rgb uint8 [H, W, 3]
    with stride(2) == 1 and stride(1) == 3, depth torch.uint16 (mm) or torch.float32 (scaled by depth_scale, converted
    to u16 mm on the device) [H, W] with stride(1) == 1, masks [] or [mask_color, mask_depth], each None, empty or uint8
    [H, W] with stride(1) == 1 and one row pitch; every tensor CUDA on `device`.  Row pitches are free (crop views).
    The frame is read in order on `stream` (device_stream)."""

    def __init__(self, rgb, depth, masks, depth_scale, stream, device):
        import torch
        if not (is_tensor(rgb) and is_tensor(depth)):
            raise TypeError("sources mix numpy arrays and torch tensors: pass both as CUDA tensors or both as numpy arrays")
        if rgb.dtype != torch.uint8 or rgb.dim() != 3 or rgb.shape[2] != 3:
            raise TypeError("sources[0] must be a uint8 HxWx3 colour tensor, got %s %s" % (rgb.dtype, tuple(rgb.shape)))
        if rgb.stride(2) != 1 or rgb.stride(1) != 3:
            raise ValueError("sources[0]: pixels must be packed within a row (strides (*, 3, 1)), got %s" % (rgb.stride(),))
        if depth.dtype not in (torch.uint16, torch.float32) or depth.dim() != 2:
            raise TypeError("sources[1] must be a uint16 (mm) or float32 HxW depth tensor, got %s %s" % (depth.dtype, tuple(depth.shape)))
        if tuple(depth.shape) != tuple(rgb.shape[:2]):
            raise ValueError("sources[1] is %s, the colour image %s" % (tuple(depth.shape), tuple(rgb.shape[:2])))
        if depth.stride(1) != 1:
            raise ValueError("sources[1]: depth must be packed within a row (stride(1) == 1), got %s" % (depth.stride(),))
        f32 = depth.dtype == torch.float32
        scale = depth_scale_value(depth_scale)
        if not f32 and scale != 1.0:
            raise ValueError("depth_scale applies to float32 depth; uint16 depth is in mm (depth_scale=%r)" % depth_scale)
        rows, cols = int(rgb.shape[0]), int(rgb.shape[1])
        mk = [None, None]
        if masks:
            if len(masks) != 2:
                raise RuntimeError("masks.size() == modalities.size()")
            for i, m in enumerate(masks):
                if m is None:
                    continue
                if not is_tensor(m):
                    if np.asarray(m).size:
                        raise TypeError("masks[%d] is not a tensor: masks of a device frame are CUDA tensors too" % i)
                    continue
                if m.numel() == 0:
                    continue
                if m.dtype != torch.uint8 or tuple(m.shape) != (rows, cols):
                    raise RuntimeError("mask.size() == source.size()")
                if m.stride(1) != 1:
                    raise ValueError("masks[%d] must be packed within a row (stride(1) == 1), got %s" % (i, m.stride()))
                mk[i] = m
            if mk[0] is not None and mk[1] is not None and mk[0].stride(0) != mk[1].stride(0):
                raise ValueError("the two masks must share one row pitch, got %d and %d" % (mk[0].stride(0), mk[1].stride(0)))
        for name, t in (("sources[0]", rgb), ("sources[1]", depth), ("masks[0]", mk[0]), ("masks[1]", mk[1])):
            if t is not None and (not t.is_cuda or t.device.index != int(device)):
                raise ValueError("%s is on %s; the detector runs on cuda:%d" % (name, t.device, int(device)))
        mask_pitch = next((m.stride(0) for m in mk if m is not None), cols)
        self.rows, self.cols = rows, cols
        self.tensors = [t for t in (rgb, depth, mk[0], mk[1]) if t is not None]
        self.pitches = (rgb.stride(0), depth.stride(0) * depth.element_size(), mask_pitch)
        self.rgb, self.depth, self.masks = rgb.data_ptr(), depth.data_ptr(), [m.data_ptr() if m is not None else None for m in mk]
        self.format = DEPTH_F32 if f32 else DEPTH_U16_MM
        self.scale = scale
        self.stream = device_stream(stream, device)


class DeviceBatch:
    """DeviceFrames for lm_detect_batch_device: one size, row pitches, depth dtype, depth_scale and stream, and one row
    pitch for every mask of the batch.  ValueError otherwise, before any library call."""

    def __init__(self, frames):
        frames = list(frames)
        if not frames:
            raise ValueError("no frames")
        f0 = frames[0]
        key = lambda f: (f.rows, f.cols, f.pitches[:2], f.format, f.scale, f.stream)
        if any(key(f) != key(f0) for f in frames):
            raise ValueError("every frame's tensors must have one size, row pitch, depth dtype and depth_scale")
        masked = [f for f in frames if any(m is not None for m in f.masks)]
        if len({f.pitches[2] for f in masked}) > 1:
            raise ValueError("the masks of a batch must share one row pitch")
        vp = ctypes.c_void_p
        self.n, self.stream = len(frames), f0.stream
        self.tensors = [t for f in frames for t in f.tensors]
        masks = (vp * (2 * self.n))(*[m for f in frames for m in f.masks]) if masked else None
        self.args = (self.n, (vp * self.n)(*[f.rgb for f in frames]), f0.pitches[0], (vp * self.n)(*[f.depth for f in frames]),
                     f0.pitches[1], f0.format, ctypes.c_float(f0.scale), f0.rows, f0.cols, masks,
                     masked[0].pitches[2] if masked else f0.cols, f0.stream.cuda_stream)


def frame_inputs(rgb, depth, masks, depth_scale, stream, device):
    """A DeviceFrame for a pair of CUDA tensors (rgb itself when it is one already), None for numpy arrays (the host path,
    where depth_scale must stay 1.0 and stream None).  TypeError / ValueError before any library call."""
    if isinstance(rgb, DeviceFrame):
        return rgb
    if not (is_tensor(rgb) or is_tensor(depth)):
        host_frame_options(depth_scale, stream)
        if masks and any(is_tensor(m) for m in masks if m is not None):
            raise TypeError("masks are tensors, the frame is numpy arrays")
        return None
    return DeviceFrame(rgb, depth, masks, depth_scale, stream, device)


def host_frame_options(depth_scale, stream):
    """A frame of numpy arrays takes neither option: its depth is uint16 mm and it is copied before the call returns."""
    if stream is not None:
        raise TypeError("stream applies to frames given as CUDA tensors")
    if depth_scale_value(depth_scale) != 1.0:
        raise ValueError("depth_scale applies to float32 depth tensors; numpy depth is uint16 mm")


def _depth_plane(t, name, torch):
    """(data pointer, row pitch in bytes, format) of a uint16 (mm) or float32 [H, W] tensor packed within a row."""
    if t.dtype not in (torch.uint16, torch.float32) or t.dim() != 2:
        raise TypeError("%s must be a uint16 (mm) or float32 HxW depth tensor, got %s %s" % (name, t.dtype, tuple(t.shape)))
    if t.stride(1) != 1:
        raise ValueError("%s: depth must be packed within a row (stride(-1) == 1), got %s" % (name, t.stride()))
    return t.data_ptr(), t.stride(0) * t.element_size(), DEPTH_F32 if t.dtype == torch.float32 else DEPTH_U16_MM


def _plane_scale(f32, scale, name, what):
    s = depth_scale_value(scale, name)
    if not f32 and s != 1.0:
        raise ValueError("%s applies to float32 %s; uint16 %s is in mm (%s=%r)" % (name, what, what, name, scale))
    return s


class DeviceDepths:
    """A scene depth and its renders already on the GPU, checked for lm_icp_process_batch_device without any library call:
    the scene a torch.uint16 (mm) or torch.float32 [H, W] tensor (scaled by depth_scale), the renders uint16 or float32
    [h, w] tensors of one dtype and size (scaled by render_scale), given as a list or as one [n, h, w] tensor; every plane
    packed within a row (stride(-1) == 1) with a free row pitch, every tensor CUDA on `device`.  The planes are read in
    order on `stream` (device_stream).  n: the renders expected; host: the call's K, R and t by name (host_arrays)."""

    def __init__(self, scene, renders, depth_scale, render_scale, stream, device, n=None, host=None):
        import torch
        if is_tensor(renders):
            if renders.dim() != 3:
                raise TypeError("renders given as one tensor must be [n, H, W], got %s" % (tuple(renders.shape),))
            renders = list(renders.unbind(0))
        renders = list(renders)
        if not (is_tensor(scene) and all(is_tensor(r) for r in renders)):
            raise TypeError("depths mix numpy arrays and torch tensors: pass the scene and every render as CUDA tensors or all as numpy arrays")
        self.scene, self.scene_pitch, self.scene_format = _depth_plane(scene, "sceneDepth", torch)
        self.depth_scale = _plane_scale(self.scene_format == DEPTH_F32, depth_scale, "depth_scale", "depth")
        planes = [_depth_plane(r, "modelDepths[%d]" % i, torch) for i, r in enumerate(renders)]
        if any(r.dtype != renders[0].dtype or r.shape != renders[0].shape for r in renders):
            raise ValueError("every render must have one dtype and size, got %s" % sorted({(str(r.dtype), tuple(r.shape)) for r in renders}))
        self.format = planes[0][2] if planes else DEPTH_U16_MM
        self.render_scale = _plane_scale(self.format == DEPTH_F32, render_scale, "render_scale", "renders")
        if n is not None and len(renders) != n:
            raise TypeError("modelDepths: one render per match, got %d renders for %d matches" % (len(renders), n))
        host_arrays(**(host or {}))
        for name, t in [("sceneDepth", scene)] + [("modelDepths[%d]" % i, r) for i, r in enumerate(renders)]:
            if not t.is_cuda or t.device.index != int(device):
                raise ValueError("%s is on %s; the ICP runs on cuda:%d" % (name, t.device, int(device)))
        self.srows, self.scols = int(scene.shape[0]), int(scene.shape[1])
        self.mrows, self.mcols = (int(renders[0].shape[0]), int(renders[0].shape[1])) if renders else (1, 1)
        self.n = len(renders)
        self.renders, self.pitches = [p[0] for p in planes], [p[1] for p in planes]
        self.tensors = [scene] + renders
        self.stream = device_stream(stream, device)


def depth_inputs(scene, renders, depth_scale, render_scale, stream, device, n=None, host=None):
    """A DeviceDepths when the scene or any render is a tensor, None for numpy arrays (process_batch, where depth_scale
    and render_scale must stay 1.0 and stream None).  TypeError / ValueError before any library call."""
    if not (is_tensor(scene) or is_tensor(renders) or any(is_tensor(r) for r in renders)):
        host_frame_options(depth_scale, stream)
        if depth_scale_value(render_scale, "render_scale") != 1.0:
            raise ValueError("render_scale applies to float32 render tensors; numpy renders are uint16 mm")
        return None
    return DeviceDepths(scene, renders, depth_scale, render_scale, stream, device, n, host)


def host_arrays(**arrays):
    """K, R and t of the ICP stay host arrays whatever the depths are: TypeError for a tensor (no library call)."""
    for name, a in arrays.items():
        if is_tensor(a) or (isinstance(a, (list, tuple)) and any(is_tensor(x) for x in a)):
            raise TypeError("%s must be a host (numpy) array, got a tensor" % name)


def device_stream(stream, device):
    """The torch stream a device frame is ordered on: torch.cuda.current_stream(device) for None."""
    import torch
    if stream is None:
        return torch.cuda.current_stream(int(device))
    if not isinstance(stream, torch.cuda.Stream):
        raise TypeError("stream must be a torch.cuda.Stream or None, got %s" % type(stream).__name__)
    if stream.device.index != int(device):
        raise ValueError("stream is on %s; the detector runs on cuda:%d" % (stream.device, int(device)))
    return stream


_lib = None


class LinemodLibraryError(RuntimeError):
    pass


def load():
    """Load liblinemod_b200.so (built in-tree by `make -C 6dpose_b200/csrc` / __graft_entry__.build())."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise LinemodLibraryError(
            "%s not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(nvcc, sm_90a).  There is no CPU fallback for the LINEMOD hot path." % LIB_PATH)
    L = ctypes.CDLL(LIB_PATH)
    c_int, c_i64, c_f, vp = ctypes.c_int, ctypes.c_int64, ctypes.c_float, ctypes.c_void_p
    i32p = ctypes.POINTER(ctypes.c_int32)
    u8pp = ctypes.POINTER(ctypes.POINTER(ctypes.c_uint8))
    L.lm_last_error.restype = ctypes.c_char_p
    L.lm_create.argtypes = [c_int, c_int, ctypes.POINTER(c_int), ctypes.POINTER(vp)]
    L.lm_destroy.argtypes = [vp]
    L.lm_destroy.restype = None
    L.lm_load_bank.argtypes = [vp, c_int, i32p, c_int, i32p, i32p, c_i64]
    L.lm_select.argtypes = [vp, i32p, c_int, c_int, c_int]
    L.lm_select_layout.argtypes = [vp, i32p, c_int, c_int, c_int, c_int]
    L.lm_prepare.argtypes = [vp]
    L.lm_coarse_tasks.argtypes = [i32p, c_i64, c_int, c_i64, i32p, c_i64] + [ctypes.POINTER(c_i64)] * 3 + [i32p]
    L.lm_coarse_descriptors.argtypes = [i32p, i32p] + [c_int] * 7 + [ctypes.POINTER(ctypes.c_uint32), c_i64,
                                                                        ctypes.POINTER(c_i64), i32p, ctypes.POINTER(ctypes.c_uint8),
                                                                        ctypes.POINTER(ctypes.c_uint32)]
    L.lm_shard_range.argtypes = [vp, ctypes.POINTER(c_i64), ctypes.POINTER(c_i64)]
    L.lm_upload_quantized.argtypes = [vp, u8pp, ctypes.POINTER(c_int), ctypes.POINTER(c_int)]
    u8p_ = ctypes.POINTER(ctypes.c_uint8)
    L.lm_upload_images.argtypes = [vp, u8p_, ctypes.POINTER(ctypes.c_uint16), c_int, c_int, u8p_, u8p_]
    L.lm_match_images.argtypes = [vp, u8p_, ctypes.POINTER(ctypes.c_uint16), c_int, c_int, u8p_, u8p_, c_f, vp, c_i64,
                                  ctypes.POINTER(c_i64)]
    L.lm_debug_quantized.argtypes = [vp, c_int, c_int, u8p_, c_i64]
    L.lm_bind_quantized_device.argtypes = [vp, ctypes.POINTER(vp), ctypes.POINTER(c_int), ctypes.POINTER(c_int)]
    L.lm_run.argtypes = [vp, c_f]
    L.lm_enqueue.argtypes = [vp, c_f]
    L.lm_complete.argtypes = [vp]
    L.lm_set_result_buffer.argtypes = [vp, vp, c_i64]
    L.lm_set_boxes.argtypes = [vp, i32p, c_i64]
    L.lm_enqueue_post.argtypes = [vp, ctypes.c_double, c_int]
    L.lm_complete_post.argtypes = [vp, vp, c_i64, ctypes.POINTER(c_i64), ctypes.POINTER(c_i64)]
    L.lm_match_top.argtypes = [vp, u8pp, ctypes.POINTER(c_int), ctypes.POINTER(c_int), c_f, ctypes.c_double, c_int, vp, c_i64,
                               ctypes.POINTER(c_i64), ctypes.POINTER(c_i64)]
    L.lm_peer_export.argtypes = [vp, c_int, c_i64, u8p_]
    L.lm_peer_base.argtypes = [vp, ctypes.POINTER(vp)]
    L.lm_peer_connect.argtypes = [vp, c_int, c_int, u8p_]
    L.lm_peer_connect_local.argtypes = [vp, c_int, c_int, ctypes.POINTER(vp)]
    L.lm_peer_disconnect.argtypes = [vp]
    L.lm_peer_share_pose.argtypes = [vp, c_int]
    L.lm_pose_stats.argtypes = [vp, ctypes.POINTER(c_i64)]
    L.lm_set_pose_estimation.argtypes = [vp, c_int]
    L.lm_set_template_depths.argtypes = [vp, c_i64, c_i64, ctypes.POINTER(c_f)]
    L.lm_set_depth_gate.argtypes = [vp, c_int, ctypes.c_double]
    L.lm_depth_gate_stats.argtypes = [vp, ctypes.POINTER(c_i64)]
    L.lm_device_result.argtypes = [vp, ctypes.POINTER(vp), ctypes.POINTER(c_i64)]
    L.lm_fetch_records.argtypes = [vp, vp, c_i64, ctypes.POINTER(c_i64)]
    L.lm_finish.argtypes = [vp, vp, c_i64, vp, c_i64, ctypes.POINTER(c_i64)]
    L.lm_match_quantized.argtypes = [vp, u8pp, ctypes.POINTER(c_int), ctypes.POINTER(c_int), c_f, vp, c_i64,
                                     ctypes.POINTER(c_i64)]
    L.lm_debug_linear_memories.argtypes = [vp, c_int, c_int, ctypes.POINTER(ctypes.c_uint8), c_i64]
    L.lm_debug_time_k1.argtypes = [vp, c_int, c_int, ctypes.POINTER(c_f)]
    L.lm_debug_bit_planes.argtypes = [vp, ctypes.POINTER(ctypes.c_uint32), c_i64, ctypes.POINTER(c_i64)]
    L.lm_counters.argtypes = [vp, ctypes.POINTER(c_i64)]
    L.lm_set_timing.argtypes = [vp, c_int]
    L.lm_stage_times.argtypes = [vp, ctypes.POINTER(c_f)]
    L.lm_stream.argtypes = [vp]
    L.lm_stream.restype = vp
    L.lm_launch_count.argtypes = [vp]
    L.lm_launch_count.restype = c_i64
    f32p, f64p = ctypes.POINTER(ctypes.c_float), ctypes.POINTER(ctypes.c_double)
    u16p = ctypes.POINTER(ctypes.c_uint16)
    L.lm_set_template_renders.argtypes = [vp, c_i64, c_i64, ctypes.POINTER(u16p), c_int, c_int, f32p, f32p, f32p]
    L.lm_enqueue_pose.argtypes = [vp, f32p, c_int, c_int]
    L.lm_complete_pose.argtypes = [vp, vp, f64p, f64p, f32p, c_i64, ctypes.POINTER(c_i64), ctypes.POINTER(c_i64)]
    L.lm_enqueue_pose_nms.argtypes = [vp, ctypes.c_double]
    L.lm_complete_detect.argtypes = [vp, vp, f64p, f64p, f32p, c_i64] + [ctypes.POINTER(c_i64)] * 4
    L.lm_detect_batch.argtypes = [vp, c_int, u8p_, u16p, c_int, c_int, ctypes.POINTER(u8p_), c_f, f32p, ctypes.c_double, c_int, c_int,
                                  c_int, c_int, ctypes.c_double, vp, f64p, f64p, f32p, c_i64, ctypes.POINTER(c_i64),
                                  ctypes.POINTER(c_i64)]
    L.lm_peer_detect_batch.argtypes = L.lm_detect_batch.argtypes
    L.lm_bind_images_device.argtypes = [vp, vp, c_i64, vp, c_i64, c_int, c_f, c_int, c_int, vp, vp, c_i64, vp]
    L.lm_detect_batch_device.argtypes = [vp, c_int, ctypes.POINTER(vp), c_i64, ctypes.POINTER(vp), c_i64, c_int, c_f, c_int, c_int,
                                         ctypes.POINTER(vp), c_i64, vp] + L.lm_detect_batch.argtypes[7:]
    L.lm_debug_depth.argtypes = [vp, u16p, c_i64]
    L.lm_debug_plan.argtypes = [vp, i32p, c_i64]
    L.lm_debug_coarse.argtypes = [vp, ctypes.POINTER(ctypes.c_uint32), c_i64, u16p, c_i64, i32p]
    L.lm_debug_pose_clouds.argtypes = [vp, c_int, c_int, vp, c_i64]
    L.lm_nms_translations.argtypes = [c_int, c_i64, f64p, f64p, ctypes.c_double, i32p, ctypes.POINTER(c_i64)]
    L.lm_set_pose_verify.argtypes = [vp, c_int, ctypes.c_double, c_int, ctypes.c_double]
    L.lm_pose_verify.argtypes = [vp, f32p, i32p, c_i64, ctypes.POINTER(c_i64)]
    L.lm_pose_verify_points.argtypes = [c_int, f64p, c_i64, f64p, u16p, c_int, c_int, f32p, ctypes.c_double, i32p, f32p]
    L.lm_icp_set_verify.argtypes = [vp, c_int, ctypes.c_double]
    L.lm_icp_verify.argtypes = [vp, f32p, i32p, c_i64, ctypes.POINTER(c_i64)]
    search = [c_int, c_int, ctypes.c_double, ctypes.c_double, ctypes.c_double, ctypes.c_uint64]
    L.lm_set_pose_search.argtypes = [vp] + search
    L.lm_icp_set_pose_search.argtypes = [vp] + search
    L.lm_pose_search_points.argtypes = [c_int, f64p, c_i64, f64p, u16p, c_int, c_int, f32p] + search + [c_i64, f64p, vp, c_i64]
    track_out = [f32p, vp, c_int, c_int, c_int, f64p, f64p, f64p, f32p, i32p, i32p]
    L.lm_track.argtypes = [vp, u16p, c_int, c_int] + track_out
    L.lm_track_device.argtypes = [vp, vp, c_i64, c_int, c_f, c_int, c_int] + track_out + [vp]
    batch_out = track_out[:2] + [i32p] + track_out[3:]  # n_objects [n_frames] in place of n
    L.lm_track_batch.argtypes = [vp, c_int, u16p, c_int, c_int] + batch_out
    L.lm_track_batch_device.argtypes = [vp, c_int, ctypes.POINTER(vp), c_i64, c_int, c_f, c_int, c_int] + batch_out + [vp]
    L.lm_peer_track_batch.argtypes = L.lm_track_batch.argtypes
    L.lm_peer_track_batch_device.argtypes = L.lm_track_batch_device.argtypes
    L.lm_pose_transforms.argtypes = [vp, f64p, c_i64, ctypes.POINTER(c_i64)]
    L.lm_set_track_views.argtypes = [vp, c_int, ctypes.c_double]
    L.lm_track_templates.argtypes = [vp, i32p, c_i64, ctypes.POINTER(c_i64)]
    L.lm_track_views_points.argtypes = [c_int, c_i64, f32p, f32p, c_i64, f64p, ctypes.c_double, ctypes.POINTER(c_i64), f64p]
    L.lm_icp_create.argtypes = [c_int, ctypes.POINTER(vp)]
    L.lm_icp_destroy.argtypes = [vp]
    L.lm_icp_destroy.restype = None
    L.lm_icp_process.argtypes = [vp, u16p, c_int, c_int, u16p, c_int, c_int, f32p, f32p, f32p, f32p, c_int, c_int, c_int,
                                 f64p, f64p, f32p]
    L.lm_icp_process_batch.argtypes = [vp, c_int, u16p, c_int, c_int, ctypes.POINTER(u16p), c_int, c_int, f32p, f32p, f32p, f32p,
                                       i32p, c_int, f64p, f64p, f32p]
    L.lm_icp_last_stats.argtypes = [vp, f64p]
    L.lm_icp_set_use_scene_cloud.argtypes = [vp, c_int]
    L.lm_icp_set_estimation.argtypes = [vp, c_int]
    L.lm_icp_launch_count.argtypes = [vp]
    L.lm_icp_launch_count.restype = c_i64
    L.lm_icp_set_capture.argtypes = [vp, c_int]
    L.lm_icp_capture.argtypes = [vp, c_int, c_int, vp, c_i64]
    L.lm_icp_process_batch_device.argtypes = [vp, c_int, vp, c_i64, c_int, c_f, c_int, c_int, ctypes.POINTER(vp), ctypes.POINTER(c_i64),
                                              c_int, c_f, c_int, c_int, f32p, f32p, f32p, f32p, i32p, c_int, f64p, f64p, f32p, vp]
    for name in SYMBOLS:
        getattr(L, name)  # AttributeError if the library does not export a declared symbol
    _lib = L
    return L


def coarse_tasks(words, sm_count, plane_bytes):
    """lm_coarse_tasks: the bit-sliced coarse scan's task table for items with `words` position words each, and its launch
    shape.  Returns (table [n_entries, 2] int32, n_full, n_rem, dict(tasks, split, warps_per_cta, grid)); no device needed."""
    L = load()
    words = np.ascontiguousarray(words, np.int32)
    i32p = ctypes.POINTER(ctypes.c_int32)
    n_entries, n_full, n_rem = ctypes.c_int64(), ctypes.c_int64(), ctypes.c_int64()
    shape = np.zeros(4, np.int32)
    args = (words.ctypes.data_as(i32p), len(words), sm_count, plane_bytes)
    check(L.lm_coarse_tasks(*args, None, 0, ctypes.byref(n_entries), ctypes.byref(n_full), ctypes.byref(n_rem),
                            shape.ctypes.data_as(i32p)))
    table = np.zeros((n_entries.value, 2), np.int32)
    check(L.lm_coarse_tasks(*args, table.ctypes.data_as(i32p), n_entries.value, ctypes.byref(n_entries), ctypes.byref(n_full),
                            ctypes.byref(n_rem), None))
    return table, n_full.value, n_rem.value, dict(tasks=int(shape[0]), split=int(shape[1]), warps_per_cta=int(shape[2]),
                                                  grid=int(shape[3]))


def coarse_descriptors(feats, tmeta, M, slot_low, T, rows, cols):
    """lm_coarse_descriptors: the bit-sliced coarse scan's feature descriptors of a packed bank (feats [n, 3], tmeta
    [G, S, 4]) at the level of slots slot_low .. slot_low + M - 1 (sampling step T, rows x cols).  Returns (desc uint32,
    info [G, 2] int32 = first descriptor and feature count, fits [G] bool, zero descriptor); no device needed."""
    L = load()
    feats = np.ascontiguousarray(feats, np.int32).reshape(-1, 3)
    tmeta = np.ascontiguousarray(tmeta, np.int32)
    G = len(tmeta)
    tmeta = tmeta.reshape(G, -1, 4)
    S = tmeta.shape[1]
    i32p, u32p = ctypes.POINTER(ctypes.c_int32), ctypes.POINTER(ctypes.c_uint32)
    n_desc, zero = ctypes.c_int64(), ctypes.c_uint32()
    info = np.zeros((G, 2), np.int32)
    fits = np.zeros(G, np.uint8)
    args = (feats.ctypes.data_as(i32p), tmeta.ctypes.data_as(i32p), G, S, M, slot_low, T, rows, cols)
    check(L.lm_coarse_descriptors(*args, None, 0, ctypes.byref(n_desc), info.ctypes.data_as(i32p),
                                  fits.ctypes.data_as(ctypes.POINTER(ctypes.c_uint8)), ctypes.byref(zero)))
    desc = np.zeros(n_desc.value, np.uint32)
    check(L.lm_coarse_descriptors(*args, desc.ctypes.data_as(u32p), len(desc), ctypes.byref(n_desc), None, None, None))
    return desc, info, fits.astype(bool), int(zero.value)


def check(rc):
    if rc == LM_OK:
        return
    msg = load().lm_last_error().decode("utf-8", "replace")
    if rc == LM_E_INVALID:
        raise RuntimeError(msg)  # the reference raises cv::Exception -> RuntimeError through pybind11
    raise LinemodLibraryError("linemod_b200 error %d: %s" % (rc, msg))


class NativeDetector:
    """Thin RAII wrapper over the lm_detector handle."""

    def __init__(self, T, device=0):
        L = load()
        self._L = L
        self.T = [int(t) for t in T]
        self.levels = len(self.T)
        arr = (ctypes.c_int * self.levels)(*self.T)
        h = ctypes.c_void_p()
        check(L.lm_create(int(device), self.levels, arr, ctypes.byref(h)))
        self._h = h
        self._keep = None
        self.device = int(device)

    def close(self):
        if getattr(self, "_h", None):
            self._L.lm_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @staticmethod
    def _i32(a):
        return a.ctypes.data_as(ctypes.POINTER(ctypes.c_int32))

    def load_bank(self, packed, slots):
        cb = np.ascontiguousarray(packed["class_begin"], np.int32)
        tm = np.ascontiguousarray(packed["tmeta"], np.int32)
        ft = np.ascontiguousarray(packed["feats"], np.int32)
        check(self._L.lm_load_bank(self._h, len(cb) - 1, self._i32(cb), int(slots), self._i32(tm), self._i32(ft),
                                   int(ft.shape[0])))

    def select(self, class_indices=None, shard_index=0, shard_count=1, layout=SHARD_CONTIGUOUS):
        """layout: SHARD_CONTIGUOUS (blocks of the sequence) or SHARD_INTERLEAVED (rank r takes r, r+N, ...)."""
        if class_indices is None:
            check(self._L.lm_select_layout(self._h, None, -1, int(shard_index), int(shard_count), int(layout)))
        else:
            a = np.ascontiguousarray(class_indices, np.int32)
            check(self._L.lm_select_layout(self._h, self._i32(a), int(a.shape[0]), int(shard_index), int(shard_count), int(layout)))

    def prepare(self):
        check(self._L.lm_prepare(self._h))

    def shard_range(self):
        b, c = ctypes.c_int64(), ctypes.c_int64()
        check(self._L.lm_shard_range(self._h, ctypes.byref(b), ctypes.byref(c)))
        return b.value, c.value

    def _frame_args(self, quantized):
        qs = []
        rows, cols = [], []
        for lvl in quantized:
            if len(lvl) != 2:
                raise RuntimeError("sources.size() == modalities.size()")
            rows.append(lvl[0].shape[0])
            cols.append(lvl[0].shape[1])
            for q in lvl:
                if q.dtype != np.uint8 or q.ndim != 2 or q.shape != lvl[0].shape:
                    raise TypeError("quantized images must be uint8 HxW, same size per level")
                qs.append(np.ascontiguousarray(q))
        if len(quantized) != self.levels:
            raise RuntimeError("expected %d pyramid levels, got %d" % (self.levels, len(quantized)))
        ptrs = (ctypes.POINTER(ctypes.c_uint8) * len(qs))(*[q.ctypes.data_as(ctypes.POINTER(ctypes.c_uint8)) for q in qs])
        r = (ctypes.c_int * len(rows))(*rows)
        c = (ctypes.c_int * len(cols))(*cols)
        return qs, ptrs, r, c

    def upload_quantized(self, quantized):
        qs, ptrs, r, c = self._frame_args(quantized)
        check(self._L.lm_upload_quantized(self._h, ptrs, r, c))

    @staticmethod
    def _image_args(rgb, depth, masks):
        rgb = np.ascontiguousarray(rgb)
        depth = np.ascontiguousarray(depth)
        if rgb.dtype != np.uint8 or rgb.ndim != 3 or rgb.shape[2] != 3:
            raise TypeError("sources[0] must be a uint8 HxWx3 colour image")
        if depth.dtype != np.uint16 or depth.shape != rgb.shape[:2]:
            raise TypeError("sources[1] must be a uint16 HxW depth image of the same size")
        mk = [None, None]
        if masks:
            if len(masks) != 2:
                raise RuntimeError("masks.size() == modalities.size()")
            for i, m in enumerate(masks):
                if m is not None and np.asarray(m).size:
                    m = np.ascontiguousarray(m)
                    if m.dtype != np.uint8 or m.shape != rgb.shape[:2]:
                        raise RuntimeError("mask.size() == source.size()")
                    mk[i] = m
        u8p = ctypes.POINTER(ctypes.c_uint8)
        ptr = lambda a: a.ctypes.data_as(u8p) if a is not None else None
        return rgb, depth, mk, (ptr(rgb), depth.ctypes.data_as(ctypes.POINTER(ctypes.c_uint16)), rgb.shape[0], rgb.shape[1],
                               ptr(mk[0]), ptr(mk[1]))

    def upload_images(self, rgb, depth, masks=None):
        keep = self._image_args(rgb, depth, masks)
        check(self._L.lm_upload_images(self._h, *keep[3]))

    def bind_frame(self, frame):
        """lm_bind_images_device of a DeviceFrame, ordered on its stream."""
        for t in frame.tensors:
            # the caching allocator reuses the frame only after the stream's work, which waits for the ingest
            t.record_stream(frame.stream)
        check(self._L.lm_bind_images_device(self._h, frame.rgb, frame.pitches[0], frame.depth, frame.pitches[1], frame.format,
                                            ctypes.c_float(frame.scale), frame.rows, frame.cols, frame.masks[0], frame.masks[1],
                                            frame.pitches[2], frame.stream.cuda_stream))

    def set_frame(self, rgb, depth, masks=None, depth_scale=1.0, stream=None):
        """upload_images for numpy arrays; bind_frame for CUDA tensors, or for a DeviceFrame passed as rgb."""
        frame = frame_inputs(rgb, depth, masks, depth_scale, stream, self.device)
        if frame is None:
            self.upload_images(rgb, depth, masks)
        else:
            self.bind_frame(frame)

    def depth_image(self, shape):
        """The u16 mm depth of the frame last uploaded or bound (lm_debug_depth)."""
        out = np.zeros(shape, np.uint16)
        check(self._L.lm_debug_depth(self._h, out.ctypes.data_as(ctypes.POINTER(ctypes.c_uint16)), out.size))
        return out

    def match_images(self, rgb, depth, masks, threshold, depth_scale=1.0, stream=None):
        frame = frame_inputs(rgb, depth, masks, depth_scale, stream, self.device)
        if frame is not None:  # lm_match_images of a bound device frame
            self.bind_frame(frame)
            self.run(threshold)
            return self.finish(self.fetch_records())
        keep = self._image_args(rgb, depth, masks)
        cap = 1 << 12
        while True:
            out = np.empty(cap, MATCH_DTYPE)
            n = ctypes.c_int64()
            rc = self._L.lm_match_images(self._h, *keep[3], ctypes.c_float(threshold), out.ctypes.data_as(ctypes.c_void_p), cap,
                                         ctypes.byref(n))
            if rc == LM_E_CAPACITY:
                cap = int(n.value)
                continue
            check(rc)
            return out[:n.value].copy()

    def quantized(self, level, modality, shape):
        out = np.zeros(shape, np.uint8)
        check(self._L.lm_debug_quantized(self._h, level, modality, out.ctypes.data_as(ctypes.POINTER(ctypes.c_uint8)), out.size))
        return out

    def bind_quantized_device(self, ptrs, rows, cols):
        """ptrs: device addresses (ints) index level*2+modality; rows/cols per level."""
        p = (ctypes.c_void_p * len(ptrs))(*[int(x) for x in ptrs])
        r = (ctypes.c_int * len(rows))(*[int(x) for x in rows])
        c = (ctypes.c_int * len(cols))(*[int(x) for x in cols])
        check(self._L.lm_bind_quantized_device(self._h, p, r, c))

    @staticmethod
    def bind_args(ptrs, rows, cols):
        """The ctypes arrays of bind_quantized_device, built once for a frame that is bound many times."""
        return ((ctypes.c_void_p * len(ptrs))(*[int(x) for x in ptrs]), (ctypes.c_int * len(rows))(*[int(x) for x in rows]),
                (ctypes.c_int * len(cols))(*[int(x) for x in cols]))

    def bind_quantized_device_args(self, args):
        check(self._L.lm_bind_quantized_device(self._h, args[0], args[1], args[2]))

    def run(self, threshold):
        check(self._L.lm_run(self._h, ctypes.c_float(threshold)))

    def enqueue(self, threshold):
        check(self._L.lm_enqueue(self._h, ctypes.c_float(threshold)))

    def complete(self):
        check(self._L.lm_complete(self._h))

    def fetch_records(self):
        cap = 1 << 12
        while True:
            out = np.empty(cap, RECORD_DTYPE)
            n = ctypes.c_int64()
            rc = self._L.lm_fetch_records(self._h, out.ctypes.data_as(ctypes.c_void_p), cap, ctypes.byref(n))
            if rc == LM_E_CAPACITY:
                cap = int(n.value)
                continue
            check(rc)
            return out[:n.value].copy()

    def set_result_buffer(self, device_ptr, capacity_records):
        check(self._L.lm_set_result_buffer(self._h, ctypes.c_void_p(device_ptr) if device_ptr else None, int(capacity_records)))

    # ---- multi-GPU exchange fused into the refinement kernel (include/linemod_b200.h, lm_peer_*) ----
    def peer_export(self, world, capacity_records=8192):
        """Allocate this rank's exchange buffer; returns its CUDA IPC handle (bytes)."""
        h = (ctypes.c_uint8 * PEER_HANDLE_BYTES)()
        check(self._L.lm_peer_export(self._h, int(world), int(capacity_records), h))
        return bytes(h)

    def peer_base(self):
        b = ctypes.c_void_p()
        check(self._L.lm_peer_base(self._h, ctypes.byref(b)))
        return b.value

    def peer_connect(self, rank, world, handles):
        """handles: list of `world` IPC handles (bytes), index = rank (own entry ignored)."""
        blob = b"".join(bytes(h) for h in handles)
        if len(blob) != world * PEER_HANDLE_BYTES:
            raise ValueError("need %d handles of %d bytes" % (world, PEER_HANDLE_BYTES))
        buf = (ctypes.c_uint8 * len(blob)).from_buffer_copy(blob)
        check(self._L.lm_peer_connect(self._h, int(rank), int(world), buf))

    def peer_connect_local(self, rank, world, bases):
        arr = (ctypes.c_void_p * world)(*[int(b) for b in bases])
        check(self._L.lm_peer_connect_local(self._h, int(rank), int(world), arr))

    def peer_disconnect(self):
        check(self._L.lm_peer_disconnect(self._h))

    def peer_share_pose(self, on):
        """Divide the pose stage over the ranks of the connected exchange (lm_peer_share_pose).  Every rank must set the
        same value before its next frame and, while it is on, run the pose stage of every frame."""
        if not isinstance(on, (bool, int, np.bool_, np.integer)):
            raise TypeError("peer_share_pose(on): on must be a bool, got %s" % type(on).__name__)
        check(self._L.lm_peer_share_pose(self._h, 1 if on else 0))

    def device_result(self):
        p, cap = ctypes.c_void_p(), ctypes.c_int64()
        check(self._L.lm_device_result(self._h, ctypes.byref(p), ctypes.byref(cap)))
        return p.value, cap.value

    def finish(self, records):
        records = np.ascontiguousarray(records, RECORD_DTYPE)
        cap = max(int(records.shape[0]), 1)
        out = np.zeros(cap, MATCH_DTYPE)
        n = ctypes.c_int64()
        check(self._L.lm_finish(self._h, records.ctypes.data_as(ctypes.c_void_p), int(records.shape[0]),
                                out.ctypes.data_as(ctypes.c_void_p), cap, ctypes.byref(n)))
        return out[:n.value].copy()

    def match_quantized(self, quantized, threshold):
        qs, ptrs, r, c = self._frame_args(quantized)
        cap = 1 << 12
        while True:
            out = np.empty(cap, MATCH_DTYPE)
            n = ctypes.c_int64()
            rc = self._L.lm_match_quantized(self._h, ptrs, r, c, ctypes.c_float(threshold),
                                            out.ctypes.data_as(ctypes.c_void_p), cap, ctypes.byref(n))
            if rc == LM_E_CAPACITY:
                cap = int(n.value)
                continue
            check(rc)
            return out[:n.value].copy()

    # ---- post-match stage on the device: greedy NMS + top-k (include/linemod_b200.h, lm_*_post) ----
    def set_boxes(self, wh):
        if wh is None:
            check(self._L.lm_set_boxes(self._h, None, 0))
            return
        wh = np.ascontiguousarray(wh, np.int32).reshape(-1, 2)
        check(self._L.lm_set_boxes(self._h, self._i32(wh), wh.shape[0]))

    def enqueue_post(self, iou_threshold=0.5, top_k=3):
        check(self._L.lm_enqueue_post(self._h, float(iou_threshold), int(top_k)))

    def complete_post(self):
        out = np.empty(1024, MATCH_DTYPE)
        n, nrec = ctypes.c_int64(), ctypes.c_int64()
        check(self._L.lm_complete_post(self._h, out.ctypes.data_as(ctypes.c_void_p), out.shape[0], ctypes.byref(n),
                                       ctypes.byref(nrec)))
        return out[:n.value].copy(), int(nrec.value)

    def match_top(self, quantized, threshold, iou_threshold=0.5, top_k=3):
        qs, ptrs, r, c = self._frame_args(quantized)
        out = np.empty(1024, MATCH_DTYPE)
        n, nrec = ctypes.c_int64(), ctypes.c_int64()
        check(self._L.lm_match_top(self._h, ptrs, r, c, ctypes.c_float(threshold), float(iou_threshold), int(top_k),
                                   out.ctypes.data_as(ctypes.c_void_p), out.shape[0], ctypes.byref(n), ctypes.byref(nrec)))
        return out[:n.value].copy(), int(nrec.value)

    # ---- depth gate of the coarse scan (include/linemod_b200.h, lm_set_depth_gate) ----
    def set_template_depths(self, first, z_mm):
        """Training distances (mm) of templates [first, first + len(z_mm)) of the bank; NaN or <= 0: never gated."""
        z = np.ascontiguousarray(z_mm, np.float32).reshape(-1)
        check(self._L.lm_set_template_depths(self._h, int(first), z.shape[0], z.ctypes.data_as(ctypes.POINTER(ctypes.c_float))))

    def set_depth_gate(self, tolerance):
        """Gate the coarse scan by scene depth with this tolerance from the next frame on; None turns the gate off."""
        if tolerance is None:
            check(self._L.lm_set_depth_gate(self._h, 0, 0.0))
        else:
            check(self._L.lm_set_depth_gate(self._h, 1, depth_gate_tolerance(tolerance)))

    def depth_gate_stats(self):
        """Of the last frame, which ran gated: candidates before / after the gate, empty cells, templates with a distance."""
        a = (ctypes.c_int64 * 4)()
        check(self._L.lm_depth_gate_stats(self._h, a))
        return dict(zip(["before", "after", "empty_cells", "with_distance"], [int(v) for v in a]))

    # ---- pose stage behind the NMS (include/linemod_b200.h, lm_*_pose) ----
    def set_template_renders(self, first, depths, K, R, t):
        """Templates [first, first + len(depths)) of the bank: depths u16 HxW (one size per call), K / R [n,3,3] f32,
        t [n,3] f32 mm.  The same array may serve several templates."""
        n = len(depths)
        ds = [np.ascontiguousarray(d, np.uint16) for d in depths]
        if any(d.ndim != 2 or d.shape != ds[0].shape for d in ds):
            raise TypeError("renders must be uint16 HxW images of one size")
        u16p = ctypes.POINTER(ctypes.c_uint16)
        f32p = ctypes.POINTER(ctypes.c_float)
        ptrs = (u16p * max(n, 1))(*[d.ctypes.data_as(u16p) for d in ds])
        K = np.ascontiguousarray(K, np.float32).reshape(n, 9)
        R = np.ascontiguousarray(R, np.float32).reshape(n, 9)
        t = np.ascontiguousarray(t, np.float32).reshape(n, 3)
        rows, cols = ds[0].shape if n else (0, 0)
        check(self._L.lm_set_template_renders(self._h, int(first), n, ptrs, int(rows), int(cols), K.ctypes.data_as(f32p),
                                              R.ctypes.data_as(f32p), t.ctypes.data_as(f32p)))

    def set_pose_estimation(self, estimation):
        """"point_to_plane" (default), "point_to_point" or "pso" for the next pose stage (lm_set_pose_estimation)."""
        check(self._L.lm_set_pose_estimation(self._h, estimation_code(estimation)))

    def set_pose_search(self, particles=64, iterations=40, dt_mm=40.0, dr_deg=30.0, clamp_mm=20.0, seed=0):
        """The particle swarm of estimation="pso" for the next pose stage (lm_set_pose_search)."""
        check(self._L.lm_set_pose_search(self._h, int(particles), int(iterations), float(dt_mm), float(dr_deg), float(clamp_mm),
                                         int(seed)))

    def enqueue_pose(self, sceneK, max_iterations=30, use_scene_cloud=False, estimation="point_to_plane"):
        est = estimation_code(estimation)
        sK = np.ascontiguousarray(sceneK, np.float32).reshape(9)
        check(self._L.lm_set_pose_estimation(self._h, est))
        check(self._L.lm_enqueue_pose(self._h, sK.ctypes.data_as(ctypes.POINTER(ctypes.c_float)), int(max_iterations),
                                      1 if use_scene_cloud else 0))

    def complete_pose(self):
        """Returns (survivors, R [n,3,3] f64, t [n,3] f64 mm, residual [n] f32, records seen by the NMS); rows of an
        early return (residual -1) keep R / t at NaN."""
        cap = 1024
        out = np.empty(cap, MATCH_DTYPE)
        Ro = np.full((cap, 3, 3), np.nan, np.float64)
        to = np.full((cap, 3), np.nan, np.float64)
        res = np.zeros(cap, np.float32)
        n, nrec = ctypes.c_int64(), ctypes.c_int64()
        f64p = ctypes.POINTER(ctypes.c_double)
        check(self._L.lm_complete_pose(self._h, out.ctypes.data_as(ctypes.c_void_p), Ro.ctypes.data_as(f64p), to.ctypes.data_as(f64p),
                                       res.ctypes.data_as(ctypes.POINTER(ctypes.c_float)), cap, ctypes.byref(n), ctypes.byref(nrec)))
        k = n.value
        return out[:k].copy(), Ro[:k].copy(), to[:k].copy(), res[:k].copy(), int(nrec.value)

    def match_pose(self, rgb, depth, masks, threshold, sceneK, iou_threshold=0.5, top_k=3, max_iterations=30, use_scene_cloud=False,
                   estimation="point_to_plane", depth_scale=1.0, stream=None):
        """set_frame + enqueue + enqueue_post + enqueue_pose + complete_pose: one chain on the detector's stream."""
        estimation_code(estimation)
        self.set_frame(rgb, depth, masks, depth_scale, stream)
        self.enqueue(threshold)
        self.enqueue_post(iou_threshold, top_k)
        self.enqueue_pose(sceneK, max_iterations, use_scene_cloud, estimation)
        return self.complete_pose()

    # ---- pose NMS behind the pose stage (include/linemod_b200.h, lm_enqueue_pose_nms / lm_complete_detect) ----
    def enqueue_pose_nms(self, translation_threshold=40.0):
        check(self._L.lm_enqueue_pose_nms(self._h, float(translation_threshold)))

    def complete_detect(self):
        """Returns (kept survivors, R [n,3,3] f64, t [n,3] f64 mm, residual [n] f32, counts) in keep order; counts is a
        dict of survivors (box NMS), posed (survivors with a pose) and records (kept records the box NMS saw)."""
        cap = 1024
        out = np.empty(cap, MATCH_DTYPE)
        Ro = np.empty((cap, 3, 3), np.float64)
        to = np.empty((cap, 3), np.float64)
        res = np.empty(cap, np.float32)
        n, ns, npo, nrec = ctypes.c_int64(), ctypes.c_int64(), ctypes.c_int64(), ctypes.c_int64()
        f64p = ctypes.POINTER(ctypes.c_double)
        check(self._L.lm_complete_detect(self._h, out.ctypes.data_as(ctypes.c_void_p), Ro.ctypes.data_as(f64p), to.ctypes.data_as(f64p),
                                         res.ctypes.data_as(ctypes.POINTER(ctypes.c_float)), cap, ctypes.byref(n), ctypes.byref(ns),
                                         ctypes.byref(npo), ctypes.byref(nrec)))
        k = n.value
        return (out[:k].copy(), Ro[:k].copy(), to[:k].copy(), res[:k].copy(),
                dict(survivors=int(ns.value), posed=int(npo.value), records=int(nrec.value)))

    def detect(self, rgb, depth, masks, threshold, sceneK, iou_threshold=0.5, top_k=0, max_iterations=30, use_scene_cloud=False,
               translation_threshold=40.0, estimation="point_to_plane", depth_scale=1.0, stream=None):
        """set_frame + enqueue + enqueue_post + enqueue_pose + enqueue_pose_nms + complete_detect: RGB-D frame (numpy, or
        CUDA tensors) to the object list in one chain on the detector's stream."""
        estimation_code(estimation)
        self.set_frame(rgb, depth, masks, depth_scale, stream)
        self.enqueue(threshold)
        self.enqueue_post(iou_threshold, top_k)
        self.enqueue_pose(sceneK, max_iterations, use_scene_cloud, estimation)
        self.enqueue_pose_nms(translation_threshold)
        return self.complete_detect()

    # ---- a batch of frames through one pose stage (include/linemod_b200.h, lm_detect_batch) ----
    def detect_batch(self, rgb, depth, masks, threshold, sceneK, iou_threshold=0.5, top_k=0, max_iterations=30, use_scene_cloud=False,
                     pose_nms=True, translation_threshold=40.0, cap=None, estimation="point_to_plane"):
        """rgb [n,H,W,3] u8, depth [n,H,W] u16, masks None or one (mask_color, mask_depth) pair per frame (None or an empty
        array: no mask), sceneK [n,3,3].  Returns one tuple per frame: what complete_detect returns (pose_nms) or what
        complete_pose returns.  cap: entries of the first attempt (default: every survivor of every frame); a larger
        batch result grows it and runs the batch again; any other LM_E_CAPACITY raises.  self.batch_counts keeps the last
        call's [n,4] frame counts (entries, survivors, posed, records).  The handle keeps the batch's buffers for the next
        one, sized for its shape: with top_k 0 that includes the pose stage's cloud buffers for 1024 survivors (as a
        single frame with top_k 0 uses), however few survivors the frames have.  estimation: the ICP's estimation step
        (set_pose_estimation)."""
        return self._batch(self._L.lm_detect_batch, rgb, depth, masks, threshold, sceneK, iou_threshold, top_k, max_iterations,
                           use_scene_cloud, pose_nms, translation_threshold, cap, estimation)

    def peer_detect_batch(self, rgb, depth, masks, threshold, sceneK, iou_threshold=0.5, top_k=0, max_iterations=30,
                          use_scene_cloud=False, pose_nms=True, translation_threshold=40.0, cap=None, estimation="point_to_plane"):
        """detect_batch over the ranks of the connected exchange (lm_peer_detect_batch): every rank calls it with the same
        frames and arguments, and every rank returns what detect_batch returns on one unconnected handle over the whole
        bank.  The retry on too small outputs happens on every rank alike; records beyond the exchange's
        capacity_records raise LinemodLibraryError on every rank (reconnect with a larger capacity).  Every rank passes the
        same estimation."""
        return self._batch(self._L.lm_peer_detect_batch, rgb, depth, masks, threshold, sceneK, iou_threshold, top_k, max_iterations,
                           use_scene_cloud, pose_nms, translation_threshold, cap, estimation)

    def _batch(self, fn, rgb, depth, masks, threshold, sceneK, iou_threshold, top_k, max_iterations, use_scene_cloud, pose_nms,
               translation_threshold, cap, estimation="point_to_plane"):
        est = estimation_code(estimation)
        rgb = np.ascontiguousarray(rgb)
        depth = np.ascontiguousarray(depth)
        if rgb.dtype != np.uint8 or rgb.ndim != 4 or rgb.shape[3] != 3:
            raise TypeError("rgb must be uint8 [n,H,W,3]")
        if depth.dtype != np.uint16 or depth.shape != rgb.shape[:3]:
            raise TypeError("depth must be uint16 [n,H,W] of the colour images' size")
        n, rows, cols = rgb.shape[:3]
        sK = np.ascontiguousarray(sceneK, np.float32)
        if sK.shape != (n, 3, 3):
            raise ValueError("sceneK must be [%d,3,3], got %s" % (n, sK.shape))
        u8p = ctypes.POINTER(ctypes.c_uint8)
        mptr, keep = None, []
        if masks is not None:
            if len(masks) != n:
                raise ValueError("%d mask pairs for %d frames" % (len(masks), n))
            mptr = (u8p * (2 * n))()
            for f, pair in enumerate(masks):
                if len(pair) != 2:
                    raise RuntimeError("masks.size() == modalities.size()")
                for m, a in enumerate(pair):
                    if a is not None and np.asarray(a).size:
                        a = np.ascontiguousarray(a)
                        if a.dtype != np.uint8 or a.shape != (rows, cols):
                            raise RuntimeError("mask.size() == source.size()")
                        keep.append(a)
                        mptr[2 * f + m] = a.ctypes.data_as(u8p)
        return self._batch_run(fn, (n, rgb.ctypes.data_as(u8p), depth.ctypes.data_as(ctypes.POINTER(ctypes.c_uint16)), rows, cols, mptr),
                               n, threshold, sK, iou_threshold, top_k, max_iterations, use_scene_cloud, pose_nms, translation_threshold,
                               cap, est)

    def detect_batch_device(self, batch, threshold, sceneK, iou_threshold=0.5, top_k=0, max_iterations=30, use_scene_cloud=False,
                            pose_nms=True, translation_threshold=40.0, cap=None, estimation="point_to_plane"):
        """detect_batch of a DeviceBatch (lm_detect_batch_device), ordered on its stream.  Returns what detect_batch returns."""
        est = estimation_code(estimation)
        sK = np.ascontiguousarray(sceneK, np.float32)
        if sK.shape != (batch.n, 3, 3):
            raise ValueError("sceneK must be [%d,3,3], got %s" % (batch.n, sK.shape))
        for t in batch.tensors:
            t.record_stream(batch.stream)
        return self._batch_run(self._L.lm_detect_batch_device, batch.args, batch.n, threshold, sK, iou_threshold, top_k,
                               max_iterations, use_scene_cloud, pose_nms, translation_threshold, cap, est)

    def _batch_run(self, fn, frame_args, n, threshold, sK, iou_threshold, top_k, max_iterations, use_scene_cloud, pose_nms,
                   translation_threshold, cap, est):
        bound = top_k if top_k > 0 else 1024
        cap = n * bound if cap is None else max(int(cap), 1)
        counts = np.zeros((n, 4), np.int64)
        f32p, f64p = ctypes.POINTER(ctypes.c_float), ctypes.POINTER(ctypes.c_double)
        check(self._L.lm_set_pose_estimation(self._h, est))
        while True:
            out = np.empty(cap, MATCH_DTYPE)
            Ro = np.full((cap, 3, 3), np.nan, np.float64)
            to = np.full((cap, 3), np.nan, np.float64)
            res = np.zeros(cap, np.float32)
            total = ctypes.c_int64()
            rc = fn(self._h, *frame_args, ctypes.c_float(threshold), sK.ctypes.data_as(f32p), float(iou_threshold), int(top_k), int(max_iterations),
                    1 if use_scene_cloud else 0, 1 if pose_nms else 0, float(translation_threshold), out.ctypes.data_as(ctypes.c_void_p),
                    Ro.ctypes.data_as(f64p), to.ctypes.data_as(f64p), res.ctypes.data_as(f32p), cap, ctypes.byref(total),
                    counts.ctypes.data_as(ctypes.POINTER(ctypes.c_int64)))
            if rc == LM_E_CAPACITY and total.value > cap:  # only the outputs were too small: retry with the total
                cap = int(total.value)
                continue
            # any other LM_E_CAPACITY (records beyond the exchange or the result block) would recur on every retry
            check(rc)
            break
        self.batch_counts = counts
        frames, at = [], 0
        for f in range(n):
            k = int(counts[f, 0])
            sl = slice(at, at + k)
            at += k
            if pose_nms:
                extra = dict(survivors=int(counts[f, 1]), posed=int(counts[f, 2]), records=int(counts[f, 3]))
            else:
                extra = int(counts[f, 3])
            frames.append((out[sl].copy(), Ro[sl].copy(), to[sl].copy(), res[sl].copy(), extra))
        return frames

    def linear_memories(self, level, modality, shape):
        out = np.zeros(shape, np.uint8)
        check(self._L.lm_debug_linear_memories(self._h, level, modality, out.ctypes.data_as(ctypes.POINTER(ctypes.c_uint8)),
                                               out.size))
        return out

    def bit_planes(self):
        """The lowest level's spread bit-planes of the last run (lm_debug_bit_planes): uint32 [M * 8 * lbw]."""
        n = ctypes.c_int64()
        rc = self._L.lm_debug_bit_planes(self._h, None, 0, ctypes.byref(n))
        if rc != LM_E_CAPACITY:
            check(rc)
        out = np.zeros(int(n.value), np.uint32)
        if out.size:
            check(self._L.lm_debug_bit_planes(self._h, out.ctypes.data_as(ctypes.POINTER(ctypes.c_uint32)), out.size,
                                              ctypes.byref(n)))
        return out

    def time_k1_us(self, level, reps):
        """Mean device time of `reps` launches of the K1 blocks of `level` (-1: all of K1), as the last run planned them."""
        us = ctypes.c_float()
        check(self._L.lm_debug_time_k1(self._h, int(level), int(reps), ctypes.byref(us)))
        return float(us.value)

    def counters(self):
        a = (ctypes.c_int64 * 8)()
        check(self._L.lm_counters(self._h, a))
        keys = ["templates", "coarse_candidates", "scan_bytes", "refine_bytes", "kept", "refine_bytes_read",
                "filter_dropped_bytes", "filter_bytes_read"]
        return dict(zip(keys, [int(v) for v in a]))

    PLAN_KEYS = ["k1_band", "planes_level", "pseg", "k1_smem", "rounds", "bit_planes", "packed_templates", "byte_templates",
                 "k2_smem", "split", "plane_bytes", "k2_tasks", "filter_ok", "use_bits", "filter_templates", "gated",
                 "filter_items", "refine_bits_items", "refine_filtered_items", "refine_items", "refine_bits_ctas", "k1_low_mode"]

    def plan(self):
        """The kernels and launch shapes of the last run (lm_debug_plan); -1: that kernel did not run."""
        a = np.zeros(len(self.PLAN_KEYS), np.int32)
        check(self._L.lm_debug_plan(self._h, self._i32(a), a.size))
        return dict(zip(self.PLAN_KEYS, [int(v) for v in a]))

    def coarse(self):
        """The coarse scan's outputs of the last run (lm_debug_coarse): pass masks uint32 [n_work, nwords] and raw scores
        uint16 [n_work, plane], 0 wherever the pass bit is clear; work items in this handle's shard order."""
        dims = np.zeros(3, np.int32)
        u32p, u16p = ctypes.POINTER(ctypes.c_uint32), ctypes.POINTER(ctypes.c_uint16)
        rc = self._L.lm_debug_coarse(self._h, None, 0, None, 0, self._i32(dims))  # dims only
        if rc != LM_E_CAPACITY:
            check(rc)
        mask = np.zeros((int(dims[0]), int(dims[1])), np.uint32)
        raw = np.zeros((int(dims[0]), int(dims[2])), np.uint16)
        if rc == LM_E_CAPACITY:
            check(self._L.lm_debug_coarse(self._h, mask.ctypes.data_as(u32p), mask.size, raw.ctypes.data_as(u16p), raw.size,
                                          self._i32(dims)))
        return mask, raw

    def _pose_item(self, slot, what, out):
        check(self._L.lm_debug_pose_clouds(self._h, int(slot), CAPTURE_ITEMS[what], out.ctypes.data_as(ctypes.c_void_p), out.nbytes))
        return out

    def pose_clouds(self):
        """The clouds of the last pose-stage chunk this handle enqueued (lm_debug_pose_clouds): (head, slots).  head is a
        dict of the chunk's slots, rank, world and first (slot i holds survivor first + rank + i * world); slots has one
        dict per slot: posed (bool) and, where posed, counts (src, tgt), source / target [n,3] f64 (down-sampled), init
        [4,4] f64, raw_model / raw_scene [n,3] f64 (before down-sampling); a track chunk's slots also window (x, y, w, h)
        and status."""
        head = self._pose_item(-1, "slots", np.zeros(4, np.int32))
        out = []
        for i in range(int(head[0])):
            posed = bool(self._pose_item(i, "posed", np.zeros(1, np.uint8))[0])
            d = dict(posed=posed)
            w = np.zeros(5, np.int32)
            if self._L.lm_debug_pose_clouds(self._h, i, CAPTURE_ITEMS["window"], w.ctypes.data_as(ctypes.c_void_p), w.nbytes) == LM_OK:
                d["window"], d["status"] = w[:4].copy(), int(w[4])  # a track chunk's (lm_track)
            if posed:
                n, nt = self._pose_item(i, "counts", np.zeros(2, np.int32)).tolist()
                d.update(counts=(n, nt), source=self._pose_item(i, "source", np.zeros((n, 3))),
                         target=self._pose_item(i, "target", np.zeros((nt, 3))), init=self._pose_item(i, "init", np.zeros((4, 4))))
                for item in ("raw_model", "raw_scene"):  # sized by asking: LM_E_CAPACITY names the bytes
                    d[item] = self._pose_raw(i, item)
            out.append(d)
        return dict(zip(("slots", "rank", "world", "first"), [int(v) for v in head])), out

    def _pose_raw(self, slot, what):
        rc = self._L.lm_debug_pose_clouds(self._h, int(slot), CAPTURE_ITEMS[what], ctypes.byref(ctypes.c_uint8()), 0)
        if rc == LM_OK:
            return np.zeros((0, 3))
        if rc != LM_E_CAPACITY:
            check(rc)
        need = int(re.search(r"needs (\d+) bytes", self._L.lm_last_error().decode()).group(1))
        return self._pose_item(slot, what, np.zeros((need // 24, 3)))

    def set_timing(self, slots):
        check(self._L.lm_set_timing(self._h, int(slots)))

    def stage_times_us(self):
        a = (ctypes.c_float * 8)()
        check(self._L.lm_stage_times(self._h, a))
        keys = ["linear_memories", "coarse_scan", "offsets", "refine", "total", "refine_prep", "refine_filter", "refine_exact"]
        return dict(zip(keys, [float(v) for v in a]))

    def stream(self):
        return self._L.lm_stream(self._h)

    def launch_count(self):
        return int(self._L.lm_launch_count(self._h))

    def set_pose_verify(self, on, inlier_mm=10.0, rank_by=0, min_score=-math.inf):
        """lm_set_pose_verify for the next pose stage: on, the inlier distance (mm), the pose NMS's ranking (0 fitness, 1
        score) and its minimum score (-inf: none)."""
        check(self._L.lm_set_pose_verify(self._h, 1 if on else 0, float(inlier_mm), int(rank_by), float(min_score)))

    def pose_verify(self):
        """The verification of the last completed frame or batch (lm_pose_verify): (score [n] f32, counts [n,6] int32) in
        the order of its entries."""
        return _verify_results(self._L.lm_pose_verify, self._h)

    def pose_stats(self):
        """[survivors, hypotheses this rank refined, launches, 1 if shared] of the last completed pose stage (lm_pose_stats)."""
        a = (ctypes.c_int64 * 4)()
        check(self._L.lm_pose_stats(self._h, a))
        return [int(v) for v in a]

    def pose_transforms(self):
        """The 4x4 T of every entry of the last finished pose run (lm_pose_transforms): f64 [n,4,4], NaN without a pose."""
        n = ctypes.c_int64()
        f64p = ctypes.POINTER(ctypes.c_double)
        rc = self._L.lm_pose_transforms(self._h, None, 0, ctypes.byref(n))
        if rc != LM_E_CAPACITY:
            check(rc)
        out = np.empty((int(n.value), 4, 4), np.float64)
        if out.size:
            check(self._L.lm_pose_transforms(self._h, out.ctypes.data_as(f64p), out.shape[0], ctypes.byref(n)))
        return out

    def set_track_views(self, on, turn_deg=0.0):
        """lm_set_track_views for the next track calls: view following on or off, and the turn (degrees) from the
        template's view beyond which an object re-chooses its template."""
        check(self._L.lm_set_track_views(self._h, 1 if on else 0, float(turn_deg)))

    def track_templates(self):
        """The template (within its class) of every entry of the last finished track run (lm_track_templates): int32 [n]."""
        n = ctypes.c_int64()
        i32p = ctypes.POINTER(ctypes.c_int32)
        rc = self._L.lm_track_templates(self._h, None, 0, ctypes.byref(n))
        if rc != LM_E_CAPACITY:
            check(rc)
        out = np.zeros(int(n.value), np.int32)
        if out.size:
            check(self._L.lm_track_templates(self._h, out.ctypes.data_as(i32p), out.size, ctypes.byref(n)))
        return out

    @staticmethod
    def track_objects(objects):
        """lm_track_object [n] of (class_index, template_id, T [4,4] f64) triples."""
        arr = (TrackObject * max(len(objects), 1))()
        for i, (c, t, T) in enumerate(objects):
            arr[i].class_index, arr[i].template_id = int(c), int(t)
            arr[i].T[:] = [float(v) for v in np.asarray(T, np.float64).reshape(16)]
        return arr

    def track(self, depth, sceneK, objects, max_iterations=30, margin_px=4, estimation="point_to_plane"):
        """lm_track on a u16 HxW numpy depth (mm).  objects: (class_index, template_id, T) triples.  Returns (status [n]
        int32, T [n,4,4], R [n,3,3], t [n,3] mm, residual [n] f32, box [n,4] int32); an entry not tracked keeps its input
        T and R / t NaN."""
        depth = np.ascontiguousarray(depth)
        if depth.dtype != np.uint16 or depth.ndim != 2:
            raise TypeError("depth must be a uint16 HxW image (mm)")
        return self._track(lambda *a: self._L.lm_track(self._h, depth.ctypes.data_as(ctypes.POINTER(ctypes.c_uint16)), depth.shape[0],
                                                       depth.shape[1], *a), sceneK, objects, max_iterations, margin_px, estimation)

    def track_device(self, depth, pitch, depth_format, depth_scale, rows, cols, stream, sceneK, objects, max_iterations=30, margin_px=4,
                     estimation="point_to_plane"):
        """lm_track_device on a pitched device plane (u16 mm or f32 scaled by depth_scale) ordered on `stream` (a CUDA stream
        handle).  Returns what track returns."""
        return self._track(lambda *a: self._L.lm_track_device(self._h, depth, int(pitch), int(depth_format), ctypes.c_float(depth_scale),
                                                              int(rows), int(cols), *a, stream), sceneK, objects, max_iterations,
                           margin_px, estimation)

    def track_batch(self, depth, sceneK, objects, max_iterations=30, margin_px=4, estimation="point_to_plane"):
        """lm_track_batch on u16 [n,H,W] numpy depths (mm), sceneK [n,3,3].  objects: one list of (class_index, template_id,
        T) triples per frame.  Returns one tuple per frame, each what track returns for that frame."""
        return self._track_host(self._L.lm_track_batch, depth, sceneK, objects, max_iterations, margin_px, estimation)

    def track_batch_device(self, planes, pitch, depth_format, depth_scale, rows, cols, stream, sceneK, objects, max_iterations=30,
                           margin_px=4, estimation="point_to_plane"):
        """lm_track_batch_device on device planes (data pointers, one pitch, format and depth_scale) ordered on `stream`.
        Returns what track_batch returns."""
        return self._track_device(self._L.lm_track_batch_device, planes, pitch, depth_format, depth_scale, rows, cols, stream, sceneK,
                                  objects, max_iterations, margin_px, estimation)

    def peer_track_batch(self, depth, sceneK, objects, max_iterations=30, margin_px=4, estimation="point_to_plane"):
        """track_batch over the ranks of the connected exchange (lm_peer_track_batch): every rank calls it with the same
        frames, objects and estimation, and every rank returns what track_batch returns on one unconnected handle."""
        return self._track_host(self._L.lm_peer_track_batch, depth, sceneK, objects, max_iterations, margin_px, estimation)

    def peer_track_batch_device(self, planes, pitch, depth_format, depth_scale, rows, cols, stream, sceneK, objects, max_iterations=30,
                                margin_px=4, estimation="point_to_plane"):
        """track_batch_device over the ranks of the connected exchange (lm_peer_track_batch_device), as peer_track_batch."""
        return self._track_device(self._L.lm_peer_track_batch_device, planes, pitch, depth_format, depth_scale, rows, cols, stream, sceneK,
                                  objects, max_iterations, margin_px, estimation)

    def _track_host(self, fn, depth, sceneK, objects, max_iterations, margin_px, estimation):
        # lm_track_batch or lm_peer_track_batch on host depths
        depth = np.ascontiguousarray(depth)
        if depth.dtype != np.uint16 or depth.ndim != 3:
            raise TypeError("depth must be uint16 [n,H,W] images (mm)")
        n, rows, cols = depth.shape
        return self._track(lambda *a: fn(self._h, n, depth.ctypes.data_as(ctypes.POINTER(ctypes.c_uint16)), rows, cols, *a), sceneK, objects,
                           max_iterations, margin_px, estimation, n)

    def _track_device(self, fn, planes, pitch, depth_format, depth_scale, rows, cols, stream, sceneK, objects, max_iterations, margin_px,
                      estimation):
        # lm_track_batch_device or lm_peer_track_batch_device on device planes
        n = len(planes)
        ptrs = (ctypes.c_void_p * max(n, 1))(*planes)
        return self._track(lambda *a: fn(self._h, n, ptrs, int(pitch), int(depth_format), ctypes.c_float(depth_scale), int(rows), int(cols), *a,
                                         stream), sceneK, objects, max_iterations, margin_px, estimation, n)

    def _track(self, fn, sceneK, objects, max_iterations, margin_px, estimation, n_frames=None):
        # n_frames None: one frame's objects (lm_track); else one list of objects per frame, and one result tuple per frame
        est = estimation_code(estimation)
        sK = np.ascontiguousarray(sceneK, np.float32).reshape(-1)
        counts = None if n_frames is None else np.ascontiguousarray([len(o) for o in objects], np.int32)
        if counts is not None:
            if len(counts) != n_frames or sK.size != 9 * n_frames:
                raise ValueError("%d frames, %d object lists and %d intrinsics" % (n_frames, len(counts), sK.size // 9))
            objects = [o for frame in objects for o in frame]
        n = len(objects)
        arr = self.track_objects(objects)
        T = np.stack([np.asarray(o[2], np.float64).reshape(4, 4) for o in objects]) if n else np.zeros((0, 4, 4))
        T = np.ascontiguousarray(T)
        Ro = np.full((max(n, 1), 3, 3), np.nan)
        to = np.full((max(n, 1), 3), np.nan)
        res = np.zeros(max(n, 1), np.float32)
        status = np.zeros(max(n, 1), np.int32)
        box = np.zeros((max(n, 1), 4), np.int32)
        f32p, f64p = ctypes.POINTER(ctypes.c_float), ctypes.POINTER(ctypes.c_double)
        Tout = T if n else np.zeros((1, 4, 4))
        check(self._L.lm_set_pose_estimation(self._h, est))
        check(fn(sK.ctypes.data_as(f32p), ctypes.cast(arr, ctypes.c_void_p), n if counts is None else self._i32(counts), int(max_iterations),
                 int(margin_px), Tout.ctypes.data_as(f64p), Ro.ctypes.data_as(f64p), to.ctypes.data_as(f64p), res.ctypes.data_as(f32p),
                 self._i32(status), self._i32(box)))
        got = status[:n].copy(), Tout[:n].copy(), Ro[:n].copy(), to[:n].copy(), res[:n].copy(), box[:n].copy()
        if counts is None:
            return got
        starts = np.cumsum(np.concatenate([[0], counts]))
        return [tuple(a[s:e] for a in got) for s, e in zip(starts[:-1], starts[1:])]


class TrackObject(ctypes.Structure):
    """lm_track_object of include/linemod_b200.h."""
    _fields_ = [("class_index", ctypes.c_int32), ("template_id", ctypes.c_int32), ("T", ctypes.c_double * 16)]


class NativeIcp:
    """RAII wrapper over the lm_icp handle (poseRefine compute)."""

    def __init__(self, device=0):
        L = load()
        self._L = L
        h = ctypes.c_void_p()
        check(L.lm_icp_create(int(device), ctypes.byref(h)))
        self._h = h
        self.device = int(device)
        self._estimation = "point_to_plane"  # the handle's estimation (lm_icp_set_estimation)
        self._search = pose_search_options()  # its swarm settings (lm_icp_set_pose_search)
        self._captured = None               # the estimation of the last call (capture())
        self._captured_search = None        # and its swarm settings

    def close(self):
        if getattr(self, "_h", None):
            self._L.lm_icp_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def process_batch(self, scene_depth, model_depths, sceneK, modelKs, Rs, ts, detect_xy, max_iterations=30, estimation=None):
        """scene u16 HxW; model_depths list of u16 HxW (same size); modelKs/Rs [n,3,3] f32; ts [n,3] f32;
        detect_xy [n,2] int.  estimation: "point_to_plane", "point_to_point" or "pso" for this call and the next ones (None:
        as set before, point-to-plane on a new handle).  The scene and each distinct render are copied to the device once,
        then the call runs as process_batch_device.  Returns (R [n,3,3] f64, t [n,3] f64 mm, residual [n] f32)."""
        if estimation is not None:
            self.set_estimation(estimation)
        n = len(model_depths)
        scene = np.ascontiguousarray(scene_depth, np.uint16)
        models = [np.ascontiguousarray(m, np.uint16) for m in model_depths]
        for m in models:
            if m.shape != models[0].shape:
                raise TypeError("model depth images must share one size")
        u16p = ctypes.POINTER(ctypes.c_uint16)
        f32p, f64p = ctypes.POINTER(ctypes.c_float), ctypes.POINTER(ctypes.c_double)
        mp = (u16p * max(n, 1))(*[m.ctypes.data_as(u16p) for m in models])
        sK = np.ascontiguousarray(sceneK, np.float32).reshape(9)
        mK = np.ascontiguousarray(modelKs, np.float32).reshape(n, 9)
        R = np.ascontiguousarray(Rs, np.float32).reshape(n, 9)
        t = np.ascontiguousarray(ts, np.float32).reshape(n, 3)
        xy = np.ascontiguousarray(detect_xy, np.int32).reshape(n, 2)
        Ro = np.full((n, 3, 3), np.nan, np.float64)
        to = np.full((n, 3), np.nan, np.float64)
        res = np.zeros(n, np.float32)
        mrows, mcols = (models[0].shape if n else (1, 1))
        check(self._L.lm_icp_process_batch(self._h, n, scene.ctypes.data_as(u16p), scene.shape[0], scene.shape[1], mp, mrows, mcols,
                                           sK.ctypes.data_as(f32p), mK.ctypes.data_as(f32p), R.ctypes.data_as(f32p),
                                           t.ctypes.data_as(f32p), xy.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)),
                                           int(max_iterations), Ro.ctypes.data_as(f64p), to.ctypes.data_as(f64p),
                                           res.ctypes.data_as(f32p)))
        self._captured = self._estimation
        self._captured_search = self._search
        return Ro, to, res

    def process_batch_device(self, depths, sceneK, modelKs, Rs, ts, detect_xy, max_iterations=30, estimation=None):
        """process_batch for a DeviceDepths (lm_icp_process_batch_device), read where they lie: the same outputs, bit for
        bit, as process_batch on the u16 images the depths convert to; sceneK, modelKs, Rs, ts and detect_xy as there."""
        if estimation is not None:
            self.set_estimation(estimation)
        n = depths.n
        f32p, f64p, vp = ctypes.POINTER(ctypes.c_float), ctypes.POINTER(ctypes.c_double), ctypes.c_void_p
        sK = np.ascontiguousarray(sceneK, np.float32).reshape(9)
        mK = np.ascontiguousarray(modelKs, np.float32).reshape(n, 9)
        R = np.ascontiguousarray(Rs, np.float32).reshape(n, 9)
        t = np.ascontiguousarray(ts, np.float32).reshape(n, 3)
        xy = np.ascontiguousarray(detect_xy, np.int32).reshape(n, 2)
        Ro = np.full((n, 3, 3), np.nan, np.float64)
        to = np.full((n, 3), np.nan, np.float64)
        res = np.zeros(n, np.float32)
        ptrs = (vp * max(n, 1))(*depths.renders)
        pitches = (ctypes.c_int64 * max(n, 1))(*depths.pitches)
        check(self._L.lm_icp_process_batch_device(self._h, n, depths.scene, depths.scene_pitch, depths.scene_format,
                                                  ctypes.c_float(depths.depth_scale), depths.srows, depths.scols, ptrs, pitches,
                                                  depths.format, ctypes.c_float(depths.render_scale), depths.mrows, depths.mcols,
                                                  sK.ctypes.data_as(f32p), mK.ctypes.data_as(f32p), R.ctypes.data_as(f32p),
                                                  t.ctypes.data_as(f32p), xy.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)),
                                                  int(max_iterations), Ro.ctypes.data_as(f64p), to.ctypes.data_as(f64p),
                                                  res.ctypes.data_as(f32p), depths.stream.cuda_stream))
        self._captured = self._estimation
        self._captured_search = self._search
        return Ro, to, res

    def set_use_scene_cloud(self, on):
        check(self._L.lm_icp_set_use_scene_cloud(self._h, 1 if on else 0))

    def set_estimation(self, estimation):
        """"point_to_plane" (the reference's active branch, default), "point_to_point" or "pso" (lm_icp_set_estimation)."""
        check(self._L.lm_icp_set_estimation(self._h, estimation_code(estimation)))
        self._estimation = estimation

    def set_pose_search(self, particles=64, iterations=40, dt_mm=40.0, dr_deg=30.0, clamp_mm=20.0, seed=0):
        """The particle swarm of estimation="pso" for the next calls (lm_icp_set_pose_search)."""
        opts = (int(particles), int(iterations), float(dt_mm), float(dr_deg), float(clamp_mm), int(seed))
        check(self._L.lm_icp_set_pose_search(self._h, *opts))
        self._search = opts

    def set_verify(self, inlier_mm):
        """Pose verification for the next calls (lm_icp_set_verify): the inlier distance in mm, or None for off."""
        d = 10.0 if inlier_mm is None else float(inlier_mm)
        check(self._L.lm_icp_set_verify(self._h, 0 if inlier_mm is None else 1, d))

    def verify(self):
        """The verification of the last call (lm_icp_verify): (score [n] f32, counts [n,6] int32) per hypothesis."""
        return _verify_results(self._L.lm_icp_verify, self._h)

    def set_capture(self, on):
        check(self._L.lm_icp_set_capture(self._h, 1 if on else 0))

    def _capture_item(self, hyp, what, out):
        check(self._L.lm_icp_capture(self._h, int(hyp), what, out.ctypes.data_as(ctypes.c_void_p), out.nbytes))
        return out

    def capture(self, hyp):
        """What the kernels saw and kept for hypothesis `hyp` of the last call with capture on (see lm_icp_capture): source
        / target [n,3] f64, normals [nt,3] f64, init [4,4] f64, T [4,4] f64, fitness, rmse, iterations, knn [nt,30] int32
        (-1 padded), corr_first / corr_last [n] int32 (-1: no correspondence), search the swarm record (search_record).
        An item is None where the call's estimation computed nothing: normals and knn but under "point_to_plane", the
        correspondences under "pso", search but under "pso"."""
        n, nt = self._capture_item(hyp, 0, np.zeros(2, np.int32)).tolist()
        res = self._capture_item(hyp, 5, np.zeros(19, np.float64))
        p2pl, pso = self._captured == "point_to_plane", self._captured == "pso"
        P, I = self._captured_search[:2]
        return dict(source=self._capture_item(hyp, 1, np.zeros((n, 3), np.float64)),
                    target=self._capture_item(hyp, 2, np.zeros((nt, 3), np.float64)),
                    normals=self._capture_item(hyp, 3, np.zeros((nt, 3), np.float64)) if p2pl else None,
                    init=self._capture_item(hyp, 4, np.zeros((4, 4), np.float64)),
                    T=res[:16].reshape(4, 4).copy(), fitness=float(res[16]), rmse=float(res[17]), iterations=int(res[18]),
                    knn=self._capture_item(hyp, 6, np.zeros((nt, 30), np.int32)) if p2pl else None,
                    corr_first=None if pso else self._capture_item(hyp, 7, np.zeros(n, np.int32)),
                    corr_last=None if pso else self._capture_item(hyp, 8, np.zeros(n, np.int32)),
                    search=search_record(self._capture_item(hyp, 13, np.zeros(6 + I + 19 * P, np.int64)), P, I) if pso else None)

    def last_stats(self):
        a = (ctypes.c_double * 4)()
        check(self._L.lm_icp_last_stats(self._h, a))
        return dict(points=int(a[0]), iterations=int(a[1]), rmse=float(a[2]), kernel_us=float(a[3]))

    def launch_count(self):
        return int(self._L.lm_icp_launch_count(self._h))


def nms_translations(t, score, thr, device=0):
    """The pose NMS's greedy pass (lm_nms_translations) on caller arrays: t [n,3] f64, score [n] f64, n <= 1024.
    Returns the kept indices (int64) in keep order."""
    L = load()
    t = np.ascontiguousarray(t, np.float64).reshape(-1, 3)
    score = np.ascontiguousarray(score, np.float64).reshape(-1)
    if score.shape[0] != t.shape[0]:
        raise ValueError("%d translations, %d scores" % (t.shape[0], score.shape[0]))
    n = t.shape[0]
    keep = np.empty(max(n, 1), np.int32)
    nk = ctypes.c_int64()
    f64p = ctypes.POINTER(ctypes.c_double)
    check(L.lm_nms_translations(int(device), n, t.ctypes.data_as(f64p), score.ctypes.data_as(f64p), float(thr),
                                keep.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)), ctypes.byref(nk)))
    return keep[:nk.value].astype(np.int64)


def _verify_results(fn, h):
    n = ctypes.c_int64()
    f32p, i32p = ctypes.POINTER(ctypes.c_float), ctypes.POINTER(ctypes.c_int32)
    rc = fn(h, None, None, 0, ctypes.byref(n))
    if rc != LM_E_CAPACITY:
        check(rc)
    score = np.zeros(n.value, np.float32)
    counts = np.zeros((n.value, 6), np.int32)
    if n.value:
        check(fn(h, score.ctypes.data_as(f32p), counts.ctypes.data_as(i32p), n.value, ctypes.byref(n)))
    return score, counts


def pose_search_points(pts, start_t, scene, sceneK, job=0, device=0, **search):
    """k_pose_pso on caller arrays (lm_pose_search_points): pts [n,3] f64 (m), start_t [3] f64 (the start pose's
    translation, m), scene HxW u16 mm, sceneK 3x3 f32, job the job number of the draws, search as pose_search_options.
    Returns (T [4,4] f64, the swarm record as search_record gives it)."""
    L = load()
    opts = pose_search_options(**search)
    pts = np.ascontiguousarray(pts, np.float64).reshape(-1, 3)
    st = np.ascontiguousarray(start_t, np.float64).reshape(3)
    scene = np.ascontiguousarray(scene)
    if scene.dtype != np.uint16 or scene.ndim != 2:
        raise TypeError("scene must be a uint16 HxW depth image (mm)")
    sK = np.ascontiguousarray(sceneK, np.float32).reshape(9)
    P, I = opts[:2]
    words = np.zeros(6 + I + 19 * P, np.int64)
    T = np.zeros(16, np.float64)
    f64p = ctypes.POINTER(ctypes.c_double)
    check(L.lm_pose_search_points(int(device), pts.ctypes.data_as(f64p), pts.shape[0], st.ctypes.data_as(f64p),
                                  scene.ctypes.data_as(ctypes.POINTER(ctypes.c_uint16)), scene.shape[0], scene.shape[1],
                                  sK.ctypes.data_as(ctypes.POINTER(ctypes.c_float)), *opts, int(job), T.ctypes.data_as(f64p),
                                  words.ctypes.data_as(ctypes.c_void_p), words.nbytes))
    return T.reshape(4, 4), search_record(words, P, I)


def pose_verify_points(pts, T, scene, sceneK, inlier_mm=10.0, device=0):
    """Steps 3-5 of the pose verification on caller arrays (lm_pose_verify_points): pts [n,3] f64 (m), T [4,4] f64,
    scene HxW u16 mm, sceneK 3x3 f32.  Returns (score, counts [6] int32)."""
    L = load()
    pts = np.ascontiguousarray(pts, np.float64).reshape(-1, 3)
    T = np.ascontiguousarray(T, np.float64).reshape(16)
    scene = np.ascontiguousarray(scene)
    if scene.dtype != np.uint16 or scene.ndim != 2:
        raise TypeError("scene must be a uint16 HxW depth image (mm)")
    sK = np.ascontiguousarray(sceneK, np.float32).reshape(9)
    counts = np.zeros(6, np.int32)
    score = ctypes.c_float()
    f64p = ctypes.POINTER(ctypes.c_double)
    check(L.lm_pose_verify_points(int(device), pts.ctypes.data_as(f64p), pts.shape[0], T.ctypes.data_as(f64p),
                                  scene.ctypes.data_as(ctypes.POINTER(ctypes.c_uint16)), scene.shape[0], scene.shape[1],
                                  sK.ctypes.data_as(ctypes.POINTER(ctypes.c_float)), float(inlier_mm),
                                  counts.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)), ctypes.byref(score)))
    return float(score.value), counts


def track_views_points(R_b, t_b, k, T, turn_deg, device=0):
    """View following on caller arrays (lm_track_views_points): one object at template k with T [4,4] f64 among the
    templates R_b [n,3,3], t_b [n,3] f32 of one class.  Returns (chosen template, T [4,4] f64)."""
    L = load()
    Rb = np.ascontiguousarray(R_b, np.float32).reshape(-1, 9)
    tb = np.ascontiguousarray(t_b, np.float32).reshape(-1, 3)
    if Rb.shape[0] != tb.shape[0]:
        raise ValueError("%d rotations and %d translations" % (Rb.shape[0], tb.shape[0]))
    T = np.ascontiguousarray(T, np.float64).reshape(16)
    out = np.zeros(16, np.float64)
    chosen = ctypes.c_int64()
    f32p, f64p = ctypes.POINTER(ctypes.c_float), ctypes.POINTER(ctypes.c_double)
    check(L.lm_track_views_points(int(device), Rb.shape[0], Rb.ctypes.data_as(f32p), tb.ctypes.data_as(f32p), int(k), T.ctypes.data_as(f64p),
                                  float(turn_deg), ctypes.byref(chosen), out.ctypes.data_as(f64p)))
    return int(chosen.value), out.reshape(4, 4)
