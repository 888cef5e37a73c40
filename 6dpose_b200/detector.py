"""Host-side mirror of the reference's Python surface (linemodLevelup/pybind11.cpp:7-35).

`Detector`, `Match` and `poseRefine` keep the reference's names, argument order, keyword names and
error behaviour; underneath, `Detector.match` calls the C-ABI library (CUDA, sm_90a) through
ctypes.  The quantization front-end (cv2) and template extraction run on the host, as SURVEY.md
section 8 rows a14 / f2 describe.
"""
import os

import numpy as np

from . import _lib, frontend
from .bank import TemplateBank


class Match:
    """linemodLevelup::Match (pybind11.cpp:16-22): default-constructible, read/write attributes."""
    __slots__ = ("x", "y", "similarity", "class_id", "template_id")

    def __init__(self, x=0, y=0, similarity=0.0, class_id="", template_id=0):
        # the reference binds only the default constructor; the arguments are this module's fast path
        self.x = x
        self.y = y
        self.similarity = similarity
        self.class_id = class_id
        self.template_id = template_id

    def __repr__(self):
        return "Match(x=%d, y=%d, similarity=%.4f, class_id=%r, template_id=%d)" % (
            self.x, self.y, self.similarity, self.class_id, self.template_id)


def _default_device():
    for key in ("LINEMOD_B200_DEVICE", "LOCAL_RANK"):
        v = os.environ.get(key)
        if v is not None and v != "":
            return int(v)
    return 0


class Detector:
    """linemodLevelup::Detector as bound at pybind11.cpp:25-34.

    Detector()                      -> 63 features, T = [5, 8]          (LL.cpp:1663-1672)
    Detector(T)                     -> 63 features, T as given          (LL.cpp:1674-1682)
    Detector(num_features, T)       -> ColorGradient(10, nf, 55), DepthNormal(2000, 50, nf, 2)  (LL.cpp:1684-1692)
    """

    def __init__(self, *args):
        if len(args) == 0:
            nf, T = 63, [5, 8]
        elif len(args) == 1:
            nf, T = 63, list(args[0])
        elif len(args) == 2:
            nf, T = int(args[0]), list(args[1])
        else:
            raise TypeError("Detector(): incompatible constructor arguments")
        if not all(isinstance(t, (int, np.integer)) for t in T):
            raise TypeError("Detector(): T must be a list of ints")
        self.num_features = nf
        self.T_at_level = [int(t) for t in T]
        self.pyramid_levels = len(self.T_at_level)
        self.bank = TemplateBank()
        self._native = None
        self._bank_dirty = True
        self._class_order = []
        self._selection = None
        self._template_depths = None  # training distances registered with the native handle (setTemplateDepths)
        self._peers = None  # (rank, world) once dist.connect_peers has wired the fused exchange
        self._verify = _lib.verify_options(None)  # lm_set_pose_verify's arguments (setPoseVerification)
        self._views = _lib.track_views_option(None)  # lm_set_track_views's arguments (setTrackViews)
        self._search = _lib.pose_search_options()  # lm_set_pose_search's arguments (setPoseSearch)
        self._render_poses = {}  # class_id -> (R [n,3,3], t [n,3]) f32 of its registered renders (track's dict starts)
        self.device = _default_device()
        self.shard = (0, 1)  # (index, count): template shard matched by this process (multi-GPU)
        self.shard_layout = _lib.SHARD_CONTIGUOUS
        # quantization front-end used by match(): "gpu" (CUDA, lm_match_images) or "cv2" (host, frontend.py);
        # both produce the same label images (tests/test_gpu_frontend.py)
        self.frontend = os.environ.get("LINEMOD_B200_FRONTEND", "gpu")

    # ---- template IO ----------------------------------------------------------------------
    def readClasses(self, class_ids, format):
        """Detector::readClasses, LL.cpp:2124-2134 (format is a printf pattern with one %s).

        Beyond the reference: a pattern ending in ".lmb" names packed bank files (bank.py), and with
        LINEMOD_B200_BANK_CACHE=1 a YAML is read through a packed sibling `<file>.lmb` (built on first use)."""
        for cid in class_ids:
            self.bank.read_any(format % cid, self.pyramid_levels)
        self._bank_dirty = True

    def writeClasses(self, format):
        """Detector::writeClasses, LL.cpp:2136-2146 (".lmb" pattern: packed bank files)."""
        from .bank import PACKED_SUFFIX
        for cid in self.bank.class_ids():
            if (format % cid).endswith(PACKED_SUFFIX):
                self.bank.write_packed(cid, format % cid, self.pyramid_levels)
            else:
                self.bank.write_class(cid, format % cid, self.pyramid_levels)

    def addTemplate(self, sources, class_id, object_mask):
        """Detector::addTemplate, LL.cpp:1943-1975: returns the template id, or -1 on failure."""
        from . import training
        tid = training.add_template(self, sources, class_id, object_mask)
        if tid >= 0:
            self._bank_dirty = True
        return tid

    def getTemplates(self, class_id, template_id):
        # The reference returns std::vector<Template>, a type pybind11.cpp never registers: calling it
        # from Python raises TypeError.  Kept for surface parity.
        raise TypeError("Unable to convert function return value to a Python type! (Template is not bound)")

    def numTemplates(self, class_id=None):
        return self.bank.num_templates(class_id)

    def classIds(self):
        return self.bank.class_ids()

    # ---- matching -------------------------------------------------------------------------
    def _ensure_native(self):
        if self._native is None:
            self._native = _lib.NativeDetector(self.T_at_level, self.device)
            self._bank_dirty = True
        if self._bank_dirty:
            self._class_order = self.bank.class_ids()  # std::map iteration order
            packed = self.bank.pack(self._class_order, self.pyramid_levels * 2)
            self._native.load_bank(packed, self.pyramid_levels * 2)
            self._bank_dirty = False
            self._selection = None
            self._template_depths = None  # lm_load_bank drops them
        return self._native

    def _select(self, class_ids):
        nat = self._ensure_native()
        if not class_ids:
            sel = None  # all classes, map order (LL.cpp:1753-1759)
        else:
            index = {c: i for i, c in enumerate(self._class_order)}
            sel = [index[c] for c in class_ids if c in index]  # unknown ids are skipped (LL.cpp:1765-1767)
        key = (None if sel is None else tuple(sel), self.shard, self.shard_layout)
        if key != self._selection:
            nat.select(sel, self.shard[0], self.shard[1], self.shard_layout)
            self._selection = key
        return nat

    def _whole_bank_only(self, what):
        # a detector left holding ONE template shard (dist.py) would silently return that shard's matches only
        if self.shard[1] > 1 and self._peers is None:
            raise RuntimeError("%s on a detector that holds template shard %d of %d without a connected peer exchange: "
                               "use dist.match_quantized_sharded, or reset detector.shard = (0, 1)" % (what, self.shard[0], self.shard[1]))

    def quantize(self, sources, masks=None):
        """The host front-end: list over levels of [color_labels, normal_labels] (u8)."""
        return frontend.quantize_pyramid(sources, self.pyramid_levels, masks, self.num_features)

    def match(self, sources, threshold, class_ids, masks=None, depth_scale=1.0, stream=None):
        """Detector::match (LL.cpp:1702-1777) -> list[Match], sorted, duplicates pruned.

        As in the reference binding the declared default for `masks` is not convertible; every caller
        passes masks=[] (linemod_and_levelup_test.py:324).

        Beyond the reference: sources may be [rgb, depth] CUDA tensors on the detector's device (a frame already on the
        GPU; see _lib.DeviceFrame for dtypes and strides, masks then tensors too).  float32 depth is scaled by depth_scale
        and converted to u16 mm on the device as the driver converts it on the host; the frame is read in order on
        `stream` (None: torch.cuda.current_stream) without a host synchronise.  Tensors always take the GPU front-end,
        whatever `frontend` says."""
        if masks is None:
            raise TypeError("match(): incompatible function arguments (masks must be a list; pass masks=[])")
        if len(sources) != 2:
            raise RuntimeError("sources.size() == modalities.size()")  # CV_Assert LL.cpp:1707
        sources = self._frame_sources(sources, masks, depth_scale, stream)
        if isinstance(sources[0], _lib.DeviceFrame):
            self._whole_bank_only("match()")
            nat = self._select(list(class_ids))
            return self._to_matches(nat.match_images(sources[0], None, None, float(threshold)))
        self._whole_bank_only("match()")
        if self.frontend == "gpu" and self.shard[1] == 1:
            nat = self._select(list(class_ids))
            return self._to_matches(nat.match_images(sources[0], sources[1], list(masks), float(threshold)))
        quantized = self.quantize(sources, list(masks))
        return self.match_quantized(quantized, threshold, class_ids)

    def match_quantized(self, quantized, threshold, class_ids=()):
        """Same as match() but starting from quantized label images (the accelerated path proper)."""
        self._whole_bank_only("match_quantized()")
        nat = self._select(list(class_ids))
        out = nat.match_quantized(quantized, float(threshold))
        return self._to_matches(out)

    # ---- post-match stage (SURVEY.md 8f-3; the reference's drivers do this on the host) ----
    def setBoxes(self, sizes):
        """Box size (width, height) per template for the NMS: dict class_id -> array [n_templates, 2], as the
        drivers' template-info files give it (linemod_and_levelup_test.py:248-249, 337-338).  None = the
        templates' own width/height."""
        nat = self._ensure_native()
        if sizes is None:
            nat.set_boxes(None)
            return
        rows = []
        for cid in self._class_order:
            wh = np.asarray(sizes[cid], np.int32).reshape(-1, 2)
            if wh.shape[0] != self.bank.num_templates(cid):
                raise ValueError("class %s: %d box sizes for %d templates" % (cid, wh.shape[0], self.bank.num_templates(cid)))
            rows.append(wh)
        nat.set_boxes(np.concatenate(rows, 0))

    # ---- depth gate of the coarse scan (include/linemod_b200.h, lm_set_depth_gate) ----
    def setTemplateDepths(self, depths):
        """Training distance (mm) per template for the depth gate: dict class_id -> sequence [n_templates] indexed by
        template id.  Classes left out, NaN and values <= 0 are never gated.  Loading another bank drops them."""
        order = self.bank.class_ids()
        unknown = [c for c in depths if c not in order]
        if unknown:
            raise ValueError("setTemplateDepths: classes %s are not in the bank" % ", ".join(repr(c) for c in unknown))
        rows = []
        for cid in order:
            n = self.bank.num_templates(cid)
            if cid in depths:
                z = np.asarray(depths[cid], np.float32).reshape(-1)
                if z.shape[0] != n:
                    raise ValueError("class %s: %d distances for %d templates" % (cid, z.shape[0], n))
            else:
                z = np.full(n, np.nan, np.float32)
            rows.append(z)
        z = np.concatenate(rows) if rows else np.zeros(0, np.float32)
        nat = self._ensure_native()
        nat.set_template_depths(0, z)
        self._template_depths = z

    @staticmethod
    def templateDepthsFromInfo(infos):
        """The drivers' template-info files (dict class_id -> {template_id: {"cam_t_w2c": [x, y, z], ...}}, as yaml.load
        reads <class>_info.yaml) to setTemplateDepths' argument: the distance of template i is cam_t_w2c[2] of entry i."""
        out = {}
        for cid, info in infos.items():
            ids = sorted(int(k) for k in info)
            if ids != list(range(len(ids))):
                raise ValueError("class %s: info entries are not the template ids 0..%d" % (cid, len(ids) - 1))
            get = lambda i: info[i] if i in info else info[str(i)]
            out[cid] = np.asarray([float(get(i)["cam_t_w2c"][2]) for i in ids], np.float32)
        return out

    def setDepthGate(self, tolerance):
        """Gate the coarse scan by scene depth (include/linemod_b200.h): a template's candidates only where the depth
        around its centre lies within [z (1 - tolerance), z (1 + tolerance)] of its training distance z.  Every match
        path that takes a depth image (match, match_refine, detect, the batch calls, dist's sharded calls) picks it up
        from the next frame on; paths from quantized images (match_top, match_quantized) have no depth and refuse to run
        while it is on.  None turns it off."""
        if tolerance is not None:
            _lib.depth_gate_tolerance(tolerance)
            z = self._template_depths
            if self._bank_dirty or z is None or not (z > 0).any():
                raise RuntimeError("setDepthGate: no training distances registered for this bank (setTemplateDepths first)")
        self._ensure_native().set_depth_gate(tolerance)

    def depthGateStats(self):
        """Of the last frame, which ran gated: dict(before, after, empty_cells, with_distance) (lm_depth_gate_stats)."""
        return self._ensure_native().depth_gate_stats()

    def match_top(self, quantized, threshold, class_ids=(), iou_threshold=0.5, top_k=3):
        """match + nms(dets, iou_threshold)[:top_k] of the reference's drivers (linemod_and_levelup_test.py:
        34-61, 325-350) in one call; the NMS runs on the GPU and only the survivors are copied back.
        Returns (list[Match] best first, number of raw matches before sort/unique)."""
        self._whole_bank_only("match_top()")
        nat = self._select(list(class_ids))
        out, nrec = nat.match_top(quantized, float(threshold), float(iou_threshold), int(top_k))
        return self._to_matches(out), nrec

    # ---- pose stage on the device (the drivers' poseRefine loop over the NMS survivors) ----
    RENDER_CHUNK = 64

    def setTemplateRenders(self, renders):
        """Model render and pose per template for match_refine: dict class_id -> (depths, K, R, t), every class of
        the bank.  depths is a sequence of u16 HxW renders, one per template (the drivers' render(model, im_size, K, R,
        t) of the template's info entry; it may produce them lazily), K / R [n,3,3], t [n,3] mm.  Renders are
        registered RENDER_CHUNK at a time: only their crops are kept."""
        from .pose_refine import poseRefine
        nat = self._ensure_native()
        first = 0
        for cid in self._class_order:
            depths, K, R, t = renders[cid]
            n = self.bank.num_templates(cid)
            K = np.asarray(K, np.float32).reshape(-1, 3, 3)
            R = np.asarray(R, np.float32).reshape(-1, 3, 3)
            t = np.asarray(t, np.float32).reshape(-1, 3)
            if not (K.shape[0] == R.shape[0] == t.shape[0] == n):
                raise ValueError("class %s: K / R / t for %d templates, the bank has %d" % (cid, K.shape[0], n))
            chunk, got = [], 0
            for d in depths:
                chunk.append(poseRefine._depth(d, "render"))
                if len(chunk) == self.RENDER_CHUNK:
                    nat.set_template_renders(first + got, chunk, K[got:got + len(chunk)], R[got:got + len(chunk)], t[got:got + len(chunk)])
                    got += len(chunk)
                    chunk = []
            if chunk:
                nat.set_template_renders(first + got, chunk, K[got:got + len(chunk)], R[got:got + len(chunk)], t[got:got + len(chunk)])
                got += len(chunk)
            if got != n:
                raise ValueError("class %s: %d renders for %d templates" % (cid, got, n))
            self._render_poses[cid] = (R.copy(), t.copy())
            first += n

    def setPoseVerification(self, inlier_mm=10.0, rank_by="fitness", min_score=None):
        """Verify every refined pose against the scene depth (include/linemod_b200.h, lm_set_pose_verify), for
        match_refine, detect, the batch calls and dist's sharded calls: the poseRefine objects they return then carry
        getScore() and getVerification().  inlier_mm: the distance (mm) within which a model point's depth agrees with the
        scene's; None turns verification off (the default).  rank_by: the pose NMS's order in detect / detect_batch,
        "fitness" (-residual, as without verification) or "score" (score descending).  min_score: detect's posed
        survivors scoring below it are dropped before the pose NMS.  A pose stage shared over the ranks verifies too."""
        self._verify = _lib.verify_options(inlier_mm, rank_by, min_score)

    def setTrackViews(self, turn_deg=None):
        """View following for track, track_batch and dist.track_batch_sharded (include/linemod_b200.h,
        lm_set_track_views): once an object has turned more than turn_deg degrees from its template's training view,
        it switches to the template of its class whose view is closest to its current orientation before its clouds are
        built, so the ICP keeps registering the surface the camera now sees.  The returned Match.template_id is the
        template chosen, and the poseRefine's R, t and transformation belong to it, so feeding the pairs back continues
        from it.  None turns view following off (the default).  Checked here, before any device work."""
        self._views = _lib.track_views_option(turn_deg)

    def setPoseSearch(self, particles=64, iterations=40, dt_mm=40.0, dr_deg=30.0, clamp_mm=20.0, seed=0):
        """The particle swarm of estimation="pso" (include/linemod_b200.h, LM_POSE_PSO / lm_set_pose_search) for
        match_refine, detect, the batch calls and dist's unshared sharded calls: particles, iterations, the bounds of the
        search about the ICP's initial guess (translation dt_mm per axis, rotation dr_deg per axis about the cloud's
        centroid), the per-point cost clamp in mm and the seed of its random numbers.  Checked here, before any device
        work; the defaults are 64, 40, 40 mm, 30 degrees, 20 mm and 0."""
        self._search = _lib.pose_search_options(particles, iterations, dt_mm, dr_deg, clamp_mm, seed)

    def _pose_native(self, class_ids):
        nat = self._select(list(class_ids))
        nat.set_pose_verify(*self._verify)
        nat.set_pose_search(*self._search)
        nat.set_track_views(*self._views)
        return nat

    def _verification(self, nat, sizes):
        # per run of `sizes` entries, the [(score, counts)] of the last completed pose stage; None without verification
        if not self._verify[0]:
            return [None] * len(sizes)
        pairs = _lib.verify_arrays(*nat.pose_verify())
        out, at = [], 0
        for k in sizes:
            out.append(pairs[at:at + k])
            at += k
        return out

    def match_refine(self, sources, threshold, class_ids, sceneK, iou_threshold=0.5, top_k=3, max_iterations=30,
                     use_scene_cloud=False, masks=[], estimation="point_to_plane", depth_scale=1.0, stream=None):
        """match + nms + poseRefine().process for every survivor, as the drivers do (linemod_and_levelup_test.py:
        324-367), in one chain on the GPU: front-end, match, NMS/top-k, cloud building, normals and ICP.  Needs
        setTemplateRenders.  Returns [(Match, poseRefine)] in pick order; each poseRefine is in the state
        refine_matches leaves it in (residual -1, R / t None where the model box does not fit the frame).
        estimation (not in the reference's surface): the ICP's estimation step, "point_to_plane" (the reference's
        active branch) or "point_to_point" (its other branch, LL.cpp:131-135: no normals, a closed-form rigid fit).
        sources, depth_scale and stream as match: a frame may be CUDA tensors."""
        from .pose_refine import poseRefine
        _lib.estimation_code(estimation)
        sources = self._frame_sources(sources, masks, depth_scale, stream)
        self._whole_bank_only("match_refine()")
        sK = poseRefine._mat(sceneK, np.float32, (3, 3), "sceneK")
        nat = self._pose_native(class_ids)
        out, R, t, res, _ = nat.match_pose(sources[0], sources[1], list(masks), float(threshold), sK, float(iou_threshold),
                                           int(top_k), int(max_iterations), bool(use_scene_cloud), estimation)
        return self._pose_pairs(out, R, t, res, self._verification(nat, [len(out)])[0], nat.pose_transforms())

    def detect(self, sources, threshold, class_ids, sceneK, iou_threshold=0.5, translation_threshold=40.0, top_k=0,
               max_iterations=30, use_scene_cloud=False, masks=[], estimation="point_to_plane", depth_scale=1.0, stream=None):
        """The whole frame of linemod_ros/detect.py (:91-141): match, box NMS, poseRefine of every survivor (top_k=0)
        and the greedy translation NMS nms_norms(ts, -residual, translation_threshold) (:41-50, :130-131), in one chain
        on the GPU; only the kept objects are copied back.  Needs setTemplateRenders.  Returns [(Match, poseRefine)] in
        keep order, as match_refine(top_k) followed by pose_refine.nms_translations would.  Survivors whose model box
        does not fit the frame (no pose) are not returned; equal residuals keep box-NMS pick order.  estimation as
        match_refine; sources, depth_scale and stream as match: a frame may be CUDA tensors."""
        from .pose_refine import poseRefine
        _lib.estimation_code(estimation)
        sources = self._frame_sources(sources, masks, depth_scale, stream)
        self._whole_bank_only("detect()")
        sK = poseRefine._mat(sceneK, np.float32, (3, 3), "sceneK")
        nat = self._pose_native(class_ids)
        out, R, t, res, _ = nat.detect(sources[0], sources[1], list(masks), float(threshold), sK, float(iou_threshold), int(top_k),
                                       int(max_iterations), bool(use_scene_cloud), float(translation_threshold), estimation)
        # every kept pose has one: residual >= 0
        return self._pose_pairs(out, R, t, res, self._verification(nat, [len(out)])[0], nat.pose_transforms())

    # ---- a batch of RGB-D frames through one pose stage (lm_detect_batch) ----
    def match_refine_batch(self, frames, threshold, class_ids, sceneK, iou_threshold=0.5, top_k=3, max_iterations=30,
                           use_scene_cloud=False, masks=[], estimation="point_to_plane", depth_scale=1.0, stream=None):
        """match_refine for many frames in one call: each frame's match and box NMS, then one pose stage for the survivors
        of all of them, which fills the GPU where one frame's few survivors cannot.  frames: a sequence of [rgb, depth]
        pairs of one size; sceneK: one 3x3 matrix or one per frame; masks: [] or one masks list per frame.  Returns one
        list per frame, each equal to match_refine on that frame.  The handle keeps the batch's device buffers, sized
        for the batch's shape (frames, size, top_k; with top_k=0 the pose buffers of 1024 survivors), for the next one.
        estimation as match_refine.  frames may be CUDA tensor pairs (match), all of one size, row pitches and depth dtype,
        with depth_scale and stream as match."""
        _lib.estimation_code(estimation)
        inputs, K = self._batch_inputs(frames, sceneK, masks, "match_refine_batch()", depth_scale, stream)
        self._whole_bank_only("match_refine_batch()")
        nat = self._pose_native(class_ids)
        call, inputs = (nat.detect_batch_device, (inputs,)) if isinstance(inputs, _lib.DeviceBatch) else (nat.detect_batch, inputs)
        got = call(*inputs, float(threshold), K, float(iou_threshold), int(top_k), int(max_iterations), bool(use_scene_cloud),
                   pose_nms=False, estimation=estimation)
        return self._batch_pairs(nat, got, transforms=True)

    def detect_batch(self, frames, threshold, class_ids, sceneK, iou_threshold=0.5, translation_threshold=40.0, top_k=0,
                     max_iterations=30, use_scene_cloud=False, masks=[], estimation="point_to_plane", depth_scale=1.0, stream=None):
        """detect for many frames in one call: each frame's match and box NMS, then one pose stage and one pose NMS for all
        of them.  Arguments as match_refine_batch; returns one list per frame, each equal to detect on that frame."""
        _lib.estimation_code(estimation)
        inputs, K = self._batch_inputs(frames, sceneK, masks, "detect_batch()", depth_scale, stream)
        self._whole_bank_only("detect_batch()")
        nat = self._pose_native(class_ids)
        call, inputs = (nat.detect_batch_device, (inputs,)) if isinstance(inputs, _lib.DeviceBatch) else (nat.detect_batch, inputs)
        got = call(*inputs, float(threshold), K, float(iou_threshold), int(top_k), int(max_iterations), bool(use_scene_cloud),
                   pose_nms=True, translation_threshold=float(translation_threshold), estimation=estimation)
        return self._batch_pairs(nat, got, transforms=True)

    def _batch_pairs(self, nat, got, transforms=False):
        # one [(Match, poseRefine)] list per frame of a batch call's result; transforms: with each pose's T
        # (lm_pose_transforms)
        sizes = [len(g[0]) for g in got]
        ver = self._verification(nat, sizes)
        T = nat.pose_transforms() if transforms else None
        starts = np.cumsum([0] + sizes)
        return [self._pose_pairs(out, R, t, res, v, None if T is None else T[a:b])
                for (out, R, t, res, _), v, a, b in zip(got, ver, starts[:-1], starts[1:])]

    def _batch_args(self, frames, class_ids, sceneK, masks, what):
        # the sharded batch calls (dist.py), which take numpy frames: the handle, then (rgb, depth, mask pairs, K)
        inputs, K = self._batch_inputs(frames, sceneK, masks, what)
        if isinstance(inputs, _lib.DeviceBatch):
            raise TypeError("%s takes numpy frames" % what)
        self._whole_bank_only(what)
        return self._pose_native(class_ids), inputs + (K,)

    def _batch_inputs(self, frames, sceneK, masks, what, depth_scale=1.0, stream=None):
        # every check that needs no device, before the native handle exists.  Returns (inputs, K): inputs is a
        # _lib.DeviceBatch for CUDA tensor frames, else (rgb [n,H,W,3], depth [n,H,W], mask pairs or None)
        frames = list(frames)
        if not frames:
            raise ValueError("%s: no frames" % what)
        for sources in frames:
            if len(sources) != 2:
                raise RuntimeError("sources.size() == modalities.size()")
        on_device = [_lib.is_tensor(s[0]) or _lib.is_tensor(s[1]) for s in frames]
        if any(on_device) and not all(on_device):
            raise TypeError("%s: frames mix numpy arrays and torch tensors" % what)
        rgb, depth = [], []
        if not on_device[0]:
            _lib.host_frame_options(depth_scale, stream)
            for sources in frames:
                rgb.append(self._as_source(sources[0], 0))
                depth.append(self._as_source(sources[1], 1))
            if any(r.shape != rgb[0].shape or d.shape != rgb[0].shape[:2] for r, d in zip(rgb, depth)):
                raise ValueError("%s: every frame's colour and depth images must have one size" % what)
        n = len(frames)
        K = self._frame_ks(sceneK, n, what)
        if masks is None:
            raise TypeError("%s: masks must be a list; pass masks=[]" % what)
        masks = list(masks)
        if masks and len(masks) != n:
            raise ValueError("%s: %d masks lists for %d frames" % (what, len(masks), n))
        pairs = None
        if masks:
            pairs = []
            for m in masks:
                m = list(m)
                if m and len(m) != 2:
                    raise RuntimeError("masks.size() == modalities.size()")
                pairs.append(m if m else [None, None])
        if on_device[0]:
            try:
                return _lib.DeviceBatch([_lib.DeviceFrame(s[0], s[1], pairs[f] if pairs else None, depth_scale, stream, self.device)
                                         for f, s in enumerate(frames)]), K
            except ValueError as e:
                raise ValueError("%s: %s" % (what, e)) from None
        return (np.stack(rgb), np.stack(depth), pairs), K

    @staticmethod
    def _frame_ks(sceneK, n, what):
        # one 3x3 f32 intrinsics per frame of a batch call, from one matrix or n of them
        from .pose_refine import poseRefine
        K = np.asarray(sceneK)
        if K.size == 9:
            return np.repeat(poseRefine._mat(K, np.float32, (3, 3), "sceneK")[None], n, 0)
        if K.shape == (n, 3, 3):
            return poseRefine._mat(K, np.float32, (n, 3, 3), "sceneK")
        raise ValueError("%s: sceneK must be one 3x3 matrix or %d of them, got shape %s" % (what, n, K.shape))

    def _pose_pairs(self, out, R, t, res, ver=None, T=None):
        # [(Match, poseRefine)]; a survivor without a pose (residual -1, only without the pose NMS) keeps R / t None.
        # ver: per entry (score, counts) of the pose verification, or None; T: per entry its transformation, or None
        from .pose_refine import poseRefine
        pairs = []
        for i, m in enumerate(self._to_matches(out)):
            p = poseRefine()
            p._residual = float(res[i])
            if ver is not None:
                p._score, p._verification = ver[i]
            if res[i] != -1.0:
                p._R = R[i].copy()
                p._t = t[i].reshape(3, 1).copy()
                if T is not None:
                    p._T = T[i].copy()
            pairs.append((m, p))
        return pairs

    # ---- tracking (include/linemod_b200.h, lm_track / lm_track_device) ----
    def track(self, depth, sceneK, objects, max_iterations=30, margin_px=4, estimation="point_to_plane", depth_scale=1.0, stream=None):
        """Refine each object's last pose against a new depth frame, with no match: the ICP starts from the object's T and
        registers its template's model cloud against the scene pixels of the window the model projects to (its projected
        box grown by margin_px).  Not in the reference, whose live loop detects again on every frame (linemod_ros/
        detect.py:167-168).  depth: a uint16 HxW numpy image (mm), or a CUDA tensor as in match (uint16 mm, or float32
        scaled by depth_scale, read in order on `stream`).  objects: (Match, poseRefine) pairs of match_refine, detect,
        the batch calls or track itself, and/or dicts {class_id, template_id, R, t (mm)} converted to T with the
        template's registered pose (include/linemod_b200.h).  estimation: "point_to_plane" or "point_to_point".
        Returns [(Match, poseRefine)], one per object in order: Match.x / .y the projected box's top-left, similarity
        carried over (0.0 for a dict); poseRefine.getTrackStatus() "tracked", "outside", "window" or "no_depth", the
        last three with residual -1 and the start's R, t and T.  With setPoseVerification, every entry carries its score.
        TypeError for a pair whose poseRefine has no transformation (refine_matches / process), ValueError for an unknown
        class or template; both before any device work."""
        from .pose_refine import poseRefine
        _lib.estimation_code(estimation)
        starts = self._track_starts(objects, "track")
        sK = poseRefine._mat(sceneK, np.float32, (3, 3), "sceneK")
        triples = [(c, t, T) for c, t, T, _, _, _ in starts]
        if _lib.is_tensor(depth):
            plane = self._depth_planes([depth], ["depth"], depth_scale, stream)
            nat = self._pose_native(())
            got = nat.track_device(plane[0][0], *plane[1:], sK, triples, max_iterations, margin_px, estimation)
        else:
            _lib.host_frame_options(depth_scale, stream)
            depth = np.asarray(depth)
            if depth.dtype != np.uint16 or depth.ndim != 2:
                raise TypeError("depth must be a uint16 HxW depth image (mm)")
            nat = self._pose_native(())
            got = nat.track(depth, sK, triples, max_iterations, margin_px, estimation)
        return self._track_pairs(starts, got, self._verification(nat, [len(starts)])[0], nat.track_templates(), estimation)

    def track_batch(self, depths, sceneK, objects, max_iterations=30, margin_px=4, estimation="point_to_plane", depth_scale=1.0,
                    stream=None):
        """track for many frames in one call (lm_track_batch): several cameras, or several independent sequences at one time
        step, whose objects then share one pose-stage run and fill the GPU where one frame's few objects cannot.  depths: a
        sequence of uint16 HxW numpy images of one size, or of CUDA tensors of one size, row pitch and dtype (as track takes
        them, with depth_scale and stream); sceneK: one 3x3 matrix or one per frame; objects: one list per frame, each entry
        any kind track takes, at most 1024 per frame.  Returns one [(Match, poseRefine)] list per frame, each equal to track
        on that frame alone.  TypeError / ValueError before any device work."""
        return self._track_batch(depths, sceneK, objects, max_iterations, margin_px, estimation, depth_scale, stream, False, "track_batch")

    def _track_batch(self, depths, sceneK, objects, max_iterations, margin_px, estimation, depth_scale, stream, peers, what):
        # track_batch, and (peers) dist.track_batch_sharded on a connected detector; messages name `what`
        _lib.estimation_code(estimation)
        depths, objects = list(depths), [list(o) for o in objects]
        n = len(depths)
        if not n:
            raise ValueError("%s: no frames" % what)
        if len(objects) != n:
            raise ValueError("%s: %d object lists for %d frames" % (what, len(objects), n))
        starts = [self._track_starts(o, "%s: frame %d" % (what, f)) for f, o in enumerate(objects)]
        K = self._frame_ks(sceneK, n, what + "()")
        triples = [[(c, t, T) for c, t, T, _, _, _ in s] for s in starts]
        on_device = [_lib.is_tensor(d) for d in depths]
        if any(on_device) and not all(on_device):
            raise TypeError("%s: depths mix numpy arrays and torch tensors" % what)
        if on_device[0]:
            planes = self._depth_planes(depths, ["depths[%d]" % f for f in range(n)], depth_scale, stream)
            nat = self._pose_native(())
            run = nat.peer_track_batch_device if peers else nat.track_batch_device
            got = run(*planes, K, triples, max_iterations, margin_px, estimation)
        else:
            _lib.host_frame_options(depth_scale, stream)
            depths = [np.asarray(d) for d in depths]
            for f, d in enumerate(depths):
                if d.dtype != np.uint16 or d.ndim != 2:
                    raise TypeError("%s: depths[%d] must be a uint16 HxW depth image (mm)" % (what, f))
                if d.shape != depths[0].shape:
                    raise ValueError("%s: depths[%d] is %s, depths[0] %s" % (what, f, d.shape, depths[0].shape))
            nat = self._pose_native(())
            run = nat.peer_track_batch if peers else nat.track_batch
            got = run(np.stack(depths), K, triples, max_iterations, margin_px, estimation)
        ver = self._verification(nat, [len(s) for s in starts])
        tpl = nat.track_templates()
        at = np.cumsum([0] + [len(s) for s in starts])
        return [self._track_pairs(s, g, v, tpl[a:b], estimation) for s, g, v, a, b in zip(starts, got, ver, at[:-1], at[1:])]

    def _track_starts(self, objects, what):
        # track's objects as (class_index, template_id, T, Match, R, t); TypeError / ValueError naming `what`
        from .pose_refine import poseRefine, pose_to_transform
        objects = list(objects)
        if len(objects) > _lib.TRACK_MAX:
            raise ValueError("%s: %d objects, at most %d per frame" % (what, len(objects), _lib.TRACK_MAX))
        order = self.bank.class_ids()
        index = {c: i for i, c in enumerate(order)}
        starts = []
        for k, o in enumerate(objects):
            if isinstance(o, dict):
                cid, tid = o["class_id"], int(o["template_id"])
                m, R, t = Match(0, 0, 0.0, cid, tid), np.asarray(o["R"], np.float64).reshape(3, 3), np.asarray(o["t"], np.float64).reshape(3)
                T = None
            else:
                m, p = o
                cid, tid = m.class_id, int(m.template_id)
                T = p.getTransformation() if isinstance(p, poseRefine) else None
                if T is None:
                    raise TypeError("%s: object %d's poseRefine has no transformation (only match_refine, detect, the batch calls "
                                    "and track return one)" % (what, k))
                R, t = p.getR(), p.getT()
            if cid not in index:
                raise ValueError("%s: object %d: class %r is not in the bank" % (what, k, cid))
            if not 0 <= tid < self.bank.num_templates(cid):
                raise ValueError("%s: object %d: template %d outside class %r's %d templates" % (what, k, tid, cid, self.bank.num_templates(cid)))
            if T is None:
                if cid not in self._render_poses:
                    raise ValueError("%s: object %d: class %r has no registered renders (setTemplateRenders)" % (what, k, cid))
                Rb, tb = self._render_poses[cid]
                T = pose_to_transform(R, t, Rb[tid], tb[tid])
            starts.append((index[cid], tid, np.asarray(T, np.float64).reshape(4, 4), m, R, t))
        return starts

    def _depth_planes(self, tensors, names, depth_scale, stream):
        # CUDA depth tensors of one size, row pitch and dtype on the detector's device: (pointers, pitch, format, scale,
        # rows, cols, stream handle)
        import torch
        planes = [_lib._depth_plane(t, name, torch) for t, name in zip(tensors, names)]
        for t, name, pl in zip(tensors, names, planes):
            if not t.is_cuda or t.device.index != int(self.device):
                raise ValueError("%s is on %s; the detector runs on cuda:%d" % (name, t.device, int(self.device)))
            if tuple(t.shape) != tuple(tensors[0].shape) or pl[1:] != planes[0][1:]:
                raise ValueError("%s: every depth tensor must have one size, row pitch and dtype" % name)
        fmt = planes[0][2]
        scale = _lib._plane_scale(fmt == _lib.DEPTH_F32, depth_scale, "depth_scale", names[0])
        st = _lib.device_stream(stream, self.device)
        return ([pl[0] for pl in planes], planes[0][1], fmt, scale, int(tensors[0].shape[0]), int(tensors[0].shape[1]), st.cuda_stream)

    def _track_pairs(self, starts, got, ver, templates, estimation):
        # [(Match, poseRefine)] of one frame's track results, one per start; templates: each entry's (lm_track_templates)
        from .pose_refine import poseRefine
        status, T, R, t, res, box = got
        pairs = []
        for i, (_, _, T0, m0, R0, t0) in enumerate(starts):
            p = poseRefine(estimation)
            p._track_status = _lib.TRACK_STATUS[int(status[i])]
            p._residual = float(res[i])
            if ver is not None:
                p._score, p._verification = ver[i]
            x, y = (int(box[i, 0]), int(box[i, 1])) if status[i] != 1 else (m0.x, m0.y)
            if status[i] == 0:
                p._R, p._t, p._T = R[i].copy(), t[i].reshape(3, 1).copy(), T[i].copy()
            else:
                p._R = None if R0 is None else np.asarray(R0, np.float64).reshape(3, 3).copy()
                p._t = None if t0 is None else np.asarray(t0, np.float64).reshape(3, 1).copy()
                p._T = T0.copy()
            pairs.append((Match(x, y, m0.similarity, m0.class_id, int(templates[i])), p))
        return pairs

    def _to_matches(self, out):
        # column-wise conversion + map(): building ~1400 objects field by field from numpy scalars costs 10x the
        # GPU match itself
        names = self._class_order
        return list(map(Match, out["x"].tolist(), out["y"].tolist(), out["similarity"].tolist(),
                        [names[c] for c in out["class_index"].tolist()], out["template_id"].tolist()))

    def _frame_sources(self, sources, masks, depth_scale, stream):
        # [DeviceFrame, None] for CUDA tensors, checked here once, before any library call; the numpy sources otherwise
        if len(sources) != 2:
            raise RuntimeError("sources.size() == modalities.size()")
        frame = _lib.frame_inputs(sources[0], sources[1], list(masks) if masks is not None else None, depth_scale, stream, self.device)
        if frame is not None:
            return [frame, None]
        return [self._as_source(s, i) for i, s in enumerate(sources)]

    @staticmethod
    def _as_source(a, i):
        a = np.asarray(a)
        if i == 0:
            if a.dtype != np.uint8 or a.ndim != 3 or a.shape[2] != 3:
                raise TypeError("sources[0] must be a uint8 HxWx3 colour image")
        else:
            if a.dtype != np.uint16 or a.ndim != 2:
                raise TypeError("sources[1] must be a uint16 HxW depth image (mm)")
        return np.ascontiguousarray(a)
