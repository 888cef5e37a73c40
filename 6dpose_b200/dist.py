"""Template-bank sharding over the GPUs of one box (SURVEY.md section 8e).

The reference matches templates in a serial loop (Detector::matchClass, LL.cpp:1797); templates are
independent, so rank r of W scans a contiguous, feature-balanced slice of the selected template
sequence (lm_select).  Every rank sees every frame.  The only exchange is ONE all-gather of the
per-rank result blocks (kept records, 16 bytes each, with their global (work, seq) sort keys); any
rank can then run the host finisher (lm_finish = the reference's std::sort + std::unique) on the
concatenation.  Backends: NCCL on device tensors (GPUs), gloo on host tensors (CPU tests).

On GPUs the exchange is FUSED into the exact refinement kernels (connect_peers): k_refine_bits / k_refine store every kept
record straight into every rank's exchange buffer with peer stores over NVLink, a collector kernel on
the same stream waits for all ranks' frame flags and packs the blocks -- the ordinary result block of
each rank then already holds all shards' records; the process group only carries the one-time IPC
handle exchange.
"""
import numpy as np

from . import _lib


def shard_of(rank, world):
    return (int(rank), int(world))


def gather_records(records, group=None):
    """All-gather variable-length lm_record arrays; returns the concatenation (same on every rank)."""
    import torch
    import torch.distributed as dist
    records = np.ascontiguousarray(records, _lib.RECORD_DTYPE)
    world = dist.get_world_size(group)
    backend = dist.get_backend(group)
    dev = torch.device("cuda", torch.cuda.current_device()) if backend == "nccl" else torch.device("cpu")
    n = torch.tensor([records.shape[0]], dtype=torch.int64, device=dev)
    counts = [torch.zeros(1, dtype=torch.int64, device=dev) for _ in range(world)]
    dist.all_gather(counts, n, group=group)
    counts = [int(c.item()) for c in counts]
    cap = max(max(counts), 1)
    buf = torch.zeros(cap * 16, dtype=torch.uint8, device=dev)
    if records.shape[0]:
        buf[:records.shape[0] * 16] = torch.from_numpy(records.view(np.uint8).reshape(-1).copy()).to(dev)
    out = torch.zeros(world * cap * 16, dtype=torch.uint8, device=dev)
    dist.all_gather_into_tensor(out, buf, group=group)
    host = out.cpu().numpy().reshape(world, cap * 16)
    parts = [host[r, :counts[r] * 16].copy().view(_lib.RECORD_DTYPE) for r in range(world)]
    return np.concatenate(parts) if parts else np.zeros(0, _lib.RECORD_DTYPE)


def connect_peers(detector, group=None, capacity_records=8192, class_ids=(), share_pose=False):
    """One-time setup of the fused exchange: every rank exports its buffer's CUDA IPC handle, the
    handles travel through the process group (any backend), every rank maps the others' buffers.

    share_pose: divide the pose stage of Detector.detect / match_refine and of detect_batch_sharded /
    match_refine_batch_sharded / track_batch_sharded over the ranks (lm_peer_share_pose).  Only for callers whose every
    rank runs the pose stage of every frame."""
    import torch.distributed as dist
    if not isinstance(share_pose, (bool, int, np.bool_, np.integer)):
        raise TypeError("connect_peers(share_pose=...): a bool, got %s" % type(share_pose).__name__)
    rank, world = dist.get_rank(group), dist.get_world_size(group)
    detector.shard = shard_of(rank, world)
    nat = detector._select(list(class_ids))
    handle = nat.peer_export(world, capacity_records)
    handles = [None] * world
    dist.all_gather_object(handles, handle, group=group)
    nat.peer_connect(rank, world, handles)
    dist.barrier(group=group)
    nat.peer_share_pose(bool(share_pose))
    detector._peers = (rank, world)
    return nat


def disconnect_peers(detector, group=None):
    import torch.distributed as dist
    if getattr(detector, "_peers", None) is None:
        return
    dist.barrier(group=group)  # nobody may still be storing into a buffer that is about to be unmapped
    detector._native.peer_disconnect()
    detector._peers = None
    detector.shard = (0, 1)
    dist.barrier(group=group)


def _check_connected(detector, group, what):
    # RuntimeError unless the detector is connected to the peer exchange of this rank and world
    import torch.distributed as dist
    rank, world = dist.get_rank(group), dist.get_world_size(group)
    if getattr(detector, "_peers", None) != (rank, world):
        raise RuntimeError("%s needs a detector connected to the peer exchange of rank %d of %d (dist.connect_peers)" % (what, rank, world))


def _connected_batch(detector, frames, class_ids, sceneK, masks, group, what):
    # the native handle and its arguments for lm_peer_detect_batch; nothing touches a device before the checks
    _check_connected(detector, group, what)
    return detector._batch_args(frames, class_ids, sceneK, masks, what)


def match_refine_batch_sharded(detector, frames, threshold, class_ids, sceneK, iou_threshold=0.5, top_k=3, max_iterations=30,
                               use_scene_cloud=False, masks=[], group=None, estimation="point_to_plane"):
    """Detector.match_refine_batch with the bank sharded over the connected peer exchange (lm_peer_detect_batch); with
    connect_peers(share_pose=True) the pose stage is divided over the ranks too.  Every rank calls it with the same
    arguments (estimation included) and returns the whole result, equal to match_refine_batch on one unconnected
    detector."""
    _lib.estimation_code(estimation)
    nat, (rgb, depth, mk, K) = _connected_batch(detector, frames, class_ids, sceneK, masks, group, "match_refine_batch_sharded()")
    got = nat.peer_detect_batch(rgb, depth, mk, float(threshold), K, float(iou_threshold), int(top_k), int(max_iterations),
                                bool(use_scene_cloud), pose_nms=False, estimation=estimation)
    return detector._batch_pairs(nat, got)


def detect_batch_sharded(detector, frames, threshold, class_ids, sceneK, iou_threshold=0.5, translation_threshold=40.0, top_k=0,
                         max_iterations=30, use_scene_cloud=False, masks=[], group=None, estimation="point_to_plane"):
    """Detector.detect_batch with the bank sharded over the connected peer exchange (lm_peer_detect_batch), as
    match_refine_batch_sharded: every rank calls it and returns the whole result, equal to detect_batch on one
    unconnected detector."""
    _lib.estimation_code(estimation)
    nat, (rgb, depth, mk, K) = _connected_batch(detector, frames, class_ids, sceneK, masks, group, "detect_batch_sharded()")
    got = nat.peer_detect_batch(rgb, depth, mk, float(threshold), K, float(iou_threshold), int(top_k), int(max_iterations),
                                bool(use_scene_cloud), pose_nms=True, translation_threshold=float(translation_threshold),
                                estimation=estimation)
    return detector._batch_pairs(nat, got)


def track_batch_sharded(detector, depths, sceneK, objects, max_iterations=30, margin_px=4, estimation="point_to_plane", depth_scale=1.0,
                        stream=None, group=None):
    """Detector.track_batch over the connected peer exchange (lm_peer_track_batch); with connect_peers(share_pose=True)
    each rank tracks its share of every chunk's objects and the results travel to every rank.  Every rank calls it with
    the same depths, objects and arguments (estimation included), in the same order as its other pose exchanges, and
    returns the whole result, equal to track_batch on one unconnected detector.  A single frame is a one-frame batch.
    RuntimeError when the detector is not connected for this rank and world, and track_batch's TypeError / ValueError,
    all before any device work."""
    _check_connected(detector, group, "track_batch_sharded()")
    return detector._track_batch(depths, sceneK, objects, max_iterations, margin_px, estimation, depth_scale, stream, True,
                                 "track_batch_sharded")


def match_quantized_sharded(detector, quantized, threshold, class_ids=(), group=None):
    """Detector.match_quantized with the bank sharded over the process group: every rank returns the
    full, finished match list (identical to the single-GPU result)."""
    import torch.distributed as dist
    rank, world = dist.get_rank(group), dist.get_world_size(group)
    connected = getattr(detector, "_peers", None) == (rank, world)
    before = detector.shard
    detector.shard = shard_of(rank, world)
    try:
        nat = detector._select(list(class_ids))
        nat.upload_quantized(quantized)
        nat.run(float(threshold))
        if connected:
            allrec = nat.fetch_records()  # fused exchange: the result block already holds every shard's records
        else:
            allrec = gather_records(nat.fetch_records(), group)
        return detector._to_matches(nat.finish(allrec))
    finally:
        if not connected:
            detector.shard = before  # a later plain match() on this detector sees the whole bank again
