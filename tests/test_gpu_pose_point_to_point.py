"""The device pose stage with the point-to-point estimation (lm_set_pose_estimation(LM_ICP_POINT_TO_POINT)): on the
recorded driver frame against the allScales bank, every path -- single frame, pose NMS, batch, shared stage and peer
batch -- must equal lm_icp_process_batch in point-to-point mode (or one unconnected handle), bit for bit, as the
point-to-plane mode does in tests/test_gpu_pose_stage.py, tests/test_gpu_detect_batch.py and tests/test_gpu_peer_batch.py,
whose data and helpers are reused."""
import importlib

import numpy as np
import pytest

import pose_nms_model
import test_gpu_peer_batch as pb
import test_gpu_pose_stage as ps

pytestmark = pytest.mark.gpu
lib = importlib.import_module("6dpose_b200._lib")
P2P, P2PL = "point_to_point", "point_to_plane"
FRAMES = ["recorded", "rolled", "mirrored", "blank", "masked"]


@pytest.fixture(scope="module")
def data():
    return pb.load_data()


def host_poses(data, surv, max_iterations, use_scene, renders=None, which=None, estimation=P2P):
    renders = data["renders"] if renders is None else renders
    which = data["which"] if which is None else which
    icp = lib.NativeIcp()
    icp.set_use_scene_cloud(use_scene)
    tid = surv["template_id"].astype(np.int64)
    xy = np.stack([surv["x"], surv["y"]], 1)
    return icp.process_batch(data["g"]["depth"], [renders[k] for k in which[tid]], data["sK"], data["K"][tid], data["R"][tid],
                             data["t"][tid], xy, max_iterations, estimation)


def chain(nat, data, thr, top_k, iters, use_scene, estimation=P2P):
    g = data["g"]
    return nat.match_pose(g["rgb"], g["depth"], None, thr, data["sK"], 0.5, top_k, iters, use_scene, estimation)


@pytest.mark.parametrize("max_iterations", [30, 10])
@pytest.mark.parametrize("use_scene", [False, True])
def test_device_chain_equals_process_batch(data, use_scene, max_iterations):
    nat = ps.detector(data)
    found, differ = 0, 0
    for thr, top_k in ((75.0, 3), (65.0, 0)):
        want_surv, nrec = ps.survivors(nat, data, thr, top_k)
        got = chain(nat, data, thr, top_k, max_iterations, use_scene)
        assert np.array_equal(got[0], want_surv) and got[4] == nrec
        want = host_poses(data, want_surv, max_iterations, use_scene)
        ps.same_poses(got, want)
        found += int((got[3] > 0).sum())
        plane = host_poses(data, want_surv, max_iterations, use_scene, estimation=P2PL)
        differ += int(not np.array_equal(want[0], plane[0], equal_nan=True))
        # the pose NMS on top equals the numpy model on lm_complete_pose's output
        g = data["g"]
        nat.upload_images(g["rgb"], g["depth"], None)
        nat.enqueue(thr)
        nat.enqueue_post(0.5, top_k)
        nat.enqueue_pose(data["sK"], max_iterations, use_scene, P2P)
        nat.enqueue_pose_nms(40.0)
        out, R, t, res, counts = nat.complete_detect()
        ws, wR, wt, wr = pose_nms_model.detect(want_surv, want[0], want[1], want[2], 40.0)
        assert np.array_equal(out, ws) and np.array_equal(res, wr)
        assert np.array_equal(R, wR, equal_nan=True) and np.array_equal(t, wt, equal_nan=True)
        assert counts["survivors"] == len(want_surv)
    assert found > 0 and differ > 0  # some hypotheses find correspondences, and their poses are the point-to-point ones


def test_early_returns_zero_anchor_and_retry(data):
    g = data["g"]
    wide = np.zeros_like(g["render"])
    wide[200:260, 10:600] = 1000
    renders = data["renders"] + [wide]
    which = data["which"].copy()
    which[::2] = len(renders) - 1
    nat = ps.detector(data, renders, which)
    got = chain(nat, data, 62.0, 0, 30, False)
    assert (got[3] == -1.0).any() and (got[3] != -1.0).any()
    ps.same_poses(got, host_poses(data, got[0], 30, False, renders, which))
    off = [data["renders"][2]]
    assert off[0][240, 320] == 0
    which0 = np.zeros(data["G"], np.int64)
    nat = ps.detector(data, off, which0)
    for use_scene in (False, True):
        got = chain(nat, data, 70.0, 0, 30, use_scene)
        want = host_poses(data, got[0], 30, use_scene, off, which0)
        assert np.isnan(want[0]).any()
        ps.same_poses(got, want)
    # the result block overflows on the first frame of a fresh handle: the rerun keeps the frame's estimation, even
    # though the handle's setting changed between enqueue and complete
    probe = ps.detector(data)
    thr = next(c for c in (55.0, 50.0, 45.0, 40.0) if ps.survivors(probe, data, c, 3)[1] > (1 << 16))
    nat = ps.detector(data)
    nat.upload_images(g["rgb"], g["depth"], None)
    nat.enqueue(thr)
    nat.enqueue_post(0.5, 5)
    nat.enqueue_pose(data["sK"], 30, True, P2P)
    nat.set_pose_estimation(P2PL)
    got = nat.complete_pose()
    want_surv, _ = ps.survivors(probe, data, thr, 5)
    assert np.array_equal(got[0], want_surv)
    ps.same_poses(got, host_poses(data, want_surv, 30, True))


def test_switching_modes_and_launches(data):
    g = data["g"]
    nat = ps.detector(data)
    chain(nat, data, 45.0, 1, 30, True, P2PL)  # the first frame grows the result block
    p2p = chain(nat, data, 65.0, 0, 30, True, P2P)
    plane = chain(nat, data, 65.0, 0, 30, True, P2PL)
    for est, got in ((P2P, p2p), (P2PL, plane)):
        want = chain(ps.detector(data), data, 65.0, 0, 30, True, est)
        ps.same_poses(got, want[1:4])
    # a frame enqueued in one mode completes in that mode after the setting changed
    nat.upload_images(g["rgb"], g["depth"], None)
    nat.enqueue(65.0)
    nat.enqueue_post(0.5, 0)
    nat.enqueue_pose(data["sK"], 30, True, P2P)
    nat.set_pose_estimation(P2PL)
    ps.same_poses(nat.complete_pose(), p2p[1:4])
    # launches: 4 per unshared frame in point-to-point mode, 5 in point-to-plane mode, whatever the survivor count
    for est, n in ((P2P, 4), (P2PL, 5)):
        for top_k in (1, 50):
            nat.upload_images(g["rgb"], g["depth"], None)
            nat.enqueue(45.0)
            nat.enqueue_post(0.5, top_k)
            before = nat.launch_count()
            nat.enqueue_pose(data["sK"], 30, True, est)
            nat.complete_pose()
            assert nat.launch_count() - before == n, (est, top_k)
            assert nat.pose_stats()[2] == n
    L = lib.load()
    for bad in (2, -1, 7):
        assert L.lm_set_pose_estimation(nat._h, bad) == lib.LM_E_INVALID
    assert L.lm_set_pose_estimation(None, 0) == lib.LM_E_INVALID


def test_batch_equals_single_frames(data):
    nat = pb.handle(data)
    single = ps.detector(data)
    K = pb.scene_ks(data, len(FRAMES))
    for pose_nms in (False, True):
        for top_k, thr in ((0, 75.0), (3, 65.0)):
            args = pb.batch_args(data, FRAMES, K, thr, top_k, True, pose_nms)
            before = nat.launch_count()
            got = nat.detect_batch(*args, estimation=P2P)
            S = int(nat.batch_counts[:, 1].sum())
            chunks = len(pb.chunk_sizes(S))
            assert nat.launch_count() - before >= chunks * 4
            for f, name in enumerate(FRAMES):
                rgb, depth, masks = data["frames"][name]
                single.upload_images(rgb, depth, list(masks) if masks else None)
                single.enqueue(thr)
                single.enqueue_post(0.5, top_k)
                single.enqueue_pose(K[f], 30, True, P2P)
                if pose_nms:
                    single.enqueue_pose_nms(40.0)
                    want = single.complete_detect()
                else:
                    want = single.complete_pose()
                assert np.array_equal(got[f][0], want[0]), (name, pose_nms, top_k)
                for a, b in zip(got[f][1:4], want[1:4]):
                    assert np.array_equal(a, b, equal_nan=True), (name, pose_nms, top_k)


@pytest.mark.parametrize("world", [2, 3])
def test_shared_stage_and_peer_batch_equal_one_handle(data, world):
    ref = pb.handle(data)
    K = pb.scene_ks(data, len(FRAMES))
    dets = pb.connected(data, [0] * world)
    try:
        for share in (True, False):
            for d in dets:
                d.peer_share_pose(share)
            for pose_nms in (False, True):
                args = pb.batch_args(data, FRAMES, K, 75.0, 0, True, pose_nms)
                want = (ref.detect_batch(*args, estimation=P2P), ref.batch_counts.copy())
                got = pb.on_every_rank(dets, lambda r, d: (d.peer_detect_batch(*args, estimation=P2P), d.batch_counts.copy()))
                for gr in got:
                    pb.same(gr, want)
                S = int(want[1][:, 1].sum())
                for r, d in enumerate(dets):
                    st = d.pose_stats()
                    assert st[2] == len(pb.chunk_sizes(S)) * (5 if share else 4) and st[3] == int(share), (r, st)
            # a shared single frame: every rank returns the unconnected handle's poses
            g = data["g"]
            for d in dets:
                d.upload_images(g["rgb"], g["depth"], None)
            for d in dets:
                d.enqueue(65.0)
            for d in dets:
                d.enqueue_post(0.5, 0)
                d.enqueue_pose(data["sK"], 30, True, P2P)
            got = [d.complete_pose() for d in dets]
            want = chain(ref, data, 65.0, 0, 30, True, P2P)
            for gr in got:
                assert np.array_equal(gr[0], want[0])
                ps.same_poses(gr, want[1:4])
            for d in dets:
                assert d.pose_stats()[2] == (5 if share else 4)
    finally:
        pb.close(dets)


def test_distinct_devices(data):
    import torch
    n = min(torch.cuda.device_count(), 3)
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    ref = pb.handle(data)
    K = pb.scene_ks(data, len(FRAMES))
    dets = pb.connected(data, list(range(n)))
    try:
        args = pb.batch_args(data, FRAMES, K, 75.0, 0, True, True)
        want = (ref.detect_batch(*args, estimation=P2P), ref.batch_counts.copy())
        for gr in pb.on_every_rank(dets, lambda r, d: (d.peer_detect_batch(*args, estimation=P2P), d.batch_counts.copy())):
            pb.same(gr, want)
    finally:
        pb.close(dets)
