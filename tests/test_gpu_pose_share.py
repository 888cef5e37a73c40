"""The pose stage shared over the ranks of the peer exchange (lm_peer_share_pose): rank r refines survivors r, r + world,
... of the box NMS, the results travel to every rank, and every rank's lm_complete_pose / lm_complete_detect must equal,
bit for bit, one unconnected handle over the whole bank -- early returns, NaN patterns and the pose NMS's counts
included.  The frame is the recorded driver frame (tests/golden/driver_trace.npz) against the allScales bank, with the
per-template renders of tests/test_gpu_pose_stage.py: the recorded render shifted by a few pixels."""
import importlib
import os
import socket

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
lib = importlib.import_module("6dpose_b200._lib")

SHIFTS = [(0, 0), (-68, -19), (-180, 57), (3, -2), (-2, 4)]  # (rows, cols): two of them put the model where survivors lie
CAPACITY = 1 << 17                                          # records per rank and frame: the bank's at threshold 62


def load_data():
    g = np.load(os.path.join(ROOT, "tests", "golden", "driver_trace.npz"))
    b = np.load(os.path.join(ROOT, "tests", "golden", "bank_allScales_full.npz"))
    packed = dict(class_begin=b["class_begin"], tmeta=b["tmeta"].astype(np.int32), feats=b["feats"].astype(np.int32))
    G = packed["tmeta"].shape[0]
    renders = [np.ascontiguousarray(np.roll(np.roll(g["render"], dy, 0), dx, 1)) for dy, dx in SHIFTS]
    K = np.repeat(g["rf0_modelK"][None], G, 0).astype(np.float32)
    R = np.repeat(g["rf0_modelR"][None], G, 0).astype(np.float32)
    t = np.repeat(g["rf0_modelT"].reshape(1, 3), G, 0).astype(np.float32)
    t[:, 0] += (np.arange(G) % 7) - 3.0
    t[:, 2] += np.arange(G) % 11
    return dict(g=g, packed=packed, T=b["T"].tolist(), G=G, renders=renders, which=np.arange(G) % len(renders), K=K, R=R, t=t,
                sK=g["rf0_sceneK"].astype(np.float32), nf=int(g["num_features"]))


@pytest.fixture(scope="module")
def data():
    return load_data()


def handle(data, device=0, shard=(0, 1), renders=None, which=None):
    renders = data["renders"] if renders is None else renders
    which = data["which"] if which is None else which
    nat = lib.NativeDetector(data["T"], device)
    nat.load_bank(data["packed"], 4)
    nat.select(None, shard[0], shard[1])
    nat.set_template_renders(0, [renders[k] for k in which], data["K"], data["R"], data["t"])
    return nat


def connected(data, devices, share=True, renders=None, which=None):
    world = len(devices)
    dets = [handle(data, dev, (r, world), renders, which) for r, dev in enumerate(devices)]
    for d in dets:
        d.peer_export(world, CAPACITY)
    bases = [d.peer_base() for d in dets]
    for r, d in enumerate(dets):
        d.peer_connect_local(r, world, bases)
    # ranks of one process on one device: an unshared frame at the largest bound grows every pose stage's buffers first
    # (growing frees device memory, which waits for the whole device, a peer's pose collector included)
    frame(dets, data, 75.0, 0, False, False)
    for d in dets:
        d.peer_share_pose(share)
    return dets


def close(dets):
    for d in dets:
        d.peer_disconnect()
    for d in dets:
        d.close()


def frame(dets, data, thr, top_k, use_scene, nms, depth=None, max_iterations=30):
    """One frame on every rank: every match is enqueued before any post / pose stage (lm_enqueue_pose may synchronise)."""
    g = data["g"]
    for d in dets:
        d.upload_images(g["rgb"], g["depth"] if depth is None else depth, None)
    for d in dets:
        d.enqueue(thr)
    for d in dets:
        d.enqueue_post(0.5, top_k)
        d.enqueue_pose(data["sK"], max_iterations, use_scene)
        if nms:
            d.enqueue_pose_nms(40.0)
    return [d.complete_detect() if nms else d.complete_pose() for d in dets]


def same(got, want):
    assert np.array_equal(got[0], want[0])
    for x, y in zip(got[1:4], want[1:4]):
        assert np.array_equal(x, y, equal_nan=True)
    assert got[4] == want[4]


def expect_state(fn):
    with pytest.raises(lib.LinemodLibraryError) as e:
        fn()
    assert ("error %d" % lib.LM_E_STATE) in str(e.value), e.value
    return str(e.value)


@pytest.mark.parametrize("world", [2, 3, 4])
def test_every_rank_returns_the_single_gpu_result(data, world):
    single = handle(data)
    dets = connected(data, [0] * world)
    sizes = {}
    try:
        for thr in (62.0, 65.0, 75.0):
            for top_k in (0, 3):
                for use_scene in (False, True):
                    for nms in (False, True):
                        want = frame([single], data, thr, top_k, use_scene, nms)[0]
                        for got in frame(dets, data, thr, top_k, use_scene, nms):
                            same(got, want)
                        if nms:
                            sizes[(thr, top_k, use_scene)] = want[4]["survivors"]
                            assert all(d.pose_stats()[3] == 1 for d in dets)
    finally:
        close(dets)
    assert sizes[(65.0, 0, False)] > 100 and sizes[(75.0, 3, True)] == 3, sizes


def test_fewer_survivors_than_ranks_and_no_match(data):
    single = handle(data)
    dets = connected(data, [0] * 4)
    try:
        for nms in (False, True):
            want = frame([single], data, 75.0, 1, True, nms)[0]
            for got in frame(dets, data, 75.0, 1, True, nms):
                same(got, want)
            assert [d.pose_stats()[1] for d in dets] == [1, 0, 0, 0]
            blank = np.zeros_like(data["g"]["depth"])
            want = frame([single], data, 100.0, 0, False, nms, depth=blank)[0]
            assert len(want[0]) == 0
            for got in frame(dets, data, 100.0, 0, False, nms, depth=blank):
                same(got, want)
            assert [d.pose_stats()[:2] for d in dets] == [[0, 0]] * 4
    finally:
        close(dets)


def test_early_returns_and_zero_anchor_depth(data):
    g = data["g"]
    wide = np.zeros_like(g["render"])
    wide[200:260, 10:600] = 1000                               # a 598 x 68 box: fits only survivors with x < 42
    renders = data["renders"] + [wide]
    which = data["which"].copy()
    which[::2] = len(renders) - 1
    single = handle(data, renders=renders, which=which)
    dets = connected(data, [0, 0], renders=renders, which=which)
    try:
        want = frame([single], data, 62.0, 0, False, False)[0]
        early = want[3] == -1.0
        assert early.any() and (~early).any() and np.isnan(want[1][early]).all()
        for got in frame(dets, data, 62.0, 0, False, False):
            same(got, want)
        want = frame([single], data, 62.0, 0, False, True)[0]
        assert want[4]["posed"] < want[4]["survivors"]
        for got in frame(dets, data, 62.0, 0, False, True):
            same(got, want)
    finally:
        close(dets)
    off = [data["renders"][2]]                                 # shifted far from the centre: render[240, 320] == 0
    assert off[0][240, 320] == 0
    zeros = np.zeros(data["G"], np.int64)
    single = handle(data, renders=off, which=zeros)
    dets = connected(data, [0, 0], renders=off, which=zeros)
    try:
        for use_scene in (False, True):
            for nms in (False, True):
                want = frame([single], data, 70.0, 0, use_scene, nms)[0]
                if not nms:
                    assert np.isnan(want[1]).any()
                for got in frame(dets, data, 70.0, 0, use_scene, nms):
                    same(got, want)
    finally:
        close(dets)


def test_work_is_divided_and_launches_stay_fixed(data):
    single = handle(data)
    world = 3
    dets = connected(data, [0] * world)
    try:
        for top_k in (1, 50, 0):
            want = frame([single], data, 65.0, top_k, True, False)[0]
            S = len(want[0])
            got = frame(dets, data, 65.0, top_k, True, False)
            stats = [d.pose_stats() for d in dets]
            for r, (d, s) in enumerate(zip(dets, stats)):
                same(got[r], want)
                assert s == [S, len(range(r, S, world)), 6, 1], (r, s)
            assert sum(s[1] for s in stats) == S
            if top_k:
                assert S == top_k
        for d in dets:
            d.peer_share_pose(False)
        for top_k in (1, 50):
            want = frame([single], data, 65.0, top_k, True, True)[0]
            for d, got in zip(dets, frame(dets, data, 65.0, top_k, True, True)):
                same(got, want)
                assert d.pose_stats() == [top_k, top_k, 5, 0]
    finally:
        close(dets)
    # launches of the pose stage alone: enqueue_pose + complete_pose
    dets = connected(data, [0, 0])
    try:
        for share in (True, False):
            for d in dets:
                d.peer_share_pose(share)
            for top_k in (1, 50):
                g = data["g"]
                for d in dets:
                    d.upload_images(g["rgb"], g["depth"], None)
                for d in dets:
                    d.enqueue(65.0)
                for d in dets:
                    d.enqueue_post(0.5, top_k)
                before = [d.launch_count() for d in dets]
                for d in dets:
                    d.enqueue_pose(data["sK"], 30, True)
                for d, b in zip(dets, before):
                    assert len(d.complete_pose()[0]) == top_k
                    assert d.launch_count() - b == (6 if share else 5)
    finally:
        close(dets)


def test_twenty_frames_toggling_the_share(data):
    single = handle(data)
    dets = connected(data, [0, 0, 0], share=False)
    # threshold, top_k, use_scene_cloud, pose NMS; sharing off on every third frame: both frame slots of the pose area
    # are used with sharing on either side of a frame without it
    plan = [((62.0, 65.0, 75.0)[k % 3], (0, 3, 1, 17)[k % 4], k % 2 == 0, k % 5 < 2) for k in range(20)]
    want = {}
    try:
        for k, key in enumerate(plan):
            share = k % 3 != 1
            for d in dets:
                d.peer_share_pose(share)
            if key not in want:
                want[key] = frame([single], data, *key)[0]
            for d, got in zip(dets, frame(dets, data, *key)):
                same(got, want[key])
                assert d.pose_stats()[3] == int(share)
    finally:
        close(dets)


def test_errors(data):
    g = data["g"]
    nat = handle(data)
    expect_state(lambda: nat.peer_share_pose(True))            # not connected
    expect_state(lambda: nat.peer_share_pose(False))
    dets = connected(data, [0, 0])
    try:
        cfg = (65.0, 0, False, False)
        frame(dets, data, *cfg)
        assert all(d.pose_stats()[3] == 1 for d in dets)
        for d in dets:                                         # the batch stays single-GPU
            expect_state(lambda: d.detect_batch(g["rgb"][None], g["depth"][None], None, 65.0, data["sK"].reshape(1, 3, 3)))
    finally:
        for d in dets:
            d.peer_disconnect()
    for d in dets:                                             # disconnected: sharing is off, and cannot be turned on
        expect_state(lambda: d.peer_share_pose(True))
    for d in dets:
        d.peer_export(2, CAPACITY)
    bases = [d.peer_base() for d in dets]
    for r, d in enumerate(dets):
        d.peer_connect_local(r, 2, bases)
    try:
        frame(dets, data, *cfg)
        assert all(d.pose_stats()[2:] == [5, 0] for d in dets)  # reconnected: off until turned on again
    finally:
        close(dets)


def test_distinct_devices(data):
    import torch
    n = min(torch.cuda.device_count(), 4)
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    single = handle(data)
    dets = connected(data, list(range(n)))
    try:
        for thr, top_k in ((65.0, 0), (75.0, 3)):
            for nms in (False, True):
                want = frame([single], data, thr, top_k, True, nms)[0]
                for got in frame(dets, data, thr, top_k, True, nms):
                    same(got, want)
    finally:
        close(dets)


# ---- two processes: gloo for the IPC handles, Detector.detect on each rank ----
def free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def detector(data, bank_path):
    pkg = importlib.import_module("6dpose_b200")
    det = pkg.Detector(data["nf"], data["T"])
    det.device = 0
    det.readClasses(["06_template"], bank_path)
    det.setTemplateRenders({"06_template": ((data["renders"][k] for k in data["which"]), data["K"], data["R"], data["t"])})
    return det


def flatten(pairs):
    return dict(xy=np.asarray([(m.x, m.y, m.template_id) for m, _ in pairs], np.int64).reshape(-1, 3),
                sim=np.asarray([m.similarity for m, _ in pairs], np.float64),
                cls=np.asarray([m.class_id for m, _ in pairs]),
                res=np.asarray([p.getResidual() for _, p in pairs], np.float64),
                R=np.asarray([p.getR() for _, p in pairs], np.float64).reshape(-1, 3, 3),
                t=np.asarray([p.getT() for _, p in pairs], np.float64).reshape(-1, 3))


def detect_worker(rank, world, port, out_dir, bank_path):
    import sys
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    os.environ.pop("LINEMOD_B200_DEVICE", None)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    sys.path.insert(0, ROOT)
    dmod = importlib.import_module("6dpose_b200.dist")
    data = load_data()
    det = detector(data, bank_path)
    dmod.connect_peers(det, capacity_records=CAPACITY, share_pose=True)
    g = data["g"]
    out = {}
    for k, (thr, top_k) in enumerate(((65.0, 0), (75.0, 0), (65.0, 3))):
        got = flatten(det.detect([g["rgb"], g["depth"]], thr, ["06_template"], data["sK"], top_k=top_k))
        out.update({"%d_%s" % (k, key): v for key, v in got.items()})
    out["stats"] = np.asarray(det._native.pose_stats())
    dmod.disconnect_peers(det)
    np.savez(os.path.join(out_dir, "rank%d.npz" % rank), **out)
    dist.destroy_process_group()


def test_two_processes_detect(data, tmp_path):
    import torch.multiprocessing as mp
    bk = importlib.import_module("6dpose_b200.bank")
    bank = bk.TemplateBank()
    bank.classes["06_template"] = bk.PackedPyramids(data["packed"]["tmeta"], data["packed"]["feats"], 2)
    bank.write_packed("06_template", str(tmp_path / "06_template.lmb"), 2)
    bank_path = str(tmp_path / "%s.lmb")
    det = detector(data, bank_path)
    g = data["g"]
    want = {}
    for k, (thr, top_k) in enumerate(((65.0, 0), (75.0, 0), (65.0, 3))):
        got = flatten(det.detect([g["rgb"], g["depth"]], thr, ["06_template"], data["sK"], top_k=top_k))
        want.update({"%d_%s" % (k, key): v for key, v in got.items()})
    assert len(want["0_res"]) > 0
    mp.spawn(detect_worker, args=(2, free_port(), str(tmp_path), bank_path), nprocs=2, join=True)
    for r in range(2):
        got = np.load(str(tmp_path / ("rank%d.npz" % r)))
        for key, v in want.items():
            assert np.array_equal(got[key], v, equal_nan=v.dtype.kind == "f"), (r, key)
        assert got["stats"][3] == 1 and got["stats"][1] == len(range(r, int(got["stats"][0]), 2))
