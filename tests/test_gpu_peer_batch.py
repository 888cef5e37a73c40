"""A batch of RGB-D frames over the ranks of the peer exchange (lm_peer_detect_batch, dist.detect_batch_sharded /
match_refine_batch_sharded): each frame's match runs the fused record exchange, the batch's pose stage runs in chunks
-- divided over the ranks with lm_peer_share_pose -- and every rank must return, bit for bit, what one unconnected
handle over the whole bank returns from lm_detect_batch on the same frames: entries, R, t, residual (NaN patterns
included) and all four frame counts.  The data are those of tests/test_gpu_detect_batch.py: the recorded driver frame
(rolled, mirrored, blank and masked variants, a sceneK per frame) against the allScales bank, with per-template
renders that are the recorded render shifted by a few pixels.  Ranks that are handles of one process on one device
call from their own host threads, each after one unconnected batch of the largest shape it runs."""
import ctypes
import importlib
import os
import socket
import threading

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
lib = importlib.import_module("6dpose_b200._lib")

SHIFTS = [(0, 0), (-68, -19), (-180, 57), (3, -2), (-2, 4)]  # (rows, cols): two of them put the model where survivors lie
CAPACITY = 1 << 17                                          # records per rank and frame: the bank's at threshold 62
WARM = 5                                                    # frames of the warm-up batch: the largest batch below


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
    rgb, depth = g["rgb"], g["depth"]
    H, W = depth.shape
    mask = np.zeros((H, W), np.uint8)
    mask[:, W // 3:] = 255
    frames = dict(
        recorded=(rgb, depth, None),
        rolled=(np.roll(rgb, (17, -23), (0, 1)), np.roll(depth, (17, -23), (0, 1)), None),
        mirrored=(np.ascontiguousarray(rgb[:, ::-1]), np.ascontiguousarray(depth[:, ::-1]), None),
        blank=(np.zeros_like(rgb), np.zeros_like(depth), None),
        masked=(rgb, depth, (mask, mask)),
    )
    return dict(g=g, packed=packed, T=b["T"].tolist(), G=G, renders=renders, which=np.arange(G) % len(renders), K=K, R=R, t=t,
                sK=g["rf0_sceneK"].astype(np.float32), frames=frames, nf=int(g["num_features"]))


@pytest.fixture(scope="module")
def data():
    return load_data()


def scene_ks(data, n):
    # a different focal length and principal point per frame: the scene clouds and centroids depend on them
    K = np.repeat(data["sK"][None], n, 0).copy()
    K[:, 0, 0] *= 1.0 + 0.01 * np.arange(n)
    K[:, 1, 2] += np.arange(n)
    return K


def handle(data, device=0, shard=(0, 1)):
    nat = lib.NativeDetector(data["T"], device)
    nat.load_bank(data["packed"], 4)
    nat.select(None, shard[0], shard[1])
    nat.set_template_renders(0, [data["renders"][k] for k in data["which"]], data["K"], data["R"], data["t"])
    return nat


def batch_args(data, names, K, thr, top_k, use_scene, pose_nms, iters=30):
    frames = [data["frames"][n] for n in names]
    masks = [list(f[2]) if f[2] else [None, None] for f in frames]
    return (np.stack([f[0] for f in frames]), np.stack([f[1] for f in frames]), masks, thr, K, 0.5, top_k, iters, use_scene,
            pose_nms, 40.0)


def connected(data, devices, share=True, capacity=CAPACITY, warm_frame=True):
    """Handles over shards (r, world); each runs one unconnected batch of the largest shape first (it uploads the renders
    and grows every buffer: a free waits for the whole device, a peer's collector included), then the exchange is wired,
    every rank's result block grows to the exchange's size (lm_prepare, before any rank's collector runs) and (warm_frame)
    one connected single frame runs on every rank."""
    world = len(devices)
    dets = [handle(data, dev, (r, world)) for r, dev in enumerate(devices)]
    names = ["recorded", "rolled", "mirrored", "blank", "masked"][:WARM]
    for d in dets:
        d.detect_batch(*batch_args(data, names, scene_ks(data, WARM), 62.0, 0, True, True))
    for d in dets:
        d.peer_export(world, capacity)
    bases = [d.peer_base() for d in dets]
    for r, d in enumerate(dets):
        d.peer_connect_local(r, world, bases)
    for d in dets:
        d.prepare()
    if warm_frame:
        frame(dets, data, 75.0, 0, False, False)
    for d in dets:
        d.peer_share_pose(share)
    return dets


def close(dets):
    for d in dets:
        d.peer_disconnect()
    for d in dets:
        d.close()


def frame(dets, data, thr, top_k, use_scene, nms):
    """One shared single frame on every rank from one thread: every match is enqueued before any post / pose stage."""
    g = data["g"]
    for d in dets:
        d.upload_images(g["rgb"], g["depth"], None)
    for d in dets:
        d.enqueue(thr)
    for d in dets:
        d.enqueue_post(0.5, top_k)
        d.enqueue_pose(data["sK"], 30, use_scene)
        if nms:
            d.enqueue_pose_nms(40.0)
    return [d.complete_detect() if nms else d.complete_pose() for d in dets]


def on_every_rank(dets, fn):
    """fn(rank, handle) on every rank, each from its own host thread; returns the results (or raises the first error)."""
    got, errs = [None] * len(dets), [None] * len(dets)

    def run(r):
        try:
            got[r] = fn(r, dets[r])
        except BaseException as e:  # re-raised below, on the test's thread
            errs[r] = e

    threads = [threading.Thread(target=run, args=(r,)) for r in range(len(dets))]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    for e in errs:
        if e is not None:
            raise e
    return got


def peer_batch(dets, args, cap=None):
    """lm_peer_detect_batch on every rank: [(frames, frame counts)] per rank."""
    def one(r, d):
        frames = d.peer_detect_batch(*args, cap=cap)
        return frames, d.batch_counts.copy()
    return on_every_rank(dets, one)


@pytest.fixture(scope="module")
def ref(data):
    """One unconnected handle over the whole bank, and its lm_detect_batch results by configuration."""
    nat = handle(data)
    cache = {}

    def want(names, thr, top_k, use_scene, pose_nms, K=None):
        K = scene_ks(data, len(names)) if K is None else K
        key = (tuple(names), thr, top_k, use_scene, pose_nms, K.tobytes())
        if key not in cache:
            frames = nat.detect_batch(*batch_args(data, names, K, thr, top_k, use_scene, pose_nms))
            cache[key] = (frames, nat.batch_counts.copy())
        return cache[key]

    want.nat = nat
    return want


def same(got, want):
    frames, counts = got
    wframes, wcounts = want
    assert np.array_equal(counts, wcounts), (counts, wcounts)
    assert len(frames) == len(wframes)
    for (out, R, t, res, extra), w in zip(frames, wframes):
        assert np.array_equal(out, w[0])
        assert np.array_equal(res, w[3], equal_nan=True)
        assert np.array_equal(R, w[1], equal_nan=True)
        assert np.array_equal(t, w[2], equal_nan=True)
        assert extra == w[4]


def chunk_sizes(S):
    return [min(1024, S - c0) for c0 in range(0, S, 1024)]


def expect_stats(dets, S, share):
    chunks = chunk_sizes(S)
    world = len(dets)
    stats = [d.pose_stats() for d in dets]
    for r, s in enumerate(stats):
        mine = sum(len(range(r, C, world)) for C in chunks) if share else S
        assert s == [S, mine, len(chunks) * (6 if share else 5), int(share)], (r, s, S)
    if share:
        assert sum(s[1] for s in stats) == S


FRAMES = ["recorded", "rolled", "mirrored", "blank", "masked"]


@pytest.mark.parametrize("world", [2, 3, 4])
def test_every_rank_returns_the_single_gpu_batch(data, ref, world):
    dets = connected(data, [0] * world)
    try:
        for share in (True, False):
            for d in dets:
                d.peer_share_pose(share)
            for top_k in (0, 3):
                for use_scene in (False, True):
                    for pose_nms in (False, True):
                        want = ref(FRAMES, 75.0, top_k, use_scene, pose_nms)
                        args = batch_args(data, FRAMES, scene_ks(data, len(FRAMES)), 75.0, top_k, use_scene, pose_nms)
                        for got in peer_batch(dets, args):
                            same(got, want)
                        expect_stats(dets, int(want[1][:, 1].sum()), share)
        n = ref(FRAMES, 75.0, 0, False, True)[1][:, 1]
        assert n[3] == 0 and min(n[0], n[1], n[2], n[4]) > 0, n  # the blank frame has no match, the others do
    finally:
        close(dets)


def test_two_chunks_few_survivors_and_a_blank_batch(data, ref):
    dets = connected(data, [0] * 3)
    try:
        names = ["recorded", "rolled", "recorded", "mirrored"]
        for share in (True, False):
            for d in dets:
                d.peer_share_pose(share)
            for pose_nms in (True, False):
                # more than 1024 survivors: two chunks, so both slots of the pose area serve one call
                want = ref(names, 65.0, 0, False, pose_nms)
                S = int(want[1][:, 1].sum())
                assert S > 1024 and want[1][:, 1].max() <= 1024, S
                for got in peer_batch(dets, batch_args(data, names, scene_ks(data, 4), 65.0, 0, False, pose_nms)):
                    same(got, want)
                expect_stats(dets, S, share)
                # top_k 1 over two frames: 2 survivors for 3 ranks, one rank refines none and still publishes
                want = ref(["recorded", "mirrored"], 75.0, 1, True, pose_nms)
                assert want[1][:, 1].tolist() == [1, 1]
                for got in peer_batch(dets, batch_args(data, ["recorded", "mirrored"], scene_ks(data, 2), 75.0, 1, True, pose_nms)):
                    same(got, want)
                expect_stats(dets, 2, share)
                if share:
                    assert [d.pose_stats()[1] for d in dets] == [1, 1, 0]
                # every frame blank: no survivor, no pose exchange, every rank returns
                want = ref(["blank", "blank"], 75.0, 0, True, pose_nms)
                assert want[1][:, 1].sum() == 0
                for got in peer_batch(dets, batch_args(data, ["blank", "blank"], scene_ks(data, 2), 75.0, 0, True, pose_nms)):
                    same(got, want)
                expect_stats(dets, 0, share)
    finally:
        close(dets)


def test_twenty_steps_mixing_frames_and_batches(data, ref):
    single = ref.nat
    dets = connected(data, [0] * 3, share=False)
    g = data["g"]
    try:
        for k in range(20):
            share = k % 4 != 3
            for d in dets:
                d.peer_share_pose(share)
            thr, top_k, use_scene, nms = (65.0, 75.0, 70.0)[k % 3], (0, 3, 1)[k % 3], k % 2 == 0, k % 5 < 3
            if k % 3 == 1:                                     # a shared single frame: detect or match_pose
                if nms:
                    want = single.detect(g["rgb"], g["depth"], None, thr, data["sK"], 0.5, top_k, 30, use_scene, 40.0)
                else:
                    want = single.match_pose(g["rgb"], g["depth"], None, thr, data["sK"], 0.5, top_k, 30, use_scene)
                for got in frame(dets, data, thr, top_k, use_scene, nms):
                    assert np.array_equal(got[0], want[0])
                    for x, y in zip(got[1:4], want[1:4]):
                        assert np.array_equal(x, y, equal_nan=True)
                    assert got[4] == want[4]
                assert all(d.pose_stats()[3] == int(share) for d in dets)
            else:                                              # a sharded batch of 1 to 4 frames
                names = [FRAMES[(k + j) % len(FRAMES)] for j in range(1 + k % 4)]
                K = scene_ks(data, len(names))
                want = ref(names, thr, top_k, use_scene, nms, K)
                for got in peer_batch(dets, batch_args(data, names, K, thr, top_k, use_scene, nms)):
                    same(got, want)
                expect_stats(dets, int(want[1][:, 1].sum()), share)
    finally:
        close(dets)


def match_launches(dets, data, thr):
    g = data["g"]
    before = [d.launch_count() for d in dets]
    for d in dets:
        d.upload_images(g["rgb"], g["depth"], None)
    for d in dets:
        d.enqueue(thr)
    for d in dets:
        d.enqueue_post(0.5, 0)
    for d in dets:
        d.complete_post()
    return [d.launch_count() - b for d, b in zip(dets, before)]


def test_launches(data, ref):
    dets = connected(data, [0] * 3)
    try:
        for thr, n_frames in ((75.0, 1), (75.0, 4), (65.0, 3)):
            match_launches(dets, data, thr)                    # first use of this threshold
            per_frame = match_launches(dets, data, thr)
            names = ["recorded"] * n_frames
            for share in (True, False):
                for d in dets:
                    d.peer_share_pose(share)
                for pose_nms in (False, True):
                    args = batch_args(data, names, scene_ks(data, n_frames), thr, 0, False, pose_nms)
                    before = [d.launch_count() for d in dets]
                    got = peer_batch(dets, args)
                    S = int(got[0][1][:, 1].sum())
                    chunks = len(chunk_sizes(S))
                    assert chunks == (2 if thr == 65.0 else 1), S
                    for d, b, p in zip(dets, before, per_frame):
                        assert d.launch_count() - b == n_frames * p + chunks * (6 if share else 5) + (1 if pose_nms else 0)
                    expect_stats(dets, S, share)
    finally:
        close(dets)


def expect_code(fn, code):
    with pytest.raises(RuntimeError) as e:
        fn()
    if code == lib.LM_E_INVALID:
        assert not isinstance(e.value, lib.LinemodLibraryError), e.value
    else:
        assert ("error %d" % code) in str(e.value), e.value
    return str(e.value)


def test_errors_and_capacity(data, ref):
    names = ["recorded", "mirrored"]
    K = scene_ks(data, 2)
    args = batch_args(data, names, K, 75.0, 0, False, True)
    expect_code(lambda: ref.nat.peer_detect_batch(*args), lib.LM_E_STATE)  # no exchange
    dets = connected(data, [0] * 3)
    try:
        for d in dets:                                          # argument errors: before any device work, rank by rank
            bad = list(args)
            bad[10] = float("nan")
            expect_code(lambda: d.peer_detect_batch(*bad), lib.LM_E_INVALID)
            bad[10] = -1.0
            expect_code(lambda: d.peer_detect_batch(*bad), lib.LM_E_INVALID)
            empty = (np.zeros((0, 480, 640, 3), np.uint8), np.zeros((0, 480, 640), np.uint16), None, 75.0,
                     np.zeros((0, 3, 3), np.float32))
            expect_code(lambda: d.peer_detect_batch(*empty), lib.LM_E_INVALID)
            expect_code(lambda: d.detect_batch(*args), lib.LM_E_STATE)  # the unconnected call still refuses
        L = lib.load()
        for pose_nms in (False, True):
            want = ref(names, 75.0, 0, False, pose_nms)
            total = int(want[1][:, 0].sum())
            assert total > 1
            rgb = np.ascontiguousarray(np.stack([data["frames"][n][0] for n in names]))
            depth = np.ascontiguousarray(np.stack([data["frames"][n][1] for n in names]))
            Kc = np.ascontiguousarray(K)

            def raw(r, d):
                n, counts = ctypes.c_int64(), np.zeros((2, 4), np.int64)
                rc = L.lm_peer_detect_batch(d._h, 2, rgb.ctypes.data_as(ctypes.POINTER(ctypes.c_uint8)),
                                            depth.ctypes.data_as(ctypes.POINTER(ctypes.c_uint16)), 480, 640, None, ctypes.c_float(75.0),
                                            Kc.ctypes.data_as(ctypes.POINTER(ctypes.c_float)), 0.5, 0, 30, 0, 1 if pose_nms else 0, 40.0,
                                            None, None, None, None, 0, ctypes.byref(n), counts.ctypes.data_as(ctypes.POINTER(ctypes.c_int64)))
                return rc, n.value, counts

            for rc, n, counts in on_every_rank(dets, raw):     # LM_E_CAPACITY with the needed total on every rank
                assert rc == lib.LM_E_CAPACITY and n == total
                assert np.array_equal(counts, want[1])
            for got in peer_batch(dets, batch_args(data, names, K, 75.0, 0, False, pose_nms), cap=1):  # the binding grows it
                same(got, want)
    finally:
        close(dets)


def test_records_beyond_the_exchange_raise_on_every_rank(data):
    """A shard that keeps more records than the exchange holds fails the batch on every rank with the exchange's
    message: growing the output capacity cannot help, so the binding raises instead of calling again."""
    dets = connected(data, [0] * 3, capacity=16, warm_frame=False)  # 16 records per shard: any frame outgrows them
    args = batch_args(data, ["recorded", "mirrored"], scene_ks(data, 2), 62.0, 0, False, True)
    try:
        for share in (True, False):
            for d in dets:
                d.peer_share_pose(share)

            def one(r, d):
                try:
                    d.peer_detect_batch(*args)
                except lib.LinemodLibraryError as e:
                    return str(e)
                return None
            msgs = on_every_rank(dets, one)
            for m in msgs:
                assert m is not None and ("error %d" % lib.LM_E_CAPACITY) in m and "peer exchange" in m, msgs
    finally:
        close(dets)


def test_distinct_devices(data, ref):
    import torch
    n = min(torch.cuda.device_count(), 4)
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    dets = connected(data, list(range(n)))
    try:
        for share in (True, False):
            for d in dets:
                d.peer_share_pose(share)
            for thr, top_k, names in ((65.0, 0, ["recorded", "rolled", "recorded", "mirrored"]), (75.0, 3, FRAMES)):
                for pose_nms in (False, True):
                    want = ref(names, thr, top_k, True, pose_nms)
                    for got in peer_batch(dets, batch_args(data, names, scene_ks(data, len(names)), thr, top_k, True, pose_nms)):
                        same(got, want)
                    expect_stats(dets, int(want[1][:, 1].sum()), share)
    finally:
        close(dets)


# ---- two processes: gloo for the IPC handles, dist.detect_batch_sharded / match_refine_batch_sharded on each rank ----
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


def flatten(per_frame):
    out = {}
    for f, pairs in enumerate(per_frame):
        out.update({"%d_xy" % f: np.asarray([(m.x, m.y, m.template_id) for m, _ in pairs], np.int64).reshape(-1, 3),
                    "%d_sim" % f: np.asarray([m.similarity for m, _ in pairs], np.float64),
                    "%d_cls" % f: np.asarray([m.class_id for m, _ in pairs]),
                    "%d_res" % f: np.asarray([p.getResidual() for _, p in pairs], np.float64),
                    "%d_R" % f: np.asarray([np.full((3, 3), -7.0) if p.getR() is None else p.getR() for _, p in pairs],
                                           np.float64).reshape(-1, 3, 3),
                    "%d_t" % f: np.asarray([np.full((3, 1), -7.0) if p.getT() is None else p.getT() for _, p in pairs],
                                           np.float64).reshape(-1, 3)})
    return out


def sources(data):
    fr = data["frames"]
    frames = [[fr[n][0], fr[n][1]] for n in ("recorded", "mirrored", "blank", "masked")]
    masks = [[], [], [], list(fr["masked"][2])]
    return frames, masks, scene_ks(data, len(frames))


def dist_worker(rank, world, port, out_dir, bank_path):
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
    frames, masks, K = sources(data)
    out = {}
    for key, v in flatten(dmod.detect_batch_sharded(det, frames, 75.0, ["06_template"], K, masks=masks)).items():
        out["detect_" + key] = v
    out["stats"] = np.asarray(det._native.pose_stats())
    det._native.peer_share_pose(False)
    for key, v in flatten(dmod.match_refine_batch_sharded(det, frames, 75.0, ["06_template"], K, top_k=3, masks=masks)).items():
        out["refine_" + key] = v
    try:
        det.detect_batch(frames, 75.0, ["06_template"], K, masks=masks)  # the unconnected call keeps refusing
        out["refused"] = np.asarray(0)
    except lib.LinemodLibraryError:
        out["refused"] = np.asarray(1)
    dmod.disconnect_peers(det)
    np.savez(os.path.join(out_dir, "rank%d.npz" % rank), **out)
    dist.destroy_process_group()


def test_two_processes_sharded_batches(data, tmp_path):
    import torch.multiprocessing as mp
    bk = importlib.import_module("6dpose_b200.bank")
    bank = bk.TemplateBank()
    bank.classes["06_template"] = bk.PackedPyramids(data["packed"]["tmeta"], data["packed"]["feats"], 2)
    bank.write_packed("06_template", str(tmp_path / "06_template.lmb"), 2)
    bank_path = str(tmp_path / "%s.lmb")
    det = detector(data, bank_path)
    frames, masks, K = sources(data)
    want = {}
    want.update({"detect_" + k: v for k, v in flatten(det.detect_batch(frames, 75.0, ["06_template"], K, masks=masks)).items()})
    want.update({"refine_" + k: v for k, v in
                 flatten(det.match_refine_batch(frames, 75.0, ["06_template"], K, top_k=3, masks=masks)).items()})
    assert len(want["detect_0_res"]) > 0 and len(want["refine_0_res"]) == 3 and len(want["detect_2_res"]) == 0
    mp.spawn(dist_worker, args=(2, free_port(), str(tmp_path), bank_path), nprocs=2, join=True)
    for r in range(2):
        got = np.load(str(tmp_path / ("rank%d.npz" % r)))
        for key, v in want.items():
            assert np.array_equal(got[key], v, equal_nan=v.dtype.kind == "f"), (r, key)
        S = int(got["stats"][0])
        assert got["stats"][3] == 1 and got["stats"][1] == len(range(r, S, 2)) and S > 0
        assert int(got["refused"]) == 1
