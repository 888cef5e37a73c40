"""Tracking a batch of depth frames over the ranks of the peer exchange (lm_peer_track_batch / lm_peer_track_batch_device,
dist.track_batch_sharded): sharing off, every rank tracks every object; sharing on, each chunk's objects are divided over
the ranks and their results and window records travel through the pose area.  Either way every rank must return, bit for
bit, what one unconnected handle holding the same renders returns from lm_track_batch: status, box, T, R, t, residual,
lm_pose_transforms and lm_pose_verify.

Data: the recorded driver frame and its variants with a K per frame, each frame's objects as detect keeps them
(tests/test_gpu_track_batch.py), and the synthetic sequences of tests/pso_scenes.py.  Ranks that are handles of one
process on one device call from their own host threads, each after one run of the largest shape with sharing off."""
import importlib
import os
import socket

import numpy as np
import pytest
import torch

import pso_scenes
import test_gpu_peer_batch as pb
import test_gpu_track as gt
import test_gpu_track_batch as tb
import track_model as tm

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
lib = importlib.import_module("6dpose_b200._lib")

same_bits = gt.same_bits
WARM_COUNTS = [1000, 0, 1000, 100, 0, 0, 0, 0]  # the largest run below: 2100 objects over 8 frames


def make_handle(data, device, shard, one_render):
    if not one_render:
        return pb.handle(data, device, shard)
    # every template with the unshifted render: the window cap is the object's own, so WINDOW can be reached
    nat = lib.NativeDetector(data["T"], device)
    nat.load_bank(data["packed"], 4)
    nat.select(None, shard[0], shard[1])
    nat.set_template_renders(0, [data["g"]["render"]] * data["G"], data["K"], data["R"], data["t"])
    return nat


@pytest.fixture(scope="module")
def data():
    return pb.load_data()


@pytest.fixture(scope="module")
def ref(data):
    return make_handle(data, 0, (0, 1), False)


@pytest.fixture(scope="module")
def ref_one(data):
    return make_handle(data, 0, (0, 1), True)


@pytest.fixture(scope="module")
def pool(data, ref):
    """Every object detect keeps at threshold 65 on the recorded, rolled and mirrored frames."""
    out = []
    for name, K in zip(["recorded", "rolled", "mirrored"], pb.scene_ks(data, 3)):
        rgb, depth, _ = data["frames"][name]
        out += tb.detected(ref, rgb, depth, K, 65.0)
    assert out
    return out


def ragged(data, pool, counts):
    """(depths, Ks, objects) of frames cycling over the recorded, rolled and mirrored depths, counts[f] objects each."""
    names = ["recorded", "rolled", "mirrored"]
    depths = np.stack([data["frames"][names[f % 3]][1] for f in range(len(counts))])
    return depths, pb.scene_ks(data, len(counts)), tb.repeated(pool, counts)


def connected(data, pool, devices, one_render=False, warm_detect=False):
    """Handles over shards (r, world), connected on one exchange with sharing off; each has run the largest track run of
    these tests with sharing off and verification on, which grows every buffer a track run needs while no collector
    spins (warm_detect: and first one unconnected detect batch of the largest shape, then one connected frame, as
    tests/test_gpu_peer_batch.py's ranks)."""
    world = len(devices)
    dets = [make_handle(data, dev, (r, world), one_render) for r, dev in enumerate(devices)]
    if warm_detect:
        names = ["recorded", "rolled", "mirrored", "blank", "masked"][:pb.WARM]
        for d in dets:
            d.detect_batch(*pb.batch_args(data, names, pb.scene_ks(data, pb.WARM), 62.0, 0, True, True))
    for d in dets:
        d.peer_export(world, pb.CAPACITY)
    bases = [d.peer_base() for d in dets]
    for r, d in enumerate(dets):
        d.peer_connect_local(r, world, bases)
    if warm_detect:  # the result block grows to the exchange's size before any rank's collector runs
        for d in dets:
            d.prepare()
        pb.frame(dets, data, 75.0, 0, False, False)
    depths, Ks, objects = ragged(data, pool, WARM_COUNTS)
    for d in dets:
        d.set_pose_verify(True, 10.0)
        d.peer_track_batch(depths, Ks, objects, 30, 4)
        d.set_pose_verify(False)
    return dets


def unconnected(nat, depths, Ks, objects, estimation="point_to_plane", verify=False, margin=4):
    """lm_track_batch on one unconnected handle: (outputs per frame, transformations, verification or None)."""
    nat.set_pose_verify(verify, 10.0)
    try:
        got = nat.track_batch(depths, Ks, objects, 30, margin, estimation)
        return got, nat.pose_transforms(), nat.pose_verify() if verify else None
    finally:
        nat.set_pose_verify(False)


def peer_track(dets, depths, Ks, objects, estimation="point_to_plane", verify=False, margin=4, device=None):
    """lm_peer_track_batch on every rank from its own thread (device: per rank (planes, pitch, format, scale, stream) of
    lm_peer_track_batch_device): per rank (outputs, transformations, verification, pose stats, SLOTS item, launches)."""
    def one(r, d):
        d.set_pose_verify(verify, 10.0)
        try:
            before = d.launch_count()
            if device is None:
                got = d.peer_track_batch(depths, Ks, objects, 30, margin, estimation)
            else:
                planes, pitch, fmt, scale, st = device[r]
                got = d.peer_track_batch_device(planes, pitch, fmt, scale, depths.shape[1], depths.shape[2], st, Ks, objects, 30, margin,
                                                estimation)
            launches = d.launch_count() - before
            slots = d._pose_item(-1, "slots", np.zeros(4, np.int32)) if sum(map(len, objects)) else None
            return got, d.pose_transforms(), d.pose_verify() if verify else None, d.pose_stats(), slots, launches
        finally:
            d.set_pose_verify(False)
    return pb.on_every_rank(dets, one)


def same_run(got, want):
    (frames, T, ver), (wframes, wT, wver) = got[:3], want
    assert len(frames) == len(wframes)
    for f, (g, w) in enumerate(zip(frames, wframes)):
        for k, (a, b) in enumerate(zip(g, w)):
            assert same_bits(a, b), (f, k)
    assert same_bits(T, wT)
    assert (ver is None) == (wver is None)
    if ver is not None:
        assert same_bits(ver[0], wver[0]) and same_bits(ver[1], wver[1])


def expect_division(results, n, share, estimation="point_to_plane", verify=False, conversions=0):
    """pose stats, the last chunk's SLOTS item and the launches of every rank."""
    chunks = pb.chunk_sizes(n)
    world = len(results)
    per = (6 if share else 5) - (estimation == "point_to_point") + verify
    for r, (_, _, _, stats, slots, launches) in enumerate(results):
        mine = sum(len(range(r, C, world)) for C in chunks) if share else n
        assert stats == [n, mine, len(chunks) * per, int(share)], (r, stats, n)
        assert launches == len(chunks) * per + conversions, (r, launches)
        if n:
            C = chunks[-1]
            want = [-(-C // world), r, world] if share else [C, 0, 1]
            assert list(slots[:3]) == want and slots[3] == n - C, (r, slots)
    if share:
        assert sum(res[3][1] for res in results) == n


def status_run(ref_one, data):
    """tests/test_gpu_track_batch.py's status frames, with the first frame's first object also moved over every frame edge
    and behind the camera (tests/test_gpu_track.py)."""
    depths, Ks, objects = tb.status_frames(ref_one, data)
    c, t, T0 = objects[0][0]
    rows, cols = depths[0].shape
    objects[0] = objects[0] + [(c, t, T) for T in gt.edge_objects(T0, Ks[0], rows, cols)[1:]]
    return np.stack(depths), Ks, objects


@pytest.mark.parametrize("world", [2, 3, 4])
def test_every_rank_returns_the_unconnected_run(data, ref_one, pool, world):
    depths, Ks, objects = status_run(ref_one, data)
    n = sum(map(len, objects))
    dets = connected(data, pool, [0] * world, one_render=True)
    try:
        for share in (True, False):
            for d in dets:
                d.peer_share_pose(share)
            for estimation in ("point_to_plane", "point_to_point"):
                for verify in (False, True):
                    want = unconnected(ref_one, depths, Ks, objects, estimation, verify)
                    statuses = np.concatenate([w[0] for w in want[0]])
                    assert set(statuses.tolist()) == {tm.TRACKED, tm.OUTSIDE, tm.WINDOW, tm.NO_DEPTH}
                    results = peer_track(dets, depths, Ks, objects, estimation, verify)
                    for got in results:
                        same_run(got, want)
                    expect_division(results, n, share, estimation, verify)
        # the entries not tracked keep their box, residual -1 and their start T
        flat = [o for objs in objects for o in objs]
        got = results[-1][0]
        status, T, box, res = (np.concatenate([g[k] for g in got]) for k in (0, 1, 5, 4))
        lost = np.nonzero(status != tm.TRACKED)[0]
        assert len(lost) and np.all(res[lost] == -1.0)
        for i in lost:
            assert same_bits(T[i], flat[i][2])
            assert (status[i] == tm.OUTSIDE) == (not box[i].any())
    finally:
        pb.close(dets)


# more than 1024 objects with frames straddling the chunk boundary and an empty frame; fewer objects than ranks; frames
# without objects; no objects at all
RAGGED = [[1000, 0, 1000, 100], [1024, 1], [0, 2, 0], [1], [0, 0]]


def test_ragged_runs(data, ref, pool):
    dets = connected(data, pool, [0] * 3)
    try:
        for share in (True, False):
            for d in dets:
                d.peer_share_pose(share)
            for counts in RAGGED:
                depths, Ks, objects = ragged(data, pool, counts)
                want = unconnected(ref, depths, Ks, objects, verify=sum(counts) == 2100)
                results = peer_track(dets, depths, Ks, objects, verify=sum(counts) == 2100)
                for got in results:
                    same_run(got, want)
                expect_division(results, sum(counts), share, verify=sum(counts) == 2100)
    finally:
        pb.close(dets)


def test_twenty_steps_mixing_frames_batches_and_tracking(data, ref, pool):
    dets = connected(data, pool, [0] * 3, warm_detect=True)
    g = data["g"]
    try:
        for k in range(20):
            share = k % 4 != 3
            for d in dets:
                d.peer_share_pose(share)
            thr, top_k = (65.0, 75.0, 70.0)[k % 3], (0, 3, 1)[k % 3]
            if k % 3 == 0:                                     # a shared single frame
                want = ref.detect(g["rgb"], g["depth"], None, thr, data["sK"], 0.5, top_k, 30, True, 40.0)
                for got in pb.frame(dets, data, thr, top_k, True, True):
                    assert np.array_equal(got[0], want[0])
                    for x, y in zip(got[1:4], want[1:4]):
                        assert np.array_equal(x, y, equal_nan=True)
            elif k % 3 == 1:                                   # a sharded batch
                names = [pb.FRAMES[(k + j) % len(pb.FRAMES)] for j in range(1 + k % 4)]
                K = pb.scene_ks(data, len(names))
                args = pb.batch_args(data, names, K, thr, top_k, True, k % 2 == 0)
                want = (ref.detect_batch(*args), ref.batch_counts.copy())
                for got in pb.peer_batch(dets, args):
                    pb.same(got, want)
            else:                                              # a tracked batch, one or two chunks
                counts = [[30, 0, 7], [1000, 50], [5], [0, 3]][(k // 3) % 4]
                depths, Ks, objects = ragged(data, pool, counts)
                estimation = ("point_to_plane", "point_to_point")[k % 2]
                want = unconnected(ref, depths, Ks, objects, estimation)
                results = peer_track(dets, depths, Ks, objects, estimation)
                for got in results:
                    same_run(got, want)
                expect_division(results, sum(counts), share, estimation)
    finally:
        pb.close(dets)


def test_device_frames_equal_the_host_form(data, ref, pool):
    depths, Ks, objects = ragged(data, pool, [40, 0, 25])
    want = unconnected(ref, depths, Ks, objects)
    dets = connected(data, pool, [0] * 2)
    try:
        for share in (True, False):
            for d in dets:
                d.peer_share_pose(share)
            for f32, fmt, scale in ((False, lib.DEPTH_U16_MM, 1.0), (True, lib.DEPTH_F32, 1000.0)):
                streams = [torch.cuda.Stream() for _ in dets]
                ts = [[tb.pitched(d, f32, st) for d in depths] for st in streams]
                for st in streams:
                    st.synchronize()
                pitch = ts[0][0].stride(0) * ts[0][0].element_size()
                device = [([t.data_ptr() for t in tr], pitch, fmt, scale, st.cuda_stream) for tr, st in zip(ts, streams)]
                results = peer_track(dets, depths, Ks, objects, device=device)
                for got in results:
                    same_run(got, want)
                expect_division(results, 65, share, conversions=len(depths))
                for st in streams:
                    st.synchronize()
    finally:
        pb.close(dets)


def test_distinct_devices(data, ref, pool):
    n = min(torch.cuda.device_count(), 4)
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    dets = connected(data, pool, list(range(n)))
    try:
        for share in (True, False):
            for d in dets:
                d.peer_share_pose(share)
            for counts in ([1000, 0, 1000, 100], [3, 0]):
                depths, Ks, objects = ragged(data, pool, counts)
                want = unconnected(ref, depths, Ks, objects)
                results = peer_track(dets, depths, Ks, objects)
                for got in results:
                    same_run(got, want)
                expect_division(results, sum(counts), share)
    finally:
        pb.close(dets)


# ---- two processes: gloo for the IPC handles, dist.track_batch_sharded on each rank ----
def free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


MOTIONS = [(np.radians([0.6, -0.8, 0.5]), np.array([2.0, -1.0, 1.5])), (np.radians([-0.4, 0.3, 0.9]), np.array([-1.5, 2.0, -1.0]))]


def sequence_scene(sc, k, m):
    """Frame k of synthetic sequence m (the motions of tests/test_gpu_track_batch.py's lockstep test) and its truth."""
    w, v = MOTIONS[m]
    Rt = pso_scenes.rodrigues(w * k)
    tt = sc.cM + v * k / 1000.0 - Rt @ sc.cM
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = Rt, tt
    return pso_scenes.splat(sc.M @ Rt.T + tt, sc.sK, sc.rows, sc.cols, sc.table), T


def flatten(frames):
    pairs = [p for frame in frames for p in frame]
    return dict(n=np.asarray([len(f) for f in frames], np.int64),
                xy=np.asarray([(m.x, m.y, m.template_id) for m, _ in pairs], np.int64).reshape(-1, 3),
                status=np.asarray([p.getTrackStatus() for _, p in pairs]),
                res=np.asarray([p.getResidual() for _, p in pairs], np.float64),
                R=np.asarray([p.getR() for _, p in pairs], np.float64).reshape(-1, 3, 3),
                t=np.asarray([p.getT() for _, p in pairs], np.float64).reshape(-1, 3),
                T=np.asarray([p.getTransformation() for _, p in pairs], np.float64).reshape(-1, 4, 4))


def track_steps(det, data, track_batch):
    """detect on the recorded and rolled frames, track those objects on both frames, then the two synthetic sequences
    tracked in lockstep for four steps: the flattened results of every call, keyed by step."""
    pkg = importlib.import_module("6dpose_b200")
    pr = importlib.import_module("6dpose_b200.pose_refine")
    fr = data["frames"]
    names = ["recorded", "rolled"]
    pairs = [det.detect([fr[n][0], fr[n][1]], 75.0, [], data["sK"]) for n in names]
    out = {}
    got = track_batch([fr[n][1] for n in names], data["sK"], pairs)
    out.update({"0_" + k: v for k, v in flatten(got).items()})
    sc = pso_scenes.Scenes(data["g"])
    cid = det.classIds()[0]
    batch = []
    for m in range(len(MOTIONS)):
        p = pr.poseRefine()
        p._T = sequence_scene(sc, 0, m)[1]
        batch.append([(pkg.Match(0, 0, 1.0, cid, 0), p)])
    for k in range(1, 5):
        batch = track_batch([sequence_scene(sc, k, m)[0] for m in range(len(MOTIONS))], sc.sK.astype(np.float32), batch)
        out.update({"%d_%s" % (k, key): v for key, v in flatten(batch).items()})
    return out


def track_worker(rank, world, port, out_dir, bank_path):
    import sys
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    os.environ.pop("LINEMOD_B200_DEVICE", None)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    sys.path.insert(0, ROOT)
    dmod = importlib.import_module("6dpose_b200.dist")
    data = pb.load_data()
    det = pb.detector(data, bank_path)
    dmod.connect_peers(det, capacity_records=pb.CAPACITY, share_pose=True)
    out = track_steps(det, data, lambda depths, K, objects: dmod.track_batch_sharded(det, depths, K, objects))
    out["stats"] = np.asarray(det._native.pose_stats())
    dmod.disconnect_peers(det)
    np.savez(os.path.join(out_dir, "rank%d.npz" % rank), **out)
    dist.destroy_process_group()


def test_two_processes_track(data, tmp_path):
    import torch.multiprocessing as mp
    bk = importlib.import_module("6dpose_b200.bank")
    bank = bk.TemplateBank()
    bank.classes["06_template"] = bk.PackedPyramids(data["packed"]["tmeta"], data["packed"]["feats"], 2)
    bank.write_packed("06_template", str(tmp_path / "06_template.lmb"), 2)
    bank_path = str(tmp_path / "%s.lmb")
    det = pb.detector(data, bank_path)
    want = track_steps(det, data, det.track_batch)
    assert len(want["0_res"]) > 0 and (want["4_status"] == "tracked").all()
    mp.spawn(track_worker, args=(2, free_port(), str(tmp_path), bank_path), nprocs=2, join=True)
    for r in range(2):
        got = np.load(str(tmp_path / ("rank%d.npz" % r)))
        for key, v in want.items():
            assert np.array_equal(got[key], v, equal_nan=v.dtype.kind == "f"), (r, key)
        assert got["stats"][3] == 1 and got["stats"][1] == len(range(r, int(got["stats"][0]), 2))
