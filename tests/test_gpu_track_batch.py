"""Tracking a batch of depth frames (include/linemod_b200.h, lm_track_batch / lm_track_batch_device, Detector.track_batch):
every frame's entries bit for bit against a separate lm_track call on that frame -- status, box, T, R, t, residual, the
transformations and the verification -- across statuses, both ICP estimations, verification off and on, chunk boundaries
and device frames; the clouds of a chunk whose slots come from different frames against tests/track_model.py; launch
counts; and two synthetic sequences tracked in lockstep.

Data: the recorded driver frame and its rolled / mirrored variants with a K per frame (tests/test_gpu_peer_batch.py),
and the synthetic scenes of tests/pso_scenes.py."""
import importlib

import numpy as np
import pytest
import torch

import pso_scenes
import test_gpu_peer_batch as pb
import test_gpu_track as gt
import track_model as tm
from oracle import icp_oracle

pytestmark = pytest.mark.gpu
lib = importlib.import_module("6dpose_b200._lib")
pkg = importlib.import_module("6dpose_b200")
pr = importlib.import_module("6dpose_b200.pose_refine")

same_bits = gt.same_bits
shifted = gt.shifted


@pytest.fixture(scope="module")
def data():
    d = pb.load_data()
    d["cap"] = 4 * max(int(np.prod(icp_oracle.model_bbox(r)[2:])) for r in d["renders"])
    return d


@pytest.fixture(scope="module")
def nat(data):
    return pb.handle(data)


@pytest.fixture(scope="module")
def one_render(data):
    # every template with the unshifted render: the window cap is the object's own, so WINDOW can be reached
    nat = lib.NativeDetector(data["T"], 0)
    nat.load_bank(data["packed"], 4)
    nat.select(None, 0, 1)
    nat.set_template_renders(0, [data["g"]["render"]] * data["G"], data["K"], data["R"], data["t"])
    return nat


def detected(nat, rgb, depth, K, thr):
    out, *_ = nat.detect(rgb, depth, None, thr, K, 0.5, 0, 30, False, 40.0)
    T = nat.pose_transforms()
    return [(int(o["class_index"]), int(o["template_id"]), T[k]) for k, o in enumerate(out)]


def singles(nat, depths, Ks, objects, margin=4, estimation="point_to_plane", verify=False):
    """Each frame's lm_track alone: (outputs, transformations, verification or None) per frame."""
    out = []
    for d, K, objs in zip(depths, Ks, objects):
        got = nat.track(d, K, objs, 30, margin, estimation)
        out.append((got, nat.pose_transforms(), nat.pose_verify() if verify else None))
    return out


def check_batch(nat, got, want, verify):
    """The batch's per-frame outputs, lm_pose_transforms and lm_pose_verify against the single calls', bit for bit."""
    T = nat.pose_transforms()
    ver = nat.pose_verify() if verify else None
    assert len(got) == len(want)
    at = 0
    for f, (g, (w, wT, wv)) in enumerate(zip(got, want)):
        n = len(w[0])
        for k, (a, b) in enumerate(zip(g, w)):
            assert same_bits(a, b), (f, k)
        assert same_bits(T[at:at + n], wT), f
        if verify:
            assert same_bits(ver[0][at:at + n], wv[0]) and same_bits(ver[1][at:at + n], wv[1]), f
        at += n
    assert at == len(T)
    if verify:
        assert len(ver[0]) == at


def status_frames(nat, data):
    """The recorded, rolled and mirrored frames, the recorded one with its first object's window zeroed, a synthetic
    scene and a blank frame without objects, a K per frame; per frame its detect poses at 75, plus copies of its first
    object moved out of the frame and close to the camera."""
    fr = data["frames"]
    names = ["recorded", "rolled", "mirrored"]
    Ks = list(pb.scene_ks(data, 4))
    blankK = pb.scene_ks(data, 5)[4]
    depths, objects = [], []
    base = None
    for name, K in zip(names, Ks):
        rgb, depth, _ = fr[name]
        objs = detected(nat, rgb, depth, K, 75.0)
        if objs and base is None:
            base = (objs[0], depth, K)
        depths.append(depth)
        objects.append(objs)
    assert base is not None
    (c, t, T0), depth0, K0 = base
    nat.track(depth0, K0, [(c, t, T0)], 30, 4)
    slot = nat.pose_clouds()[1][0]
    raw = slot["raw_model"]
    x, y, w, h = (int(v) for v in slot["window"])
    zeroed = depth0.copy()
    zeroed[y:y + h, x:x + w] = 0
    depths.append(zeroed)
    Ks[3] = K0
    objects.append([(c, t, T0)])
    for f in range(len(objects)):
        if not objects[f]:
            continue
        c, t, T = objects[f][0]
        centroid = (raw @ T[:3, :3].T + T[:3, 3]).mean(0)
        objects[f] = objects[f] + [(c, t, shifted(T, 10.0)), (c, t, shifted(T, *(-0.75 * centroid)))]
    blank = fr["blank"][1]
    depths.insert(2, blank)
    Ks.insert(2, blankK)
    objects.insert(2, [])
    sc = pso_scenes.Scenes(data["g"])
    if (sc.rows, sc.cols) == depth0.shape:
        scene, _, T_true = sc.case(10, np.random.default_rng(7))
        depths.append(scene)
        Ks.append(sc.sK.astype(np.float32))
        objects.append([(0, 0, T_true), (0, 0, shifted(T_true, 10.0))])
    return depths, np.stack(Ks).astype(np.float32), objects


@pytest.mark.parametrize("verify", [False, True])
@pytest.mark.parametrize("estimation", ["point_to_plane", "point_to_point"])
def test_every_frame_equals_its_own_track(one_render, data, estimation, verify):
    nat = one_render
    depths, Ks, objects = status_frames(nat, data)
    nat.set_pose_verify(verify, 10.0)
    try:
        want = singles(nat, depths, Ks, objects, 4, estimation, verify)
        statuses = set(np.concatenate([w[0][0] for w in want]).tolist())
        assert statuses == {tm.TRACKED, tm.OUTSIDE, tm.WINDOW, tm.NO_DEPTH}, statuses
        got = nat.track_batch(np.stack(depths), Ks, objects, 30, 4, estimation)
        check_batch(nat, got, want, verify)
    finally:
        nat.set_pose_verify(False)


def repeated(objects, counts):
    """counts[f] objects for frame f, cycling through the pool `objects`."""
    out, at = [], 0
    for n in counts:
        out.append([objects[(at + k) % len(objects)] for k in range(n)])
        at += n
    return out


# totals 1023, 1024, 1025, 1050 (the last chunk's slots from two frames) and 2100, empty frames first, in the middle and
# last, and frames straddling the boundaries at 1024 and 2048
COUNTS = [[0, 700, 0, 323], [1024, 0], [0, 700, 0, 325, 0], [1000, 0, 30, 20, 0], [1000, 0, 1000, 100]]


@pytest.mark.parametrize("counts", COUNTS, ids=[str(sum(c)) for c in COUNTS])
def test_chunk_boundaries(nat, data, counts):
    names = ["recorded", "rolled", "mirrored"]
    Ks = pb.scene_ks(data, len(counts))
    pool = []
    for name, K in zip(names, Ks):
        rgb, depth, _ = data["frames"][name]
        pool += detected(nat, rgb, depth, K, 65.0)
    assert pool
    depths = np.stack([data["frames"][names[f % 3]][1] for f in range(len(counts))])
    objects = repeated(pool, counts)
    verify = sum(counts) == 1025
    nat.set_pose_verify(verify, 10.0)
    try:
        want = singles(nat, depths, Ks, objects, 4, "point_to_plane", verify)
        before = nat.launch_count()
        got = nat.track_batch(depths, Ks, objects, 30, 4)
        chunks = -(-sum(counts) // 1024)
        assert nat.launch_count() - before == chunks * (6 if verify else 5)
        check_batch(nat, got, want, verify)
        first = (chunks - 1) * 1024
        head = nat._pose_item(-1, "slots", np.zeros(4, np.int32))
        assert head[0] == sum(counts) - first and head[3] == first
    finally:
        nat.set_pose_verify(False)
    if counts != [1000, 0, 30, 20, 0]:
        return
    _, slots = nat.pose_clouds()
    # the last chunk's slots against the model, each with its own frame's depth and K
    frame_of = np.repeat(np.arange(len(counts)), counts)
    flat = [o for objs in objects for o in objs]
    frames_seen = set()
    for i, s in enumerate(slots):
        e = first + i
        f = int(frame_of[e])
        frames_seen.add(f)
        c, tid, T = flat[e]
        g = int(data["packed"]["class_begin"][c]) + tid
        w = tm.track(depths[f], Ks[f], data["renders"][data["which"][g]], data["K"][g], T, 4, data["cap"])
        assert s["status"] == w["status"] and tuple(int(v) for v in s["window"]) == w["window"], (i, f)
        if s["posed"]:
            for k in ("raw_model", "raw_scene", "source", "target", "init"):
                assert same_bits(s[k], w[k]), (i, k)
    assert frames_seen == {2, 3}


def test_launches_and_empty_batches(nat, data):
    rgb, depth, _ = data["frames"]["recorded"]
    objs = detected(nat, rgb, depth, data["sK"], 75.0)
    Ks = pb.scene_ks(data, 3)
    depths = np.stack([depth] * 3)
    for estimation, per in (("point_to_plane", 5), ("point_to_point", 4)):
        before = nat.launch_count()
        nat.track_batch(depths, Ks, [objs, [], objs], 30, 4, estimation)
        assert nat.launch_count() - before == per
    before = nat.launch_count()
    got = nat.track_batch(depths, Ks, [[], [], []], 30, 4)
    assert nat.launch_count() - before == 0 and all(len(g[0]) == 0 for g in got)
    assert len(nat.pose_transforms()) == 0
    # a one-frame batch is lm_track
    want = nat.track(depth, Ks[0], objs, 30, 4)
    got = nat.track_batch(depth[None], Ks[:1], [objs], 30, 4)
    assert all(same_bits(a, b) for a, b in zip(got[0], want))


def pitched(depth, f32, st):
    """depth as a CUDA tensor view with a row pitch wider than its row: u16 mm, or f32 metres."""
    H, W = depth.shape
    with torch.cuda.stream(st):
        if f32:
            wide = torch.zeros(H, W + 24, dtype=torch.float32, device="cuda")
            wide[:, :W] = torch.from_numpy(depth.astype(np.float32)).cuda() / 1000.0
        else:
            wide = torch.zeros(H, W + 40, dtype=torch.int16, device="cuda").view(torch.uint16)
            wide.view(torch.int16)[:, :W] = torch.from_numpy(depth.view(np.int16)).cuda()
    return wide[:, :W]


def test_device_frames_equal_the_host_batch(nat, data):
    names = ["recorded", "rolled", "mirrored"]
    Ks = pb.scene_ks(data, 3)
    depths = np.stack([data["frames"][n][1] for n in names])
    objects = [detected(nat, data["frames"][n][0], data["frames"][n][1], K, 75.0) for n, K in zip(names, Ks)]
    objects[1] = []
    want = nat.track_batch(depths, Ks, objects, 30, 4)
    wT = nat.pose_transforms()
    st = torch.cuda.Stream()
    for f32, fmt, scale in ((False, lib.DEPTH_U16_MM, 1.0), (True, lib.DEPTH_F32, 1000.0)):
        ts = [pitched(d, f32, st) for d in depths]
        pitch = ts[0].stride(0) * ts[0].element_size()
        assert pitch > depths.shape[2] * ts[0].element_size()
        before = nat.launch_count()
        got = nat.track_batch_device([t.data_ptr() for t in ts], pitch, fmt, scale, depths.shape[1], depths.shape[2], st.cuda_stream, Ks,
                                     objects, 30, 4)
        assert nat.launch_count() - before == 3 + 5
        for g, w in zip(got, want):
            assert all(same_bits(a, b) for a, b in zip(g, w))
        assert same_bits(nat.pose_transforms(), wT)
        st.synchronize()


# ---- the Python surface -----------------------------------------------------------------------------------------------
def same_pairs(a, b):
    assert len(a) == len(b)
    for (ma, pa), (mb, pb_) in zip(a, b):
        assert (ma.x, ma.y, ma.similarity, ma.class_id, ma.template_id) == (mb.x, mb.y, mb.similarity, mb.class_id, mb.template_id)
        assert pa.getTrackStatus() == pb_.getTrackStatus() and same_bits(pa.getResidual(), pb_.getResidual())
        for x, y in ((pa.getR(), pb_.getR()), (pa.getT(), pb_.getT()), (pa.getTransformation(), pb_.getTransformation())):
            assert (x is None and y is None) or same_bits(x, y)


def test_detector_track_batch_equals_track(data, tmp_path):
    det = gt.det_public(data, tmp_path)
    names = ["recorded", "rolled", "mirrored"]
    Ks = pb.scene_ks(data, 3)
    frames = [data["frames"][n] for n in names]
    pairs = [det.detect([f[0], f[1]], 75.0, [], K) for f, K in zip(frames, Ks)]
    pairs[2] = pairs[2] + [dict(class_id=m.class_id, template_id=m.template_id, R=p.getR(), t=p.getT()) for m, p in pairs[0][:2]]
    depths = [f[1] for f in frames]
    for estimation in ("point_to_plane", "point_to_point"):
        want = [det.track(d, K, p, estimation=estimation) for d, K, p in zip(depths, Ks, pairs)]
        got = det.track_batch(depths, Ks, pairs, estimation=estimation)
        for g, w in zip(got, want):
            same_pairs(g, w)
    tensors = [torch.from_numpy(d.view(np.int16)).cuda().view(torch.uint16) for d in depths]
    got = det.track_batch(tensors, Ks, pairs)
    for g, w in zip(got, [det.track(d, K, p) for d, K, p in zip(depths, Ks, pairs)]):
        same_pairs(g, w)
    # one K for every frame
    got = det.track_batch(depths, data["sK"], pairs)
    for g, d, p in zip(got, depths, pairs):
        same_pairs(g, det.track(d, data["sK"], p))


def test_two_sequences_in_lockstep(data, tmp_path):
    # two synthetic sequences with different motions, tracked one step at a time as a batch of their frames, equal the
    # two sequences tracked on their own
    det = gt.det_public(data, tmp_path)
    sc = pso_scenes.Scenes(data["g"])
    sK = sc.sK.astype(np.float32)
    motions = [(np.radians([0.6, -0.8, 0.5]), np.array([2.0, -1.0, 1.5])), (np.radians([-0.4, 0.3, 0.9]), np.array([-1.5, 2.0, -1.0]))]

    def scene(k, m):
        w, v = motions[m]
        Rt = pso_scenes.rodrigues(w * k)
        tt = sc.cM + v * k / 1000.0 - Rt @ sc.cM
        T = np.eye(4)
        T[:3, :3], T[:3, 3] = Rt, tt
        return pso_scenes.splat(sc.M @ Rt.T + tt, sc.sK, sc.rows, sc.cols, sc.table), T

    cid = det.classIds()[0]
    batch = []
    for m in range(len(motions)):
        p = pr.poseRefine()
        p._T = scene(0, m)[1]  # the first frame's truth starts each sequence
        batch.append([(pkg.Match(0, 0, 1.0, cid, 0), p)])
    single = list(batch)
    for k in range(1, 5):
        scenes = [scene(k, m)[0] for m in range(len(motions))]
        batch = det.track_batch(scenes, sK, batch)
        single = [det.track(s, sK, objs) for s, objs in zip(scenes, single)]
        for g, w in zip(batch, single):
            same_pairs(g, w)
            assert g[0][1].getTrackStatus() == "tracked"
