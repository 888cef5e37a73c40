"""Tracking on the device (include/linemod_b200.h, lm_track / lm_track_device / lm_pose_transforms): the clouds of a
track chunk bit for bit against tests/track_model.py, the ICP against the oracle, the transformations of the existing
pose calls, the round trip from detect, sequences of synthetic frames, the statuses, device depth and verification.

Data: the recorded driver frame (tests/golden/driver_trace.npz) against the allScales bank with per-template renders
(tests/test_gpu_peer_batch.py), and the synthetic scenes of tests/pso_scenes.py (the recorded render moved and splatted
over a tilted table)."""
import importlib

import numpy as np
import pytest
import torch

import pose_verify_model as pvm
import pso_scenes
import test_gpu_peer_batch as pb
import track_model as tm
from oracle import icp_oracle

pytestmark = pytest.mark.gpu
lib = importlib.import_module("6dpose_b200._lib")
pkg = importlib.import_module("6dpose_b200")
bk = importlib.import_module("6dpose_b200.bank")


@pytest.fixture(scope="module")
def data():
    d = pb.load_data()
    d["cap"] = 4 * max(int(np.prod(icp_oracle.model_bbox(r)[2:])) for r in d["renders"])
    return d


@pytest.fixture(scope="module")
def nat(data):
    return pb.handle(data)


def detected(nat, data, thr=65.0, use_scene=False):
    g = data["g"]
    out, R, t, res, _ = nat.detect(g["rgb"], g["depth"], None, thr, data["sK"], 0.5, 0, 30, use_scene, 40.0)
    return out, R, t, res, nat.pose_transforms()


def shifted(T, dx_m, dy_m=0.0, dz_m=0.0):
    T = np.array(T, np.float64).reshape(4, 4)
    T[0, 3] += dx_m
    T[1, 3] += dy_m
    T[2, 3] += dz_m
    return T


def same_bits(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and a.tobytes() == b.tobytes()


def check_chunk(nat, data, depth, sK, objects, margin):
    """Every slot of the last (track) chunk against track_model; returns the model's results."""
    head, slots = nat.pose_clouds()
    assert head["slots"] == len(objects)
    want_all = []
    for i, (c, tid, T) in enumerate(objects):
        g = int(data["packed"]["class_begin"][c]) + tid
        want = tm.track(depth, sK, data["renders"][data["which"][g]], data["K"][g], T, margin, data["cap"])
        s = slots[i]
        assert s["status"] == want["status"], (i, s["status"], want["status"])
        assert tuple(int(v) for v in s["window"]) == want["window"], (i, s["window"], want["window"])
        assert s["posed"] == (want["status"] == tm.TRACKED)
        if s["posed"]:
            for k in ("raw_model", "raw_scene", "source", "target", "init"):
                assert same_bits(s[k], want[k]), (i, k)
        want_all.append(want)
    return want_all


def edge_objects(T0, sK, rows, cols):
    """T0 moved so that the object straddles each frame edge, lies wholly outside, and stays put."""
    z = T0[2, 3] + 0.0
    fx, fy = float(sK[0, 0]), float(sK[1, 1])
    out = [T0]
    for dx, dy in ((-1, 0), (1, 0), (0, -1), (0, 1)):
        # the translation that moves the projected centre about half a frame in that direction
        out.append(shifted(T0, dx * 0.5 * cols * z / fx, dy * 0.5 * rows * z / fy))
    out.append(shifted(T0, 0.0, 0.0, -5.0))  # behind the camera
    return out


# ---- clouds pinned -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("margin", [0, 4, 13])
def test_clouds_equal_the_model_on_the_recorded_frame(nat, data, margin):
    out, _, _, _, T = detected(nat, data)
    assert len(out) > 0
    objects = [(int(o["class_index"]), int(o["template_id"]), T[k]) for k, o in enumerate(out)]
    c0, t0 = objects[0][:2]
    objects += [(c0, t0, Te) for Te in edge_objects(T[0], data["sK"], *data["g"]["depth"].shape)]
    status, *_ = nat.track(data["g"]["depth"], data["sK"], objects, 30, margin)
    want = check_chunk(nat, data, data["g"]["depth"], data["sK"], objects, margin)
    assert [w["status"] for w in want] == status.tolist()
    assert tm.OUTSIDE in status.tolist() and tm.TRACKED in status.tolist()


@pytest.mark.parametrize("seed", [0, 1])
def test_clouds_equal_the_model_on_synthetic_scenes(nat, data, seed):
    sc = pso_scenes.Scenes(data["g"])
    rng = np.random.default_rng(seed)
    scene, _, T_true = sc.case(10, rng)
    sK = sc.sK.astype(np.float32)
    objects = [(0, 0, T_true)] + [(0, 0, Te) for Te in edge_objects(T_true, sK, *scene.shape)]
    for margin in (0, 4, 9):
        nat.track(scene, sK, objects, 30, margin)
        check_chunk(nat, data, scene, sK, objects, margin)


# ---- ICP against the oracle -------------------------------------------------------------------------------------------
def rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-12))


# On the synthetic scenes every object is compared.  On the recorded frame only detect's best-ranked object is: the others
# are false detections of this bank (its renders are shifted copies of one render), whose models slide along the table
# with a few pairs where the point-to-plane system is ill-conditioned, and one rounding difference (the normals' eigen
# solver, a correspondence at the 1 cm radius) sends device and oracle on different paths, as on any pose path (measured
# on an H100: the best object agrees to 1.6e-13, another pairing 58 % of its points differs by 2.5e-2).
@pytest.mark.parametrize("estimation", ["point_to_plane"])
def test_icp_equals_the_oracle(nat, data, estimation):
    out, _, _, _, T = detected(nat, data, 75.0, True)
    sc = pso_scenes.Scenes(data["g"])
    cases = [(data["g"]["depth"], data["sK"], [(int(out[0]["class_index"]), int(out[0]["template_id"]), T[0])])]
    for seed in (3, 4, 5):
        scene, _, T_true = sc.case(10, np.random.default_rng(seed))
        cases.append((scene, sc.sK.astype(np.float32), [(0, 0, T_true)]))
    for depth, sK, objs in cases:
        status, Tn, _, _, res, _ = nat.track(depth, sK, objs, 30, 4, estimation)
        assert status[0] == tm.TRACKED
        s = nat.pose_clouds()[1][0]
        tgt = s["target"]
        Tw, fit, _, _ = icp_oracle.registration_icp_p2pl(s["source"], tgt, icp_oracle.estimate_normals(tgt), icp_oracle.MAX_DIST,
                                                          s["init"], 30)
        assert rel(Tn[0], Tw) <= 1e-4, rel(Tn[0], Tw)
        assert abs(float(res[0]) - fit) <= 1e-4, (float(res[0]), fit)


# ---- transformations of the existing pose calls -------------------------------------------------------------------------
def det_public(data, tmp_path):
    g, packed = data["g"], data["packed"]
    bank = bk.TemplateBank()
    bank.classes["06_template"] = bk.PackedPyramids(packed["tmeta"], packed["feats"], 2)
    bank.write_packed("06_template", str(tmp_path / "06_template.lmb"), 2)
    det = pkg.Detector(int(g["num_features"]), data["T"])
    det.readClasses(["06_template"], str(tmp_path / "%s.lmb"))
    det.setTemplateRenders({"06_template": ((data["renders"][k] for k in data["which"]), data["K"], data["R"], data["t"])})
    return det


def composes(data, pairs):
    n = 0
    for m, p in pairs:
        if p.getResidual() == -1.0:
            assert p.getTransformation() is None
            continue
        T = p.getTransformation()
        R, t = tm.compose(T, data["R"][m.template_id], data["t"][m.template_id])
        assert same_bits(R, p.getR()) and same_bits(t, p.getT().reshape(3)), m
        assert p.getTrackStatus() is None
        n += 1
    return n


def test_transformations_compose_to_the_poses(data, tmp_path):
    det = det_public(data, tmp_path)
    g = data["g"]
    frame = [g["rgb"], g["depth"]]
    assert composes(data, det.match_refine(frame, 65.0, [], data["sK"], top_k=0)) > 0
    assert composes(data, det.detect(frame, 65.0, [], data["sK"])) > 0
    assert composes(data, det.detect(frame, 65.0, [], data["sK"], estimation="point_to_point")) > 0
    for frames in ([frame, frame], [[torch.from_numpy(g["rgb"]).cuda(), torch.from_numpy(g["depth"].view(np.int16)).cuda().view(torch.uint16)]] * 2):
        for got in (det.detect_batch(frames, 65.0, [], data["sK"]), det.match_refine_batch(frames, 65.0, [], data["sK"], top_k=0)):
            assert all(composes(data, f) > 0 for f in got)
    # asking for the transformations changes nothing the pose calls return
    nat = pb.handle(data)
    out, R, t, res, _ = nat.detect(g["rgb"], g["depth"], None, 65.0, data["sK"], 0.5, 0, 30, False, 40.0)
    nat.pose_transforms()
    out2, R2, t2, res2, _ = nat.detect(g["rgb"], g["depth"], None, 65.0, data["sK"], 0.5, 0, 30, False, 40.0)
    assert same_bits(R, R2) and same_bits(t, t2) and same_bits(res, res2)


# ---- round trip -------------------------------------------------------------------------------------------------------
# Tracking the detection frame from detect's own pairs (threshold 75) tracks every object.  detect registers the model
# against itself (the reference's target, LL.cpp:109), so its pose is the centroid start, and tracking, which registers
# against the scene, moves it by as much as the scene asks: this bank's detections are false ones (its renders are
# shifted copies of one render) whose models slide along the table, by up to 1.2 m from detect's pose and by 2 mm to
# 0.54 m more on a second track of the same frame (measured on an H100; some leave the frame), so no distance bounds
# those steps.  A dict start
# (R, t converted to T) gives the pair start's result (T itself) to within DICT_MM, for the objects whose tracked pose
# pairs at least half of the model's points (measured: 9e-5 mm at most).
DICT_MM = 1e-3


def test_round_trip_from_detect(data, tmp_path):
    det = det_public(data, tmp_path)
    g = data["g"]
    pairs = det.detect([g["rgb"], g["depth"]], 75.0, [], data["sK"])
    assert pairs
    got = det.track(g["depth"], data["sK"], pairs)
    assert [p.getTrackStatus() for _, p in got] == ["tracked"] * len(pairs)
    for (m, p), (m0, _) in zip(got, pairs):
        assert m.similarity == m0.similarity and (m.class_id, m.template_id) == (m0.class_id, m0.template_id)
        assert (m.x, m.y) != (0, 0)
    real = [k for k, (_, p) in enumerate(got) if p.getResidual() >= 0.5]
    assert real
    # a track result starts the next call; a model that slid out of the frame comes back OUTSIDE with its T carried
    again = det.track(g["depth"], data["sK"], got)
    for (_, a), (_, b) in zip(again, got):
        assert a.getTrackStatus() in ("tracked", "outside")
        if a.getTrackStatus() == "outside":
            assert a.getResidual() == -1.0 and same_bits(a.getTransformation(), b.getTransformation())
    dicts = [dict(class_id=m.class_id, template_id=m.template_id, R=p.getR(), t=p.getT()) for m, p in pairs]
    from_dicts = det.track(g["depth"], data["sK"], dicts)
    assert [p.getTrackStatus() for _, p in from_dicts] == ["tracked"] * len(pairs)
    diff = [float(np.abs(from_dicts[k][1].getT() - got[k][1].getT()).max()) for k in real]
    assert max(diff) <= DICT_MM, diff


# ---- sequences --------------------------------------------------------------------------------------------------------
FRAMES = 20
STEP_DEG, STEP_MM = 0.75, 2.5   # the object's motion per frame, about its centroid
# Tracking stays within these of the truth on every frame.  Measured on an H100 80GB HBM3 (700 W): worst 1.541 degrees
# and 0.899 mm point to plane, 2.162 degrees and 0.985 mm point to point; carrying frame 0's T unchanged ends 14.25
# degrees and 47.5 mm off.
BOUNDS = {"point_to_plane": (2.0, 1.5), "point_to_point": (2.75, 1.5)}


def rot_err(Ta, Tb):
    dR = Ta[:3, :3] @ Tb[:3, :3].T
    return float(np.degrees(np.arccos(np.clip((np.trace(dR) - 1) / 2, -1, 1))))


def centroid_err(sc, Ta, Tb):
    return float(np.linalg.norm((Ta[:3, :3] @ sc.cM + Ta[:3, 3]) - (Tb[:3, :3] @ sc.cM + Tb[:3, 3])) * 1000.0)


@pytest.mark.parametrize("estimation", ["point_to_plane", "point_to_point"])
def test_sequence_stays_with_the_truth(nat, data, estimation):
    sc = pso_scenes.Scenes(data["g"])
    yy, xx = np.mgrid[0:sc.rows, 0:sc.cols]
    table = (sc.cM[2] * 1000.0 + 60.0) + 0.12 * (yy - sc.rows / 2) - 0.05 * (xx - sc.cols / 2)
    w = np.radians(np.array([0.6, -0.8, 0.5]))
    w = w / np.linalg.norm(w) * np.radians(STEP_DEG)
    v = np.array([1.0, -0.6, 0.8])
    v = v / np.linalg.norm(v) * STEP_MM / 1000.0
    sK = sc.sK.astype(np.float32)
    T = None
    worst = [0.0, 0.0]
    carried = [0.0, 0.0]
    for k in range(FRAMES):
        Rt = pso_scenes.rodrigues(w * k)
        tt = sc.cM + v * k - Rt @ sc.cM
        truth = np.eye(4)
        truth[:3, :3], truth[:3, 3] = Rt, tt
        scene = pso_scenes.splat(sc.M @ Rt.T + tt, sc.sK, sc.rows, sc.cols, table)
        if T is None:
            T, T0 = truth.copy(), truth.copy()
            continue
        status, Tn, _, _, res, _ = nat.track(scene, sK, [(0, 0, T)], 30, 4, estimation)
        assert status[0] == tm.TRACKED, k
        T = Tn[0]
        worst = [max(worst[0], rot_err(T, truth)), max(worst[1], centroid_err(sc, T, truth))]
        carried = [max(carried[0], rot_err(T0, truth)), max(carried[1], centroid_err(sc, T0, truth))]
    print("%s: tracked worst %.3f deg %.3f mm; carried %.3f deg %.3f mm" % (estimation, *worst, *carried))
    deg, mm = BOUNDS[estimation]
    assert worst[0] <= deg and worst[1] <= mm, worst
    assert carried[0] > deg and carried[1] > mm, carried


# ---- statuses on the device ---------------------------------------------------------------------------------------------
def test_statuses(data):
    # every template with the unshifted render: the largest crop, and so the window cap, is the object's own
    nat = lib.NativeDetector(data["T"], 0)
    nat.load_bank(data["packed"], 4)
    nat.select(None, 0, 1)
    nat.set_template_renders(0, [data["g"]["render"]] * data["G"], data["K"], data["R"], data["t"])
    out, _, _, _, T = detected(nat, data, 75.0)
    depth = data["g"]["depth"].copy()
    c, t = int(out[0]["class_index"]), int(out[0]["template_id"])
    rows, cols = depth.shape
    base = [(c, t, T[0])]
    nat.track(depth, data["sK"], base, 30, 4)
    slot = nat.pose_clouds()[1][0]
    win = slot["window"]
    ref = nat.track(depth, data["sK"], base, 30, 4)
    # OUTSIDE: moved far to the side; NO_DEPTH: the window zeroed; WINDOW: brought along its line of sight to a quarter
    # of its distance, 16 times its image area
    far = shifted(T[0], 10.0)
    centroid = (slot["raw_model"] @ T[0][:3, :3].T + T[0][:3, 3]).mean(0)
    near = shifted(T[0], *(-0.75 * centroid))
    zeroed = depth.copy()
    x, y, w, h = (int(v) for v in win)
    zeroed[y:y + h, x:x + w] = 0
    for objs, d, want in (([(c, t, far)], depth, tm.OUTSIDE), ([(c, t, T[0])], zeroed, tm.NO_DEPTH), ([(c, t, near)], depth, tm.WINDOW)):
        mixed = base + objs + base
        status, Tn, R, tt, res, box = nat.track(d, data["sK"], mixed, 30, 4)
        assert status[1] == want, (status, want)
        assert res[1] == -1.0 and same_bits(Tn[1], np.asarray(objs[0][2])) and np.isnan(R[1]).all() and np.isnan(tt[1]).all()
        if d is depth:
            for k in (0, 2):
                assert status[k] == tm.TRACKED and same_bits(Tn[k], ref[1][0]) and same_bits(res[k], ref[4][0])


# ---- device and host depth ----------------------------------------------------------------------------------------------
def test_device_depth_equals_host_depth(nat, data):
    out, _, _, _, T = detected(nat, data)
    objects = [(int(o["class_index"]), int(o["template_id"]), T[k]) for k, o in enumerate(out)]
    depth = data["g"]["depth"]
    want = nat.track(depth, data["sK"], objects, 30, 4)
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        u16 = torch.from_numpy(depth.view(np.int16)).cuda().view(torch.uint16)
        f32 = (torch.from_numpy(depth.astype(np.float32)).cuda() / 1000.0)
    for t, fmt, scale in ((u16, lib.DEPTH_U16_MM, 1.0), (f32, lib.DEPTH_F32, 1000.0)):
        ptr, pitch, f = lib._depth_plane(t, "depth", torch)
        got = nat.track_device(ptr, pitch, f, scale, depth.shape[0], depth.shape[1], st.cuda_stream, data["sK"], objects, 30, 4)
        for a, b in zip(got, want):
            assert same_bits(a, b)
    # converted as the host converts float depth: round(d * 1000) equals the u16 image here
    assert same_bits(np.round(depth.astype(np.float32) / np.float32(1000.0) * np.float32(1000.0)).astype(np.uint16), depth)


# ---- verification -----------------------------------------------------------------------------------------------------
def test_verification_equals_the_model(data):
    nat = pb.handle(data)
    out, _, _, _, T = detected(nat, data)
    objects = [(int(o["class_index"]), int(o["template_id"]), T[k]) for k, o in enumerate(out)]
    objects.append((objects[0][0], objects[0][1], shifted(T[0], 10.0)))  # OUTSIDE: score -1
    nat.set_pose_verify(True, 10.0)
    status, Tn, *_ = nat.track(data["g"]["depth"], data["sK"], objects, 30, 4)
    score, counts = nat.pose_verify()
    _, slots = nat.pose_clouds()
    assert len(score) == len(objects)
    for i, s in enumerate(slots):
        if not s["posed"]:
            assert score[i] == np.float32(-1.0)
            continue
        ws, wc = pvm.verify(s["raw_model"], Tn[i], data["g"]["depth"], data["sK"], 10.0)
        assert score[i] == ws and (counts[i] == wc).all(), i
    nat.set_pose_verify(False)
