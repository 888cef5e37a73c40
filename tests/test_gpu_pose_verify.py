"""Pose verification on the device (include/linemod_b200.h, lm_set_pose_verify): the counts and score of every refined
pose equal the numpy model of tests/pose_verify_model.py, through every path that refines poses, and turning it on
changes no match, pose or residual -- one launch more per chunk, nothing else.

Inputs: the boundary cases of pose_verify_model.py (lm_pose_verify_points), the recorded ICP case
(tests/golden/icp_case1.npz) through the lm_icp handle, and the recorded driver frame (tests/golden/driver_trace.npz)
against the allScales bank with the shifted renders of tests/test_gpu_pose_stage.py."""
import importlib
import os

import numpy as np
import pytest
import torch

import pose_nms_model
import pose_verify_model as pvm

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
lib = importlib.import_module("6dpose_b200._lib")
pr = importlib.import_module("6dpose_b200.pose_refine")

SHIFTS = [(0, 0), (-68, -19), (-180, 57), (3, -2), (-2, 4)]
MODES = [(e, s) for e in ("point_to_plane", "point_to_point") for s in (False, True)]
ICP_SCENES = ["scene_a", "scene_b", "scene_edge", "shift_0", "shift_1", "shift_2", "shift_3"]


def same_verify(got, want):
    gs, gc = got
    ws, wc = want
    assert np.asarray(gc).tolist() == np.asarray(wc).tolist()
    assert np.asarray(gs, np.float32).tobytes() == np.asarray(ws, np.float32).tobytes(), (gs, ws)


# ---- 1. the device routine on caller arrays -----------------------------------------------------------------------
def test_points_equal_the_model_on_every_boundary_case():
    for name, (pts, T, scene, sK, delta, want) in pvm.boundary_cases().items():
        s, c = lib.pose_verify_points(pts, T, scene, sK, delta)
        same_verify((s, c), pvm.verify(pts, T, scene, sK, delta))
        for k in range(len(pts)):  # one point at a time: its class
            s, c = lib.pose_verify_points(pts[k:k + 1], T, scene, sK, delta)
            assert c[1 + want[k]] == 1, (name, k, c)


# ---- 2. the lm_icp handle on the recorded ICP case ----------------------------------------------------------------
@pytest.fixture(scope="module")
def gold():
    return np.load(os.path.join(GOLD, "icp_case1.npz"))


def icp_scene(gold, name):
    return gold["scene"] if name.startswith("scene") else gold["scene_" + name]


def icp_call(icp, gold, scene, xy, device=False, verify=True):
    args = (gold["K"], gold["K"][None], gold["R"][None], gold["t"].reshape(1, 3), [xy], 30)
    if device:
        dev = lib.DeviceDepths(torch.from_numpy(scene.view(np.int16)).cuda().view(torch.uint16),
                               [torch.from_numpy(gold["model"].view(np.int16)).cuda().view(torch.uint16)], 1.0, 1.0, None, 0)
        out = icp.process_batch_device(dev, *args)
    else:
        out = icp.process_batch(scene, [gold["model"]], *args)
    return out, icp.verify() if verify else None


@pytest.mark.parametrize("mode", MODES)
def test_icp_calls_equal_the_model_through_the_pose_stage(gold, mode):
    icp = lib.NativeIcp(0)
    icp.set_estimation(mode[0])
    icp.set_use_scene_cloud(mode[1])
    pts = pvm.model_cloud(gold["model"], gold["K"])
    for name in ICP_SCENES:
        scene = icp_scene(gold, name)
        for moved in (0, 30):
            sc = np.where(scene > 0, scene + moved, 0).astype(np.uint16)
            xy = [int(v) for v in gold["xy_" + name]]
            icp.set_capture(False)
            icp.set_verify(None)
            plain = icp_call(icp, gold, sc, xy, verify=False)[0]
            icp.set_capture(True)
            icp.set_verify(10.0)
            n0 = icp.launch_count()
            out, (score, counts) = icp_call(icp, gold, sc, xy)
            assert [a.tobytes() for a in out] == [a.tobytes() for a in plain]  # verification changes no pose
            if out[2][0] == -1.0:  # early return
                assert name == "scene_edge"
                same_verify((score[0], counts[0]), pvm.no_pose())
            else:
                T = icp.capture(0)["T"]
                same_verify((score[0], counts[0]), pvm.verify(pts, T, sc, gold["K"], 10.0))
                assert counts[0][0] == len(pts)
                assert icp.launch_count() - n0 == (9 if mode[0] == "point_to_plane" else 8)
            icp.set_capture(False)
            dev_out, dev_ver = icp_call(icp, gold, sc, xy, device=True)
            assert [a.tobytes() for a in dev_out] == [a.tobytes() for a in out]
            same_verify((dev_ver[0][0], dev_ver[1][0]), (score[0], counts[0]))


def test_own_scene_scores_higher_than_the_scene_moved_back(gold):
    """Sanity only, as an inequality: a recorded pose agrees better with its own scene than with that scene 30 mm deeper."""
    icp = lib.NativeIcp(0)
    pts = pvm.model_cloud(gold["model"], gold["K"])
    icp.set_capture(True)
    for name in ("scene_a", "shift_0"):
        scene = icp_scene(gold, name)
        xy = [int(v) for v in gold["xy_" + name]]
        icp.process_batch(scene, [gold["model"]], gold["K"], gold["K"][None], gold["R"][None], gold["t"].reshape(1, 3), [xy], 30)
        T = icp.capture(0)["T"]
        own = pvm.verify(pts, T, scene, gold["K"], 10.0)[0]
        back = pvm.verify(pts, T, np.where(scene > 0, scene + 30, 0).astype(np.uint16), gold["K"], 10.0)[0]
        s_own = lib.pose_verify_points(pts, T, scene, gold["K"], 10.0)[0]
        assert s_own == own and own > back, (name, own, back)


# ---- 3-5. the detector's pose stage ------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def data():
    g = np.load(os.path.join(GOLD, "driver_trace.npz"))
    b = np.load(os.path.join(GOLD, "bank_allScales_full.npz"))
    packed = dict(class_begin=b["class_begin"], tmeta=b["tmeta"].astype(np.int32), feats=b["feats"].astype(np.int32))
    G = packed["tmeta"].shape[0]
    renders = [np.ascontiguousarray(np.roll(np.roll(g["render"], dy, 0), dx, 1)) for dy, dx in SHIFTS]
    K = np.repeat(g["rf0_modelK"][None], G, 0).astype(np.float32)
    R = np.repeat(g["rf0_modelR"][None], G, 0).astype(np.float32)
    t = np.repeat(g["rf0_modelT"].reshape(1, 3), G, 0).astype(np.float32)
    t[:, 0] += (np.arange(G) % 7) - 3.0
    t[:, 2] += np.arange(G) % 11
    return dict(g=g, packed=packed, T=b["T"].tolist(), G=G, renders=renders, which=np.arange(G) % len(renders), K=K, R=R, t=t,
                sK=g["rf0_sceneK"].astype(np.float32))


@pytest.fixture(scope="module")
def nat(data):
    n = lib.NativeDetector(data["T"], 0)
    n.load_bank(data["packed"], 4)
    n.select(None, 0, 1)
    n.set_template_renders(0, [data["renders"][k] for k in data["which"]], data["K"], data["R"], data["t"])
    return n


def cuda_frame(g):
    return torch.from_numpy(g["rgb"]).cuda(), torch.from_numpy(g["depth"].view(np.int16)).cuda().view(torch.uint16)


def host_verify(data, surv, use_scene, estimation="point_to_plane"):
    """refine_matches' lm_icp path on the same survivors: poses and verification."""
    icp = lib.NativeIcp(0)
    icp.set_use_scene_cloud(use_scene)
    icp.set_verify(10.0)
    tid = surv["template_id"].astype(np.int64)
    xy = np.stack([surv["x"], surv["y"]], 1)
    out = icp.process_batch(data["g"]["depth"], [data["renders"][k] for k in data["which"][tid]], data["sK"], data["K"][tid],
                            data["R"][tid], data["t"][tid], xy, 30, estimation)
    return out, icp.verify()


@pytest.mark.parametrize("use_scene", [False, True])
def test_every_path_gives_the_same_scores(data, nat, use_scene):
    g = data["g"]
    thr = 65.0
    nat.set_pose_verify(True, 10.0)
    single = nat.match_pose(g["rgb"], g["depth"], None, thr, data["sK"], 0.5, 0, 30, use_scene)
    ver = nat.pose_verify()
    surv = single[0]
    assert len(surv) > 16 and (ver[0] > 0).any() and (ver[0] == -1).any() == (single[3] == -1).any()
    # the lm_icp path on the same survivors
    (R, t, res), hv = host_verify(data, surv, use_scene)
    assert res.tobytes() == single[3].tobytes()
    same_verify(hv, ver)
    # CUDA tensor frame
    rgb_t, depth_t = cuda_frame(g)
    dev = nat.match_pose(rgb_t, depth_t, None, thr, data["sK"], 0.5, 0, 30, use_scene)
    assert dev[0].tobytes() == surv.tobytes()
    same_verify(nat.pose_verify(), ver)
    # a batch of the frame, the frame rolled off and the frame again: frames 0 and 2 give the single frame's
    rolled = np.ascontiguousarray(np.roll(g["depth"], 5, 1))
    rgb = np.stack([g["rgb"], g["rgb"], g["rgb"]])
    depth = np.stack([g["depth"], rolled, g["depth"]])
    K = np.repeat(data["sK"][None], 3, 0)
    got = nat.detect_batch(rgb, depth, None, thr, K, 0.5, 0, 30, use_scene, pose_nms=False)
    bs, bc = nat.pose_verify()
    n0, n1 = len(got[0][0]), len(got[1][0])
    assert n0 == len(surv) and len(bs) == n0 + n1 + len(got[2][0])
    same_verify((bs[:n0], bc[:n0]), ver)
    same_verify((bs[n0 + n1:], bc[n0 + n1:]), ver)
    # the batch of device frames
    batch = lib.DeviceBatch([lib.DeviceFrame(*cuda_frame(g), None, 1.0, None, 0)] * 2)
    got = nat.detect_batch_device(batch, thr, K[:2], 0.5, 0, 30, use_scene, pose_nms=False)
    bs, bc = nat.pose_verify()
    same_verify((bs[:n0], bc[:n0]), ver)
    same_verify((bs[n0:], bc[n0:]), ver)
    # the pose NMS passes each kept pose's verification through
    kept = nat.detect(g["rgb"], g["depth"], None, thr, data["sK"], 0.5, 0, 30, use_scene, 40.0)
    ks, kc = nat.pose_verify()
    idx = [int(np.flatnonzero((surv["x"] == m["x"]) & (surv["y"] == m["y"]) & (surv["template_id"] == m["template_id"]))[0])
           for m in kept[0]]
    same_verify((ks, kc), (ver[0][idx], ver[1][idx]))
    # a peer exchange of one rank, its pose stage unshared and shared: the same scores
    one = lib.NativeDetector(data["T"], 0)
    try:
        one.load_bank(data["packed"], 4)
        one.select(None, 0, 1)
        one.set_template_renders(0, [data["renders"][k] for k in data["which"]], data["K"], data["R"], data["t"])
        one.set_pose_verify(True, 10.0)
        one.detect_batch(rgb[:1], depth[:1], None, thr, K[:1], 0.5, 0, 30, use_scene, pose_nms=False)  # grows every buffer
        one.peer_export(1, 1 << 17)
        one.peer_connect_local(0, 1, [one.peer_base()])
        one.prepare()
        one.match_pose(g["rgb"], g["depth"], None, thr, data["sK"], 0.5, 0, 30, use_scene)  # a connected frame first
        for share in (False, True):
            one.peer_share_pose(share)
            got = one.peer_detect_batch(rgb[:1], depth[:1], None, thr, K[:1], 0.5, 0, 30, use_scene, pose_nms=False)
            assert got[0][0].tobytes() == surv.tobytes() and got[0][3].tobytes() == single[3].tobytes()
            same_verify(one.pose_verify(), ver)
            got = one.match_pose(g["rgb"], g["depth"], None, thr, data["sK"], 0.5, 0, 30, use_scene)
            assert got[3].tobytes() == single[3].tobytes()
            same_verify(one.pose_verify(), ver)
            got = one.detect(g["rgb"], g["depth"], None, thr, data["sK"], 0.5, 0, 30, use_scene, 40.0)
            assert got[0].tobytes() == kept[0].tobytes()
            same_verify(one.pose_verify(), (ks, kc))
    finally:
        one.peer_disconnect()
        one.close()


@pytest.mark.parametrize("world", [2, 3])
def test_shared_pose_stage_gives_the_unshared_scores(data, nat, world):
    """The pose stage divided over `world` ranks on one device: each rank verifies the survivors it refines, and every rank
    returns the unshared scores and counts -- single frames, the pose NMS, and a batch of two chunks."""
    import test_gpu_peer_batch as pb
    pdata = pb.load_data()
    names = ["recorded", "rolled", "recorded", "mirrored"]
    K = pb.scene_ks(pdata, len(names))
    nat.set_pose_verify(True, 10.0)
    want = {}
    for nms in (False, True):
        frames = nat.detect_batch(*pb.batch_args(pdata, names, K, 65.0, 0, False, nms))
        want[nms] = (frames, nat.pose_verify())
    assert sum(len(f[0]) for f in want[False][0]) > 1024  # two chunks, so both slots of the pose area serve one call
    dets = [pb.handle(pdata, 0, (r, world)) for r in range(world)]
    try:
        for d in dets:  # verifying from the start: every buffer is grown before the exchange is wired
            d.set_pose_verify(True, 10.0)
            d.detect_batch(*pb.batch_args(pdata, pb.FRAMES, pb.scene_ks(pdata, 5), 62.0, 0, True, True))
        for d in dets:
            d.peer_export(world, pb.CAPACITY)
        bases = [d.peer_base() for d in dets]
        for r, d in enumerate(dets):
            d.peer_connect_local(r, world, bases)
        for d in dets:
            d.prepare()
        pb.frame(dets, pdata, 75.0, 0, False, False)
        for share in (True, False):
            for d in dets:
                d.peer_share_pose(share)
            for nms in (False, True):
                for frames, _ in pb.peer_batch(dets, pb.batch_args(pdata, names, K, 65.0, 0, False, nms)):
                    for f, w in zip(frames, want[nms][0]):
                        assert f[0].tobytes() == w[0].tobytes() and f[3].tobytes() == w[3].tobytes()
                for d in dets:
                    same_verify(d.pose_verify(), want[nms][1])
                # a single frame on every rank
                nat.match_pose(pdata["g"]["rgb"], pdata["g"]["depth"], None, 65.0, pdata["sK"], 0.5, 0, 30, False)
                one = nat.pose_verify()
                if nms:
                    nat.detect(pdata["g"]["rgb"], pdata["g"]["depth"], None, 65.0, pdata["sK"], 0.5, 0, 30, False, 40.0)
                    one = nat.pose_verify()
                pb.frame(dets, pdata, 65.0, 0, False, nms)
                for d in dets:
                    same_verify(d.pose_verify(), one)
                if share:
                    assert sum(d.pose_stats()[1] for d in dets) == dets[0].pose_stats()[0]  # each rank verified its share
    finally:
        pb.close(dets)


@pytest.mark.parametrize("estimation", ["point_to_plane", "point_to_point"])
def test_results_and_launches_do_not_change(data, nat, estimation):
    g = data["g"]
    for thr, top_k in ((75.0, 3), (65.0, 0)):
        for nms in (False, True):
            runs = {}
            for on in (False, True):
                nat.set_pose_verify(on, 10.0)
                nat.set_pose_estimation(estimation)
                l0 = nat.launch_count()
                if nms:
                    out = nat.detect(g["rgb"], g["depth"], None, thr, data["sK"], 0.5, top_k, 30, False, 40.0, estimation)
                else:
                    out = nat.match_pose(g["rgb"], g["depth"], None, thr, data["sK"], 0.5, top_k, 30, False, estimation)
                runs[on] = (out, nat.launch_count() - l0, nat.pose_stats()[2])
            (off, l_off, p_off), (on_, l_on, p_on) = runs[False], runs[True]
            for a, b in zip(off[:4], on_[:4]):
                assert a.tobytes() == b.tobytes()
            assert l_on == l_off + 1 and p_on == p_off + 1, (l_off, l_on, p_off, p_on)
    # a batch of two chunks: one launch more per chunk
    nat.set_pose_verify(False)
    n1 = len(nat.match_pose(g["rgb"], g["depth"], None, 62.0, data["sK"], 0.5, 0, 30, False, estimation)[0])
    nf = 1024 // max(n1, 1) + 1
    rgb = np.stack([g["rgb"]] * nf)
    depth = np.stack([g["depth"]] * nf)
    K = np.repeat(data["sK"][None], nf, 0)
    runs = {}
    for on in (False, True):
        nat.set_pose_verify(on, 10.0)
        l0 = nat.launch_count()
        got = nat.detect_batch(rgb, depth, None, 62.0, K, 0.5, 0, 30, False, pose_nms=False, estimation=estimation)
        runs[on] = (got, nat.launch_count() - l0)
    S = sum(len(f[0]) for f in runs[True][0])
    assert S > 1024, S
    assert runs[True][1] == runs[False][1] + (S + 1023) // 1024
    for fa, fb in zip(runs[False][0], runs[True][0]):
        for a, b in zip(fa[:4], fb[:4]):
            assert a.tobytes() == b.tobytes()
    assert len(nat.pose_verify()[0]) == S


def test_rank_by_score_and_min_score_equal_the_pose_nms_model(data, nat):
    g = data["g"]
    thr, tthr = 65.0, 40.0
    # zero-anchor renders for every third template: NaN poses among the survivors
    nan_render = data["renders"][0].copy()
    nan_render[nan_render.shape[0] // 2, nan_render.shape[1] // 2] = 0
    renders = [nan_render if k % 3 == 0 else data["renders"][data["which"][k]] for k in range(data["G"])]
    nat.set_template_renders(0, renders, data["K"], data["R"], data["t"])
    try:
        nat.set_pose_verify(True, 10.0)
        surv, R, t, res, _ = nat.match_pose(g["rgb"], g["depth"], None, thr, data["sK"], 0.5, 0, 30, False)
        score, counts = nat.pose_verify()
        posed = res != np.float32(-1.0)
        assert np.isnan(t[posed]).any() and (score[posed] == 0).any()
        for rank_by, key in (("fitness", -res.astype(np.float64)), ("score", score.astype(np.float64))):
            for lo in (-np.inf, 0.0, 0.3, float(np.median(score[posed])), 2.0):
                cand = np.flatnonzero(posed & ~(score.astype(np.float64) < lo))
                keep = cand[np.asarray(pose_nms_model.nms(t[cand], key[cand], tthr), np.int64)] if cand.size else cand
                nat.set_pose_verify(True, 10.0, lib.VERIFY_RANKS[rank_by], lo)
                out, Rk, tk, rk, cnt = nat.detect(g["rgb"], g["depth"], None, thr, data["sK"], 0.5, 0, 30, False, tthr)
                assert out.tobytes() == surv[keep].tobytes(), (rank_by, lo)
                assert Rk.tobytes() == R[keep].tobytes() and rk.tobytes() == res[keep].tobytes()
                assert cnt["posed"] == int(posed.sum())
                same_verify(nat.pose_verify(), (score[keep], counts[keep]))
    finally:
        nat.set_pose_verify(False)
        nat.set_template_renders(0, [data["renders"][k] for k in data["which"]], data["K"], data["R"], data["t"])


def test_python_surface(data, tmp_path):
    pkg = importlib.import_module("6dpose_b200")
    g = data["g"]
    # refine_matches and poseRefine.process carry the lm_icp handle's results
    icp = lib.NativeIcp(0)
    icp.set_verify(10.0)
    gold = np.load(os.path.join(GOLD, "icp_case1.npz"))
    xy = [int(v) for v in gold["xy_scene_a"]]
    icp.process_batch(gold["scene"], [gold["model"]], gold["K"], gold["K"][None], gold["R"][None], gold["t"].reshape(1, 3), [xy], 30)
    ws, wc = icp.verify()
    p = pr.poseRefine()
    p.process(gold["scene"], gold["model"], gold["K"], gold["K"], gold["R"], gold["t"], xy[0], xy[1], verify_mm=10.0)
    assert p.getScore() == float(ws[0]) and list(p.getVerification().values()) == wc[0].tolist()
    p.process(gold["scene"], gold["model"], gold["K"], gold["K"], gold["R"], gold["t"], xy[0], xy[1])
    assert p.getScore() is None and p.getVerification() is None

    class M:
        x, y = xy

    got = pr.refine_matches(gold["scene"], gold["K"], [M(), M()], [gold["model"]] * 2, [gold["K"]] * 2, [gold["R"]] * 2,
                            [gold["t"]] * 2, verify_mm=10.0)
    assert [q.getScore() for q in got] == [float(ws[0])] * 2
    assert all(q.getVerification()["n_model"] == int(wc[0][0]) for q in got)
