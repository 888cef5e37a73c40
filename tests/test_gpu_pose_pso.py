"""The particle-swarm estimation on the device (include/linemod_b200.h, LM_POSE_PSO): k_pose_pso's objective and its whole
trajectory equal the numpy model of tests/pose_pso_model.py bit for bit, its invariants hold on the recorded driver
frame, and every path that refines poses returns the same poses.

Inputs: crafted clouds and scenes (lm_pose_search_points), the recorded driver frame (tests/golden/driver_trace.npz)
against the allScales bank with the shifted renders of tests/test_gpu_pose_stage.py, and the frames of
tests/test_gpu_peer_batch.py."""
import importlib
import os

import numpy as np
import pytest
import torch

import pose_nms_model
import pose_pso_model as pm
import pose_verify_model as pvm
import test_gpu_peer_batch as pb
import test_gpu_pose_stage as ps

pytestmark = pytest.mark.gpu
lib = importlib.import_module("6dpose_b200._lib")
pr = importlib.import_module("6dpose_b200.pose_refine")
PSO = "pso"
FAST = dict(particles=16, iterations=8)  # the path tests: every survivor searched, few iterations
SK = np.array([[80.0, 0.0, 32.0], [0.0, 80.0, 24.0], [0.0, 0.0, 1.0]], np.float32)


def same_record(got, want):
    for k in ("cost_start", "cost", "best"):
        assert got[k] == want[k], (k, got[k], want[k])
    for k in ("c", "x", "v", "p"):
        assert np.asarray(got[k], np.float64).tobytes() == np.asarray(want[k], np.float64).tobytes(), k
    for k in ("trace", "cost_best"):
        assert np.array_equal(got[k], want[k]), (k, got[k], want[k])


def scene_steps(rows=48, cols=64):
    """A plane at 500 mm with a 20 mm step, a 40 mm step and a hole: costs of every kind."""
    sc = np.full((rows, cols), 500, np.uint16)
    sc[:, 40:] = 520
    sc[:, 52:] = 460
    sc[10:16, 8:20] = 0
    return sc


def cloud(n, seed):
    rng = np.random.default_rng(seed)
    return np.stack([rng.uniform(-0.1, 0.1, n), rng.uniform(-0.08, 0.08, n), rng.uniform(0.47, 0.53, n)], 1)


# ---- 1. the objective ---------------------------------------------------------------------------------------------
def objective_cases():
    cases = {}
    for name, (pts, T, scene, sK, delta, _) in pvm.boundary_cases().items():
        if len(pts) and np.array_equal(T[:3, :3], np.eye(3)):  # a start pose is a translation
            cases[name] = (pts, T[:3, 3].copy(), scene, sK, 20.0)
    # |d| = clamp exactly (z_q = 500 mm) and the clamp one double either side
    for zs in (520, 480):
        for clamp in (20.0, np.nextafter(20.0, 0.0), np.nextafter(20.0, np.inf)):
            cases["d_eq_clamp_%d_%r" % (zs, clamp)] = ([pvm._pt(3, 2)], np.zeros(3), np.full((6, 8), zs, np.uint16), pvm.SK, clamp)
    cases["clamp_zero"] = ([pvm._pt(3, 2), pvm._pt(4, 2)], np.zeros(3), np.full((6, 8), 510, np.uint16), pvm.SK, 0.0)
    cases["cloud"] = (cloud(3000, 1), np.array([0.003, -0.004, 0.01]), scene_steps(), SK, 20.0)
    return cases


def test_objective_equals_the_model():
    for name, (pts, s, scene, sK, clamp) in objective_cases().items():
        pts = np.asarray(pts, np.float64).reshape(-1, 3)
        S = np.eye(4)
        S[:3, 3] = s
        T, rec = lib.pose_search_points(pts, s, scene, sK, particles=1, iterations=0, clamp_mm=clamp)
        assert rec["cost_start"] == pm.cost(pts, S, scene, sK, clamp), name
        assert T.tobytes() == S.tobytes(), name
        # every particle's first evaluation: its personal best after one iteration
        T, rec = lib.pose_search_points(pts, s, scene, sK, job=5, particles=24, iterations=1, clamp_mm=clamp, seed=3)
        for i in range(24):
            assert rec["cost_best"][i] == pm.cost(pts, pm.pose(rec["x"][i], rec["c"], s), scene, sK, clamp), (name, i)


# ---- 2. the trajectory --------------------------------------------------------------------------------------------
TRAJ = [(P, I, 300, (P + I) % 2 * 77, {}) for P in (1, 2, 33, 64, 130) for I in (0, 1, 40)]
TRAJ += [(33, 5, n, seed, {}) for n in (1, 2047, 2048, 2049, 6000) for seed in (0, 77)]
TRAJ += [(16, 6, 500, 0, dict(dt_mm=0.0, dr_deg=0.0)), (16, 6, 500, 0, dict(dt_mm=0.0)), (16, 6, 500, 0, dict(dr_deg=0.0)),
         (64, 40, 800, 5, dict(dt_mm=25.0, dr_deg=45.0, clamp_mm=7.5))]


@pytest.mark.parametrize("P,I,n,seed,extra", TRAJ)
def test_trajectory_equals_the_model(P, I, n, seed, extra):
    pts = cloud(n, n + P)
    s = np.array([0.006, -0.003, 0.012])
    opts = dict(particles=P, iterations=I, seed=seed, **extra)
    T, rec = lib.pose_search_points(pts, s, scene_steps(), SK, job=11, **opts)
    Tm, want = pm.search(pts, s, scene_steps(), SK, job=11, **opts)
    same_record(rec, want)
    assert T.tobytes() == Tm.tobytes()
    assert rec["cost"] <= rec["cost_start"] and np.all(np.diff(rec["trace"]) <= 0)


# ---- 3. invariants on the recorded frame ----------------------------------------------------------------------------
@pytest.fixture(scope="module")
def data():
    return pb.load_data()


def host(data, surv, icp=None, use_scene=False, verify=None, search=None, device=False):
    icp = lib.NativeIcp() if icp is None else icp
    icp.set_use_scene_cloud(use_scene)
    icp.set_verify(verify)
    icp.set_pose_search(**(FAST if search is None else search))
    tid = surv["template_id"].astype(np.int64)
    xy = np.stack([surv["x"], surv["y"]], 1)
    renders = [data["renders"][k] for k in data["which"][tid]]
    args = (data["sK"], data["K"][tid], data["R"][tid], data["t"][tid], xy, 30, PSO)
    if device:
        dev = lib.DeviceDepths(torch.from_numpy(data["g"]["depth"].view(np.int16)).cuda().view(torch.uint16),
                               [torch.from_numpy(r.view(np.int16)).cuda().view(torch.uint16) for r in renders], 1.0, 1.0, None, 0)
        return icp.process_batch_device(dev, *args)
    return icp.process_batch(data["g"]["depth"], renders, *args)


def detector(data, search=None, verify=False):
    nat = pb.handle(data)
    nat.set_pose_search(**(FAST if search is None else search))
    nat.set_pose_verify(verify)
    return nat


@pytest.mark.parametrize("thr", [75.0, 65.0])
def test_invariants_on_the_recorded_frame(data, thr):
    nat = detector(data)
    surv, _ = ps.survivors(nat, data, thr, 0)
    assert len(surv) > 0
    icp = lib.NativeIcp()
    icp.set_capture(True)
    for search in (dict(), dict(particles=1, iterations=40)):
        R, t, res = host(data, surv, icp, search=search)
        posed = np.flatnonzero(res != -1.0)
        assert posed.size > 0
        for i in posed:
            c = icp.capture(int(i))
            rec = c["search"]
            assert rec["cost"] <= rec["cost_start"] and c["fitness"] <= c["rmse"]
            assert np.float32(c["fitness"]) == res[i]
            if search.get("particles") == 1:
                assert c["T"].tobytes() == c["init"].tobytes() and rec["best"] == -1
    # one posed survivor's whole search on its real cloud, default settings, against the model (its job number is its
    # index in the call)
    k = int(posed[0])
    R, t, res = host(data, surv[:k + 1], icp, search=dict())
    assert res[k] != -1.0
    c = icp.capture(k)
    Tm, want = pm.search(c["source"], c["init"][:3, 3], data["g"]["depth"], data["sK"], job=k)
    same_record(c["search"], want)
    assert c["T"].tobytes() == Tm.tobytes()


# ---- 5. every path agrees -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("verify", [False, True])
def test_frame_chain_equals_process_batch(data, verify):
    nat = detector(data, verify=verify)
    g = data["g"]
    for thr, top_k in ((75.0, 3), (65.0, 0)):
        got = nat.match_pose(g["rgb"], g["depth"], None, thr, data["sK"], 0.5, top_k, 30, False, PSO)
        want = host(data, got[0], verify=10.0 if verify else None)
        ps.same_poses(got, want)
        assert (got[3] > 0).any()
        # the ICP's poses differ: the swarm ran
        plane = ps.host_poses(data, got[0], 30, False)
        assert not np.array_equal(want[0], plane[0], equal_nan=True)
        # use_scene_cloud has no effect
        again = nat.match_pose(g["rgb"], g["depth"], None, thr, data["sK"], 0.5, top_k, 30, True, PSO)
        ps.same_poses(again, want)
        # process_batch_device equals process_batch, verification and swarm records included
        icp, hv = lib.NativeIcp(), lib.NativeIcp()
        for h in (icp, hv):
            h.set_capture(True)
        dev = host(data, got[0], icp, verify=10.0 if verify else None, device=True)
        assert [a.tobytes() for a in dev] == [a.tobytes() for a in want]
        staged = host(data, got[0], hv, verify=10.0 if verify else None)
        assert [a.tobytes() for a in staged] == [a.tobytes() for a in want]
        for i in np.flatnonzero(want[2] != -1.0):
            same_record(icp.capture(int(i))["search"], hv.capture(int(i))["search"])
        if verify:
            assert [a.tobytes() for a in icp.verify()] == [a.tobytes() for a in hv.verify()]
            assert [a.tobytes() for a in nat.pose_verify()] == [a.tobytes() for a in hv.verify()]
        # the pose NMS on top equals the model on those poses; 4 launches for the pose stage
        nat.upload_images(g["rgb"], g["depth"], None)
        nat.enqueue(thr)
        nat.enqueue_post(0.5, top_k)
        before = nat.launch_count()
        nat.enqueue_pose(data["sK"], 30, False, PSO)
        assert nat.launch_count() - before == (5 if verify else 4)
        nat.enqueue_pose_nms(40.0)
        out, R, t, res, counts = nat.complete_detect()
        ws, wR, wt, wr = pose_nms_model.detect(got[0], want[0], want[1], want[2], 40.0)
        assert np.array_equal(out, ws) and np.array_equal(res, wr)
        assert np.array_equal(R, wR, equal_nan=True) and np.array_equal(t, wt, equal_nan=True)


def test_refine_matches_equals_process_batch(data):
    nat = detector(data)
    surv, _ = ps.survivors(nat, data, 75.0, 3)
    tid = surv["template_id"].astype(np.int64)

    class M:
        def __init__(self, m):
            self.x, self.y = int(m["x"]), int(m["y"])
    got = pr.refine_matches(data["g"]["depth"], data["sK"], [M(m) for m in surv], [data["renders"][k] for k in data["which"][tid]],
                            data["K"][tid], data["R"][tid], data["t"][tid], estimation=PSO, pose_search=FAST)
    R, t, res = host(data, surv)
    for i, p in enumerate(got):
        assert np.float32(p.getResidual()) == res[i]
        if res[i] != -1.0:
            assert p.getR().tobytes() == R[i].tobytes() and p.getT().reshape(3).tobytes() == t[i].tobytes()


@pytest.mark.parametrize("pose_nms", [False, True])
def test_batch_equals_single_frames(data, pose_nms):
    nat = detector(data, verify=pose_nms)
    single = detector(data, verify=pose_nms)
    names = ["recorded", "rolled", "mirrored", "blank", "masked"]
    K = pb.scene_ks(data, len(names))
    for top_k, thr in ((0, 75.0), (3, 65.0)):
        got = nat.detect_batch(*pb.batch_args(data, names, K, thr, top_k, False, pose_nms), estimation=PSO)
        for f, name in enumerate(names):
            rgb, depth, masks = data["frames"][name]
            single.upload_images(rgb, depth, masks)
            single.enqueue(thr)
            single.enqueue_post(0.5, top_k)
            single.enqueue_pose(K[f], 30, False, PSO)
            if pose_nms:
                single.enqueue_pose_nms(40.0)
                want = single.complete_detect()
            else:
                want = single.complete_pose()
            out, R, t, res = got[f][:4]
            assert np.array_equal(out, want[0]) and np.array_equal(res, want[3])
            assert np.array_equal(R, want[1], equal_nan=True) and np.array_equal(t, want[2], equal_nan=True)


def test_sharded_unshared_batch_equals_the_unconnected_batch(data):
    names = ["recorded", "rolled", "mirrored"]
    K = pb.scene_ks(data, len(names))
    want = {}
    for verify in (False, True):
        ref = detector(data, verify=verify)
        frames = ref.detect_batch(*pb.batch_args(data, names, K, 65.0, 0, False, True), estimation=PSO)
        want[verify] = (frames, ref.batch_counts.copy()), ref.pose_verify() if verify else None
    for world in (2, 3):
        dets = pb.connected(data, [0] * world, share=False)
        try:
            for verify in (False, True):
                for d in dets:
                    d.set_pose_search(**FAST)
                    d.set_pose_verify(verify)

                def one(r, d):
                    frames = d.peer_detect_batch(*pb.batch_args(data, names, K, 65.0, 0, False, True), estimation=PSO)
                    return (frames, d.batch_counts.copy()), d.pose_verify() if verify else None
                for g, ver in pb.on_every_rank(dets, one):
                    pb.same(g, want[verify][0])
                    if verify:
                        assert [a.tobytes() for a in ver] == [a.tobytes() for a in want[verify][1]]
            for d in dets:
                d.set_pose_verify(False)
            # the shared stage refuses the swarm, before any device work
            for d in dets:
                d.peer_share_pose(True)
                with pytest.raises(lib.LinemodLibraryError, match="error -3"):
                    d.peer_detect_batch(*pb.batch_args(data, names, K, 65.0, 0, False, True), estimation=PSO)
                d.set_pose_estimation(PSO)
                assert lib.load().lm_enqueue_pose(d._h, data["sK"].ctypes.data_as(lib.ctypes.POINTER(lib.ctypes.c_float)), 30, 0) \
                    == lib.LM_E_STATE
                assert "LM_POSE_PSO" in lib.load().lm_last_error().decode()
                d.set_pose_estimation("point_to_plane")
                d.peer_share_pose(False)
        finally:
            pb.close(dets)


def test_frame_keeps_its_search_settings(data):
    g = data["g"]
    nat = detector(data)
    want = nat.match_pose(g["rgb"], g["depth"], None, 65.0, data["sK"], 0.5, 0, 30, False, PSO)
    nat.upload_images(g["rgb"], g["depth"], None)
    nat.enqueue(65.0)
    nat.enqueue_post(0.5, 0)
    nat.enqueue_pose(data["sK"], 30, False, PSO)
    nat.set_pose_search(particles=3, iterations=2, seed=9)
    nat.set_pose_estimation("point_to_point")
    ps.same_poses(nat.complete_pose(), want[1:4])


# ---- 4. recovery of a known pose ------------------------------------------------------------------------------------
# The default search on the synthetic scenes of tests/pso_scenes.py, the same 100 seeded cases per level as
# tools/pso_probe.py, measured on an H100 (DESIGN.md section 9):
#   U{10,10}  every case within 0.9 degrees and 0.8 mm: bound 1.5 degrees and 1.5 mm for every case.
#   U{20,20}  90th percentiles 1.14 degrees and 0.76 mm, 94 of 100 cases within 2 degrees and 1.5 mm at once, the worst
#             48.9 degrees and 72.4 mm (the search settles in another minimum of the objective; every setting measured has
#             such cases): bound 2 degrees and 1.5 mm for at least 90 cases, 50 degrees and 75 mm for every case.
@pytest.mark.parametrize("a,deg,mm,at_least,deg_all,mm_all", [(10, 1.5, 1.5, 100, 1.5, 1.5), (20, 2.0, 1.5, 90, 50.0, 75.0)])
def test_recovery_on_synthetic_scenes(data, a, deg, mm, at_least, deg_all, mm_all):
    import pso_scenes
    sc = pso_scenes.Scenes(data["g"])
    rng = np.random.default_rng(1000 + a)  # the probe's seed for U{a,a}
    icp = lib.NativeIcp()
    icp.set_estimation(PSO)
    icp.set_pose_search()
    close = 0
    for k in range(100):
        scene, xy, T = sc.case(a, rng)
        rot, cen = sc.errors(T, *sc.refine(icp, scene, xy))
        assert rot <= deg_all and cen <= mm_all, (k, rot, cen)
        close += rot <= deg and cen <= mm
    assert close >= at_least, close


# ---- 6. the existing estimations are untouched ----------------------------------------------------------------------
@pytest.fixture(scope="module")
def parent_poses():
    return np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "existing_modes_poses.npz"))


@pytest.mark.parametrize("est", ["point_to_plane", "point_to_point"])
@pytest.mark.parametrize("use_scene", [False, True])
def test_existing_modes_equal_the_recorded_build(data, parent_poses, est, use_scene):
    """The default and point-to-point poses are those the build before LM_POSE_PSO computed
    (tests/golden/make_existing_modes_golden.py), bit for bit, on every case of tests/icp_clouds.py and the driver frame."""
    import icp_clouds
    key = "%s_%d" % (est, use_scene)
    icp = lib.NativeIcp()
    icp.set_use_scene_cloud(use_scene)
    for i, c in enumerate(icp_clouds.all_cases()):
        Ro, to, res = icp.process_batch(c.scene, [c.model], c.K, c.K[None], c.R[None], c.t[None], [c.xy], 30, est)
        assert Ro[0].tobytes() == parent_poses["icp_%s_R" % key][i].tobytes(), c.name
        assert to[0].tobytes() == parent_poses["icp_%s_t" % key][i].tobytes(), c.name
        assert res[0].tobytes() == parent_poses["icp_%s_res" % key][i].tobytes(), c.name
    nat = pb.handle(data)
    g = data["g"]
    for thr in (75, 65):
        got = nat.match_pose(g["rgb"], g["depth"], None, float(thr), data["sK"], 0.5, 0, 30, use_scene, est)
        k = "frame_%s_%d" % (key, thr)
        for a, name in zip(got[:4], ("surv", "R", "t", "res")):
            assert a.tobytes() == parent_poses[k + "_" + name].tobytes(), (k, name)


# ---- the public surface ---------------------------------------------------------------------------------------------
def test_detector_detect_equals_the_native_chain(data, tmp_path):
    pkg = importlib.import_module("6dpose_b200")
    bk = importlib.import_module("6dpose_b200.bank")
    g, packed = data["g"], data["packed"]
    bank = bk.TemplateBank()
    bank.classes["06_template"] = bk.PackedPyramids(packed["tmeta"], packed["feats"], 2)
    bank.write_packed("06_template", str(tmp_path / "06_template.lmb"), 2)
    det = pkg.Detector(int(g["num_features"]), data["T"])
    det.readClasses(["06_template"], str(tmp_path / "%s.lmb"))
    det.setTemplateRenders({"06_template": ((data["renders"][k] for k in data["which"]), data["K"], data["R"], data["t"])})
    det.setPoseSearch(**FAST)
    nat = detector(data)
    for verify in (None, 10.0):
        det.setPoseVerification(verify)
        nat.set_pose_verify(verify is not None, 10.0)
        pairs = det.detect([g["rgb"], g["depth"]], 65.0, ["06_template"], data["sK"], estimation=PSO)
        out, R, t, res, _ = nat.detect(g["rgb"], g["depth"], None, 65.0, data["sK"], 0.5, 0, 30, False, 40.0, PSO)
        assert len(pairs) == len(out) > 0
        score = nat.pose_verify()[0] if verify else None
        for k, (m, p) in enumerate(pairs):
            assert (m.x, m.y, m.template_id) == (int(out[k]["x"]), int(out[k]["y"]), int(out[k]["template_id"]))
            assert np.float32(p.getResidual()) == res[k]
            assert p.getR().tobytes() == R[k].tobytes() and p.getT().reshape(3).tobytes() == t[k].tobytes()
            if verify:
                assert np.float32(p.getScore()) == score[k]
