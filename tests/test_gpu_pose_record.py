"""What the pose stage keeps of the run it last finished (6dpose_b200/csrc/lm_pose.h): on one handle, what
lm_pose_verify, lm_pose_transforms and lm_track_templates return or raise after each kind of run -- a frame with and
without the pose NMS, a batch with and without it, a track run with view following on, a frame enqueued but not
finished, and a finish that fails with LM_E_CAPACITY -- and what lm_icp_verify returns after lm_icp_process_batch calls
with and without verification, with every hypothesis returning early, and without hypotheses.  Every transformation
composes, bit for bit, to the R and t its run returned, with the render of the template the getters name; a kept pose's
(detect, detect_batch) is that of the same survivor without the pose NMS (match_refine, match_refine_batch).

Data: the allScales bank and driver frames of tests/test_gpu_peer_batch.py with every template's R_b a seeded rotation
(as tests/test_gpu_track_views.py), so that turned objects switch templates, and the recorded ICP case
(tests/golden/icp_case1.npz)."""
import ctypes
import importlib
import os

import numpy as np
import pytest

import test_gpu_peer_batch as pb
import test_gpu_track as gt
import test_gpu_track_views as tv
import track_model as tm

pytestmark = pytest.mark.gpu
lib = importlib.import_module("6dpose_b200._lib")
same_bits = gt.same_bits
THR = 65.0
TRACKED = 0  # LM_TRACK_TRACKED


@pytest.fixture(scope="module")
def data():
    d = pb.load_data()
    d["R"] = tv.random_rotations(d["G"], np.random.default_rng(3)).astype(np.float32)
    return d


def composes(data, T, cls, tpl, R, t):
    """T of entry k composes to R[k], t[k] with the render of template tpl[k] of class cls[k]."""
    cb = np.asarray(data["packed"]["class_begin"])
    for k in range(len(T)):
        g = int(cb[cls[k]]) + int(tpl[k])
        Rk, tk = tm.compose(T[k], data["R"][g], data["t"][g])
        assert same_bits(Rk, R[k]) and same_bits(tk, t[k]), k


def answers(nat):
    """verify, T and tpl: each getter's result, or the error code it returns."""
    got = {}
    for name, fn, nulls, get in (("verify", nat._L.lm_pose_verify, 2, nat.pose_verify), ("T", nat._L.lm_pose_transforms, 1, nat.pose_transforms),
                                 ("tpl", nat._L.lm_track_templates, 1, nat.track_templates)):
        n = ctypes.c_int64()
        rc = fn(nat._h, *([None] * nulls), 0, ctypes.byref(n))
        got[name] = get() if rc in (lib.LM_OK, lib.LM_E_CAPACITY) else rc
    return got


def same_verify(got, want):
    assert same_bits(got[0], want[0]) and same_bits(got[1], want[1])


def survivor_of(surv, m):
    return int(np.flatnonzero((surv["x"] == m["x"]) & (surv["y"] == m["y"]) & (surv["class_index"] == m["class_index"]) &
                              (surv["template_id"] == m["template_id"]))[0])


def expect_poses(got, data, surv, R, t, res, verified):
    """A frame or batch without the pose NMS (survivors surv, outputs R, t, res): every entry's T, NaN without a pose."""
    n = len(surv)
    assert got["T"].shape == (n, 4, 4)
    assert np.isnan(got["T"][res == -1]).all()
    posed = res != -1
    composes(data, got["T"][posed], surv["class_index"][posed], surv["template_id"][posed], R[posed], t[posed])
    if verified:
        assert len(got["verify"][0]) == n
    else:
        assert got["verify"] == lib.LM_E_STATE
    assert got["tpl"] == lib.LM_E_STATE


def expect_kept(got, kept, want, idx):
    """A frame with the pose NMS: the kept entries of want (the frame without it) at the survivor indices idx."""
    assert len(idx) == len(kept) > 0
    assert same_bits(got["T"], want["T"][idx])
    same_verify(got["verify"], (want["verify"][0][idx], want["verify"][1][idx]))
    assert got["tpl"] == lib.LM_E_STATE


def test_getters_after_every_kind_of_run(data):
    g = data["g"]
    sK = data["sK"]
    nat = pb.handle(data)
    try:
        # a frame without verification, then with it
        single = nat.match_pose(g["rgb"], g["depth"], None, THR, sK, 0.5, 0, 30, False)
        surv, res = single[0], single[3]
        assert len(surv) > 16 and (res == -1).any()
        expect_poses(answers(nat), data, *single[:4], False)
        nat.set_pose_verify(True, 10.0)
        single = nat.match_pose(g["rgb"], g["depth"], None, THR, sK, 0.5, 0, 30, False)
        assert same_bits(single[3], res)
        frame = answers(nat)
        expect_poses(frame, data, *single[:4], True)

        # the frame with the pose NMS: each kept pose is its survivor's
        kept, kR, kt = nat.detect(g["rgb"], g["depth"], None, THR, sK, 0.5, 0, 30, False, 40.0)[:3]
        kidx = [survivor_of(surv, m) for m in kept]
        assert same_bits(kR, single[1][kidx]) and same_bits(kt, single[2][kidx])
        expect_kept(answers(nat), kept, frame, kidx)

        # a batch of the frame, the frame rolled and the frame again, without and with the pose NMS
        names = ["recorded", "rolled", "recorded"]
        K = np.repeat(sK[None], len(names), 0)
        rgb = np.stack([data["frames"][k][0] for k in names])
        depth = np.stack([data["frames"][k][1] for k in names])
        frames = nat.detect_batch(rgb, depth, None, THR, K, 0.5, 0, 30, False, pose_nms=False)
        sizes = [len(f[0]) for f in frames]
        batch = answers(nat)
        expect_poses(batch, data, *(np.concatenate([f[k] for f in frames]) for k in range(4)), True)
        at = np.cumsum([0] + sizes)
        for f in (0, 2):  # the recorded frame: the single frame's entries
            assert same_bits(batch["T"][at[f]:at[f + 1]], frame["T"])
            same_verify((batch["verify"][0][at[f]:at[f + 1]], batch["verify"][1][at[f]:at[f + 1]]), frame["verify"])
        kept_frames = nat.detect_batch(rgb, depth, None, THR, K, 0.5, 0, 30, False, pose_nms=True)
        idx = [at[f] + survivor_of(frames[f][0], m) for f, k in enumerate(kept_frames) for m in k[0]]
        expect_kept(answers(nat), np.concatenate([k[0] for k in kept_frames]), batch, idx)
        assert same_bits(kept_frames[0][0], kept)

        # a track run with view following on, from the kept poses, each also turned, and one moved out of the frame
        objects = [(int(m["class_index"]), int(m["template_id"]), T) for m, T in zip(kept, frame["T"][kidx])]
        objects = tv.turned(objects, np.random.default_rng(17))
        objects.append((objects[0][0], objects[0][1], gt.shifted(objects[0][2], 5.0)))
        chosen = [j for _, j, _ in tv.rechosen(data, objects)[0]]
        nat.set_track_views(True, tv.TURN)
        status, T_out, R_out, t_out = nat.track(g["depth"], sK, objects)[:4]
        nat.set_track_views(False)
        tracked = status == TRACKED
        assert tracked.any() and not tracked.all()
        track = answers(nat)
        assert same_bits(track["T"], np.where(tracked[:, None, None], T_out, np.nan))
        assert len(track["verify"][0]) == len(objects)
        start = np.asarray([t for _, t, _ in objects], np.int32)
        assert same_bits(track["tpl"], np.where(tracked, np.asarray(chosen, np.int32), start))
        assert (track["tpl"] != start).any()  # view following switched some objects
        cls = [c for c, _, _ in objects]
        composes(data, track["T"][tracked], np.asarray(cls)[tracked], track["tpl"][tracked], R_out[tracked], t_out[tracked])

        # a frame enqueued and not finished: the track run's verification, no transformations and no templates
        nat.set_frame(g["rgb"], g["depth"], None)
        nat.enqueue(THR)
        nat.enqueue_post(0.5, 0)
        nat.enqueue_pose(sK, 30, False)
        pending = answers(nat)
        same_verify(pending["verify"], track["verify"])
        assert pending["T"] == lib.LM_E_STATE and pending["tpl"] == lib.LM_E_STATE
        done = nat.complete_pose()
        assert same_bits(done[3], res)
        expect_poses(answers(nat), data, *done[:4], True)
        same_verify(answers(nat)["verify"], frame["verify"])

        # a finish whose outputs are too small: nothing answers
        nat.set_frame(g["rgb"], g["depth"], None)
        nat.enqueue(THR)
        nat.enqueue_post(0.5, 0)
        nat.enqueue_pose(sK, 30, False)
        nat.enqueue_pose_nms(40.0)
        n = ctypes.c_int64()
        assert nat._L.lm_complete_detect(nat._h, None, None, None, None, 0, ctypes.byref(n), None, None, None) == lib.LM_E_CAPACITY
        assert n.value == len(kept)
        assert answers(nat) == {"verify": lib.LM_E_STATE, "T": lib.LM_E_STATE, "tpl": lib.LM_E_STATE}

        # and the next frame answers again
        again = nat.detect(g["rgb"], g["depth"], None, THR, sK, 0.5, 0, 30, False, 40.0)[0]
        assert same_bits(again, kept)
        expect_kept(answers(nat), kept, frame, kidx)
    finally:
        nat.close()


def test_icp_verify_after_every_kind_of_call():
    gold = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "icp_case1.npz"))
    scene, model = gold["scene"], gold["model"]
    rows, cols = scene.shape
    xy = [int(v) for v in gold["xy_scene_a"]]
    icp = lib.NativeIcp(0)

    def call(points):
        n = len(points)
        return icp.process_batch(scene, [model] * n, gold["K"], np.repeat(gold["K"][None], n, 0), np.repeat(gold["R"][None], n, 0),
                                 np.repeat(gold["t"].reshape(1, 3), n, 0), np.asarray(points, np.int32).reshape(n, 2), 30)

    def verify_code():
        n = ctypes.c_int64()
        return icp._L.lm_icp_verify(icp._h, None, None, 0, ctypes.byref(n))

    try:
        posed = call([xy, xy])[2]
        assert (posed != -1).all()
        assert verify_code() == lib.LM_E_STATE
        icp.set_verify(10.0)
        assert same_bits(call([xy, xy])[2], posed)
        score, counts = icp.verify()
        assert len(score) == 2 and (score >= 0).all() and (counts[:, 0] > 0).all()
        edge = [cols - 1, rows - 1]  # the render's box leaves the frame: the early return
        assert (call([edge, edge, edge])[2] == -1).all()
        score, counts = icp.verify()
        assert score.tolist() == [-1.0] * 3 and not counts.any()
        assert call([])[2].size == 0
        score, counts = icp.verify()
        assert score.size == 0 and counts.shape == (0, 6)
        icp.set_verify(None)
        call([])
        assert verify_code() == lib.LM_E_STATE
        assert (call([edge])[2] == -1).all()
        assert verify_code() == lib.LM_E_STATE
    finally:
        icp.close()
