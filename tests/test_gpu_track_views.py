"""View following on the device (include/linemod_b200.h, lm_set_track_views / k_track_views): lm_track_views_points
against tests/track_views_model.py bit for bit; every track entry point with view following on against the same call
with it off on the objects the model re-chose (status, box, T, R, t, residual, lm_pose_transforms, lm_pose_verify and
lm_track_templates); the INIT item of the chunk; launch counts; lm_peer_track_batch at worlds 2 and 3; and the
synthetic sequence of tests/view_object.py, held with view following on and lost with it off.

Data: the allScales bank and driver frame of tests/test_gpu_peer_batch.py with every template's R_b replaced by a
seeded rotation, so that objects switch, and the status frames of tests/test_gpu_track_batch.py."""
import importlib
import math

import numpy as np
import pytest
import torch

import test_gpu_peer_batch as pb
import test_gpu_peer_track as pt
import test_gpu_track as gt
import test_gpu_track_batch as tb
import test_track_views_model as tvm
import track_model as tm
import track_views_model as vm
import view_object as vo

pytestmark = pytest.mark.gpu
lib = importlib.import_module("6dpose_b200._lib")
synth = importlib.import_module("6dpose_b200.synth")
same_bits = gt.same_bits
TURN = 25.0


def random_rotations(n, rng):
    q = rng.normal(size=(n, 4))
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    w, x, y, z = q.T
    return np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w), 2 * (x * y + z * w), 1 - 2 * (x * x + z * z),
                     2 * (y * z - x * w), 2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)], 1).reshape(n, 3, 3)


# ---- lm_track_views_points ----
def adversarial():
    """(R_b, t_b, k, T, turn) cases at the rule's edges."""
    rng = np.random.default_rng(5)
    R = random_rotations(6, rng).astype(np.float32)
    t = rng.uniform(-50, 700, (6, 3)).astype(np.float32)
    T = np.eye(4)
    T[:3, :3] = R[2].astype(np.float64) @ R[0].astype(np.float64).T
    T[:3, 3] = (0.01, 0.02, 0.5)
    Rt = np.stack([R[0], R[2], R[2], R[2]])  # ties: the lowest of 1..3
    out = [(Rt, t[:4], 0, T, 10.0), (R, t, 0, T, 0.0), (R[:1], t[:1], 0, T, 0.0), (R, t, 2, T, 0.0), (R, t, 2, T, 179.9)]
    Rn = R.copy()
    Rn[3, 1, 1] = np.nan
    out.append((Rn, t, 0, T, 5.0))
    Ri = R.copy()
    Ri[4, 0, 0] = np.inf
    out.append((Ri, t, 0, T, 5.0))
    out.append((np.stack([R[0], -R[0], R[0]]), t[:3], 1, T, 0.0))  # scores with -0.0 and +0.0 terms
    sk = vm.scores(vm.rotation(T, R[0]), R)[0]
    deg = math.degrees(math.acos(min(max((sk - 1.0) / 2.0, -1.0), 1.0)))
    out += [(R, t, 0, T, deg + i * 2e-14) for i in range(-8, 9)]  # s_k on either side of tau
    return out


def test_points_equal_the_model():
    rng = np.random.default_rng(11)
    cases = adversarial()
    for n in (1, 2, 7, 256, 257, 3000):
        R = random_rotations(n, rng).astype(np.float32)
        t = rng.uniform(-100, 900, (n, 3)).astype(np.float32)
        for _ in range(4):
            k = int(rng.integers(n))
            T = np.eye(4)
            T[:3, :3] = random_rotations(1, rng)[0]
            T[:3, 3] = rng.uniform(-0.3, 0.9, 3)
            cases.append((R, t, k, T, float(rng.uniform(0, 90))))
    switched = 0
    for R, t, k, T, turn in cases:
        j, T2 = lib.track_views_points(R, t, k, T, turn)
        mj, mT, *_ = vm.choose(R, t, k, T, turn)
        assert j == mj and same_bits(T2, mT), (len(R), k, turn)
        switched += j != k
    assert switched > len(cases) // 3


# ---- every entry point against the off-run on the re-chosen objects ----
@pytest.fixture(scope="module")
def data():
    d = pb.load_data()
    d["R"] = random_rotations(d["G"], np.random.default_rng(3)).astype(np.float32)
    return d


@pytest.fixture(scope="module")
def nat(data):
    return pt.make_handle(data, 0, (0, 1), True)


def class_of(data, c):
    cb = np.asarray(data["packed"]["class_begin"])
    return int(cb[c]), int(cb[c + 1])


def rechosen(data, objects):
    """The model's (class, j*, T') per object, and whether it switched."""
    out, sw = [], []
    for c, t, T in objects:
        b, e = class_of(data, c)
        j, T2, *_ = vm.choose(data["R"][b:e], data["t"][b:e], t, T, TURN)
        out.append((c, j, T2))
        sw.append(j != t)
    return out, sw


def turned(objects, rng):
    """Each object also turned about its translation by a seeded rotation, so that its view changes."""
    out = list(objects)
    for c, t, T in objects:
        T2 = np.array(T, np.float64)
        T2[:3, :3] = random_rotations(1, rng)[0] @ T2[:3, :3]
        out.append((c, t, T2))
    return out


@pytest.fixture(scope="module")
def frames(nat, data):
    depths, Ks, objects = tb.status_frames(nat, data)
    rng = np.random.default_rng(17)
    objects = [turned(o, rng) for o in objects]
    return depths, Ks, objects


def run(nat, fn, verify, views):
    nat.set_pose_verify(verify, 10.0)
    nat.set_track_views(views, TURN)
    try:
        got = fn()
        return got, nat.pose_transforms(), nat.pose_verify() if verify else None, nat.track_templates()
    finally:
        nat.set_pose_verify(False)
        nat.set_track_views(False)


def expect_reduction(on, off, starts, chosen):
    """The on-run equals the off-run on the re-chosen objects; an entry not tracked keeps its start T and template."""
    (g_on, T_on, v_on, tpl_on), (g_off, T_off, v_off, tpl_off) = on, off
    status = g_on[0]
    assert same_bits(status, g_off[0]) and same_bits(g_on[5], g_off[5])
    for k in (2, 3, 4):
        assert same_bits(g_on[k], g_off[k]), k
    tracked = status == tm.TRACKED
    want_T = np.where(tracked[:, None, None], g_off[1], np.stack([T for _, _, T in starts]) if len(starts) else g_off[1])
    assert same_bits(g_on[1], want_T)
    assert same_bits(T_on, T_off)
    if v_on is not None:
        assert same_bits(v_on[0], v_off[0]) and same_bits(v_on[1], v_off[1])
    assert same_bits(tpl_off, np.asarray([j for _, j, _ in chosen], np.int32))
    want_tpl = np.where(tracked, tpl_off, np.asarray([t for _, t, _ in starts], np.int32))
    assert same_bits(tpl_on, want_tpl.astype(np.int32))


def cat(per_frame):
    return tuple(np.concatenate([f[k] for f in per_frame]) for k in range(6))


@pytest.mark.parametrize("estimation", ["point_to_plane", "point_to_point"])
def test_every_entry_point_reduces_to_the_off_run(nat, data, frames, estimation):
    depths, Ks, objects = frames
    flat = [o for objs in objects for o in objs]
    chosen, sw = rechosen(data, flat)
    assert sum(sw) > len(flat) // 4
    per = [rechosen(data, o)[0] for o in objects]
    seen = set()
    for verify in (False, True):
        # lm_track, frame by frame
        for f, (d, K, objs) in enumerate(zip(depths, Ks, objects)):
            if not objs:
                continue
            on = run(nat, lambda: nat.track(d, K, objs, 30, 4, estimation), verify, True)
            for i, s in enumerate(nat.pose_clouds()[1]):  # the chunk's INIT is the model's T'
                if s["posed"]:
                    assert same_bits(s["init"], per[f][i][2]), (f, i)
            off = run(nat, lambda: nat.track(d, K, per[f], 30, 4, estimation), verify, False)
            expect_reduction(on, off, objs, per[f])
            seen |= set(on[0][0].tolist())
        # lm_track_batch
        on = run(nat, lambda: nat.track_batch(np.stack(depths), Ks, objects, 30, 4, estimation), verify, True)
        off = run(nat, lambda: nat.track_batch(np.stack(depths), Ks, per, 30, 4, estimation), verify, False)
        expect_reduction((cat(on[0]),) + on[1:], (cat(off[0]),) + off[1:], flat, chosen)
        # lm_track_device (u16 and f32) and lm_track_batch_device
        st = torch.cuda.Stream()
        for f32, fmt, scale in ((False, lib.DEPTH_U16_MM, 1.0), (True, lib.DEPTH_F32, 1000.0)):
            ts = [tb.pitched(d, f32, st) for d in depths]
            st.synchronize()
            pitch = ts[0].stride(0) * ts[0].element_size()
            rows, cols = depths[0].shape
            f = next(f for f, o in enumerate(objects) if o)
            on = run(nat, lambda: nat.track_device(ts[f].data_ptr(), pitch, fmt, scale, rows, cols, st.cuda_stream, Ks[f], objects[f], 30, 4,
                                                   estimation), verify, True)
            off = run(nat, lambda: nat.track_device(ts[f].data_ptr(), pitch, fmt, scale, rows, cols, st.cuda_stream, Ks[f], per[f], 30, 4,
                                                    estimation), verify, False)
            expect_reduction(on, off, objects[f], per[f])
            ptrs = [t.data_ptr() for t in ts]
            on = run(nat, lambda: nat.track_batch_device(ptrs, pitch, fmt, scale, rows, cols, st.cuda_stream, Ks, objects, 30, 4, estimation),
                     verify, True)
            off = run(nat, lambda: nat.track_batch_device(ptrs, pitch, fmt, scale, rows, cols, st.cuda_stream, Ks, per, 30, 4, estimation),
                      verify, False)
            expect_reduction((cat(on[0]),) + on[1:], (cat(off[0]),) + off[1:], flat, chosen)
            st.synchronize()
    assert seen == {tm.TRACKED, tm.OUTSIDE, tm.WINDOW, tm.NO_DEPTH}


def test_launches_one_more_per_chunk(nat, data, frames):
    depths, Ks, objects = frames
    pool = [o for objs in objects for o in objs]
    counts = [1000, 0, 30, 20, 0, 0, 0]  # two chunks
    objs = tb.repeated(pool, counts)
    dd = np.stack([depths[f % len(depths)] for f in range(len(counts))])
    KK = np.stack([Ks[f % len(Ks)] for f in range(len(counts))])
    got = {}
    for views in (False, True):
        nat.set_track_views(views, TURN)
        before = nat.launch_count()
        nat.track_batch(dd, KK, objs, 30, 4)
        got[views] = nat.launch_count() - before
        before = nat.launch_count()
        nat.track(depths[0], Ks[0], objects[0], 30, 4)
        got[views, 1] = nat.launch_count() - before
    nat.set_track_views(False)
    assert got[False] == 2 * 5 and got[True] == 2 * 6
    assert got[False, 1] == 5 and got[True, 1] == 6


@pytest.mark.parametrize("world", [2, 3])
def test_peer_ranks_equal_the_unconnected_on_run(nat, data, frames, world):
    depths, Ks, objects = frames
    dd = np.stack(depths)
    pool = [o for objs in objects for o in objs if o]
    dets = pt.connected(data, pool, [0] * world, one_render=True)
    try:
        for d in dets:
            d.set_track_views(True, TURN)
        nat.set_track_views(True, TURN)
        for share in (True, False):
            for d in dets:
                d.peer_share_pose(share)
            for verify in (False, True):
                want = pt.unconnected(nat, dd, Ks, objects, verify=verify)
                want_tpl = nat.track_templates()
                results = pt.peer_track(dets, dd, Ks, objects, verify=verify)
                n = sum(map(len, objects))
                for r, got in enumerate(results):
                    pt.same_run(got, want)
                    assert got[5] == (6 if share else 5) + 1 + verify, (r, got[5])
                    assert got[3][2] == got[5]
                for d in dets:
                    assert same_bits(d.track_templates(), want_tpl)
                assert len(want_tpl) == n
    finally:
        nat.set_track_views(False)
        pb.close(dets)


# ---- the synthetic sequence on the device ----
def sequence_handle(Rb, tb_, Kb, renders):
    G = len(Rb)
    bank = synth.synth_bank(G, num_features=30, seed=1, variants=35)
    nat = lib.NativeDetector([4, 8], 0)
    nat.load_bank(bank.pack(bank.class_ids(), 4), 4)
    nat.set_template_renders(0, renders, Kb, Rb, tb_)
    return nat


def test_sequence_held_with_views_and_lost_without():
    Rb, tb_, Kb = vo.templates()
    renders = [vo.template_render(Rb[g], tb_[g]) for g in range(len(Rb))]
    nat = sequence_handle(Rb, tb_, Kb, renders)
    seq = vo.sequence(Rb[tvm.START].astype(np.float64), tvm.FRAMES, tvm.STEP_DEG)
    sK = vo.K.astype(np.float32)
    worst = {}
    for views in (False, True):
        nat.set_track_views(views, tvm.TURN_DEG)
        g, T = tvm.START, vo.start_T(seq[0][1], seq[0][2], Rb[tvm.START], tb_[tvm.START])
        errs, switches = [], 0
        for scene, R, b in seq[1:]:
            status, T_out, *_ = nat.track(scene, sK, [(0, g, T)], 30, 4)
            j = int(nat.track_templates()[0])
            if status[0] != tm.TRACKED:
                errs.append((math.inf, math.inf))
                break
            switches += j != g
            g, T = j, T_out[0]
            errs.append(vo.errors(T, Rb[g], tb_[g], R, b))
        e = np.array(errs)
        worst[views] = (e[:, 0].max(), e[:, 1].max(), switches, len(e))
    print("view following off / on: (worst rotation deg, worst position mm, switches, frames)", worst)
    rot_on, pos_on, sw_on, n_on = worst[True]
    assert n_on == tvm.FRAMES and sw_on >= 3 and rot_on <= tvm.HELD_ROT_DEG and pos_on <= tvm.HELD_POS_MM
    rot_off, pos_off, sw_off, _ = worst[False]
    assert sw_off == 0 and (rot_off > tvm.HELD_ROT_DEG or pos_off > tvm.HELD_POS_MM)
    nat.set_track_views(True, tvm.TURN_DEG)
    with pytest.raises(RuntimeError, match="PSO"):
        nat.track(seq[0][0], sK, [(0, tvm.START, np.eye(4))], 30, 4, "pso")
