"""The device pose stage's clouds (k_pose_cloud, the segmented sort, k_pose_voxel) against the float64 model of
tests/pose_cloud_model.py, bit for bit: per slot the posed flag, the counts, the raw model and scene clouds, the
down-sampled source and target and the initial guess, NaN patterns included.  Survivors are crafted: a frame's result
block, held by the caller, is overwritten on the handle's stream between lm_enqueue and lm_enqueue_post (IoU 1.0, distinct
similarities: the box NMS keeps every record), then lm_enqueue_pose; lm_debug_pose_clouds reads what the stage built.
Batches, shared stages and lm_icp_process_batch_device are held to the same model through their own survivors."""
import importlib
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import icp_clouds as ic  # noqa: E402
import pose_cloud_model as pcm  # noqa: E402
import test_pose_cloud_model as cases  # noqa: E402
from test_gpu_icp_device import cuda  # noqa: E402
from test_pose_cloud_model import CLASS_BEGIN, PER_CLASS, same_bits  # noqa: E402

pytestmark = pytest.mark.gpu

lib = importlib.import_module("6dpose_b200._lib")
synth = importlib.import_module("6dpose_b200.synth")

CAP = 2048          # records the caller's result block holds
ITEMS = ("counts", "raw_model", "raw_scene", "source", "target", "init")


@pytest.fixture(scope="module")
def bank():
    bk = synth.synth_bank(PER_CLASS, num_features=63, seed=5, class_ids=("01_template", "02_template", "03_template"))
    packed = bk.pack(bk.class_ids(), 4)
    assert np.array_equal(packed["class_begin"], CLASS_BEGIN)
    return packed


class Handle:
    """A detector over the crafted bank with a caller-held result block."""

    def __init__(self, packed, select=None):
        import torch
        self.nat = lib.NativeDetector([4, 8], 0)
        self.nat.load_bank(packed, 4)
        self.nat.select(select, 0, 1)
        self.block = torch.zeros(16 + 16 * CAP, dtype=torch.uint8, device="cuda")
        self.nat.set_result_buffer(self.block.data_ptr(), CAP)
        classes = range(len(CLASS_BEGIN) - 1) if select is None else select
        self.sel = [g for k in classes for g in range(CLASS_BEGIN[k], CLASS_BEGIN[k + 1])]  # record work -> template

    def close(self):
        self.nat.set_result_buffer(0, 0)
        self.nat.close()

    def register(self, renders):
        for g, (r, k) in sorted(renders.items()):
            self.nat.set_template_renders(g, [r], k[None], np.eye(3, dtype=np.float32)[None], np.array([[1.0, -2.0, 900.0]], np.float32))

    def run(self, scene, sK, surv, use_scene, top_k=None, estimation="point_to_plane", max_iterations=30, verify=False):
        """surv: (x, y, g) in pick order.  Returns complete_pose's outputs.  top_k (default: the survivors) sizes the chunk:
        its slots times the largest crop are the stage's cloud buffers."""
        import torch
        n = len(surv)
        recs = np.zeros(n, lib.RECORD_DTYPE)
        recs["x"] = [s[0] for s in surv]
        recs["y"] = [s[1] for s in surv]
        recs["similarity"] = 100.0 - 0.25 * np.arange(n)        # distinct: pick order is surv's
        recs["work"] = [self.sel.index(s[2]) for s in surv]
        recs["seq"] = np.arange(n)
        src = torch.from_numpy(np.concatenate([np.array([n], np.int32).view(np.uint8), recs.view(np.uint8)])).cuda()
        torch.cuda.synchronize()
        self.nat.set_pose_verify(verify)
        self.nat.upload_images(np.zeros(scene.shape + (3,), np.uint8), scene)
        self.nat.enqueue(99.0)
        with torch.cuda.stream(torch.cuda.ExternalStream(self.nat.stream())):
            self.block[0:4].copy_(src[0:4])
            self.block[16:16 + 16 * n].copy_(src[4:])
        self.nat.enqueue_post(1.0, n if top_k is None else top_k)
        self.nat.enqueue_pose(sK, max_iterations, use_scene, estimation)
        return self.nat.complete_pose()


def first_difference(a, b):
    """The first row (point) where a and the model b differ."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    if a.shape != b.shape:
        return "shape %s, model %s" % (a.shape, b.shape)
    rows_a, rows_b = a.reshape(a.shape[0] if a.ndim > 1 else -1, -1), b.reshape(b.shape[0] if b.ndim > 1 else -1, -1)
    for k in range(rows_a.shape[0]):
        if not same_bits(rows_a[k], rows_b[k]):
            return "row %d: %r, model %r" % (k, rows_a[k], rows_b[k])
    return "equal"


def same_slot(where, got, want):
    """One slot of lm_debug_pose_clouds against the model's clouds."""
    assert got["posed"] == want["posed"], (where, "posed", got["posed"], want["posed"])
    if not want["posed"]:
        return
    for item in ITEMS:
        g, w = np.asarray(got[item]), np.asarray(want[item])
        if item == "counts":
            assert tuple(g) == tuple(w), (where, item, tuple(g), tuple(w))
        else:
            assert same_bits(g, w), (where, item, first_difference(g, w))


def model_of(scene, renders, sK, m, use_scene):
    g = int(CLASS_BEGIN[m["class_index"]] + m["template_id"])
    return pcm.clouds(scene, renders[g][0], sK, renders[g][1], int(m["x"]), int(m["y"]), use_scene)


def check_frame(name, h, c, use_scene, out):
    """Every slot of the frame's chunk against the model of its survivor; slots past the survivors have no pose."""
    surv, R, t, res, nrec = out
    assert sorted((int(s["x"]), int(s["y"]), int(CLASS_BEGIN[s["class_index"]] + s["template_id"])) for s in surv) == sorted(c.surv)
    head, slots = h.nat.pose_clouds()
    assert head["rank"] == 0 and head["world"] == 1 and head["first"] == 0 and head["slots"] >= len(surv), head
    for i, got in enumerate(slots):
        if i >= len(surv):
            assert not got["posed"], (name, i)
            continue
        want = model_of(c.scene, c.renders, c.sK, surv[i], use_scene)
        same_slot((name, use_scene, "slot", i), got, want)
        assert (res[i] != -1) == want["posed"]
    return slots


@pytest.mark.parametrize("use_scene", [False, True])
@pytest.mark.parametrize("name", sorted(cases.CASES))
def test_crafted_survivors_equal_the_model(bank, name, use_scene):
    c = cases.CASES[name]
    h = Handle(bank, c.select)
    try:
        h.register(c.renders)
        out = h.run(c.scene, c.sK, c.surv, use_scene, top_k=0 if name == "edges" else None)  # edges: 1024 slots, small crops
        slots = check_frame(name, h, c, use_scene, out)
        assert any(s["posed"] for s in slots)
        if name == "edges":
            assert not all(s["posed"] for s in slots[:len(c.surv)])
    finally:
        h.close()


def test_slot_strides_after_re_registration(bank):
    """Large renders, then small ones (the slot stride stays the largest crop's), then larger ones again."""
    c = cases.CASES["edges"]
    h = Handle(bank)
    try:
        wide = cases.blob(480, 640, 50, 330, 100, 400, 1000, 7)
        small = cases.blob(480, 640, 236, 246, 315, 327, 1010, 5)
        wider = cases.blob(480, 640, 10, 460, 20, 620, 1000, 9)
        surv = [(2, 3, 0), (10, 20, 5), (200, 100, 0)]
        for r in (wide, small, wider):
            renders = cases.default_renders({0: (r, cases.RK), 5: (r, cases.K(500.0, 500.0, 320.0, 240.0))})
            h.register(renders)
            for use_scene in (False, True):
                out = h.run(c.scene, c.sK, surv, use_scene)
                check_frame("strides", h, cases.Case("strides", c.scene, c.sK, renders, surv), use_scene, out)
    finally:
        h.close()


def test_compaction_limit(bank):
    """A fully non-zero render of 2359 x 889 = 2^21 - 1 box pixels, every one a model, scene and centroid point; a box of
    2^21 pixels is refused at registration."""
    scene = cases.limit_scene()
    renders = cases.default_renders({0: (cases.limit_render(), cases.LIMIT_K)})
    h = Handle(bank)
    try:
        h.register(renders)
        c = cases.Case("limit", scene, cases.SK, renders, [(10, 5, 0)])
        for use_scene in (False, True):
            out = h.run(scene, cases.SK, c.surv, use_scene, top_k=1, estimation="point_to_point", max_iterations=1)
            slots = check_frame("limit", h, c, use_scene, out)
            assert slots[0]["raw_model"].shape[0] == (1 << 21) - 1
        over = np.full((1024, 2048), 1000, np.uint16)
        with pytest.raises(RuntimeError, match="too large"):
            h.nat.set_template_renders(1, [over], cases.RK[None], np.eye(3, dtype=np.float32)[None], np.zeros((1, 3), np.float32))
    finally:
        h.close()


def test_voxel_overflow_fails_the_frame_and_the_next_frame_is_clean(bank):
    c = cases.CASES["edges"]
    bad = dict(c.renders)
    bad[0] = (c.renders[0][0], cases.K(1e-3, 1e-3, 320.0, 240.0))   # metres per pixel in the kilometres
    h, fresh = Handle(bank), Handle(bank)
    try:
        h.register(bad)
        with pytest.raises(RuntimeError, match="spans more than 2\\^21 voxels"):
            h.run(c.scene, c.sK, c.surv, False)
        h.register(c.renders)
        fresh.register(c.renders)
        for use_scene in (False, True):
            got = h.run(c.scene, c.sK, c.surv, use_scene)
            want = fresh.run(c.scene, c.sK, c.surv, use_scene)
            for x, y in zip(got[1:4], want[1:4]):
                assert np.array_equal(x, y, equal_nan=True)
            check_frame("after_overflow", h, c, use_scene, got)
            hg, sg = h.nat.pose_clouds()
            hw, sw = fresh.nat.pose_clouds()
            assert hg == hw
            for i, (a, b) in enumerate(zip(sg, sw)):
                assert a["posed"] == b["posed"] and all(same_bits(a[k], b[k]) for k in ITEMS[1:] if a["posed"]), i
    finally:
        h.close()
        fresh.close()


def test_unkeyable_intrinsics_are_refused_alike_by_both_icp_calls():
    """A zero or NaN render K gives clouds that span more than 2^21 voxels: lm_icp_process_batch and
    lm_icp_process_batch_device refuse alike."""
    c = ic.size_case(257)
    icp = lib.NativeIcp()
    try:
        for K in (cases.K(0.0, 100.0, 320.0, 240.0), cases.K(np.nan, 100.0, 320.0, 240.0), cases.K(100.0, 100.0, np.nan, 240.0)):
            args = (c.K, K[None], c.R[None], c.t[None], [c.xy])
            with pytest.raises(RuntimeError, match="spans more than"):
                icp.process_batch(c.scene, [c.model], *args)
            d = lib.DeviceDepths(cuda(c.scene), [cuda(c.model)], 1.0, 1.0, None, 0)
            with pytest.raises(RuntimeError, match="spans more than"):
                icp.process_batch_device(d, *args)
        R, t, res = icp.process_batch(c.scene, [c.model], c.K, c.K[None], c.R[None], c.t[None], [c.xy])  # the handle still works
        assert res[0] != -1
    finally:
        icp.close()


# ---- batches and shared stages: the survivors the frames give ----------------------------------------------------
@pytest.fixture(scope="module")
def driver():
    import test_gpu_pose_share as share
    return share.load_data()


def renders_of(data):
    return {g: (data["renders"][data["which"][g]], data["K"][g]) for g in range(data["G"])}


def test_batch_slots_follow_the_survivor_offsets(driver):
    """Three frames of one batch, each with its own depth and intrinsics: slot i is the run's survivor i, modelled
    against its frame's depth and K."""
    data = driver
    g = data["g"]
    depth = np.stack([g["depth"], np.roll(g["depth"], 3, 1), np.where(g["depth"] > 0, g["depth"] + 7, 0).astype(np.uint16)])
    rgb = np.stack([g["rgb"]] * 3)
    sK = np.stack([data["sK"], data["sK"] * np.float32(1.01), data["sK"] * np.float32(0.98)])
    sK[:, 2, 2] = 1.0
    nat = lib.NativeDetector(data["T"], 0)
    try:
        nat.load_bank(data["packed"], 4)
        nat.select(None, 0, 1)
        nat.set_template_renders(0, [data["renders"][k] for k in data["which"]], data["K"], data["R"], data["t"])
        renders = renders_of(data)
        for use_scene in (False, True):
            frames = nat.detect_batch(rgb, depth, None, 65.0, sK, 0.5, 3, pose_nms=False, use_scene_cloud=use_scene)
            head, slots = nat.pose_clouds()
            surv = np.concatenate([f[0] for f in frames])
            frame_of = np.repeat(np.arange(3), [len(f[0]) for f in frames])
            assert head == dict(slots=len(surv), rank=0, world=1, first=0) and len(surv) == 9
            for i, got in enumerate(slots):
                f = int(frame_of[i])
                want = model_of(depth[f], renders, sK[f], surv[i], use_scene)
                same_slot(("batch", use_scene, "slot", i, "frame", f), got, want)
            assert sum(s["posed"] for s in slots) >= 3
    finally:
        nat.close()


@pytest.mark.parametrize("world", [2, 3])
def test_shared_stage_slots_are_rank_plus_i_world(driver, world):
    import test_gpu_pose_share as share
    data = driver
    renders = renders_of(data)
    single = share.handle(data)
    dets = share.connected(data, [0] * world)
    try:
        for use_scene in (False, True):
            want = share.frame([single], data, 65.0, 0, use_scene, False)[0]
            got = share.frame(dets, data, 65.0, 0, use_scene, False)
            surv = want[0]
            assert len(surv) > 2 * world
            seen = set()
            for r, d in enumerate(dets):
                share.same(got[r], want)
                head, slots = d.pose_clouds()
                assert head["rank"] == r and head["world"] == world and head["first"] == 0, head
                for i, s in enumerate(slots):
                    k = r + i * world
                    if k >= len(surv):
                        assert not s["posed"]
                        continue
                    same_slot(("shared", world, "rank", r, "slot", i), s, model_of(data["g"]["depth"], renders, data["sK"], surv[k], use_scene))
                    seen.add(k)
            assert seen == set(range(len(surv)))
    finally:
        share.close(dets)
        single.close()


# ---- lm_icp_process_batch_device: its capture equals lm_icp_process_batch's ----------------------------------------
def device_pairs():
    """(name, scene, renders, sK, mKs, xy) groups: the ICP cases, and the crafted cases' survivors by render size."""
    out = [(c.name, c.scene, [c.model], c.K, c.K[None], [c.xy]) for c in ic.all_cases()]
    for c in cases.CASES.values():
        by = {}
        for x, y, g in c.surv:
            by.setdefault(c.renders[g][0].shape, []).append((x, y, g))
        for shape, ss in sorted(by.items()):
            out.append(("%s_%dx%d" % (c.name, shape[1], shape[0]), c.scene, [c.renders[g][0] for _, _, g in ss], c.sK,
                        np.stack([c.renders[g][1] for _, _, g in ss]), [(x, y) for x, y, _ in ss]))
    return out


def test_device_icp_capture_equals_the_host_capture():
    host, dev = lib.NativeIcp(), lib.NativeIcp()
    try:
        for h in (host, dev):
            h.set_capture(True)
        for use_scene in (False, True):
            for h in (host, dev):
                h.set_use_scene_cloud(use_scene)
            for k, (name, scene, renders, sK, mKs, xy) in enumerate(device_pairs()):
                n = len(renders)
                R = np.repeat(np.eye(3, dtype=np.float32)[None], n, 0)
                t = np.tile(np.float32([1.0, 2.0, 800.0]), (n, 1))
                want = host.process_batch(scene, renders, sK, mKs, R, t, xy)
                if k % 2:   # float32 planes that convert exactly to the u16 ones
                    d = lib.DeviceDepths(cuda(scene).float() * 4.0, [cuda(r).float() * 2.0 for r in renders], 0.25, 0.5, None, 0)
                else:
                    d = lib.DeviceDepths(cuda(scene), [cuda(r) for r in renders], 1.0, 1.0, None, 0)
                got = dev.process_batch_device(d, sK, mKs, R, t, xy)
                for a, b in zip(got, want):
                    assert np.array_equal(a, b, equal_nan=True), name
                for i in range(n):
                    if want[2][i] == -1:
                        for h in (host, dev):
                            with pytest.raises(lib.LinemodLibraryError, match="early return"):
                                h.capture(i)
                        continue
                    cg, cw = dev.capture(i), host.capture(i)
                    for item in ("source", "target", "normals", "init", "T", "knn", "corr_first", "corr_last"):
                        assert same_bits(cg[item], cw[item]), (name, use_scene, i, item, first_difference(cg[item], cw[item]))
                    assert (cg["fitness"], cg["rmse"], cg["iterations"]) == (cw["fitness"], cw["rmse"], cw["iterations"]) or \
                        np.isnan(cg["fitness"]) and np.isnan(cw["fitness"])
    finally:
        host.close()
        dev.close()


# ---- no side effects ---------------------------------------------------------------------------------------------
def test_getter_and_capture_change_no_output(bank):
    c = cases.CASES["anchor"]
    a, b = Handle(bank), Handle(bank)
    try:
        for h in (a, b):
            h.register(c.renders)
        for use_scene in (False, True):
            la, lb = a.nat.launch_count(), b.nat.launch_count()
            got = a.run(c.scene, c.sK, c.surv, use_scene, verify=True)
            a.nat.pose_clouds()
            vg = a.nat.pose_verify()
            want = b.run(c.scene, c.sK, c.surv, use_scene, verify=True)
            vw = b.nat.pose_verify()
            assert a.nat.launch_count() - la == b.nat.launch_count() - lb
            assert np.array_equal(got[0], want[0])
            for x, y in zip(got[1:4], want[1:4]):
                assert np.array_equal(x, y, equal_nan=True)
            assert all(np.array_equal(x, y) for x, y in zip(vg, vw))
    finally:
        a.close()
        b.close()
    on, off = lib.NativeIcp(), lib.NativeIcp()
    try:
        on.set_capture(True)
        for h in (on, off):
            h.set_verify(10.0)
        r = [c.renders[0][0]] * 3
        args = (c.sK, np.stack([c.renders[0][1]] * 3), np.repeat(np.eye(3, dtype=np.float32)[None], 3, 0), np.zeros((3, 3), np.float32),
                [xy for xy, _ in zip(((x, y) for x, y, _ in c.surv), range(3))])
        outs = []
        for h in (on, off):
            l0 = h.launch_count()
            outs.append((h.process_batch_device(lib.DeviceDepths(cuda(c.scene), [cuda(x) for x in r], 1.0, 1.0, None, 0), *args),
                         h.verify(), h.launch_count() - l0))
        (go, gv, gl), (wo, wv, wl) = outs
        assert gl == wl and all(np.array_equal(x, y, equal_nan=True) for x, y in zip(go, wo))
        assert all(np.array_equal(x, y) for x, y in zip(gv, wv))
    finally:
        on.close()
        off.close()
