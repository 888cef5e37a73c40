"""The coarse scan (k_coarse_packed, k_coarse_bytes) bit for bit at its bounds: lm_debug_coarse (NativeDetector.coarse)
against the model of tests/coarse_frames.py, on every construction there and on every SHAPE_CASES frame.

For every case and threshold: every pass-mask word, the raw score at every pass bit (and 0 elsewhere), the per-template
pass counts, the coarse_candidates counter, and (where it says so) the final match list against oracle.match; plan()
shows the route the case is meant to take.  A wrong pass bit at a cell the refinement later drops, or a wrong raw score
that still passes, fails here although the match list would not show it."""
import importlib

import numpy as np
import pytest

import coarse_frames as cf
import depth_gate_model as dg
import match_shapes as ms
from test_gpu_match_parity import _assert_same

pytestmark = pytest.mark.gpu
lib = importlib.import_module("6dpose_b200._lib")


def _sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


class Case:
    """A bank on a quantized frame, its model and its detector."""

    def __init__(self, oracle, T, bank, q):
        self.oracle, self.T, self.q = oracle, list(T), q
        self.packed = bank.pack(bank.class_ids(), cf.M * len(T))
        self.model = cf.CoarseModel(oracle, q, T, self.packed)
        self.nat = lib.NativeDetector(T)
        self.nat.load_bank(self.packed, cf.M * len(T))

    def check(self, thr, match=True):
        """One frame at threshold thr: the coarse outputs against the model, and the match list against the oracle."""
        if match:
            got = self.nat.match_quantized(self.q, thr)
        else:
            self.nat.run(thr)
        mask, raw = self.nat.coarse()
        want_mask, want_raw = self.model.expected(thr)
        assert mask.shape == want_mask.shape and raw.shape == want_raw.shape
        bad = np.flatnonzero((mask != want_mask).any(1))
        assert len(bad) == 0, ("pass mask", float(thr), bad[:8].tolist())
        bad = np.flatnonzero((raw != want_raw).any(1))
        assert len(bad) == 0, ("raw", float(thr), bad[:8].tolist())
        per = self.model.passes(thr).sum(1)
        assert np.array_equal(np.unpackbits(mask.view(np.uint8), axis=1).sum(1), per)
        assert self.nat.counters()["coarse_candidates"] == int(per.sum())
        if match:
            want = self.oracle.match(self.q, self.T, self.packed, thr)
            _assert_same(got, want)
        return int(per.sum())

    def plan(self, **want):
        p = self.nat.plan()
        for k, v in want.items():
            assert p[k] == v, (k, p[k], v, p)
        return p

    def close(self):
        self.nat.close()


def test_threshold_sweep(oracle):
    """Every raw_min 0 .. 4 nf + 1 against every attainable raw of nf features, nf in SWEEP_NF: thresholds
    score(raw_min - 1), score(raw_min) and one ulp either side.  The match list at the lowest, middle and highest."""
    T, W, H = cf.SWEEP_SHAPE
    for nf in cf.SWEEP_NF:
        bank, q = cf.sweep_bank(nf)
        c = Case(oracle, T, bank, q)
        thrs = cf.sweep_thresholds(nf)
        c.nat.upload_quantized(q)
        for i, thr in enumerate(thrs):
            c.check(thr, match=i in (0, len(thrs) // 2, len(thrs) - 1))
        c.plan(packed_templates=c.model.G, byte_templates=0)
        c.close()


@pytest.mark.parametrize("split", [8, 4, 2, 1])
def test_counter_saturation_and_team_merges(oracle, split):
    """CH = 255, CN = 255 and the carries through 127 -> 128 and 254 -> 255, every template one full round and one
    remainder word (the remainder tasks hold lanes of templates with different nf), under team split S; fillers (raw
    0) set the task count."""
    T, W, H = cf.SAT_SHAPE
    shape = ms.frame_shape(T, W, H)
    k = cf.filler_count(shape["words"], len(cf.PATTERNS), _sm_count(), shape["plane_bytes"], split)
    c = Case(oracle, T, cf.saturation_bank(fillers=k), cf.onehot_frame(W, H, 1, cf.SAT_LABEL))
    thrs = cf.ladder() + ([np.float32(-1.0)] if k == 0 else [])
    for thr in thrs:
        c.check(thr)
    c.plan(split=split, packed_templates=len(cf.PATTERNS) + k, byte_templates=0, k2_smem=1)
    c.close()


@pytest.mark.parametrize("name", list(cf.STAGING))
def test_staging_modes(oracle, name):
    """The saturation patterns with the bit-planes in shared memory (640x624) and in global memory (640x640), two
    levels: the refinement follows."""
    T, W, H = cf.STAGING[name]
    c = Case(oracle, T, cf.saturation_bank(levels=2), cf.onehot_frame(W, H, 2, cf.SAT_LABEL))
    for thr in cf.ladder() + [np.float32(-1.0)]:
        c.check(thr)
    c.plan(k2_smem=int(name == "k2_shared"), packed_templates=len(cf.PATTERNS), byte_templates=0)
    c.close()


@pytest.mark.parametrize("frame", ["label0", "label7", "both"])
def test_label_wrap(oracle, frame):
    """Label-0 features on a label-7 frame and label-7 features on a label-0 frame respond through the wrap; on a frame
    of both, a hit with its neighbour present still counts 4.  Both kernels."""
    T, W, H = cf.WRAP_SHAPE
    o = 7 if frame == "label7" else 0
    q = cf.pair_frame(W, H, 1, 0, 7) if frame == "both" else cf.onehot_frame(W, H, 1, o)
    c = Case(oracle, T, cf.wrap_bank(o), q)
    for thr in [np.float32(-1.0), np.float32(0.0)] + [cf.score(r + d, int(nf)) for nf, r in
                                                      zip(c.model.nf, c.model.raw[:, 0]) for d in (-1, 0)]:
        c.check(thr)
    p = c.plan()
    assert p["packed_templates"] == 4 and p["byte_templates"] == 1
    c.close()


@pytest.mark.parametrize("shape", [cf.EDGE_SHAPE, cf.TINY_SHAPE], ids=["33x31", "5x3"])
def test_position_edges(oracle, shape):
    """P at every residue mod 32, P = 1, P <= 0 and a plane that is not a multiple of 32; a negative threshold passes
    every cell (positions >= P and the words past the template's last one with raw 0)."""
    T, W, H = shape
    c = Case(oracle, T, cf.edge_bank(W, H, T[0])[0], cf.random_frame(W, H, 1, seed=11))
    for thr in (-0.5, 0.0, 10.0, 30.0, 45.0):
        n = c.check(np.float32(thr))
        if thr < 0:
            assert n == c.model.G * c.model.plane
    c.plan(packed_templates=c.model.G, byte_templates=0)
    c.close()


def test_features_outside_the_level(oracle):
    """Features beyond the level's cols or rows count in nf and add nothing, in both kernels (the 700-feature template
    skips them inside its first tile)."""
    T, W, H = cf.EDGE_SHAPE
    c = Case(oracle, T, cf.outside_bank(W, H), cf.random_frame(W, H, 1, seed=12))
    for thr in (-1.0, 0.0, 10.0, 20.0, 30.0):
        c.check(np.float32(thr))
    c.plan(packed_templates=2, byte_templates=2)
    c.close()


@pytest.mark.parametrize("mixed", [False, True], ids=["hits", "mixed"])
def test_byte_kernel(oracle, mixed):
    """nf 256 and 257, per-modality counts 62 .. 189 around the 63-feature flush, tiles of 511 / 512 / 513, 8191 hits
    (raw 32 764), unequal P: every template on k_coarse_bytes."""
    T, W, H = cf.EDGE_SHAPE
    c = Case(oracle, T, cf.byte_bank(mixed=mixed), cf.onehot_frame(W, H, 1, cf.BYTE_LABEL))
    thrs = [np.float32(-1.0), np.float32(0.0)]
    for nf, r in zip(c.model.nf, c.model.raw.max(1)):
        thrs += [cf.score(int(r) - 1, int(nf)), cf.score(int(r), int(nf))]
    for thr in sorted(set(thrs)):
        c.check(thr)
    c.plan(packed_templates=0, byte_templates=c.model.G)
    c.close()


@pytest.mark.parametrize("i", range(len(ms.SHAPE_CASES)),
                         ids=["%s-%dx%d" % ("_".join(map(str, c[0])), c[1], c[2]) for c in ms.SHAPE_CASES])
def test_shape_case_coarse(synth, oracle, i):
    """Every SHAPE_CASES frame (lowest T 1 .. 16) at the coarse stage."""
    T, W, H, n, nf, size, thr = ms.SHAPE_CASES[i]
    packed, q, _ = ms.shape_case_data(synth, T, W, H, n, nf, size, thr)
    c = Case.__new__(Case)
    c.oracle, c.T, c.q, c.packed = oracle, list(T), q, packed
    c.model = cf.CoarseModel(oracle, q, T, packed)
    c.nat = lib.NativeDetector(T)
    c.nat.load_bank(packed, cf.M * len(T))
    assert c.check(np.float32(thr)) > 0
    c.check(np.float32(thr - 20), match=False)
    c.close()


@pytest.mark.parametrize("T,W,H", [([4, 8], 640, 480), ([3, 6], 384, 288)])
def test_depth_gate(synth, oracle, T, W, H):
    """The gated kernels: the gated pass mask is the ungated one AND the gate's cell mask (tests/depth_gate_model.py),
    and every gated survivor keeps the ungated raw score.  Bit-sliced and byte-wise templates."""
    import os
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "driver_trace.npz"))
    rgb = np.ascontiguousarray(g["rgb"][:H, :W, ::-1])
    bank = synth.synth_bank(12, num_features=64, levels=len(T), seed=5, size_range=((16, 60), (16, 60)))
    # 150 lowest-level features per modality: 300 in all, beyond the bit-sliced kernel
    wide = synth.synth_bank(4, num_features=300, levels=len(T), seed=6, size_range=((16, 60), (16, 60)))
    bank.classes["02_template"] = wide.classes["01_template"]
    packed = bank.pack(bank.class_ids(), 2 * len(T))
    G = int(packed["class_begin"][-1])
    z = np.random.default_rng(3).choice(np.array([700, 1000, 1500, np.nan], np.float32), G)
    depth = np.kron(np.random.default_rng(7).choice(np.array([650, 1000, 1500], np.uint16), (H // 16 + 1, W // 16 + 1)),
                    np.ones((16, 16), np.uint16))[:H, :W].copy()
    depth[np.random.default_rng(8).random((H, W)) < 0.05] = 0
    nat = lib.NativeDetector(T)
    nat.load_bank(packed, 2 * len(T))
    nat.set_template_depths(0, z)
    thr = 50.0
    nat.match_images(rgb, depth, [], thr)
    assert nat.plan()["gated"] == 0
    m_u, r_u = nat.coarse()
    q = [[nat.quantized(l, m, (H >> l, W >> l)) for m in range(2)] for l in range(len(T))]
    model = cf.CoarseModel(oracle, q, T, packed)
    want_mask, want_raw = model.expected(thr)
    assert np.array_equal(m_u, want_mask) and np.array_equal(r_u, want_raw)
    nat.set_depth_gate(0.15)
    nat.match_images(rgb, depth, [], thr)
    p = nat.plan()
    assert p["gated"] == 1 and p["packed_templates"] == 12 and p["byte_templates"] == 4, p
    m_g, r_g = nat.coarse()
    gate = cf.pack_words(dg.gate_mask(depth, packed["tmeta"], T, z, 0.15).reshape(G, -1), model.nwords)
    assert np.array_equal(m_g, m_u & gate)
    assert np.array_equal(r_g, np.where(model.passes(thr) & dg.gate_mask(depth, packed["tmeta"], T, z, 0.15).reshape(G, -1),
                                        r_u, 0))
    assert 0 < int(np.unpackbits(m_g.view(np.uint8)).sum()) < int(np.unpackbits(m_u.view(np.uint8)).sum())
    nat.close()
