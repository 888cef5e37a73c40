"""The match pipeline over its shape space: the frame size, the pyramid steps T and the bank decide which kernels run and
how they address memory.  Every case states the route it is meant to take and asserts it through lm_debug_plan
(NativeDetector.plan), then holds the device to the CPU oracle: the match list field by field (similarity with float
==), the coarse candidates, the algorithmic bytes of the coarse scan and of the refinement, and the linear memories of
every level and modality.  Every pyramid step T run here is also pinned oracle == compiled reference, at a small frame,
by tests/golden/shape_checks.npz (tests/match_shapes.py, SHAPE_CASES) or reference_checks.npz.

Which case covers which boundary (numbers from match_shapes.frame_shape; Wd x Hd = positions of a level):
  every T             SHAPE_CASES: lowest T 1..16 ([1], [1,2], [3,3], [2,4], [2,5], [3,6], [7,7], [4,8], [2,9], [5,10],
                      [4,11], [6,12], [8,13], [7,14], [5,15], [8,16], [16,16], [16]); refined T 1..8; odd T at both
                      levels ([3,3], [7,7]) and refined ([3,6], [5,10], [5,15], [7,14], [2,3,6], [1,3,2,4])
  K1 band / not       [6,8] 384x384 band | 672x480 not, only because the lowest Wd = 42 is not a multiple of 4;
                      [16] 2048x320 band (11 544 B of shared memory) | 2368x320 not, only because Wd = 148 = 4 x 37 leaves one
                      segment per row: 186 264 B > LM_BAND_SMEM_LIMIT
  pseg (planes mode)  32: [1,2] 160x128 (Wd 160) | 16: [2,4] 288x256 (Wd 144) | 8: [3,6] 384x288 | 4: [5,10] 320x240
  rounds              [4,8] 1280x1024: 80 x 64 = 5120 positions, 160 words, 5 rounds, bit-planes |
                      1296x1024: 81 x 64, 162 words, 6 rounds: no bit-planes, every template on k_coarse_bytes
  K2 bit-planes       [4,8] 640x624: 40 x 39, 204 032 B staged in shared memory | 640x640: 40 x 40, 209 152 B from global
                      (LM_BITS_SMEM_LIMIT = 200 KiB decides; the rest of LM_K2_SMEM_MAX holds the teams' counters)
  split S             [4,8] 1280x960, S = 8, 4, 2, 1: the smallest bank whose task count reaches that team size on this GPU
  filter Wd           [8,16] 128x128: refined Wd = 16, filter on | 96x128: Wd = 12, refused (k_refine<false>).  The
                      Wd = 16 side checks the host predicate, the filter's launch with no eligible template and the
                      hand-over of every candidate to k_refine<true>, not the filter's addressing at that width: a
                      template is eligible only if cols >= width + 16 T at the refined level, which Wd = 16 leaves no
                      room for, and no position there can be refined to a match.  The narrowest refined level the
                      filter and k_refine_bits take whole here is Wd = 32 ([16,16] 512x512).
  filter 2^23         [8,16] 4064x2048: 8 331 772 plane words + tail, filter on, bit-sliced refinement |
                      4096x2048: 8 397 376 > 2^23, refused (k_refine<false>)
  refinement kernels  two levels: k_refine_filter_w + k_refine_bits; three ([2,3,6]) and four ([1,3,2,4]) levels:
                      k_refine_filter_w + k_refine<true>; refused filter: k_refine<false>; one level: k_refine<false>
  depth gate          [3,6] 384x288 and [7,14] 448x336 through the GPU front-end, against tests/depth_gate_model.py
"""
import importlib
import os

import numpy as np
import pytest

import depth_gate_model as dg
import match_shapes as ms

pytestmark = pytest.mark.gpu
lib = importlib.import_module("6dpose_b200._lib")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_SYNTH_T = [[4, 8], [5, 8], [8], [2, 4, 8]]   # pinned by reference_checks.npz
NPROC = os.cpu_count() or 1

# the route of a two-level frame the filter takes whole: planes-mode K1, filter, bit-sliced refinement, nothing else
BITS = dict(filter_ok=1, use_bits=1, refine_filtered_items=-1, refine_items=-1)
UPPER = dict(filter_ok=1, use_bits=0, planes_level=-1, refine_bits_items=-1, refine_items=-1)   # >= 3 levels
REFUSED = dict(filter_ok=0, use_bits=0, planes_level=-1, filter_items=-1, refine_bits_items=-1, refine_filtered_items=-1)
SINGLE = dict(filter_ok=0, use_bits=0, planes_level=-1, filter_items=-1, refine_bits_items=-1, refine_filtered_items=-1)

# (T, W, H) of a SHAPE_CASES entry -> the plan it reaches
SHAPE_PLANS = {
    ((1, 2), 160, 128): dict(BITS, k1_band=1, planes_level=0, pseg=32, rounds=2, bit_planes=1, k2_smem=1),
    ((2, 4), 288, 256): dict(BITS, k1_band=1, planes_level=0, pseg=16, rounds=2, bit_planes=1),
    ((2, 5), 320, 240): dict(BITS, k1_band=1, planes_level=0, pseg=32, bit_planes=1),
    ((2, 9), 288, 288): dict(BITS, k1_band=1, planes_level=0, pseg=16, rounds=1),
    ((3, 3), 192, 192): dict(BITS, k1_band=1, planes_level=0, pseg=8, rounds=1),
    ((3, 6), 384, 288): dict(BITS, k1_band=1, planes_level=0, pseg=8),
    ((4, 11), 352, 352): dict(BITS, k1_band=1, planes_level=0, pseg=8),
    ((5, 10), 320, 240): dict(BITS, k1_band=1, planes_level=0, pseg=4),
    ((5, 15), 480, 480): dict(BITS, k1_band=1, planes_level=0, pseg=4),
    ((6, 8), 672, 480): dict(BITS, k1_band=0, planes_level=-1, pseg=0),
    ((6, 8), 384, 384): dict(BITS, k1_band=1, planes_level=0, pseg=4),
    ((6, 12), 384, 384): dict(BITS, k1_band=1, planes_level=0, pseg=4),
    ((7, 7), 448, 336): dict(BITS, k1_band=1, planes_level=0, pseg=4),
    ((7, 14), 448, 336): dict(BITS, k1_band=1, planes_level=0, pseg=4),
    ((8, 13), 416, 416): dict(BITS, k1_band=1, planes_level=0, pseg=4),
    ((8, 16), 384, 384): dict(BITS, k1_band=1, planes_level=0, pseg=4),
    ((16, 16), 512, 512): dict(BITS, k1_band=1, planes_level=0, pseg=4),
    ((1,), 64, 64): dict(SINGLE, k1_band=1, rounds=4, bit_planes=1),
    ((16,), 512, 320): dict(SINGLE, k1_band=1, rounds=1, bit_planes=1),
    ((2, 3, 6), 384, 288): dict(UPPER, k1_band=1),
    ((1, 3, 2, 4), 384, 384): dict(UPPER, k1_band=1),
}

# routes on frames beyond the reference's (or too large for a fixture): (name, T, W, H, templates, features, size, thr, plan)
DEFAULT_SIZE = ((20, 126), (24, 142))
ROUTES = [
    ("rounds5", [4, 8], 1280, 1024, 4, 64, DEFAULT_SIZE, 75.0,
     dict(BITS, rounds=5, bit_planes=1, byte_templates=0, k2_smem=0)),
    ("rounds6", [4, 8], 1296, 1024, 4, 64, DEFAULT_SIZE, 75.0,
     dict(rounds=6, bit_planes=0, packed_templates=0, byte_templates=8, k2_smem=-1, split=-1, k1_band=0, filter_ok=1,
          use_bits=1)),
    ("k2_shared", [4, 8], 640, 624, 10, 64, DEFAULT_SIZE, 75.0, dict(BITS, bit_planes=1, k2_smem=1, plane_bytes=204032)),
    ("k2_global", [4, 8], 640, 640, 10, 64, DEFAULT_SIZE, 75.0, dict(BITS, bit_planes=1, k2_smem=0, plane_bytes=209152)),
    ("k1_band_t16", [16], 2048, 320, 6, 64, ((16, 120), (16, 120)), 70.0, dict(SINGLE, k1_band=1)),
    ("k1_smem_limit_t16", [16], 2368, 320, 6, 64, ((16, 120), (16, 120)), 70.0, dict(SINGLE, k1_band=0, k1_smem=186264)),
    ("filter_wd16", [8, 16], 128, 128, 4, 32, ((8, 24), (8, 24)), 50.0, dict(filter_ok=1, use_bits=1, planes_level=-1,
                                                                              filter_templates=0, refine_items=-1)),
    ("filter_wd12", [8, 16], 96, 128, 4, 32, ((8, 24), (8, 24)), 50.0, dict(REFUSED)),
    ("filter_words_under", [8, 16], 4064, 2048, 4, 64, DEFAULT_SIZE, 75.0, dict(BITS, bit_planes=0, byte_templates=8)),
    ("filter_words_over", [8, 16], 4096, 2048, 4, 64, DEFAULT_SIZE, 75.0, dict(REFUSED, bit_planes=0)),
]
# frames on which no template can be refined to a match: every position lies within 8 T of a side at the refined level
NO_MATCH_ROUTES = {"filter_wd16", "filter_wd12"}


def _pinned(T):
    return T in REF_SYNTH_T or any(T == c[0] for c in ms.SHAPE_CASES)


def _same(got, want):
    assert len(got) == len(want), (len(got), len(want))
    for k in ("x", "y", "template_id"):
        assert np.array_equal(got[k], want[k]), k
    assert np.array_equal(got["class_index"], want["class_idx"])
    assert np.array_equal(got["similarity"], want["similarity"])


def _check_plan(plan, want, n_templates, shape):
    for k, v in want.items():
        assert plan[k] == v, (k, plan[k], v, plan)
    # the plan's own arithmetic against frame_shape
    assert plan["rounds"] == shape["rounds"] and plan["bit_planes"] == int(shape["bit_planes"])
    assert plan["filter_ok"] == int(shape["filter_ok"])
    k1 = shape["k1_planes"] if plan["planes_level"] >= 0 else shape["k1"]
    assert plan["k1_band"] == int(k1["band"]) and plan["k1_smem"] == k1["smem"] and plan["pseg"] == k1["pseg"]
    assert plan["packed_templates"] + plan["byte_templates"] == n_templates
    if plan["packed_templates"] > 0:
        assert plan["plane_bytes"] == shape["plane_bytes"] and plan["k2_smem"] == int(shape["k2_smem"])
    ran = [plan[k] for k in ("filter_items", "refine_bits_items", "refine_filtered_items", "refine_items")]
    assert any(v >= 0 for v in ran), plan


def _run(T, W, H, packed, q, thr, want_plan):
    shape = ms.frame_shape(T, W, H)
    nat = lib.NativeDetector(T)
    nat.load_bank(packed, 2 * len(T))
    got = nat.match_quantized(q, thr)
    n = int(packed["class_begin"][-1])
    plan = nat.plan()
    _check_plan(plan, want_plan, n, shape)
    want, st = oracle_match(q, T, packed, thr, W * H)
    _same(got, want)
    c = nat.counters()
    assert c["coarse_candidates"] == int(st["coarse_candidates"]) > 0
    assert c["scan_bytes"] == int(st["coarse_byte_adds"])
    assert c["refine_bytes"] == int(st["refine_byte_adds"])
    cand = c["coarse_candidates"]
    if plan["filter_items"] >= 0:
        assert plan["filter_items"] == cand
    if plan["refine_items"] >= 0:
        assert plan["refine_items"] == cand
    for k in ("refine_bits_items", "refine_filtered_items"):
        assert plan[k] <= cand
    for l, t in enumerate(T):
        for m in range(2):
            ref = ms_oracle().linear_memories(q[l][m], t)
            assert np.array_equal(nat.linear_memories(l, m, ref.shape), ref), (l, m)
    nat.close()
    return got, want, plan


_oracle = None


def ms_oracle():
    global _oracle
    if _oracle is None:
        from oracle import oracle
        oracle.build()
        _oracle = oracle
    return _oracle


def oracle_match(q, T, packed, thr, pixels):
    # large frames take every host core (their oracle time is not small); small ones one
    return ms_oracle().match(q, T, packed, thr, n_threads=NPROC if pixels > 1 << 20 else 1, want_stats=True)


@pytest.mark.parametrize("i", range(len(ms.SHAPE_CASES)),
                         ids=["%s-%dx%d" % ("_".join(map(str, c[0])), c[1], c[2]) for c in ms.SHAPE_CASES])
def test_shape_case(synth, i):
    T, W, H, n, nf, size, thr = ms.SHAPE_CASES[i]
    plan = SHAPE_PLANS[(tuple(T), W, H)]
    packed, q, planted = ms.shape_case_data(synth, T, W, H, n, nf, size, thr)
    got, want, p = _run(T, W, H, packed, q, thr, plan)
    assert len(planted) > 0 and len(want) > 0
    # the same list the compiled reference gave (shape_checks.npz)
    assert np.array_equal(np.load(ms.SHAPE_CHECKS)["case_%d" % i], want)
    if p["use_bits"] and p["filter_templates"] == n * 2:
        assert p["refine_bits_items"] >= len(want)


def test_shape_plans_cover_every_case():
    assert set(SHAPE_PLANS) == {(tuple(c[0]), c[1], c[2]) for c in ms.SHAPE_CASES}
    assert {c[0][-1] for c in ms.SHAPE_CASES} == set(range(1, 17))
    assert {t for c in ms.SHAPE_CASES for t in c[0][:-1]} >= set(range(1, 9))


@pytest.mark.parametrize("route", ROUTES, ids=[r[0] for r in ROUTES])
def test_route(synth, route):
    name, T, W, H, n, nf, size, thr, plan = route
    assert _pinned(T)
    bank = synth.synth_bank(n, num_features=nf, levels=len(T), seed=21, class_ids=("01_template", "02_template"),
                            size_range=size)
    q, planted = synth.synth_frame(W, H, levels=len(T), seed=9, bank=bank, plant=4, T=T, border=0)
    got, want, p = _run(T, W, H, bank.pack(bank.class_ids(), 2 * len(T)), q, thr, plan)
    if name == "filter_wd16":   # no eligible template: the filter hands every candidate to k_refine<true>
        assert p["refine_bits_items"] == 0 and p["refine_filtered_items"] == p["filter_items"] > 0, p
    if name not in NO_MATCH_ROUTES:
        assert len(planted) > 0 and len(want) > 0


def _words(packed, T, W, H):
    """Position words per template at the lowest level (prepare_bank's template_positions, in 32-position words)."""
    s = ms.frame_shape(T, W, H)
    tm = np.asarray(packed["tmeta"]).reshape(len(packed["tmeta"]), -1, 4)
    TL, Wd, Hd = T[-1], s["Wd"], s["Hd"]
    slot = 2 * (len(T) - 1)
    wf = (tm[:, slot, 0] - 1) // TL + 1
    hf = (tm[:, slot, 1] - 1) // TL + 1
    P = (Hd - hf) * Wd + (Wd - wf) + 1
    return np.minimum(np.maximum((P + 31) // 32, 1), s["words"]).astype(np.int32), s["plane_bytes"]


@pytest.mark.parametrize("split", [8, 4, 2, 1])
def test_coarse_split(synth, split):
    import torch
    T, W, H = [4, 8], 1280, 960
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    # synth_bank(k) is the first k templates of synth_bank(N): the smallest k whose tasks give this team size
    big = synth.synth_bank(5 * sm, num_features=64, levels=2, seed=5)
    words, plane_bytes = _words(big.pack(big.class_ids(), 4), T, W, H)
    S = [lib.coarse_tasks(words[:k], sm, plane_bytes)[3]["split"] for k in range(1, len(words) + 1)]
    assert S[-1] == 1
    k = 4 + S[3:].index(split)
    bank = synth.synth_bank(k, num_features=64, levels=2, seed=5)
    q, planted = synth.synth_frame(W, H, levels=2, seed=13, bank=bank, plant=4, T=T, border=0)
    got, want, p = _run(T, W, H, bank.pack(bank.class_ids(), 4), q, 75.0,
                        dict(BITS, split=split, packed_templates=k, byte_templates=0, k2_smem=0))
    assert len(planted) > 0 and len(want) > 0


def _synth_depth(seed, rows, cols, B):
    rng = np.random.default_rng(seed)
    d = rng.choice(np.array([650, 800, 1000, 1250, 1500, 1800], np.uint16), size=(rows // B + 1, cols // B + 1))
    d = np.kron(d, np.ones((B, B), np.uint16))[:rows, :cols].copy()
    d += rng.integers(0, 60, (rows, cols)).astype(np.uint16)
    d[rng.random((rows, cols)) < 0.1] = 0
    return d


@pytest.mark.parametrize("T,W,H", [([3, 6], 384, 288), ([7, 14], 448, 336)])
def test_depth_gate_at_new_steps(synth, T, W, H):
    """The gated kernels (k_depth_cells, k_coarse_packed<., true>) at pyramid steps other than [4, 8] and [5, 8]."""
    assert _pinned(T)
    g = np.load(os.path.join(ROOT, "tests", "golden", "driver_trace.npz"))
    rgb = np.ascontiguousarray(g["rgb"][:H, :W, ::-1])   # BGR, the order cv::imread gives
    bank = synth.synth_bank(20, num_features=64, levels=len(T), seed=5, size_range=((16, 60), (16, 60)))
    packed = bank.pack(bank.class_ids(), 2 * len(T))
    z = np.random.default_rng(3).choice(np.array([700, 1000, 1500, np.nan], np.float32), int(packed["class_begin"][-1]))
    depth = _synth_depth(7, H, W, dg.coarse_grid(H, W, T)[2])
    nat = lib.NativeDetector(T)
    nat.load_bank(packed, 2 * len(T))
    nat.set_template_depths(0, z)
    nat.set_depth_gate(0.15)
    got = nat.match_images(rgb, depth, [], 55.0)
    plan = nat.plan()
    assert plan["gated"] == 1 and plan["packed_templates"] == 20 and plan["use_bits"] == 1, plan
    q = [[nat.quantized(l, m, (H >> l, W >> l)) for m in range(2)] for l in range(len(T))]
    go = dg.GatedOracle(q, T, packed)
    mask = dg.gate_mask(depth, packed["tmeta"], T, z, 0.15)
    want = go.match(55.0, mask)
    _same(got, dg.as_oracle_dtype(want))
    st = nat.depth_gate_stats()
    assert st == dg.gate_stats(mask, go.coarse_pass(55.0), depth, T, z)
    assert st["before"] > st["after"] > 0 and len(want) > 0
    for l, t in enumerate(T):
        for m in range(2):
            ref = ms_oracle().linear_memories(q[l][m], t)
            assert np.array_equal(nat.linear_memories(l, m, ref.shape), ref), (l, m)
    nat.close()
