"""The depth gate of the coarse scan without a GPU: the numpy mask against its pixel-by-pixel restatement, the gated match
restatement (tests/depth_gate_model.py) against the oracle, and argument handling of the Python surface and the C-ABI."""
import importlib
import math
import os

import numpy as np
import pytest

import depth_gate_model as dg

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
lib = importlib.import_module("6dpose_b200._lib")
pkg = importlib.import_module("6dpose_b200")


def _tmeta(rng, G, T, rows, cols):
    """Random template sizes at every level; some templates so wide or tall that their sample cell leaves the grid."""
    tm = np.zeros((G, 2 * len(T), 4), np.int32)
    for l in range(len(T)):
        r, c = rows >> l, cols >> l
        tm[:, 2 * l, 0] = rng.integers(0, c + 1, G)
        tm[:, 2 * l, 1] = rng.integers(0, r + 1, G)
        tm[:, 2 * l + 1, :2] = tm[:, 2 * l, :2]
    return tm


def _depth(rng, rows, cols, B):
    """Planes at a few depths, random holes, whole empty blocks, and blocks whose range straddles 1000 mm."""
    d = rng.choice(np.array([600, 800, 1000, 1200, 1800], np.uint16), size=(rows // B + 1, cols // B + 1))
    d = np.kron(d, np.ones((B, B), np.uint16))[:rows, :cols].copy()
    d += rng.integers(0, 40, (rows, cols)).astype(np.uint16)
    d[rng.random((rows, cols)) < 0.2] = 0
    for _ in range(4):
        y, x = rng.integers(0, rows // B), rng.integers(0, cols // B)
        d[y * B:(y + 1) * B, x * B:(x + 1) * B] = 0
    d[:B, :B // 2] = 850
    d[:B, B // 2:B] = 1150
    return d


@pytest.mark.parametrize("seed,T,rows,cols", [(1, [4, 8], 128, 160), (2, [5, 8], 120, 160), (3, [2, 4, 8], 128, 192),
                                              (4, [8], 100, 120), (5, [4, 8], 132, 168)])
def test_mask_equals_the_pixel_definition(seed, T, rows, cols):
    rng = np.random.default_rng(seed)
    G = 24
    tm = _tmeta(rng, G, T, rows, cols)
    _, _, B = dg.coarse_grid(rows, cols, T)
    depth = _depth(rng, rows, cols, B)
    z = rng.choice(np.array([600, 700, 1000, 1150, 1800, np.nan, -5, 0], np.float32), G)
    z[0] = 1000.0
    for tau in (0.0, 0.1, 0.15, 0.5):
        got = dg.gate_mask(depth, tm, T, z, tau)
        want = dg.gate_mask_brute(depth, tm, T, z, tau)
        assert np.array_equal(got, want), tau
        assert 0 < got.sum() < got.size
    _, _, empty = dg.cell_summary(depth, T)
    assert empty.sum() >= 1


def test_band_edges_and_a_single_depth_band():
    # tau = 0: zlo = zhi = z; a cell holding only z + 1 fails, one holding z passes, one straddling z passes
    T = [4, 8]
    depth = np.zeros((32, 64), np.uint16)
    depth[:16, :16] = 1001
    depth[:16, 16:32] = 1000
    depth[:16, 32:40], depth[:16, 40:48] = 990, 1010
    depth[16:, 48:] = 65535
    tm = np.zeros((2, 4, 4), np.int32)
    z = np.array([1000.0, 65535.0], np.float32)
    m = dg.gate_mask(depth, tm, T, z, 0.0)
    assert m[0, 0].tolist() == [False, True, True, True]
    assert m[0, 1].tolist() == [True, True, True, False]
    assert m[1, 1].tolist() == [True, True, True, True]    # 65535 * (1 + tau) clamps to 65535
    assert np.array_equal(m, dg.gate_mask_brute(depth, tm, T, z, 0.0))
    zlo, zhi, has = dg.bands(np.array([1000.0, 0.0, np.nan, 70000.0]), 0.15)
    assert zlo.tolist()[0] == 850 and zhi.tolist()[0] == 1150 and has.tolist() == [True, False, False, True]
    assert zlo[3] == math.ceil(70000 * 0.85) and zhi[3] == 65535


CASES = [([4, 8], 640, 480, 150, 70, 75.0), ([5, 8], 640, 480, 63, 50, 70.0), ([8], 320, 240, 40, 35, 60.0),
         ([2, 4, 8], 640, 512, 96, 35, 70.0), ([4, 8], 320, 256, 32, 3, -1.0)]


def _case(synth, T, W, H, nf, n):
    bank = synth.synth_bank(n, num_features=nf, levels=len(T), seed=21, class_ids=("01_template", "02_template"))
    q, _ = synth.synth_frame(W, H, levels=len(T), seed=9, bank=bank, plant=6, T=T)
    return q, bank.pack(bank.class_ids(), 2 * len(T))


@pytest.mark.parametrize("T,W,H,nf,n,thr", CASES)
def test_all_true_mask_equals_the_oracle(oracle, synth, T, W, H, nf, n, thr):
    q, packed = _case(synth, T, W, H, nf, n)
    go = dg.GatedOracle(q, T, packed)
    want = oracle.match(q, T, packed, thr)
    assert len(want) > 0
    assert np.array_equal(dg.as_oracle_dtype(go.match(thr)), want)
    assert np.array_equal(dg.as_oracle_dtype(go.match(thr, np.ones((go.G, go.Hd, go.Wd), bool))), want)


def test_all_true_mask_equals_the_allscales_golden_lists():
    fr = np.load(os.path.join(GOLD, "frames_case1.npz"))
    b = np.load(os.path.join(GOLD, "bank_allScales_full.npz"))
    packed = dict(class_begin=b["class_begin"], tmeta=b["tmeta"].astype(np.int32), feats=b["feats"].astype(np.int32))
    exp = np.load(os.path.join(GOLD, "expected_allScales_full.npz"))
    go = dg.GatedOracle([[fr["full_l%d_m%d" % (l, m)] for m in range(2)] for l in range(2)], b["T"].tolist(), packed)
    ones = np.ones((go.G, go.Hd, go.Wd), bool)
    for thr in (75.0, 80.0):
        assert np.array_equal(dg.as_oracle_dtype(go.match(thr, ones)), exp["full_%g" % thr]), thr
        assert int(go.coarse_pass(thr).sum()) == int(exp["full_%g_stats" % thr][0])


@pytest.mark.parametrize("T,W,H,nf,n,thr", CASES[:4])
def test_gated_match_equals_the_filtered_ungated_candidates(synth, T, W, H, nf, n, thr):
    """Candidates limited before refinement == every candidate refined, then those outside the mask dropped: each
    candidate's refinement is independent, so the gate may act on the candidate list alone."""
    q, packed = _case(synth, T, W, H, nf, n)
    go = dg.GatedOracle(q, T, packed)
    rng = np.random.default_rng(len(T) * 100 + W)
    _, _, B = dg.coarse_grid(H, W, T)
    depth = _depth(rng, H, W, B)
    z = rng.choice(np.array([600, 800, 1000, 1200, 1800, np.nan], np.float32), go.G)
    mask = dg.gate_mask(depth, packed["tmeta"], T, z, 0.1)
    pre_all = go.presort(thr)
    pre = go.presort(thr, mask)
    naive = pre_all[mask[pre_all["template"], pre_all["cy"], pre_all["cx"]]]
    assert 0 < len(pre) < len(pre_all)
    assert np.array_equal(pre, naive)
    assert np.array_equal(go.finish(pre), go.finish(naive))


# ---- argument handling (no device needed) ----

@pytest.mark.parametrize("bad", [-0.01, 1.0, 1.5, float("nan"), float("inf")])
def test_bad_tolerance_is_refused(bad):
    with pytest.raises(ValueError):
        lib.depth_gate_tolerance(bad)
    nat = lib.NativeDetector([5, 8], device=-1)
    with pytest.raises(RuntimeError):   # LM_E_INVALID from the C-ABI as well
        lib.check(nat._L.lm_set_depth_gate(nat._h, 1, bad))
    with pytest.raises(RuntimeError):
        lib.check(nat._L.lm_set_depth_gate(nat._h, 0, bad))
    nat.close()


def test_tolerance_types():
    for bad in ("0.1", None, True, [0.1]):
        with pytest.raises(TypeError):
            lib.depth_gate_tolerance(bad)
    assert lib.depth_gate_tolerance(0) == 0.0 and lib.depth_gate_tolerance(np.float32(0.5)) == 0.5


def test_host_handle_checks_the_template_range():
    b = np.load(os.path.join(GOLD, "bank_allScales.npz"))
    packed = dict(class_begin=b["class_begin"], tmeta=b["tmeta"], feats=b["feats"].astype(np.int32))
    nat = lib.NativeDetector(b["T"].tolist(), device=-1)
    nat.load_bank(packed, 4)
    G = int(packed["class_begin"][-1])
    nat.set_template_depths(0, np.full(G, 1000.0))
    nat.set_template_depths(G - 2, [700.0, np.nan])
    with pytest.raises(RuntimeError):
        nat.set_template_depths(G - 1, [700.0, 800.0])
    with pytest.raises(RuntimeError):
        nat.set_template_depths(-1, [700.0])
    nat.set_depth_gate(0.15)
    nat.set_depth_gate(None)
    with pytest.raises(lib.LinemodLibraryError):   # LM_E_STATE: no frame ran, let alone a gated one
        nat.depth_gate_stats()
    nat.close()


def test_detector_refuses_bad_depths_before_any_device_work(synth):
    det = pkg.Detector(150, [4, 8])
    det.bank = synth.synth_bank(6, num_features=150, levels=2, seed=3, class_ids=("01_template", "02_template"))
    n = det.bank.num_templates("01_template")
    with pytest.raises(ValueError):
        det.setTemplateDepths({"03_template": np.full(n, 1000.0)})           # unknown class
    with pytest.raises(ValueError):
        det.setTemplateDepths({"01_template": np.full(n + 1, 1000.0)})       # wrong length
    with pytest.raises(RuntimeError):
        det.setDepthGate(0.15)                                               # gate on without distances
    with pytest.raises(ValueError):
        det.setDepthGate(1.0)
    with pytest.raises(TypeError):
        det.setDepthGate("0.15")
    assert det._native is None


def test_distances_from_the_drivers_info_files():
    info = {0: {"cam_t_w2c": [0.0, 0.0, 600.0]}, 2: {"cam_t_w2c": [1.0, 2.0, 1800.0]}, 1: {"cam_t_w2c": [0, 0, 700]}}
    z = pkg.Detector.templateDepthsFromInfo({"06_template": info})
    assert z["06_template"].tolist() == [600.0, 700.0, 1800.0]
    with pytest.raises(ValueError):
        pkg.Detector.templateDepthsFromInfo({"06_template": {0: info[0], 2: info[2]}})
    z = np.load(os.path.join(GOLD, "allScales_depths.npz"))["z_mm"]
    assert z.shape == (2989,) and sorted(set(z.tolist())) == [600, 700, 800, 900, 1000, 1200, 1400, 1600, 1800]
