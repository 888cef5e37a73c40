"""The depth gate of the coarse scan on the device (lm_set_depth_gate): the gated match list equals the gated restatement
(tests/depth_gate_model.py) on the model's mask, field by field with float ==, and lm_depth_gate_stats equals the
model's counts.  Frames go through the GPU front-end (the gate needs the depth image); the restatement reads the label
images the front-end produced."""
import importlib
import os

import numpy as np
import pytest

import depth_gate_model as dg
from test_gpu_detect_batch import batch, data, detector, single  # noqa: F401  (data is a fixture)

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
lib = importlib.import_module("6dpose_b200._lib")
GT_BOX = (331, 130, 65, 64)   # the fixture frame's ground truth, linemodLevelup/test.cpp:86


def _packed(name):
    b = np.load(os.path.join(GOLD, name))
    return dict(class_begin=b["class_begin"], tmeta=b["tmeta"].astype(np.int32), feats=b["feats"].astype(np.int32)), b["T"].tolist()


@pytest.fixture(scope="module")
def fixture():
    g = np.load(os.path.join(GOLD, "driver_trace.npz"))
    bgr = np.ascontiguousarray(g["rgb"][..., ::-1])   # the order cv::imread gave the reference's own test
    depth = g["depth"]
    h = np.load(os.path.join(GOLD, "frame_half_case1.npz"))
    bgr_h, depth_h = bgr.copy(), depth.copy()
    bgr_h.reshape(-1, 3)[h["index"]] = h["bgr"]
    depth_h.reshape(-1)[h["index"]] = h["depth"]
    packed, T = _packed("bank_allScales_full.npz")
    z = np.load(os.path.join(GOLD, "allScales_depths.npz"))["z_mm"]
    nat = lib.NativeDetector(T)
    nat.load_bank(packed, 4)
    nat.set_template_depths(0, z)
    return dict(frames=dict(full=(bgr, depth), half=(bgr_h, depth_h)), packed=packed, T=T, z=z, nat=nat, oracles={},
                exp=np.load(os.path.join(GOLD, "expected_allScales_full.npz")))


def _oracle(nat, T, packed, depth_shape, cache=None, key=None):
    if cache is not None and key in cache:
        return cache[key]
    rows, cols = depth_shape
    q = [[nat.quantized(l, m, (rows >> l, cols >> l)) for m in range(2)] for l in range(len(T))]
    go = dg.GatedOracle(q, T, packed)
    if cache is not None:
        cache[key] = go
    return go


def _same(got, want):
    assert len(got) == len(want), (len(got), len(want))
    for k in ("x", "y", "template_id", "class_index"):
        assert np.array_equal(got[k], want[k]), k
    assert np.array_equal(got["similarity"], want["similarity"])


def _gated(nat, rgb, depth, T, packed, z, thr, tau, cache=None, key=None):
    """One gated frame on the device against the restatement; returns the device's list."""
    nat.set_depth_gate(tau)
    got = nat.match_images(rgb, depth, [], thr)
    go = _oracle(nat, T, packed, depth.shape, cache, key)
    mask = dg.gate_mask(depth, packed["tmeta"], T, z, tau)
    _same(got, go.match(thr, mask))
    assert nat.depth_gate_stats() == dg.gate_stats(mask, go.coarse_pass(thr), depth, T, z)
    return got, go, mask


@pytest.mark.parametrize("thr", [75.0, 80.0])
@pytest.mark.parametrize("tau", [0.0, 0.1, 0.15, 0.5])
def test_fixture_frame_allscales(fixture, thr, tau):
    f = fixture
    rgb, depth = f["frames"]["full"]
    got, go, mask = _gated(f["nat"], rgb, depth, f["T"], f["packed"], f["z"], thr, tau, f["oracles"], "full")
    st = f["nat"].depth_gate_stats()
    assert st["after"] < st["before"] == int(f["exp"]["full_%g_stats" % thr][0]) and st["with_distance"] == 2989


def test_half_occluded_frame(fixture):
    f = fixture
    rgb, depth = f["frames"]["half"]
    _gated(f["nat"], rgb, depth, f["T"], f["packed"], f["z"], 80.0, 0.15, f["oracles"], "half")


def _iou(a, b):
    ax2, ay2, bx2, by2 = a[0] + a[2], a[1] + a[3], b[0] + b[2], b[1] + b[3]
    iw, ih = max(0, min(ax2, bx2) - max(a[0], b[0])), max(0, min(ay2, by2) - max(a[1], b[1]))
    return iw * ih / float(a[2] * a[3] + b[2] * b[3] - iw * ih)


def test_known_answer_first_match_on_the_ground_truth(fixture):
    f = fixture
    rgb, depth = f["frames"]["full"]
    f["nat"].set_depth_gate(0.15)
    got = f["nat"].match_images(rgb, depth, [], 75.0)
    tm = f["packed"]["tmeta"][got["template_id"][0]]
    assert _iou((int(got["x"][0]), int(got["y"][0]), int(tm[0, 0]), int(tm[0, 1])), GT_BOX) >= 0.5
    ungated = f["exp"]["full_75"]
    kept = set(zip(got["x"].tolist(), got["y"].tolist(), got["template_id"].tolist()))
    assert not any((int(m["x"]), int(m["y"]), int(m["template_id"])) in kept for m in ungated[:9])


def test_gate_off_moves_nothing(fixture):
    f = fixture
    nat = f["nat"]
    rgb, depth = f["frames"]["full"]
    want = f["exp"]["full_75"]
    # every band covers the frame's depths: the gated list is the ungated one
    wide = lib.NativeDetector(f["T"])
    wide.load_bank(f["packed"], 4)
    wide.set_template_depths(0, np.full(2989, 1100.0, np.float32))
    assert dg.gate_mask(depth, f["packed"]["tmeta"], f["T"], np.full(2989, 1100.0), 0.99).all()
    wide.set_depth_gate(0.99)
    _same(wide.match_images(rgb, depth, [], 75.0), _as_match(want))
    wide.close()
    # a gated frame, then the gate off: the parent's results and launches
    nat.set_depth_gate(0.15)
    nat.match_images(rgb, depth, [], 75.0)
    nat.set_depth_gate(None)
    n0 = nat.launch_count()
    got = nat.match_images(rgb, depth, [], 75.0)
    _same(got, _as_match(want))
    assert nat.counters()["coarse_candidates"] == int(f["exp"]["full_75_stats"][0])
    plain = lib.NativeDetector(f["T"])
    plain.load_bank(f["packed"], 4)
    m0 = plain.launch_count()
    plain.match_images(rgb, depth, [], 75.0)
    assert nat.launch_count() - n0 == plain.launch_count() - m0
    with pytest.raises(lib.LinemodLibraryError):
        nat.depth_gate_stats()   # the last frame ran ungated
    plain.close()


def _as_match(rec):
    out = np.zeros(len(rec), lib.MATCH_DTYPE)
    for k in ("x", "y", "similarity", "template_id"):
        out[k] = rec[k]
    out["class_index"] = rec["class_idx"]
    return out


def test_state_errors(fixture):
    f = fixture
    rgb, depth = f["frames"]["full"]
    nat = lib.NativeDetector(f["T"])
    nat.load_bank(f["packed"], 4)
    nat.set_depth_gate(0.15)
    with pytest.raises(lib.LinemodLibraryError):   # no distances
        nat.match_images(rgb, depth, [], 75.0)
    nat.set_template_depths(0, f["z"])
    fr = np.load(os.path.join(GOLD, "frames_case1.npz"))
    q = [[fr["full_l%d_m%d" % (l, m)] for m in range(2)] for l in range(2)]
    with pytest.raises(lib.LinemodLibraryError):   # a frame without depth
        nat.match_quantized(q, 75.0)
    nat.load_bank(f["packed"], 4)                 # another bank drops the distances
    with pytest.raises(lib.LinemodLibraryError):
        nat.match_images(rgb, depth, [], 75.0)
    nat.close()


def _synth_depth(seed, rows, cols, B):
    rng = np.random.default_rng(seed)
    d = rng.choice(np.array([650, 800, 1000, 1250, 1500, 1800], np.uint16), size=(rows // B + 1, cols // B + 1))
    d = np.kron(d, np.ones((B, B), np.uint16))[:rows, :cols].copy()
    d += rng.integers(0, 60, (rows, cols)).astype(np.uint16)
    d[rng.random((rows, cols)) < 0.1] = 0
    for _ in range(40):   # whole empty blocks
        y, x = rng.integers(0, rows // B), rng.integers(0, cols // B)
        d[y * B:(y + 1) * B, x * B:(x + 1) * B] = 0
    return d


def _route(fixture, T, rgb, packed, z, thr, seed, taus=(0.15,)):
    nat = lib.NativeDetector(T)
    nat.load_bank(packed, 2 * len(T))
    nat.set_template_depths(0, z)
    rows, cols = rgb.shape[:2]
    depth = _synth_depth(seed, rows, cols, dg.coarse_grid(rows, cols, T)[2])
    cache = {}
    for tau in taus:
        _gated(nat, rgb, depth, T, packed, z, thr, tau, cache, "f")
        st = nat.depth_gate_stats()
        assert st["before"] > st["after"] > 0 and st["empty_cells"] > 0
    nat.close()


def _subset(fixture):
    packed, T = _packed("bank_allScales.npz")   # every 7th template of the 2989
    z = fixture["z"][::7].copy()
    z[::5] = np.nan                             # templates without a distance are never gated
    return packed, T, z


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_synthetic_depths_allscales_subset(fixture, seed):
    packed, T, z = _subset(fixture)
    _route(fixture, T, fixture["frames"]["full"][0], packed, z, 65.0, seed, taus=(0.0, 0.15, 0.5))


ROUTES = {
    "bits_t48": ([4, 8], 480, 640, False),
    "unsafe_t48": ([4, 8], 480, 640, True),      # unsafe templates: the filter hands them to the byte-wise k_refine
    "no_filter_t44": ([4, 4], 480, 648, False),  # Wd = 162 at level 0: k_refine<false>
    "no_filter_tall": ([4, 8], 2064, 640, False),  # Hd = 516 at level 0
}


@pytest.mark.parametrize("route", list(ROUTES))
def test_refinement_routes(fixture, route):
    T, rows, cols, unsafe = ROUTES[route]
    packed, _, z = _subset(fixture)
    if unsafe:
        packed = dict(packed, feats=packed["feats"].copy())
        tm = packed["tmeta"]
        for g in range(0, tm.shape[0], 3):
            packed["feats"][tm[g, 0, 2] + 5, 0] = tm[g, 0, 0] + 6   # a level-0 feature beyond the box
    rgb = fixture["frames"]["full"][0]
    reps = (-(-rows // rgb.shape[0]), -(-cols // rgb.shape[1]), 1)
    rgb = np.ascontiguousarray(np.tile(rgb, reps)[:rows, :cols])
    _route(fixture, T, rgb, packed, z, 65.0, 7)


def test_three_levels_and_the_byte_wise_coarse_kernel(fixture, synth):
    rgb = fixture["frames"]["full"][0]
    # three levels: the filter in front of k_refine<true>, then level 0 byte-wise
    bank = synth.synth_bank(40, num_features=96, levels=3, seed=5)
    packed = bank.pack(bank.class_ids(), 6)
    z = np.random.default_rng(3).choice(np.array([700, 1000, 1500, np.nan], np.float32), int(packed["class_begin"][-1]))
    _route(fixture, [2, 4, 8], rgb, packed, z, 55.0, 11)
    # > 255 features per template: k_coarse_bytes
    bank = synth.synth_bank(30, num_features=300, levels=2, seed=6)
    packed = bank.pack(bank.class_ids(), 4)
    z = np.random.default_rng(4).choice(np.array([700, 1000, 1500, np.nan], np.float32), int(packed["class_begin"][-1]))
    _route(fixture, [4, 8], rgb, packed, z, 55.0, 12)


def test_batch_equals_single_frames(data):
    """detect_batch with the gate on equals detect frame by frame with the gate on."""
    z = np.load(os.path.join(GOLD, "allScales_depths.npz"))["z_mm"]
    frames = [data["frames"][k] for k in ("recorded", "rolled", "mirrored")]
    K = np.repeat(data["sK"][None], len(frames), 0)
    one = detector(data)
    one.set_template_depths(0, z)
    one.set_depth_gate(0.15)
    want = [single(one, fr, K[i], 65.0, 0, 30, False, True) for i, fr in enumerate(frames)]
    many = detector(data)
    many.set_template_depths(0, z)
    many.set_depth_gate(0.15)
    got = batch(many, frames, K, 65.0, 0, 30, False, True)
    for (o, R, t, r, c), (wo, wR, wt, wr, wc) in zip(got, want):
        _same(o, wo)
        assert np.array_equal(R, wR, equal_nan=True) and np.array_equal(t, wt, equal_nan=True) and np.array_equal(r, wr)
        assert c == wc
    assert one.depth_gate_stats()["after"] < one.depth_gate_stats()["before"]
    for n in (one, many):
        n.close()
