"""The edge frames of tests/frontend_frames.py certify their own edges, and the rules the GPU front-end restates hold in
cv2 at odd and ragged sizes: pyrDown with BORDER_REFLECT_101, the half-size INTER_NEAREST resize and the 5x5 median at
the image's sides.  CPU only (numpy and cv2)."""
import importlib

import cv2
import numpy as np
import pytest

import frontend_frames as ff
from test_frontend import naive_hysteresis

fe = importlib.import_module("6dpose_b200.frontend")


@pytest.mark.parametrize("masks", ff.MASK_KINDS, ids=str)
@pytest.mark.parametrize("H,W,T", ff.SHAPES, ids=["%dx%d-%s" % (h, w, "_".join(map(str, t))) for h, w, t in ff.SHAPES])
def test_edge_frames_certify_their_edges(H, W, T, masks):
    rgb, depth, mk, counts = ff.edge_frame(H, W, len(T), masks)
    print(H, W, T, masks, counts)
    assert rgb.shape == (H, W, 3) and depth.shape == (H, W)
    if masks is None:
        assert mk is None
    else:
        assert [m is not None for m in mk] == [masks in ("color", "both"), masks in ("depth", "both")]


def test_shapes_put_partial_ctas_and_odd_sources_on_every_kernel():
    facts = {(H, W, tuple(T)): ff.cta_facts(H, W, len(T)) for H, W, T in ff.SHAPES}
    for (H, W, T), f in facts.items():
        lib_rules = [(r % t == 0 and c % t == 0 and r * c % 16 == 0) for (r, c), t in zip(ff.level_dims(H, W, len(T)), T)]
        assert all(lib_rules), (H, W, T)
    assert facts[(45, 80, (5,))][0]["partial_y"] and facts[(55, 80, (5,))][0]["partial_y"]
    assert facts[(65, 80, (5, 8))][1]["odd_source"]
    assert facts[(66, 96, (1, 3, 2, 4))][1]["rows"] == 33 and facts[(66, 96, (1, 3, 2, 4))][2]["odd_source"]
    for key in ((60, 80, (2, 5)), (60, 48, (3, 6))):
        assert facts[key][0]["partial_x"] and facts[key][0]["partial_y"]
    levels = [l for f in facts.values() for l in f]
    assert any(l["partial_x"] and not l["partial_y"] for l in levels)
    assert any(l["partial_y"] and not l["partial_x"] for l in levels)
    assert all(f[0]["ingest_partial"] for f in facts.values())     # no width here is a multiple of 256
    assert (480, 640, (5, 8)) in facts


def naive_votes(q):
    """Winning vote count per interior pixel, with the loop of test_frontend.naive_hysteresis."""
    rows, cols = q.shape
    out = np.zeros((rows, cols), np.int32)
    for r in range(1, rows - 1):
        for c in range(1, cols - 1):
            hist = [0] * 8
            for v in q[r - 1:r + 2, c - 1:c + 2].ravel():
                hist[v] += 1
            out[r, c] = max(hist)
    return out


@pytest.mark.parametrize("H,W", [(45, 80), (66, 96)])
def test_colour_classes_follow_quantize_color(H, W):
    """The parts frontend_frames measures the colour edges with are quantize_color's: same magnitude, same labels, and
    vote counts equal to the naive loop's."""
    rgb = ff.color_image(H, W)
    labels, mag = fe.quantize_color(rgb)
    dx3, dy3, mag3 = ff.color_parts(rgb)
    m, angle = ff._pick(dx3, dy3, mag3, (0, 1, 2))
    assert np.array_equal(m, mag)
    assert np.array_equal(naive_hysteresis(m, angle, 100.0), labels)
    q = ff.bins(angle)
    v = naive_votes(q)
    assert np.array_equal(ff.votes(q), v)
    strong = m > 100
    assert ((v == 5) & strong).sum() >= ff.FLOORS["vote5"] and ((v == 4) & strong).sum() >= ff.FLOORS["vote4"]
    # labelled exactly where the gate passes and the winning bin has 5 or more votes
    assert np.array_equal(labels > 0, strong & (v >= 5))


def test_depth_classes_follow_quantize_depth():
    depth = ff.depth_image(45, 80)
    raw = fe.normals_before_median(depth)
    assert np.array_equal(cv2.medianBlur(raw, 5), fe.quantize_depth(depth))
    assert np.array_equal(ff.median_rank(raw, 13), fe.quantize_depth(depth))


def pyrdown_rule(src):
    """cv::pyrDown to (cols / 2, rows / 2): separable {1, 4, 6, 4, 1}, BORDER_REFLECT_101, (sum + 128) >> 8."""
    H, W = src.shape[:2]
    k = np.array([1, 4, 6, 4, 1], np.int64)
    def refl(p, n):   # BORDER_REFLECT_101 (gfedcb|abcdefgh|gfedcba), periodic with period 2 (n - 1)
        p = np.abs(p) % (2 * (n - 1))
        return np.where(p >= n, 2 * (n - 1) - p, p)

    ys = refl(2 * np.arange(H // 2)[:, None] + np.arange(-2, 3)[None, :], H)      # [Hd, 5]
    xs = refl(2 * np.arange(W // 2)[:, None] + np.arange(-2, 3)[None, :], W)      # [Wd, 5]
    s = src.astype(np.int64)
    rows = np.einsum("j,yjxc->yxc", k, s[ys])                                     # [Hd, W, 3]
    acc = np.einsum("i,yxic->yxc", k, rows[:, xs])                                # [Hd, Wd, 3]
    return ((acc + 128) >> 8).astype(np.uint8)


ODD_SIZES = [(h, w) for h in range(2, 40) for w in range(2, 40)] + [(481, 641), (239, 321), (1001, 77), (33, 997)]


def test_pyrdown_is_reflect101_at_every_size():
    rng = np.random.default_rng(4)
    for H, W in ODD_SIZES:
        src = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
        want = cv2.pyrDown(src, dstsize=(W // 2, H // 2))
        assert np.array_equal(pyrdown_rule(src), want), (H, W)


def test_half_size_nearest_resize_takes_even_rows_and_columns():
    rng = np.random.default_rng(5)
    for H, W in ODD_SIZES:
        a = rng.integers(0, 256, (H, W), dtype=np.uint8)
        got = cv2.resize(a, (W // 2, H // 2), interpolation=cv2.INTER_NEAREST)
        assert np.array_equal(got, a[: H // 2 * 2:2, : W // 2 * 2:2]), (H, W)


def test_median_is_the_13th_of_a_replicated_5x5_window():
    """cv2.medianBlur(labels, 5) == the 13th smallest of each 5x5 BORDER_REPLICATE window, down to one-pixel images."""
    rng = np.random.default_rng(6)
    for H, W in [(h, w) for h in range(1, 14) for w in range(1, 14)] + [(45, 80), (33, 48), (65, 80)]:
        for p in (0.3, 0.5, 0.7):
            a = np.where(rng.random((H, W)) < p, 1 << rng.integers(0, 8, (H, W)), 0).astype(np.uint8)
            assert np.array_equal(ff.median_rank(a, 13), cv2.medianBlur(a, 5)), (H, W, p)
