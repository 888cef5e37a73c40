"""The GPU quantization front-end (lm_upload_images, lm_bind_images_device) against cv2 (6dpose_b200/frontend.py) on the
edge frames of tests/frontend_frames.py: frames that put pixels exactly on the gradient gate, the channel pick's ties,
the 5-vote hysteresis, the normals' distance and difference thresholds, the median's 13th element, the normals' rim and
every kind of mask, at frame sizes that leave partial CTAs and odd pyramid sources (frontend_frames.SHAPES, checked by
tests/test_frontend_edges_cpu.py).  Every label image of every level and modality must equal cv2's bit for bit; a
failure names the level, the modality, the first differing pixel and the edge classes it belongs to."""
import functools
import importlib

import numpy as np
import pytest
import torch

import frontend_frames as ff

pytestmark = pytest.mark.gpu
lib = importlib.import_module("6dpose_b200._lib")
fe = importlib.import_module("6dpose_b200.frontend")
synth = importlib.import_module("6dpose_b200.synth")

SHAPE_IDS = ["%dx%d-%s" % (h, w, "_".join(map(str, t))) for h, w, t in ff.SHAPES]
DEVICE_SHAPES = [(45, 80, [5]), (66, 96, [1, 3, 2, 4]), (480, 640, [5, 8])]   # widths 80, 96, 640: partial ingest rows


@functools.lru_cache(maxsize=None)
def frame(H, W, levels, masks):
    return ff.edge_frame(H, W, levels, masks)


@functools.lru_cache(maxsize=None)
def detector(T):
    return lib.NativeDetector(list(T))


def assert_labels(nat, rgb, depth, masks, levels):
    want = fe.quantize_pyramid([rgb, depth], levels, masks)
    for l in range(levels):
        for m in range(2):
            w = want[l][m]
            got = nat.quantized(l, m, w.shape)
            bad = np.argwhere(got != w)
            if len(bad):
                y, x = (int(v) for v in bad[0])
                pytest.fail("level %d %s (%dx%d): %d pixels differ; first at (y=%d, x=%d): gpu %d, cv2 %d; classes %s" % (
                    l, ("colour", "normals")[m], w.shape[0], w.shape[1], len(bad), y, x, got[y, x], w[y, x],
                    ff.pixel_classes(rgb, depth, masks, l, m, y, x)))
    return want


@pytest.mark.parametrize("masks", ff.MASK_KINDS, ids=str)
@pytest.mark.parametrize("H,W,T", ff.SHAPES, ids=SHAPE_IDS)
def test_host_frame_labels_equal_cv2(H, W, T, masks):
    rgb, depth, mk, _ = frame(H, W, len(T), masks)
    nat = detector(tuple(T))
    nat.upload_images(rgb, depth, mk)
    want = assert_labels(nat, rgb, depth, mk, len(T))
    if mk is not None:   # the masks leave labels at every level
        assert all((w[m] > 0).any() for w in want for m in range(2))


def cuda(a, crop=False):
    """A CUDA tensor holding numpy image a; crop: a view into a larger tensor whose row pitch is no multiple of 16 bytes."""
    a = np.ascontiguousarray(a)
    src = torch.from_numpy(a.view(np.int16) if a.dtype == np.uint16 else a).cuda()
    if a.dtype == np.uint16:
        src = src.view(torch.uint16)
    if not crop:
        return src
    H, W = a.shape[:2]
    big = torch.zeros((H + 3, W + 5) + a.shape[2:], dtype=src.dtype, device=src.device)
    view = big[1:H + 1, 2:W + 2]
    view.copy_(src)
    return view


def depth_mm(d, scale):
    """lm_depth_mm (lm_depth.cuh): one float32 product, truncated; 0 outside [0, 65536)."""
    v = np.asarray(d, np.float32) * np.float32(scale)
    ok = (v >= 0) & (v < 65536)
    return np.where(ok, np.trunc(np.where(ok, v, 0)), 0).astype(np.uint16)


def float_depth(depth, scale, seed):
    """Float32 depth that lm_depth_mm maps back to `depth` (scale a power of two): fractions below one mm on a tenth of
    the pixels, and NaN, infinities, negatives and products >= 65536 where the depth is 0."""
    rng = np.random.default_rng(seed)
    d = depth.astype(np.float32) / np.float32(scale)
    frac = rng.random(depth.shape) < 0.1
    d = np.where(frac & (depth > 0), d + np.float32(0.75) / np.float32(scale), d).astype(np.float32)
    bad = np.float32([np.nan, np.inf, -np.inf, -1.0, 65536.0 / scale, 1e30, 0.0])
    holes = depth == 0
    d[holes] = bad[np.arange(int(holes.sum())) % len(bad)]
    return d


@pytest.mark.parametrize("crop", [False, True], ids=["packed", "pitched"])
@pytest.mark.parametrize("fmt", ["u16", "f32"])
@pytest.mark.parametrize("H,W,T", DEVICE_SHAPES, ids=["%dx%d" % s[:2] for s in DEVICE_SHAPES])
def test_device_frame_labels_equal_cv2(H, W, T, fmt, crop):
    rgb, depth, mk, _ = frame(H, W, len(T), "both")
    assert ff.cta_facts(H, W, len(T))[0]["ingest_partial"]
    if fmt == "u16":
        d, scale, want_depth = cuda(depth, crop), 1.0, depth
    else:
        scale = 4.0
        f = float_depth(depth, scale, H + W)
        want_depth = depth_mm(f, scale)
        assert np.array_equal(want_depth, depth)          # the frame's certified edges survive the conversion
        d = cuda(f, crop)
    r, m = cuda(rgb, crop), [cuda(x, crop) for x in mk]
    if crop:
        assert r.stride(0) % 16 and (d.stride(0) * d.element_size()) % 16 and m[0].stride(0) % 16
    nat = detector(tuple(T))
    nat.set_frame(r, d, m, depth_scale=scale)
    torch.cuda.synchronize()
    assert np.array_equal(nat.depth_image(depth.shape), want_depth)
    assert_labels(nat, rgb, want_depth, mk, len(T))


# (H, W, T, masks, templates, features, threshold): ragged frames on which the synthetic bank has matches
MATCH_CASES = [(45, 80, [5], "both", 60, 24, 40.0), (60, 80, [2, 5], None, 60, 24, 40.0)]


@pytest.mark.parametrize("case", MATCH_CASES, ids=["%dx%d" % c[:2] for c in MATCH_CASES])
def test_match_images_equals_the_oracle_on_cv2_labels(oracle, case):
    H, W, T, masks, n, nf, thr = case
    rgb, depth, mk, _ = frame(H, W, len(T), masks)
    bank = synth.synth_bank(n, num_features=nf, levels=len(T), seed=3, class_ids=("01_template", "02_template"),
                            size_range=((8, 24), (8, 24)))
    packed = bank.pack(bank.class_ids(), 2 * len(T))
    nat = lib.NativeDetector(T)
    nat.load_bank(packed, 2 * len(T))
    got = nat.match_images(rgb, depth, mk, thr)
    want = oracle.match(fe.quantize_pyramid([rgb, depth], len(T), mk), T, packed, thr)
    assert len(want) > 0 and len(got) == len(want), (len(got), len(want))
    for k in ("x", "y", "template_id", "similarity"):
        assert np.array_equal(got[k], want[k]), k
    assert np.array_equal(got["class_index"], want["class_idx"])
    nat.close()
