"""Frames given as torch tensors (Detector.match / match_refine / detect / the batch calls, lm_bind_images_device): the
Python side checks them before any library call, so these run without a GPU -- CPU tensors stand in for CUDA ones, whose
placement is checked last.  Also the float depth conversion of k_fe_ingest against the reference driver's host cast."""
import importlib

import numpy as np
import pytest
import torch

pkg = importlib.import_module("6dpose_b200")
lib = importlib.import_module("6dpose_b200._lib")

K = np.eye(3, dtype=np.float32)
H, W = 48, 64


def tframe(depth_dtype=torch.uint16):
    return [torch.zeros((H, W, 3), dtype=torch.uint8), torch.zeros((H, W), dtype=depth_dtype)]


def nframe():
    return [np.zeros((H, W, 3), np.uint8), np.zeros((H, W), np.uint16)]


def calls(det, sources, **kw):
    masks = kw.pop("masks", [])
    yield lambda: det.match(sources, 75.0, [], masks, **kw)
    yield lambda: det.match_refine(sources, 75.0, [], K, masks=masks, **kw)
    yield lambda: det.detect(sources, 75.0, [], K, masks=masks, **kw)
    yield lambda: det.match_refine_batch([sources], 75.0, [], K, masks=[masks] if masks else [], **kw)
    yield lambda: det.detect_batch([sources], 75.0, [], K, masks=[masks] if masks else [], **kw)


def rejects(sources, exc, match, **kw):
    det = pkg.Detector()
    for call in calls(det, sources, **kw):
        with pytest.raises(exc, match=match):
            call()
    assert det._native is None  # no handle was created: no library call


def test_numpy_and_torch_do_not_mix():
    t, n = tframe(), nframe()
    rejects([t[0], n[1]], TypeError, "mix")
    rejects([n[0], t[1]], TypeError, "mix")
    det = pkg.Detector()
    with pytest.raises(TypeError, match="mix"):
        det.detect_batch([tframe(), nframe()], 75.0, [], K)
    with pytest.raises(TypeError, match="masks"):
        det.detect(nframe(), 75.0, [], K, masks=[torch.zeros((H, W), dtype=torch.uint8), None])
    with pytest.raises(TypeError, match="tensors"):
        det.detect(tframe(), 75.0, [], K, masks=[np.zeros((H, W), np.uint8), None])
    assert det._native is None


def test_dtypes_and_shapes():
    rejects([torch.zeros((H, W, 3), dtype=torch.int16), tframe()[1]], TypeError, "uint8")
    rejects([torch.zeros((H, W, 4), dtype=torch.uint8), tframe()[1]], TypeError, "HxWx3")
    rejects([tframe()[0], torch.zeros((H, W), dtype=torch.int32)], TypeError, "uint16")
    rejects([tframe()[0], torch.zeros((H, W), dtype=torch.float64)], TypeError, "float32")
    rejects([tframe()[0], torch.zeros((H, W, 1), dtype=torch.uint16)], TypeError, "HxW")
    rejects([tframe()[0], torch.zeros((H, W + 8), dtype=torch.uint16)], ValueError, "colour image")
    rejects(tframe(), RuntimeError, "mask.size", masks=[torch.zeros((H, W), dtype=torch.int8), None])
    rejects(tframe(), RuntimeError, "mask.size", masks=[None, torch.zeros((H, W - 1), dtype=torch.uint8)])
    rejects(tframe(), RuntimeError, "modalities", masks=[None])


def test_strides():
    big = torch.zeros((H + 3, W + 5, 3), dtype=torch.uint8)
    planar = torch.zeros((3, H, W), dtype=torch.uint8).permute(1, 2, 0)       # strides (W, 1, H*W): not packed
    rejects([planar, tframe()[1]], ValueError, "packed")
    rejects([big[:, ::2], tframe()[1]], ValueError, "packed")                  # every other pixel
    depth_t = torch.zeros((W, H), dtype=torch.uint16).t()                     # column-major
    rejects([tframe()[0], depth_t], ValueError, "packed")
    mask_t = torch.zeros((W, H), dtype=torch.uint8).t()
    rejects(tframe(), ValueError, "packed", masks=[mask_t, None])
    wide = torch.zeros((H, W + 7), dtype=torch.uint8)
    rejects(tframe(), ValueError, "one row pitch", masks=[wide[:, :W], torch.zeros((H, W), dtype=torch.uint8)])
    # crop views with free row pitches pass every check up to the placement (CPU here)
    crop = [big[1:H + 1, 2:W + 2], torch.zeros((H + 1, W + 3), dtype=torch.float32)[:H, 1:W + 1]]
    rejects(crop, ValueError, "cuda:0", depth_scale=0.1)
    rejects(crop, ValueError, "cuda:0", masks=[wide[:, 3:W + 3], wide[:, :W]])


def test_depth_scale_rules():
    f32 = tframe(torch.float32)
    for bad in (0.0, -1.0, float("nan"), float("inf")):
        rejects(f32, ValueError, "depth_scale", depth_scale=bad)
    for bad in ("0.1", None, True):
        rejects(f32, TypeError, "depth_scale", depth_scale=bad)
    rejects(tframe(), ValueError, "float32 depth", depth_scale=0.1)           # u16 depth is mm already
    rejects(nframe(), ValueError, "depth_scale", depth_scale=0.1)             # so is numpy depth
    rejects(f32, ValueError, "cuda:0", depth_scale=0.1)                       # valid: only the placement is left
    rejects(tframe(), ValueError, "cuda:0", depth_scale=1)


def test_placement_and_stream():
    rejects(tframe(), ValueError, "is on cpu")
    rejects(nframe(), TypeError, "stream", stream=object())                  # numpy frames take no stream
    det = pkg.Detector()
    with pytest.raises(ValueError, match="one size"):
        det.detect_batch([nframe(), [np.zeros((H, W + 8, 3), np.uint8), np.zeros((H, W + 8), np.uint16)]], 75.0, [], K)
    assert det._native is None


def depth_model(d, scale):
    """k_fe_ingest's LM_DEPTH_F32 conversion: one float32 product, truncated into [0, 65536), else 0."""
    v = np.asarray(d, np.float32) * np.float32(scale)
    ok = (v >= 0) & (v < 65536)
    return np.where(ok, np.trunc(np.where(ok, v, 0)), 0).astype(np.uint16)


def driver_cast(d, scale):
    """linemod_and_levelup_test.py:315-317: depth *= depth_scale; depth.astype(np.uint16), in float32."""
    depth = np.array(d, np.float32)
    depth *= scale
    return depth.astype(np.uint16)


@pytest.mark.parametrize("scale", [1.0, 0.1, 0.25, 1000.0])
def test_float_conversion_equals_the_driver_in_range(scale):
    rng = np.random.default_rng(3)
    lim = np.float32(65536.0) / np.float32(scale)
    ints = np.arange(0, 65536, dtype=np.float32)
    d = np.concatenate([
        rng.uniform(0, float(lim), 200000).astype(np.float32),
        ints / np.float32(scale),
        np.nextafter(ints / np.float32(scale), np.float32(0)),              # just below an integer (in d)
        np.nextafter(ints, np.float32(0)) / np.float32(scale),
        np.nextafter(np.full(64, lim, np.float32), np.float32(0)) - np.arange(64, dtype=np.float32) * np.float32(lim * 2 ** -23),
        np.float32([0.0, -0.0, 0.9999, 1.9999, 65535.0, 65535.99]),
    ]).astype(np.float32)
    v = d * np.float32(scale)
    keep = (v >= 0) & (v < 65536)
    assert keep.mean() > 0.99
    d = d[keep]
    assert np.array_equal(depth_model(d, scale), driver_cast(d, scale))


def test_float_conversion_out_of_range_is_no_depth():
    d = np.float32([np.nan, -np.nan, -1.0, -1e-30, np.inf, -np.inf, 65536.0, 70000.0, 3e38])
    assert depth_model(d, 1.0).tolist() == [0] * len(d)
    assert depth_model(np.float32([655360.0]), 0.1).tolist() == [0]
    assert depth_model(np.float32([655349.9]), 0.1).tolist() == [65534]
    assert depth_model(np.float32([-0.0, 0.0, 0.99999994]), 1.0).tolist() == [0, 0, 0]
