"""Depths given as torch tensors to poseRefine.process / refine_matches (lm_icp_process_batch_device): the Python side
checks them before any library call, so these run without a GPU -- CPU tensors stand in for CUDA ones, whose placement
is checked last.  Also the C declaration and its ctypes binding, and a numpy restatement of what k_icp_render_box and
k_icp_render_crop compute per render (conversion, box, anchor, crop), held to model_box's semantics."""
import importlib
import os
import re

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
lib = importlib.import_module("6dpose_b200._lib")
pr = importlib.import_module("6dpose_b200.pose_refine")

K = np.eye(3, dtype=np.float32)
H, W = 48, 64


class M:
    x, y = 3, 4


def u16(shape=(H, W)):
    return torch.zeros(shape, dtype=torch.int16).view(torch.uint16)


def calls(scene, renders, **kw):
    n = len(renders)
    if n == 1:
        yield lambda: pr.poseRefine().process(scene, renders[0], K, K, K, np.zeros(3, np.float32), 3, 4, **kw)
    yield lambda: pr.refine_matches(scene, K, [M()] * n, renders, [K] * n, [K] * n, [np.zeros(3, np.float32)] * n, **kw)


def rejects(scene, renders, exc, match, **kw):
    pr._icp.clear()
    for call in calls(scene, renders, **kw):
        with pytest.raises(exc, match=match):
            call()
    assert not pr._icp  # no handle was created: no library call


def test_header_and_binding():
    h = open(os.path.join(ROOT, "include", "linemod_b200.h")).read()
    decl = re.search(r"int lm_icp_process_batch_device\(([^)]*)\);", h)
    assert decl, "lm_icp_process_batch_device is not declared"
    params = [p.strip() for p in decl.group(1).split(",")]
    assert len(params) == 24 and params[-1] == "void* stream" and params[8] == "const void* const* model_depths"
    assert "lm_icp_process_batch_device" in lib.SYMBOLS
    src = open(os.path.join(ROOT, "6dpose_b200", "_lib.py")).read()
    assert "L.lm_icp_process_batch_device.argtypes" in src


def test_numpy_and_torch_do_not_mix():
    n = np.zeros((H, W), np.uint16)
    rejects(u16(), [n], TypeError, "mix")
    rejects(n, [u16()], TypeError, "mix")
    rejects(u16(), [u16(), n], TypeError, "mix")


def test_dtypes_shapes_and_strides():
    rejects(torch.zeros((H, W), dtype=torch.int32), [u16()], TypeError, "uint16")
    rejects(u16(), [torch.zeros((H, W), dtype=torch.float64)], TypeError, "float32")
    rejects(u16((H, W, 1)), [u16()], TypeError, "HxW")
    rejects(u16(), [u16((2, H, W))], TypeError, "HxW")
    rejects(u16(), [u16(), torch.zeros((H, W))], ValueError, "one dtype and size")
    rejects(u16(), [u16(), u16((H, W + 2))], ValueError, "one dtype and size")
    rejects(u16((W, H)).t(), [u16()], ValueError, "packed")
    rejects(u16(), [u16((W, H)).t()], ValueError, "packed")
    with pytest.raises(TypeError, match=r"\[n, H, W\]"):
        pr.refine_matches(u16(), K, [M()], u16((1, 1, H, W)), [K], [K], [np.zeros(3, np.float32)])
    with pytest.raises(TypeError, match="one render per match"):
        pr.refine_matches(u16(), K, [M()] * 2, u16((3, H, W)), [K] * 2, [K] * 2, [np.zeros(3, np.float32)] * 2)
    # crop views with free row pitches, and one [n, H, W] tensor, pass every check up to the placement (CPU here)
    big = u16((H + 3, W + 5))
    rejects(big[1:H + 1, 2:W + 2], [big[:H, :W]], ValueError, "cuda:0")
    rejects(u16(), u16((2, H, W)), ValueError, "cuda:0")
    assert not pr._icp


def test_scales_and_stream():
    f32 = torch.zeros((H, W))
    for bad in (0.0, -1.0, float("nan"), float("inf")):
        rejects(f32, [u16()], ValueError, "depth_scale", depth_scale=bad)
        rejects(u16(), [f32], ValueError, "render_scale", render_scale=bad)
    for bad in ("0.1", None, True):
        rejects(f32, [f32], TypeError, "depth_scale", depth_scale=bad)
    rejects(u16(), [u16()], ValueError, "depth_scale", depth_scale=0.1)          # u16 depth is mm already
    rejects(u16(), [u16()], ValueError, "render_scale", render_scale=0.5)
    n = np.zeros((H, W), np.uint16)
    rejects(n, [n], ValueError, "depth_scale", depth_scale=0.1)                  # so is numpy depth
    rejects(n, [n], ValueError, "render_scale", render_scale=0.1)
    rejects(n, [n], TypeError, "stream", stream=object())                        # numpy depths take no stream
    rejects(f32, [f32], ValueError, "cuda:0", depth_scale=0.1, render_scale=2.0)  # valid: only the placement is left


def test_host_arrays():
    pr._icp.clear()
    z = np.zeros(3, np.float32)
    with pytest.raises(TypeError, match="sceneK"):
        pr.poseRefine().process(u16(), u16(), torch.eye(3), K, K, z, 3, 4)
    with pytest.raises(TypeError, match="modelT"):
        pr.poseRefine().process(u16(), u16(), K, K, K, torch.zeros(3), 3, 4)
    with pytest.raises(TypeError, match="modelRs"):
        pr.refine_matches(u16(), K, [M()], [u16()], [K], [torch.eye(3)], [z])
    assert not pr._icp


# ---- what the render kernels compute, restated ----
def depth_mm(d, scale):
    """lm_depth_mm: u16 as is; float32 d to one float32 product, truncated into [0, 65536), else 0."""
    d = np.asarray(d)
    if d.dtype == np.uint16:
        return d
    v = d.astype(np.float32) * np.float32(scale)
    ok = (v >= 0) & (v < 65536)
    return np.where(ok, np.trunc(np.where(ok, v, 0)), 0).astype(np.uint16)


def model_box(m):
    """lm_icp.cu's model_box: dilate(m > 0, 9x9) + boundingRect, by the dilation itself."""
    rows, cols = m.shape
    nz = m > 0
    dil = np.zeros_like(nz)
    for dy in range(-4, 5):
        for dx in range(-4, 5):
            src = nz[max(0, -dy):rows - max(0, dy), max(0, -dx):cols - max(0, dx)]
            dil[max(0, dy):rows - max(0, -dy), max(0, dx):cols - max(0, -dx)] |= src
    ys, xs = np.nonzero(dil)
    if len(xs) == 0:
        return (0, 0, 0, 0)
    return (int(xs.min()), int(ys.min()), int(xs.max() - xs.min() + 1), int(ys.max() - ys.min() + 1))


def render_entry(render, scale, band=16):
    """k_icp_render_box (extents merged from bands of `band` rows with min / max) + grow_box, then k_icp_render_crop."""
    mm = depth_mm(render, scale)
    rows, cols = mm.shape
    ext = [None, None, -1, -1]
    for r0 in range(0, rows, band):
        ys, xs = np.nonzero(mm[r0:r0 + band])
        if len(xs):
            ext = [min(x for x in (ext[0], int(xs.min())) if x is not None), min(y for y in (ext[1], int(ys.min()) + r0) if y is not None),
                   max(ext[2], int(xs.max())), max(ext[3], int(ys.max()) + r0)]
    box = (0, 0, 0, 0)
    if ext[2] >= 0:
        bx, by = max(ext[0] - 4, 0), max(ext[1] - 4, 0)
        box = (bx, by, min(ext[2] + 4, cols - 1) - bx + 1, min(ext[3] + 4, rows - 1) - by + 1)
    anchor = int(mm[rows // 2, cols // 2])
    crop = mm[box[1]:box[1] + box[3], box[0]:box[0] + box[2]].copy()
    return box, anchor, crop


def edge_renders():
    rng = np.random.default_rng(2)
    out = []
    for shape in ((37, 53), (48, 64), (101, 77), (1, 1), (9, 1)):
        r = np.zeros(shape, np.uint16)
        out.append(r.copy())                                                   # all zero
        r[...] = 0
        r[0, 0] = 5
        out.append(r.copy())                                                   # a corner: clipped at top and left
        r[...] = 0
        r[-1, -1] = 7
        out.append(r.copy())                                                   # clipped at bottom and right
        r = np.where(rng.random(shape) < 0.05, rng.integers(1, 3000, shape), 0).astype(np.uint16)
        out.append(r)                                                          # scattered pixels
    return out


def test_render_entry_equals_model_box():
    g = np.load(os.path.join(ROOT, "tests", "golden", "driver_trace.npz"))
    cases = [g["render"], g["rf1_modelDepth"], np.roll(g["render"], (-180, 57), (0, 1))] + edge_renders()
    for r in cases:
        box, anchor, crop = render_entry(r, 1.0)
        assert box == model_box(r), r.shape
        assert anchor == r[r.shape[0] // 2, r.shape[1] // 2]
        assert crop.shape == (box[3], box[2]) and int((crop > 0).sum()) == int((r > 0).sum())
    box, _, _ = render_entry(g["render"], 1.0)
    assert box == (292, 221, 66, 53)


def test_float_render_entry_is_the_converted_u16_entry():
    g = np.load(os.path.join(ROOT, "tests", "golden", "driver_trace.npz"))
    r = g["render"].astype(np.float32) * np.float32(4.0) + np.float32(1.5)
    r[r < 2] = 0
    r[100, 100] = np.nan                       # no depth: does not grow the box
    r[5, 600] = -3.0
    r[470, 5] = np.inf
    r[240, 300] = 262144.0                     # * 0.25 = 65536: no depth
    u = depth_mm(r, 0.25)
    assert u[100, 100] == u[5, 600] == u[470, 5] == u[240, 300] == 0
    for a, b in zip(render_entry(r, 0.25), render_entry(u, 1.0)):
        assert np.array_equal(a, b)
    assert render_entry(u, 1.0)[0] == model_box(u)
