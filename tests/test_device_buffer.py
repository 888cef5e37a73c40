"""The owners of the native library's device memory, pinned memory, streams and events (6dpose_b200/csrc/lm_buffer.h).

A small host program (tests/device_buffer_check.cu) is compiled against the header with the toolkit's compiler.  Without
a device every allocation fails: a failed reserve / assign returns the error and leaves the array empty with size 0, a
failed stream or event owner is empty, and destroying or resetting them is safe.  With a device: reserve keeps the memory
when it fits and never shrinks, assign gives exactly n, a move leaves the source empty, and growing past the device's
whole memory returns cudaErrorMemoryAllocation and leaves the array empty, not holding its old size.

On the detector, the refinement filter's H-planes are reallocated and zeroed whenever their layout changes: neither equal
plane words with a longer tail, nor an equal total size of another layout, reuses the old buffer."""
import importlib
import os
import shutil
import subprocess

import numpy as np
import pytest

import match_shapes as ms

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "6dpose_b200", "csrc")
NVCC = os.environ.get("NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"


def _check_program(tmp_path):
    exe = str(tmp_path / "device_buffer_check")
    subprocess.run([NVCC, "-std=c++17", "-O1", "-gencode", "arch=compute_90a,code=sm_90a", "-I", CSRC,
                    os.path.join(ROOT, "tests", "device_buffer_check.cu"), "-o", exe], check=True, capture_output=True)
    return exe


def _run(exe, mode, env=None):
    r = subprocess.run([exe, mode], capture_output=True, text=True, env=env, timeout=120)
    assert r.returncode == 0 and r.stdout.strip().endswith("OK"), r.stdout + r.stderr


def test_failed_allocations_leave_owners_empty(tmp_path):
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")  # no device: every allocation and creation fails
    _run(_check_program(tmp_path), "nodevice", env)


@pytest.mark.gpu
def test_owners_on_a_device(tmp_path):
    _run(_check_program(tmp_path), "device")


@pytest.mark.parametrize("snippet, compiles", [
    ("PinnedArray<int> a; DeviceArray<int> b; return a.size() ? a[0] : (int)cudaFree(b.get());", True),
    ("DeviceArray<int> a; return a[0];", False),               # host indexing: pinned arrays only
    ("DeviceArray<int> a; return (int)cudaFree(a);", False),   # no conversion to a pointer
])
def test_device_arrays_are_reached_through_get(tmp_path, snippet, compiles):
    src = tmp_path / "use.cu"
    src.write_text('#include "lm_buffer.h"\nint main() { %s }\n' % snippet)
    r = subprocess.run([NVCC, "-std=c++17", "-I", CSRC, "-c", str(src), "-o", str(tmp_path / "use.o")], capture_output=True,
                       text=True)
    assert (r.returncode == 0) == compiles, r.stderr


# (first frame, second frame) of T = [4, 8] whose filter planes (M 8 T^2 nyb Wd words + (nyb + 1) Wd + 64 zero words) differ
# in layout: refined Wd 20 x Hd 64 (nyb 4, tail 164) then Wd 40 x Hd 32 (nyb 2, tail 184), the same plane words; and
# Wd 172 x Hd 112 (nyb 7, 308 224 plane words) then Wd 1200 x Hd 24 (nyb 1, 307 200 plane words), the same 309 664 words
# in all, so that the second frame's zero tail lies where the first frame's planes were
PLANE_PAIRS = [((80, 256), (160, 128)), ((688, 448), (4800, 96))]


@pytest.mark.gpu
@pytest.mark.parametrize("pair", PLANE_PAIRS, ids=["%dx%d-%dx%d" % (a + b) for a, b in PLANE_PAIRS])
def test_filter_planes_follow_the_layout(synth, pair):
    """The filter's H-planes get a new, zeroed buffer whenever their layout changes: the second frame's match list on the
    handle that ran the first equals a fresh handle's."""
    lib = importlib.import_module("6dpose_b200._lib")
    T = [4, 8]
    for W, H in pair:
        assert ms.frame_shape(T, W, H)["filter_ok"], (W, H)
    bank = synth.synth_bank(6, num_features=32, levels=2, seed=21, class_ids=("01_template", "02_template"),
                            size_range=((16, 40), (16, 40)))
    packed = bank.pack(bank.class_ids(), 4)
    frames = [synth.synth_frame(W, H, levels=2, seed=9, bank=bank, plant=4, T=T, border=0)[0] for W, H in pair]
    reused = lib.NativeDetector(T)
    reused.load_bank(packed, 4)
    reused.match_quantized(frames[0], 70.0)
    got = reused.match_quantized(frames[1], 70.0)
    plan = reused.plan()
    reused.close()
    assert plan["filter_ok"] == 1 and plan["filter_templates"] > 0, plan  # the filter takes templates at the second size
    fresh = lib.NativeDetector(T)
    fresh.load_bank(packed, 4)
    want = fresh.match_quantized(frames[1], 70.0)
    fresh.close()
    assert len(want) > 0
    assert np.array_equal(got, want)
