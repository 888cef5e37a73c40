"""A short run of the native library for compute-sanitizer's leak check (tools/sanitize.sh, case `leaks`).

Opens a detector, runs detect_batch with the pose stage, the pose NMS and stage timing on, runs one lm_icp_process_batch
on an ICP handle, and closes both handles explicitly.  No torch CUDA tensor is created, so every device allocation left
at exit belongs to this library."""
import importlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
lib = importlib.import_module("6dpose_b200._lib")


def main():
    g = np.load(os.path.join(ROOT, "tests", "golden", "driver_trace.npz"))
    b = np.load(os.path.join(ROOT, "tests", "golden", "bank_allScales_full.npz"))
    packed = dict(class_begin=b["class_begin"], tmeta=b["tmeta"].astype(np.int32), feats=b["feats"].astype(np.int32))
    G = packed["tmeta"].shape[0]
    K = np.repeat(g["rf0_modelK"][None], G, 0).astype(np.float32)
    R = np.repeat(g["rf0_modelR"][None], G, 0).astype(np.float32)
    t = np.repeat(g["rf0_modelT"].reshape(1, 3), G, 0).astype(np.float32)
    sK = g["rf0_sceneK"].astype(np.float32)
    rgb, depth = g["rgb"], g["depth"]

    nat = lib.NativeDetector(b["T"].tolist(), 0)
    nat.load_bank(packed, 4)
    nat.select(None, 0, 1)
    nat.set_template_renders(0, [g["render"]] * G, K, R, t)
    nat.set_timing(2)
    got = nat.detect_batch(np.stack([rgb, rgb]), np.stack([depth, depth]), [[None, None], [None, None]], 75.0,
                           np.stack([sK, sK]), 0.5, 0, 30, False, True)
    nat.close()

    icp = lib.NativeIcp(0)
    Rr, tr, res = icp.process_batch(depth, [g["render"]], sK, K[:1], R[:1], t[:1], np.array([[100, 100]], np.int32))
    icp.close()
    print("frames", len(got), "icp residual", float(res[0]))


if __name__ == "__main__":
    main()
