#!/usr/bin/env python
"""Cost of the pose verification (include/linemod_b200.h, lm_set_pose_verify) on the recorded driver frame
(tests/golden/driver_trace.npz) against the allScales bank, with the shifted per-template renders of
tests/test_gpu_pose_stage.py, through Detector-level detect (front-end, match, box NMS, pose stage of every survivor,
pose NMS):

  k_pose_verify   its device time per frame, from torch.profiler's CUDA activity (a separate profiled run)
  detect          frames/s with verification off and on, three runs of each, alternated off, on, off, on, ...; host
                  clock around whole frames, each ending in a synchronise

Also checks that verification changes no kept pose, and reads the card's name and power limit.

  python tools/pose_verify_probe.py [--frames 200] [--warmup 20] [--threshold 65] [--out FILE]
"""
import argparse
import importlib
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from pose_stage_probe import SHIFTS, card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--threshold", type=float, default=65.0)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this probe only measures on the GPU")
    lib = importlib.import_module("6dpose_b200._lib")
    gold = os.path.join(ROOT, "tests", "golden")
    g = np.load(os.path.join(gold, "driver_trace.npz"))
    b = np.load(os.path.join(gold, "bank_allScales_full.npz"))
    packed = dict(class_begin=b["class_begin"], tmeta=b["tmeta"].astype(np.int32), feats=b["feats"].astype(np.int32))
    G = packed["tmeta"].shape[0]
    renders = [np.ascontiguousarray(np.roll(np.roll(g["render"], dy, 0), dx, 1)) for dy, dx in SHIFTS]
    which = np.arange(G) % len(renders)
    K = np.repeat(g["rf0_modelK"][None], G, 0).astype(np.float32)
    R = np.repeat(g["rf0_modelR"][None], G, 0).astype(np.float32)
    t = np.repeat(g["rf0_modelT"].reshape(1, 3), G, 0).astype(np.float32)
    sK = g["rf0_sceneK"].astype(np.float32)
    rgb, depth, thr = g["rgb"], g["depth"], args.threshold

    nat = lib.NativeDetector(b["T"].tolist(), 0)
    nat.load_bank(packed, 4)
    nat.select(None, 0, 1)
    nat.set_template_renders(0, [renders[k] for k in which], K, R, t)

    def frame(on):
        nat.set_pose_verify(on, 10.0)
        return nat.detect(rgb, depth, None, thr, sK, 0.5, 0, 30, False, 40.0)

    off, on = frame(False), frame(True)
    identical = all(a.tobytes() == c.tobytes() for a, c in zip(off[:4], on[:4]))
    scores = nat.pose_verify()[0]
    for _ in range(args.warmup):
        frame(False)
        frame(True)

    # k_pose_verify's device time, in a run of its own
    n_prof = min(args.frames, 50)
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(n_prof):
            frame(True)
        torch.cuda.synchronize()
    verify_us = [e.device_time for e in prof.events() if "k_pose_verify" in e.name]
    nms_us = [e.device_time for e in prof.events() if "k_pose_nms" in e.name]

    runs = {False: [], True: []}
    for _ in range(3):
        for flag in (False, True):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(args.frames):
                frame(flag)
            runs[flag].append(round(args.frames / (time.perf_counter() - t0), 1))

    results = dict(card=card(), frame="tests/golden/driver_trace.npz", bank="bank_allScales_full (%d templates)" % G,
                   threshold=thr, frames=args.frames, survivors=int(on[4]["survivors"]), posed=int(on[4]["posed"]),
                   kept=int(len(on[0])), kept_scores=[round(float(s), 4) for s in scores], identical_poses=identical,
                   k_pose_verify_us=dict(launches=len(verify_us), mean=round(float(np.mean(verify_us)), 2) if verify_us else None,
                                         max=round(float(np.max(verify_us)), 2) if verify_us else None),
                   k_pose_nms_us=round(float(np.mean(nms_us)), 2) if nms_us else None,
                   detect_frames_per_s=dict(off=runs[False], on=runs[True]))
    line = json.dumps(results)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
