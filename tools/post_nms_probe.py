"""Device time of the box NMS (k_post_nms) on the reference's fixture frame: allScales bank (427 templates), full
frame, threshold 65 (4 852 kept records), IoU 0.5, for top_k 3 and every survivor.  torch.profiler with CUDA
activities; prints one JSON line with the mean kernel time per launch, the GPU name and its power limit.

    python tools/post_nms_probe.py [--iters 200]"""
import argparse
import importlib
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
GOLD = os.path.join(ROOT, "tests", "golden")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--threshold", type=float, default=65.0)
    args = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    lib = importlib.import_module("6dpose_b200._lib")
    fr = np.load(os.path.join(GOLD, "frames_case1.npz"))
    frame = [[fr["full_l%d_m%d" % (l, m)] for m in range(2)] for l in range(2)]
    b = np.load(os.path.join(GOLD, "bank_allScales.npz"))
    packed = dict(class_begin=b["class_begin"], tmeta=b["tmeta"].astype(np.int32), feats=b["feats"].astype(np.int32))
    nat = lib.NativeDetector(b["T"].tolist(), 0)
    nat.load_bank(packed, 4)
    out = {}
    for top_k in (3, 0):
        for _ in range(10):
            got, nrec = nat.match_top(frame, args.threshold, 0.5, top_k)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.iters):
                nat.match_top(frame, args.threshold, 0.5, top_k)
            torch.cuda.synchronize()
        ts = [e.device_time for e in prof.events() if "k_post_nms" in e.name]
        out["top_k_%d" % top_k] = {"k_post_nms_us": float(np.mean(ts)) if ts else None, "launches": len(ts),
                                   "records": nrec, "survivors": len(got)}
    try:
        out["gpu"] = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                                              "--format=csv,noheader"], text=True).strip()
    except (OSError, subprocess.CalledProcessError):
        out["gpu"] = torch.cuda.get_device_name(0)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
