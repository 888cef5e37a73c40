#!/usr/bin/env python
"""Frame rate of the drivers' whole loop -- front-end, match, NMS/top-k, poseRefine of the survivors -- on the recorded
driver frame (tests/golden/driver_trace.npz) against the allScales bank, along two paths:

  host hand-off  upload_images + enqueue + enqueue_post + complete_post (what lm_match_top does on the device), then
                 lm_icp_process_batch with one full-frame render per survivor (clouds built on the host)
  device chain   the same front-end, match and NMS, then lm_enqueue_pose + lm_complete_pose (renders registered once)

at top_k = 3 and at every survivor.  Per path: frames/s (host clock around whole frames, each ending in a synchronise),
the pose stage's time (device chain: CUDA events around its kernels on the detector's stream; host hand-off: host clock
around lm_icp_process_batch, which includes its cloud building, and the device time of its kernels), and kernel
launches per frame.  Also checks that both paths return identical poses, and reads the card's name and power limit.

  python tools/pose_stage_probe.py [--frames 200] [--warmup 20] [--threshold 75] [--out FILE]
"""
import argparse
import importlib
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SHIFTS = [(0, 0), (-68, -19), (-180, 57), (3, -2), (-2, 4)]  # the per-template renders of tests/test_gpu_pose_stage.py


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    if q.returncode != 0:
        raise RuntimeError("nvidia-smi failed: %s" % q.stderr.strip())
    name, power, clock = [s.strip() for s in q.stdout.strip().split(",")]
    return dict(name=name, power_limit=power, max_sm_clock=clock)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--threshold", type=float, default=75.0)
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
    T = b["T"].tolist()
    G = packed["tmeta"].shape[0]
    renders = [np.ascontiguousarray(np.roll(np.roll(g["render"], dy, 0), dx, 1)) for dy, dx in SHIFTS]
    which = np.arange(G) % len(renders)
    K = np.repeat(g["rf0_modelK"][None], G, 0).astype(np.float32)
    R = np.repeat(g["rf0_modelR"][None], G, 0).astype(np.float32)
    t = np.repeat(g["rf0_modelT"].reshape(1, 3), G, 0).astype(np.float32)
    sK = g["rf0_sceneK"].astype(np.float32)
    rgb, depth, thr = g["rgb"], g["depth"], args.threshold

    nat = lib.NativeDetector(T, 0)
    nat.load_bank(packed, 4)
    nat.select(None, 0, 1)
    nat.set_template_renders(0, [renders[k] for k in which], K, R, t)
    icp = lib.NativeIcp(0)
    stream = torch.cuda.ExternalStream(nat.stream())
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def host_frame(top_k):
        nat.upload_images(rgb, depth, None)
        nat.enqueue(thr)
        nat.enqueue_post(0.5, top_k)
        surv, _ = nat.complete_post()
        tid = surv["template_id"].astype(np.int64)
        t0 = time.perf_counter()
        out = icp.process_batch(depth, [renders[k] for k in which[tid]], sK, K[tid], R[tid], t[tid],
                                np.stack([surv["x"], surv["y"]], 1), 30)
        return surv, out, time.perf_counter() - t0, icp.last_stats()["kernel_us"] if len(surv) else 0.0

    def device_frame(top_k):
        nat.upload_images(rgb, depth, None)
        nat.enqueue(thr)
        nat.enqueue_post(0.5, top_k)
        ev0.record(stream)
        nat.enqueue_pose(sK, 30, False)
        ev1.record(stream)
        out = nat.complete_pose()
        return out, ev0.elapsed_time(ev1) * 1000.0

    results = dict(card=card(), frame="tests/golden/driver_trace.npz", bank="bank_allScales_full (%d templates)" % G,
                   threshold=thr, frames=args.frames, runs=[])
    for top_k in (3, 0):
        # outputs must agree before anything is timed
        surv, (Rh, th, rh), _, _ = host_frame(top_k)
        out, _ = device_frame(top_k)
        identical = bool(np.array_equal(out[0], surv) and np.array_equal(out[3], rh, equal_nan=True)
                         and np.array_equal(out[1], Rh, equal_nan=True) and np.array_equal(out[2], th, equal_nan=True))
        for _ in range(args.warmup):
            host_frame(top_k)
            device_frame(top_k)
        # the two paths alternate in blocks of 10 frames, so drifts of the shared machine hit both
        host_t = dev_t = 0.0
        host_pose = host_kernel = dev_pose = 0.0
        l_host = l_dev = 0
        done = 0
        while done < args.frames:
            blk = min(10, args.frames - done)
            la, li = nat.launch_count(), icp.launch_count()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(blk):
                _, _, w, k = host_frame(top_k)
                host_pose += w
                host_kernel += k
            host_t += time.perf_counter() - t0
            l_host += nat.launch_count() - la + icp.launch_count() - li
            la = nat.launch_count()
            t0 = time.perf_counter()
            for _ in range(blk):
                _, e = device_frame(top_k)
                dev_pose += e
            dev_t += time.perf_counter() - t0
            l_dev += nat.launch_count() - la
            done += blk
        n = args.frames
        results["runs"].append(dict(
            top_k=top_k, survivors=int(len(surv)), identical_poses=identical,
            host_handoff=dict(frames_per_s=round(n / host_t, 1), pose_stage_us=round(host_pose / n * 1e6, 1),
                              pose_kernels_us=round(host_kernel / n, 1), launches_per_frame=round(l_host / n, 2)),
            device_chain=dict(frames_per_s=round(n / dev_t, 1), pose_stage_us=round(dev_pose / n, 1),
                              launches_per_frame=round(l_dev / n, 2))))
    line = json.dumps(results)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
