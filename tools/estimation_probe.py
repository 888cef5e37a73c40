#!/usr/bin/env python
"""Point-to-plane against point-to-point ICP (lm_set_pose_estimation / lm_icp_set_estimation) on the recorded driver
frame (tests/golden/driver_trace.npz) against the allScales bank with the shifted per-template renders of
tests/test_gpu_pose_stage.py.  For each estimation, in alternating blocks after warm-up, a host clock around whole calls
that end in a synchronise:

  detect@75, detect@65   Detector's whole frame with every box-NMS survivor refined and the pose NMS (NativeDetector.detect)
  match                  the same frame up to the box NMS only (the pose stage's time is detect minus match)
  refine_top3            match_pose with top_k 3
  batch8                 an 8-frame detect_batch at threshold 75 (every survivor, pose NMS)
  icp3                   lm_icp_process_batch of the three top survivors (host clouds)

and the ICP iterations to convergence of every survivor at 65 and 75 (lm_icp_process_batch with capture).  Prints one
JSON line with the card's name and power limit.

  python tools/estimation_probe.py [--calls 40] [--warmup 5] [--block 5] [--out FILE]
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
sys.path.insert(0, os.path.join(ROOT, "tests"))

EST = ("point_to_plane", "point_to_point")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    if q.returncode != 0:
        raise RuntimeError("nvidia-smi failed: %s" % q.stderr.strip())
    name, power, clock = [s.strip() for s in q.stdout.strip().split(",")]
    return dict(name=name, power_limit=power, max_sm_clock=clock)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--block", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    lib = importlib.import_module("6dpose_b200._lib")
    pb = importlib.import_module("test_gpu_peer_batch")
    data = pb.load_data()
    g = data["g"]
    nat = pb.handle(data)
    sK = data["sK"]
    K8 = np.repeat(sK[None], 8, 0)
    rgb8, depth8 = np.stack([g["rgb"]] * 8), np.stack([g["depth"]] * 8)
    icp = lib.NativeIcp()
    nat.upload_images(g["rgb"], g["depth"], None)
    nat.enqueue(75.0)
    nat.enqueue_post(0.5, 3)
    top3, _ = nat.complete_post()
    tid = top3["template_id"].astype(np.int64)
    icp_args = (g["depth"], [data["renders"][k] for k in data["which"][tid]], sK, data["K"][tid], data["R"][tid], data["t"][tid],
                np.stack([top3["x"], top3["y"]], 1), 30)

    def match(thr):
        nat.upload_images(g["rgb"], g["depth"], None)
        nat.enqueue(thr)
        nat.enqueue_post(0.5, 0)
        return nat.complete_post()

    paths = {
        "detect@75": lambda est: nat.detect(g["rgb"], g["depth"], None, 75.0, sK, 0.5, 0, 30, False, 40.0, est),
        "detect@65": lambda est: nat.detect(g["rgb"], g["depth"], None, 65.0, sK, 0.5, 0, 30, False, 40.0, est),
        "match@75": lambda est: match(75.0),
        "match@65": lambda est: match(65.0),
        "refine_top3": lambda est: nat.match_pose(g["rgb"], g["depth"], None, 75.0, sK, 0.5, 3, 30, False, est),
        "batch8": lambda est: nat.detect_batch(rgb8, depth8, None, 75.0, K8, 0.5, 0, 30, False, True, 40.0, estimation=est),
        "icp3": lambda est: icp.process_batch(*icp_args, estimation=est),
    }
    times = {(p, e): [] for p in paths for e in EST}
    for p, fn in paths.items():
        for e in EST:
            for _ in range(a.warmup):
                fn(e)
    done = 0
    while done < a.calls:
        n = min(a.block, a.calls - done)
        for p, fn in paths.items():
            for e in EST:
                for _ in range(n):
                    t0 = time.perf_counter()
                    fn(e)  # every path ends in a synchronise (complete_*, detect_batch, process_batch)
                    times[(p, e)].append(time.perf_counter() - t0)
        done += n
    res = dict(card=card(), calls=a.calls, block=a.block, ms={}, per_s={}, pose_stage_ms={}, iterations={}, survivors={})
    for (p, e), v in times.items():
        med = float(np.median(v)) * 1e3
        res["ms"]["%s/%s" % (p, e)] = round(med, 4)
        res["per_s"]["%s/%s" % (p, e)] = round(1e3 / med * (8 if p == "batch8" else 1), 2)
    for thr in ("75", "65"):
        for e in EST:
            res["pose_stage_ms"]["%s/%s" % (thr, e)] = round(res["ms"]["detect@%s/%s" % (thr, e)] - res["ms"]["match@%s/%s" % (thr, e)], 4)
    # iterations to convergence of every survivor (host clouds; the device stage refines the same clouds)
    icp.set_capture(True)
    for thr in (75.0, 65.0):
        surv, _ = match(thr)
        tid = surv["template_id"].astype(np.int64)
        res["survivors"]["%g" % thr] = int(len(surv))
        for e in EST:
            _, _, r = icp.process_batch(g["depth"], [data["renders"][k] for k in data["which"][tid]], sK, data["K"][tid], data["R"][tid],
                                        data["t"][tid], np.stack([surv["x"], surv["y"]], 1), 30, e)
            its = [icp.capture(i)["iterations"] for i in range(len(surv)) if r[i] != -1.0]
            res["iterations"]["%g/%s" % (thr, e)] = dict(mean=round(float(np.mean(its)), 3), max=int(np.max(its)),
                                                          at_cap=int(np.sum(np.asarray(its) >= 30)), n=len(its))
    icp.set_capture(False)
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
