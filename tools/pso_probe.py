#!/usr/bin/env python
"""Accuracy and cost of the particle-swarm estimation (include/linemod_b200.h, LM_POSE_PSO) against the two ICP
estimations.

  accuracy   synthetic scenes with a known pose: the recorded render's cloud (tests/golden/driver_trace.npz), supersampled
             2x, moved by a seeded perturbation U{a, a} (every rotation axis uniform in [-a, a] degrees, every translation
             axis uniform in [-a, a] mm, about the cloud's centroid) and z-buffer splatted with a scene K unlike the
             render's in front of a tilted table plane.  Each estimator refines the unmoved render at the moved object's
             match position (lm_icp_process_batch): PSO, point-to-plane and point-to-point, the ICPs with
             use_scene_cloud.  Errors: the rotation angle of R_est R_true^T (degrees) and the distance between where
             each pose puts the render's centroid (mm).  Median and 90th percentile per level and estimator.
  time       on the recorded driver frame against the allScales bank: the pose stage (lm_enqueue_pose, CUDA events on
             the detector's stream) and detect frames/s at thresholds 75 and 65 for every estimation, alternating in
             blocks; lm_icp_process_batch of 3 hypotheses (its kernel time, lm_icp_last_stats).
  scores     the verification scores of detect's kept poses under each estimation.

  python tools/pso_probe.py [--cases 100] [--frames 100] [--out FILE] [--search P,I,dt_mm,dr_deg]
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
sys.path.insert(0, os.path.join(ROOT, "tests"))

from pose_stage_probe import SHIFTS, card  # noqa: E402
from pso_scenes import ESTIMATIONS, accuracy  # noqa: E402


def timing(lib, torch, g, b, frames, search):
    packed = dict(class_begin=b["class_begin"], tmeta=b["tmeta"].astype(np.int32), feats=b["feats"].astype(np.int32))
    G = packed["tmeta"].shape[0]
    renders = [np.ascontiguousarray(np.roll(np.roll(g["render"], dy, 0), dx, 1)) for dy, dx in SHIFTS]
    which = np.arange(G) % len(renders)
    K = np.repeat(g["rf0_modelK"][None], G, 0).astype(np.float32)
    R = np.repeat(g["rf0_modelR"][None], G, 0).astype(np.float32)
    t = np.repeat(g["rf0_modelT"].reshape(1, 3), G, 0).astype(np.float32)
    sK = g["rf0_sceneK"].astype(np.float32)
    rgb, depth = g["rgb"], g["depth"]
    nat = lib.NativeDetector(b["T"].tolist(), 0)
    nat.load_bank(packed, 4)
    nat.select(None, 0, 1)
    nat.set_template_renders(0, [renders[k] for k in which], K, R, t)
    nat.set_pose_search(*search)
    st = torch.cuda.ExternalStream(nat.stream())
    out = {}
    for thr in (75.0, 65.0):
        stage = {e: [] for e in ESTIMATIONS}
        fps = {e: [] for e in ESTIMATIONS}

        def frame(e, timed):
            nat.upload_images(rgb, depth, None)
            nat.enqueue(thr)
            nat.enqueue_post(0.5, 0)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(st)
            nat.enqueue_pose(sK, 30, e != "pso", e)
            e1.record(st)
            nat.enqueue_pose_nms(40.0)
            got = nat.complete_detect()
            if timed:
                stage[e].append(e0.elapsed_time(e1) * 1000.0)
            return got

        scores, kept = {}, {}
        nat.set_pose_verify(True, 10.0)
        for e in ESTIMATIONS:
            got = frame(e, False)
            kept[e] = len(got[0])
            scores[e] = [round(float(s), 4) for s in nat.pose_verify()[0]]
        nat.set_pose_verify(False)
        for e in ESTIMATIONS:
            for _ in range(5):
                frame(e, False)
        for _ in range(3):
            for e in ESTIMATIONS:
                for _ in range(frames // 4):
                    frame(e, True)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for _ in range(frames):
                    frame(e, False)
                fps[e].append(round(frames / (time.perf_counter() - t0), 1))
        surv = frame("pso", False)[4]
        out["threshold_%d" % thr] = dict(survivors=surv["survivors"], posed=surv["posed"],
                                        pose_stage_us={e: dict(median=round(float(np.median(v)), 1), min=round(float(np.min(v)), 1))
                                                       for e, v in stage.items()},
                                        detect_frames_per_s=fps, kept=kept, kept_scores=scores)
    # lm_icp_process_batch with 3 hypotheses: the recorded frame's first three survivors
    nat.upload_images(rgb, depth, None)
    nat.enqueue(65.0)
    nat.enqueue_post(0.5, 3)
    s3, _ = nat.complete_post()
    tid = s3["template_id"].astype(np.int64)
    xy = np.stack([s3["x"], s3["y"]], 1)
    batch = {}
    for e in ESTIMATIONS:
        icp = lib.NativeIcp()
        icp.set_estimation(e)
        icp.set_use_scene_cloud(e != "pso")
        icp.set_pose_search(*search)
        us = []
        for k in range(60):
            icp.process_batch(depth, [renders[which[i]] for i in tid], sK, K[tid], R[tid], t[tid], xy, 30)
            if k >= 10:
                us.append(icp.last_stats()["kernel_us"])
        batch[e] = dict(kernel_us_median=round(float(np.median(us)), 1), points_last=icp.last_stats()["points"])
    out["icp_process_batch_3"] = batch
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cases", type=int, default=100)
    ap.add_argument("--frames", type=int, default=100)
    ap.add_argument("--search", default="64,40,40,30", help="particles,iterations,dt_mm,dr_deg")
    ap.add_argument("--skip-time", action="store_true")
    ap.add_argument("--estimations", default=",".join(ESTIMATIONS), help="the accuracy table's estimators")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this probe only measures on the GPU")
    lib = importlib.import_module("6dpose_b200._lib")
    P, I, dt, dr = (float(v) for v in args.search.split(","))
    search = (int(P), int(I), dt, dr, 20.0, 0)
    gold = os.path.join(ROOT, "tests", "golden")
    g = np.load(os.path.join(gold, "driver_trace.npz"))
    b = np.load(os.path.join(gold, "bank_allScales_full.npz"))
    results = dict(card=card(), search=dict(particles=search[0], iterations=search[1], dt_mm=dt, dr_deg=dr, clamp_mm=20.0),
                   accuracy=accuracy(lib, g, args.cases, search, estimations=args.estimations.split(",")))
    if not args.skip_time:
        results["time"] = timing(lib, torch, g, b, args.frames, search)
    line = json.dumps(results)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
