#!/usr/bin/env python
"""Frame rate of linemod_ros/detect.py's whole frame -- front-end, match, box NMS, poseRefine of EVERY survivor, then the
greedy translation NMS (nms_norms(ts, -residual, 40)) -- on the recorded driver frame (tests/golden/driver_trace.npz)
against the allScales bank with the shifted per-template renders of tests/test_gpu_pose_nms.py, along three paths:

  device     Detector.detect: one chain on the GPU, the pose NMS included (k_pose_nms); only kept objects come back
  refine     Detector.match_refine(top_k=0), every survivor's pose copied back, then the numpy pose NMS
  host loop  the box-NMS survivors from the device, then one pose_refine.refine_matches call per survivor (host clouds,
             one full render each, as the script's loop), then the numpy pose NMS

at thresholds 65 and 75.  The paths alternate in blocks after warm-up; frames/s is a host clock around whole frames,
each ending in a synchronise.  Also times k_pose_nms with CUDA events around lm_enqueue_pose_nms on the detector's stream,
reads the card's name and power limit, and exits non-zero unless the three paths return identical objects.

  python tools/detect_probe.py [--frames 200] [--warmup 20] [--block 10] [--out FILE]
"""
import argparse
import importlib
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

SHIFTS = [(0, 0), (-68, -19), (-180, 57), (3, -2), (-2, 4)]
TTHR = 40.0


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    if q.returncode != 0:
        raise RuntimeError("nvidia-smi failed: %s" % q.stderr.strip())
    name, power, clock = [s.strip() for s in q.stdout.strip().split(",")]
    return dict(name=name, power_limit=power, max_sm_clock=clock)


def objects(pairs):
    return [(m.x, m.y, m.similarity, m.class_id, m.template_id, p.getR().tobytes(), p.getT().tobytes(), p.getResidual())
            for m, p in pairs]


def model_nms(pairs):
    import pose_nms_model as pm
    posed = [(m, p) for m, p in pairs if p.getResidual() != -1.0]
    if not posed:
        return []
    ts = np.array([p.getT().reshape(3) for _, p in posed])
    keep = pm.nms(ts, -np.array([p.getResidual() for _, p in posed], np.float32).astype(np.float64), TTHR)
    return [posed[k] for k in keep]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--block", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this probe only measures on the GPU")
    pkg = importlib.import_module("6dpose_b200")
    bk = importlib.import_module("6dpose_b200.bank")
    pr = importlib.import_module("6dpose_b200.pose_refine")
    gold = os.path.join(ROOT, "tests", "golden")
    g = np.load(os.path.join(gold, "driver_trace.npz"))
    b = np.load(os.path.join(gold, "bank_allScales_full.npz"))
    tmeta, feats = b["tmeta"].astype(np.int32), b["feats"].astype(np.int32)
    G = tmeta.shape[0]
    renders = [np.ascontiguousarray(np.roll(np.roll(g["render"], dy, 0), dx, 1)) for dy, dx in SHIFTS]
    which = np.arange(G) % len(renders)
    K = np.repeat(g["rf0_modelK"][None], G, 0).astype(np.float32)
    R = np.repeat(g["rf0_modelR"][None], G, 0).astype(np.float32)
    t = np.repeat(g["rf0_modelT"].reshape(1, 3), G, 0).astype(np.float32)
    t[:, 0] += (np.arange(G) % 7) - 3.0
    t[:, 2] += np.arange(G) % 11
    sK = g["rf0_sceneK"].astype(np.float32)
    rgb, depth = g["rgb"], g["depth"]
    cid = "06_template"

    bank = bk.TemplateBank()
    bank.classes[cid] = bk.PackedPyramids(tmeta, feats, 2)
    with tempfile.TemporaryDirectory() as tmp:
        bank.write_packed(cid, os.path.join(tmp, cid + ".lmb"), 2)
        det = pkg.Detector(int(g["num_features"]), b["T"].tolist())
        det.readClasses([cid], os.path.join(tmp, "%s.lmb"))
    det.setTemplateRenders({cid: ((renders[k] for k in which), K, R, t)})
    nat = det._select([cid])
    stream = torch.cuda.ExternalStream(nat.stream())
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def device_path(thr):
        return det.detect([rgb, depth], thr, [cid], sK)

    def refine_path(thr):
        return model_nms(det.match_refine([rgb, depth], thr, [cid], sK, top_k=0))

    def host_path(thr):
        nat.upload_images(rgb, depth, None)
        nat.enqueue(thr)
        nat.enqueue_post(0.5, 0)
        surv, _ = nat.complete_post()
        ms = det._to_matches(surv)
        tid = surv["template_id"].astype(np.int64)  # one class: template id == bank index
        pairs = []
        for i, m in enumerate(ms):
            k = tid[i]
            p = pr.refine_matches(depth, sK, [m], [renders[which[k]]], K[k:k + 1], R[k:k + 1], t[k:k + 1])[0]
            pairs.append((m, p))
        return model_nms(pairs)

    def pose_nms_us(thr):
        nat.upload_images(rgb, depth, None)
        nat.enqueue(thr)
        nat.enqueue_post(0.5, 0)
        nat.enqueue_pose(sK, 30, False)
        ev0.record(stream)
        nat.enqueue_pose_nms(TTHR)
        ev1.record(stream)
        out = nat.complete_detect()
        return ev0.elapsed_time(ev1) * 1000.0, out[4]

    paths = [("device", device_path), ("refine", refine_path), ("host_loop", host_path)]
    results = dict(card=card(), frame="tests/golden/driver_trace.npz", bank="bank_allScales_full (%d templates)" % G,
                   translation_threshold=TTHR, frames=args.frames, runs=[])
    ok = True
    for thr in (65.0, 75.0):
        got = {name: objects(fn(thr)) for name, fn in paths}
        identical = got["device"] == got["refine"] == got["host_loop"]
        ok &= identical
        for _ in range(args.warmup):
            for _, fn in paths:
                fn(thr)
        elapsed = {name: 0.0 for name, _ in paths}
        done = 0
        while done < args.frames:
            blk = min(args.block, args.frames - done)
            for name, fn in paths:
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for _ in range(blk):
                    fn(thr)
                elapsed[name] += time.perf_counter() - t0
            done += blk
        us, counts = [], None
        for _ in range(args.frames):
            e, counts = pose_nms_us(thr)
            us.append(e)
        results["runs"].append(dict(
            threshold=thr, survivors=counts["survivors"], posed=counts["posed"], kept=len(got["device"]), identical_objects=identical,
            frames_per_s={name: round(args.frames / elapsed[name], 1) for name, _ in paths},
            k_pose_nms_us=dict(median=round(float(np.median(us)), 1), min=round(float(np.min(us)), 1), max=round(float(np.max(us)), 1))))
    line = json.dumps(results)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")
    if not ok:
        raise SystemExit("the three paths returned different objects")


if __name__ == "__main__":
    main()
