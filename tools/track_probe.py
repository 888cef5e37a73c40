#!/usr/bin/env python
"""What tracking (Detector.track, include/linemod_b200.h lm_track) costs against detecting again, on the reference's
fixture frame (tests/golden/driver_trace.npz, BGR) against the whole allScales bank (2989 templates, distances from
tests/golden/allScales_depths.npz) with the shifted per-template renders of tests/test_gpu_pose_nms.py, at thresholds 75
and 65:
  detect       Detector.detect of every survivor (top_k 0), depth gate off and on (tolerance 0.15), and gate off with
               use_scene_cloud (the ICP registering against the scene, as tracking does; detect's default registers
               the model against itself, LL.cpp:109, which ends after one pass)
  track        Detector.track of the objects that detect kept on that frame, starting from their own poses
for both ICP estimations, the paths alternating in blocks after a warm-up of every path.  Frames/s from a host clock
around whole calls, each of which ends in a stream synchronise; the track stage's device time (window, clouds, sort,
voxels, ICP) from CUDA events around the native lm_track call on the detector's stream.  Reads the card's name, power
limit and max SM clock in the same run.

  python tools/track_probe.py [--frames 200] [--warmup 10] [--block 20] [--out FILE]
"""
import argparse
import importlib
import json
import os
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from detect_probe import SHIFTS, card  # noqa: E402

TAU = 0.15


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--block", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this probe only measures on the GPU")
    pkg = importlib.import_module("6dpose_b200")
    bk = importlib.import_module("6dpose_b200.bank")
    gold = os.path.join(ROOT, "tests", "golden")
    g = np.load(os.path.join(gold, "driver_trace.npz"))
    b = np.load(os.path.join(gold, "bank_allScales_full.npz"))
    z = np.load(os.path.join(gold, "allScales_depths.npz"))["z_mm"]
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
    rgb, depth = np.ascontiguousarray(g["rgb"][..., ::-1]), g["depth"]
    cid = "06_template"
    bank = bk.TemplateBank()
    bank.classes[cid] = bk.PackedPyramids(tmeta, feats, 2)
    with tempfile.TemporaryDirectory() as tmp:
        bank.write_packed(cid, os.path.join(tmp, cid + ".lmb"), 2)
        det = pkg.Detector(int(g["num_features"]), b["T"].tolist())
        det.readClasses([cid], os.path.join(tmp, "%s.lmb"))
    det.setTemplateRenders({cid: ((renders[k] for k in which), K, R, t)})
    det.setTemplateDepths({cid: z})
    nat = det._select([cid])
    st = torch.cuda.ExternalStream(nat.stream())
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    results = dict(card=card(), frame="tests/golden/driver_trace.npz (BGR)", bank="bank_allScales_full (%d templates)" % G,
                   frames=args.frames, runs=[])
    for thr, est in ((t, e) for t in (75.0, 65.0) for e in ("point_to_plane", "point_to_point")):
        det.setDepthGate(None)
        objects = det.detect([rgb, depth], thr, [cid], sK, estimation=est)
        tracked = det.track(depth, sK, objects, estimation=est)
        triples = [(0, m.template_id, p.getTransformation()) for m, p in objects]

        def detect(tau, use_scene=False):
            det.setDepthGate(tau)
            return len(det.detect([rgb, depth], thr, [cid], sK, use_scene_cloud=use_scene, estimation=est))

        paths = dict(detect_gate_off=lambda: detect(None), detect_gate_on=lambda: detect(TAU),
                     detect_scene_cloud=lambda: detect(None, True),
                     track=lambda: len(det.track(depth, sK, objects, estimation=est)))
        for _ in range(args.warmup):
            for f in paths.values():
                f()
        elapsed = {k: 0.0 for k in paths}
        count = {}
        done = 0
        while done < args.frames:
            blk = min(args.block, args.frames - done)
            for name, f in paths.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for _ in range(blk):
                    count[name] = f()
                elapsed[name] += time.perf_counter() - t0
            done += blk
        det.setDepthGate(None)
        # the track stage alone on the device: events on the detector's stream around lm_track
        dev_ms = []
        for _ in range(args.frames):
            ev0.record(st)
            nat.track(depth, sK, triples, 30, 4, est)
            ev1.record(st)
            ev1.synchronize()
            dev_ms.append(ev0.elapsed_time(ev1))
        statuses = [p.getTrackStatus() for _, p in tracked]
        run = dict(threshold=thr, estimation=est, objects=len(objects), tracked=statuses.count("tracked"),
                   pairing_half=sum(p.getResidual() >= 0.5 for _, p in tracked),
                   track_device_ms_median=round(float(np.median(dev_ms)), 4))
        for name in paths:
            run[name + "_fps"] = round(args.frames / elapsed[name], 1)
            run[name + "_entries"] = count[name]
        results["runs"].append(run)
    line = json.dumps(results)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
