#!/usr/bin/env python
"""What tracking a batch of frames in one call (lm_track_batch) saves against one lm_track call per frame, on the
reference's fixture frame (tests/golden/driver_trace.npz, BGR) and its rolled / mirrored variants (each with its own K,
as tests/test_gpu_peer_batch.py builds them), against the whole allScales bank with the shifted per-template renders of
tools/track_probe.py.  Each frame's objects are the poses Detector.detect keeps on it at thresholds 75 and 65.  For
n = 1, 2, 4, 8, 16 frames and both ICP estimations:
  single   n lm_track calls, one per frame
  batch    one lm_track_batch of the same n frames
The outputs of both paths are asserted identical, bit for bit.  After a warm-up of every shape the two paths alternate in
blocks.  Frames/s comes from a host clock around whole calls, each of which ends in a stream synchronise; the stage time
(all n frames) from CUDA events on the detector's stream.  Reads the card's name, power limit and max SM clock in the
same run.

  python tools/track_batch_probe.py [--iters 40] [--warmup 3] [--block 10] [--out FILE]
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

NS = (1, 2, 4, 8, 16)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--block", type=int, default=10)
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
    tmeta, feats = b["tmeta"].astype(np.int32), b["feats"].astype(np.int32)
    G = tmeta.shape[0]
    renders = [np.ascontiguousarray(np.roll(np.roll(g["render"], dy, 0), dx, 1)) for dy, dx in SHIFTS]
    which = np.arange(G) % len(renders)
    K = np.repeat(g["rf0_modelK"][None], G, 0).astype(np.float32)
    R = np.repeat(g["rf0_modelR"][None], G, 0).astype(np.float32)
    t = np.repeat(g["rf0_modelT"].reshape(1, 3), G, 0).astype(np.float32)
    t[:, 0] += (np.arange(G) % 7) - 3.0
    t[:, 2] += np.arange(G) % 11
    rgb, depth = np.ascontiguousarray(g["rgb"][..., ::-1]), g["depth"]
    variants = [(rgb, depth), (np.roll(rgb, (17, -23), (0, 1)), np.roll(depth, (17, -23), (0, 1))),
                (np.ascontiguousarray(rgb[:, ::-1]), np.ascontiguousarray(depth[:, ::-1]))]
    nmax = max(NS)
    sK = np.repeat(g["rf0_sceneK"].astype(np.float32)[None], nmax, 0)
    sK[:, 0, 0] *= 1.0 + 0.01 * (np.arange(nmax) % 3)
    sK[:, 1, 2] += np.arange(nmax) % 3
    frames = [variants[f % 3] for f in range(nmax)]
    cid = "06_template"
    bank = bk.TemplateBank()
    bank.classes[cid] = bk.PackedPyramids(tmeta, feats, 2)
    with tempfile.TemporaryDirectory() as tmp:
        bank.write_packed(cid, os.path.join(tmp, cid + ".lmb"), 2)
        det = pkg.Detector(int(g["num_features"]), b["T"].tolist())
        det.readClasses([cid], os.path.join(tmp, "%s.lmb"))
    det.setTemplateRenders({cid: ((renders[k] for k in which), K, R, t)})
    nat = det._select([cid])
    st = torch.cuda.ExternalStream(nat.stream())
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    results = dict(card=card(), frames="tests/golden/driver_trace.npz (BGR), rolled and mirrored, a K each",
                   bank="bank_allScales_full (%d templates)" % G, iters=args.iters, runs=[])
    depths = np.stack([f[1] for f in frames])
    for thr, est in ((th, e) for th in (75.0, 65.0) for e in ("point_to_plane", "point_to_point")):
        objects = []
        for f in range(nmax):
            pairs = det.detect([frames[f][0], frames[f][1]], thr, [cid], sK[f], estimation=est)
            objects.append([(0, m.template_id, p.getTransformation()) for m, p in pairs])
        nat = det._select([cid])
        for n in NS:
            paths = dict(single=lambda: [nat.track(depths[f], sK[f], objects[f], 30, 4, est) for f in range(n)],
                         batch=lambda: nat.track_batch(depths[:n], sK[:n], objects[:n], 30, 4, est))
            a, bt = paths["single"](), paths["batch"]()
            for x, y in zip(a, bt):
                assert all(np.asarray(u).tobytes() == np.asarray(v).tobytes() for u, v in zip(x, y)), (thr, est, n)
            for _ in range(args.warmup):
                for fn in paths.values():
                    fn()
            host = {k: 0.0 for k in paths}
            dev = {k: [] for k in paths}
            done = 0
            while done < args.iters:
                blk = min(args.block, args.iters - done)
                for name, fn in paths.items():
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    for _ in range(blk):
                        ev0.record(st)
                        fn()
                        ev1.record(st)
                        ev1.synchronize()
                        dev[name].append(ev0.elapsed_time(ev1))
                    host[name] += time.perf_counter() - t0
                done += blk
            run = dict(threshold=thr, estimation=est, frames=n, objects=sum(len(o) for o in objects[:n]))
            for name in paths:
                run[name + "_fps"] = round(n * args.iters / host[name], 1)
                run[name + "_stage_ms_median"] = round(float(np.median(dev[name])), 3)
            run["speedup_fps"] = round(run["batch_fps"] / run["single_fps"], 3)
            results["runs"].append(run)
            print(json.dumps(run), flush=True)
    line = json.dumps(results)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
