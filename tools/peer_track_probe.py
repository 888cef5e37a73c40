#!/usr/bin/env python
"""What tracking a batch of frames over the ranks of the peer exchange (lm_peer_track_batch) costs or saves against one
unconnected lm_track_batch, on the workloads of tools/track_batch_probe.py: the reference's fixture frame
(tests/golden/driver_trace.npz, BGR) and its rolled / mirrored variants, each with its own K, the whole allScales bank
with the shifted per-template renders, and each frame's objects as Detector.detect keeps them at thresholds 75 and 65.
For n = 1, 4, 16 frames and both ICP estimations:
  single     one lm_track_batch on an unconnected handle
  peer_off   lm_peer_track_batch at world W with sharing off: every rank tracks every object
  peer_on    lm_peer_track_batch at world W with sharing on (lm_peer_share_pose): each rank tracks its share of each chunk
The ranks run on distinct GPUs when the machine has W of them, else all on device 0 (then they share its SMs, so sharing
cannot be faster: that arm shows the exchange's overhead).  Each rank's call runs on its own host thread.  Every rank's
outputs are asserted bit for bit equal to the single arm's.  After a warm-up of every shape (the ranks' first run of the
largest shape with sharing off) the arms alternate in blocks.  Frames/s comes from a host clock around whole calls (all
ranks returned, each call ends in a stream synchronise); the stage time from CUDA events on the stream of the single
handle and of rank 0.  Reads the card's name, power limit and max SM clock in the same run.

  python tools/peer_track_probe.py [--world 2] [--iters 30] [--warmup 3] [--block 10] [--out FILE]
"""
import argparse
import importlib
import json
import os
import sys
import tempfile
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from detect_probe import SHIFTS, card  # noqa: E402

NS = (1, 4, 16)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--world", type=int, default=2)
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--block", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this probe only measures on the GPU")
    pkg = importlib.import_module("6dpose_b200")
    bk = importlib.import_module("6dpose_b200.bank")
    lib = importlib.import_module("6dpose_b200._lib")
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
    single = det._select([cid])
    W = args.world
    distinct = torch.cuda.device_count() >= W
    devices = list(range(W)) if distinct else [0] * W
    packed = dict(class_begin=b["class_begin"], tmeta=tmeta, feats=feats)
    ranks = []
    for r, dev in enumerate(devices):
        nat = lib.NativeDetector(b["T"].tolist(), dev)
        nat.load_bank(packed, 4)
        nat.select(None, r, W)
        nat.set_template_renders(0, [renders[k] for k in which], K, R, t)
        ranks.append(nat)
    depths = np.stack([f[1] for f in frames])
    workloads = []
    for thr, est in ((th, e) for th in (75.0, 65.0) for e in ("point_to_plane", "point_to_point")):
        objects = []
        for f in range(nmax):
            pairs = det.detect([frames[f][0], frames[f][1]], thr, [cid], sK[f], estimation=est)
            objects.append([(0, m.template_id, p.getTransformation()) for m, p in pairs])
        workloads.append((thr, est, objects))
    single = det._select([cid])
    # every rank's first run of the largest shape, before it is connected: it grows the buffers while no collector spins
    largest = max(workloads, key=lambda w: sum(len(o) for o in w[2]))
    for nat in ranks:
        nat.track_batch(depths, sK, largest[2], 30, 4, largest[1])
    for nat in ranks:
        nat.peer_export(W, 1 << 12)
    bases = [nat.peer_base() for nat in ranks]
    for r, nat in enumerate(ranks):
        nat.peer_connect_local(r, W, bases)
    pool = ThreadPoolExecutor(W)

    def on_ranks(fn):
        futures = [pool.submit(fn, nat) for nat in ranks]
        return [f.result() for f in futures]

    st = torch.cuda.ExternalStream(single.stream())
    st0 = torch.cuda.ExternalStream(ranks[0].stream(), device=devices[0])
    results = dict(card=card(), world=W, ranks="distinct GPUs" if distinct else "one GPU (device 0) for every rank",
                   frames="tests/golden/driver_trace.npz (BGR), rolled and mirrored, a K each",
                   bank="bank_allScales_full (%d templates)" % G, iters=args.iters, runs=[])
    for thr, est, objects in workloads:
        for n in NS:
            def peer(share):
                def call():
                    for nat in ranks:
                        nat.peer_share_pose(share)
                    return on_ranks(lambda nat: nat.peer_track_batch(depths[:n], sK[:n], objects[:n], 30, 4, est))
                return call
            paths = dict(single=lambda: single.track_batch(depths[:n], sK[:n], objects[:n], 30, 4, est), peer_off=peer(False),
                         peer_on=peer(True))
            want = paths["single"]()
            for name in ("peer_off", "peer_on"):
                for got in paths[name]():
                    for x, y in zip(got, want):
                        assert all(np.asarray(u).tobytes() == np.asarray(v).tobytes() for u, v in zip(x, y)), (thr, est, n, name)
            for _ in range(args.warmup):
                for fn in paths.values():
                    fn()
            host = {k: 0.0 for k in paths}
            dev = {k: [] for k in paths}
            done = 0
            while done < args.iters:
                blk = min(args.block, args.iters - done)
                for name, fn in paths.items():
                    s = st if name == "single" else st0
                    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    for _ in range(blk):
                        ev0.record(s)
                        fn()
                        ev1.record(s)
                        ev1.synchronize()
                        dev[name].append(ev0.elapsed_time(ev1))
                    host[name] += time.perf_counter() - t0
                done += blk
            run = dict(threshold=thr, estimation=est, frames=n, objects=sum(len(o) for o in objects[:n]))
            for name in paths:
                run[name + "_fps"] = round(n * args.iters / host[name], 1)
                run[name + "_stage_ms_median"] = round(float(np.median(dev[name])), 3)
            results["runs"].append(run)
            print(json.dumps(run), flush=True)
    pool.shutdown()
    for nat in ranks:
        nat.peer_disconnect()
    line = json.dumps(results)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
