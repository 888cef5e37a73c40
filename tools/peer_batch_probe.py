#!/usr/bin/env python
"""Frame rate of a batch of ROS-driver frames (lm_detect_batch with the pose NMS: each frame's match and box NMS, one
pose stage over every survivor, one pose NMS) with the bank sharded over `world` ranks of the peer exchange
(lm_peer_detect_batch), the pose stage unshared (every rank refines every survivor) and shared (lm_peer_share_pose:
within each chunk, rank r refines survivors r, r + world, ...), against the unconnected batch on one GPU.  The frames
are the recorded driver frame (tests/golden/driver_trace.npz) against the allScales bank with the shifted per-template
renders of the tests.

Ranks go to distinct devices while the box has enough of them; otherwise they are handles of one process on device 0,
which measures the exchange's overhead, not scaling.  Every rank calls from its own host thread, after one unconnected
batch of the same shape.  The three paths alternate in blocks of --block batches.  Per world, threshold and path:
frames/s (host clock around whole batches, every rank's call returned), each rank's call time, and an estimate of
each rank's pose-stage time: the call time minus the time of the batch's match part (n frames of upload, match and box
NMS, each waited for) run the same way on the same handles.  Before timing, every rank's output of every path is checked against the unconnected batch.  Also reads
the card's name and power limit.

  python tools/peer_batch_probe.py [--frames-per-batch 8] [--batches 20] [--block 5] [--worlds 2,3] [--out FILE]
"""
import argparse
import importlib
import json
import os
import subprocess
import sys
import threading
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


def on_every_rank(nats, fn):
    got, errs = [None] * len(nats), [None] * len(nats)

    def run(r):
        try:
            got[r] = fn(nats[r])
        except BaseException as e:
            errs[r] = e

    threads = [threading.Thread(target=run, args=(r,)) for r in range(len(nats))]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    for e in errs:
        if e is not None:
            raise e
    return got


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames-per-batch", type=int, default=8)
    ap.add_argument("--batches", type=int, default=20)
    ap.add_argument("--block", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--worlds", default="2,3")
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
    n = args.frames_per_batch
    rgb = np.ascontiguousarray(np.repeat(g["rgb"][None], n, 0))
    depth = np.ascontiguousarray(np.repeat(g["depth"][None], n, 0))
    sKs = np.ascontiguousarray(np.repeat(sK[None], n, 0))
    n_dev = torch.cuda.device_count()

    def handle(dev, rank, world):
        nat = lib.NativeDetector(T, dev)
        nat.load_bank(packed, 4)
        nat.select(None, rank, world)
        nat.set_template_renders(0, [renders[k] for k in which], K, R, t)
        return nat

    def batch_args(thr):
        return (rgb, depth, None, thr, sKs, 0.5, 0, 30, False, True, 40.0)

    def same(a, b):
        return len(a) == len(b) and all(np.array_equal(x[0], y[0]) and all(np.array_equal(u, v, equal_nan=True) for u, v in zip(x[1:4], y[1:4]))
                                        and x[4] == y[4] for x, y in zip(a, b))

    def match_only(nats, thr, reps=1):
        # one connected frame's match chain, enqueued rank by rank from this thread
        for _ in range(reps):
            for nat in nats:
                nat.upload_images(rgb[0], depth[0], None)
            for nat in nats:
                nat.enqueue(thr)
            for nat in nats:
                nat.enqueue_post(0.5, 0)
            for nat in nats:
                nat.complete_post()

    def match_part(nats, thr, reps=3):
        # what a batch does before its pose stage: n frames of upload, match and box NMS, each waited for, every rank
        # from its own thread; seconds per batch and rank
        def one(nat):
            t0 = time.perf_counter()
            for _ in range(reps * n):
                nat.upload_images(rgb[0], depth[0], None)
                nat.enqueue(thr)
                nat.enqueue_post(0.5, 0)
                nat.complete_post()
            return (time.perf_counter() - t0) / reps
        return np.asarray(on_every_rank(nats, one))

    single = handle(0, 0, 1)
    results = dict(card=card(), devices=n_dev, frame="tests/golden/driver_trace.npz", bank="bank_allScales_full (%d templates)" % G,
                   frames_per_batch=n, batches=args.batches, runs=[])
    for world in [int(w) for w in args.worlds.split(",")]:
        devices = list(range(world)) if world <= n_dev else [0] * world
        nats = [handle(dev, r, world) for r, dev in enumerate(devices)]
        for nat in nats:                                   # unconnected, the largest shape first: no allocation later
            nat.detect_batch(*batch_args(62.0))
        for nat in nats:
            nat.peer_export(world, 1 << 17)
        bases = [nat.peer_base() for nat in nats]
        for r, nat in enumerate(nats):
            nat.peer_connect_local(r, world, bases)
        for nat in nats:                                   # the result block grows to the exchange's size on every rank
            nat.prepare()
        match_only(nats, 75.0, reps=1)                     # one connected frame, rank by rank, before the threads

        def run(path, thr):
            a = batch_args(thr)
            if path == "single":
                t0 = time.perf_counter()
                out = single.detect_batch(*a)
                return [out], [time.perf_counter() - t0]
            share = path == "shared"
            for nat in nats:
                nat.peer_share_pose(share)

            def one(nat):
                t0 = time.perf_counter()
                out = nat.peer_detect_batch(*a)
                return out, time.perf_counter() - t0
            got = on_every_rank(nats, one)
            return [x[0] for x in got], [x[1] for x in got]

        paths = ("single", "unshared", "shared")
        for thr in (65.0, 75.0):
            want = single.detect_batch(*batch_args(thr))
            survivors = int(single.batch_counts[:, 1].sum())
            identical = {}
            for path in paths:
                outs, _ = run(path, thr)
                identical[path] = all(same(o, want) for o in outs)
                for _ in range(args.warmup):
                    run(path, thr)
            match_s = dict(single=match_part([single], thr), unshared=match_part(nats, thr))
            match_s["shared"] = match_s["unshared"]
            elapsed = {p: 0.0 for p in paths}
            call_s = {p: None for p in paths}
            refined = {}
            done = 0
            while done < args.batches:
                blk = min(args.block, args.batches - done)
                for path in paths:
                    t0 = time.perf_counter()
                    for _ in range(blk):
                        _, secs = run(path, thr)
                        call_s[path] = np.asarray(secs) if call_s[path] is None else call_s[path] + secs
                    elapsed[path] += time.perf_counter() - t0
                    if path != "single":
                        refined[path] = [nat.pose_stats()[1] for nat in nats]
                done += blk
            for path in paths:
                per_call = call_s[path] / args.batches
                results["runs"].append(dict(
                    world=1 if path == "single" else world, devices=[0] if path == "single" else devices, threshold=thr, path=path,
                    survivors=survivors, identical=identical[path], frames_per_s=round(args.batches * n / elapsed[path], 1),
                    call_ms_per_rank=[round(float(v) * 1e3, 2) for v in per_call],
                    match_ms_per_rank=[round(float(v) * 1e3, 2) for v in match_s[path]],
                    pose_stage_ms_per_rank_est=[round(float(v - m) * 1e3, 2) for v, m in zip(per_call, match_s[path])],
                    refined_per_rank=refined.get(path, [survivors])))
            print(json.dumps(results["runs"][-len(paths):]), flush=True)
        for nat in nats:
            nat.peer_disconnect()
        for nat in nats:
            nat.close()
    line = json.dumps(results)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
