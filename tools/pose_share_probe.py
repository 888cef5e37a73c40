#!/usr/bin/env python
"""Frame rate of the whole ROS-driver frame (front-end, match, box NMS, poseRefine of every survivor, pose NMS: the
lm_complete_detect chain) with the bank sharded over `world` GPUs of the box, the pose stage unshared (every rank refines
every survivor) and shared over the ranks (lm_peer_share_pose: rank r refines survivors r, r + world, ...), on the
recorded driver frame (tests/golden/driver_trace.npz) against the allScales bank.

One handle per distinct device (world 1, 2, 4, 8 as far as the box has GPUs), all driven from this one host thread; the
ranks' frames are enqueued rank by rank, as tests/test_gpu_pose_share.py does.  Per world, threshold and mode: frames/s
(host clock around whole frames, each ending in every rank's synchronise), the pose stage's device time per rank (CUDA
events on the rank's stream around lm_enqueue_pose: cloud building, sort, voxels, normals, ICP and, shared, the
collector's wait), the hypotheses each rank refined and the largest share.  The two modes alternate in blocks of 10
frames.  Before timing, every rank's output of both modes is checked against one unconnected handle.  Also reads the
card's name and power limit.

  python tools/pose_share_probe.py [--frames 100] [--warmup 10] [--worlds 1,2,4,8] [--out FILE]
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
    ap.add_argument("--frames", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--worlds", default="1,2,4,8")
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
    rgb, depth = g["rgb"], g["depth"]
    n_dev = torch.cuda.device_count()

    def handle(dev, rank, world):
        nat = lib.NativeDetector(T, dev)
        nat.load_bank(packed, 4)
        nat.select(None, rank, world)
        nat.set_template_renders(0, [renders[k] for k in which], K, R, t)
        return nat

    class Rank:
        def __init__(self, nat, dev):
            self.nat, self.dev = nat, dev
            with torch.cuda.device(dev):
                self.stream = torch.cuda.ExternalStream(nat.stream(), device=torch.device("cuda", dev))
                self.ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]

    def frame(ranks, thr):
        for r in ranks:
            r.nat.upload_images(rgb, depth, None)
        for r in ranks:
            r.nat.enqueue(thr)
        for r in ranks:
            r.nat.enqueue_post(0.5, 0)
            with torch.cuda.device(r.dev):
                r.ev[0].record(r.stream)
            r.nat.enqueue_pose(sK, 30, False)
            with torch.cuda.device(r.dev):
                r.ev[1].record(r.stream)
            r.nat.enqueue_pose_nms(40.0)
        outs = [r.nat.complete_detect() for r in ranks]
        return outs, [r.ev[0].elapsed_time(r.ev[1]) * 1000.0 for r in ranks]

    def same(a, b):
        return bool(np.array_equal(a[0], b[0]) and all(np.array_equal(x, y, equal_nan=True) for x, y in zip(a[1:4], b[1:4]))
                    and a[4] == b[4])

    single = Rank(handle(0, 0, 1), 0)
    results = dict(card=card(), devices=n_dev, frame="tests/golden/driver_trace.npz", bank="bank_allScales_full (%d templates)" % G,
                   frames=args.frames, runs=[])
    for world in [int(w) for w in args.worlds.split(",")]:
        if world > n_dev:
            continue
        nats = [handle(dev, dev, world) for dev in range(world)]
        if world > 1:
            for nat in nats:
                nat.peer_export(world, 1 << 17)
            bases = [nat.peer_base() for nat in nats]
            for r, nat in enumerate(nats):
                nat.peer_connect_local(r, world, bases)
        ranks = [Rank(nat, dev) for dev, nat in enumerate(nats)]
        modes = (False, True) if world > 1 else (False,)

        def set_mode(share):
            if world > 1:
                for r in ranks:
                    r.nat.peer_share_pose(share)

        for thr in (65.0, 75.0):
            want = frame([single], thr)[0][0]
            identical = {}
            for share in modes:
                set_mode(share)
                identical[share] = all(same(o, want) for o in frame(ranks, thr)[0])
                for _ in range(args.warmup):
                    frame(ranks, thr)
            elapsed = {m: 0.0 for m in modes}
            pose_us = {m: np.zeros(world) for m in modes}
            refined = {}
            done = 0
            while done < args.frames:
                blk = min(10, args.frames - done)
                for share in modes:
                    set_mode(share)
                    t0 = time.perf_counter()
                    for _ in range(blk):
                        _, us = frame(ranks, thr)
                        pose_us[share] += us
                    elapsed[share] += time.perf_counter() - t0
                    refined[share] = [r.nat.pose_stats()[1] for r in ranks]
                done += blk
            for share in modes:
                results["runs"].append(dict(
                    world=world, threshold=thr, shared=share, survivors=int(want[4]["survivors"]), identical=identical[share],
                    frames_per_s=round(args.frames / elapsed[share], 1),
                    pose_stage_us_per_rank=[round(float(v) / args.frames, 1) for v in pose_us[share]],
                    refined_per_rank=refined[share]))
            print(json.dumps(results["runs"][-len(modes):]), flush=True)
        for r in ranks:
            if world > 1:
                r.nat.peer_disconnect()
            r.nat.close()
    line = json.dumps(results)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
