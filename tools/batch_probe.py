#!/usr/bin/env python
"""Frame rate of n single-frame calls against one batch of the same n frames (lm_detect_batch), for n in {1, 8, 32}, on the
recorded driver frame (tests/golden/driver_trace.npz) against the allScales bank with the shifted per-template renders of
tests/test_gpu_pose_stage.py:

  refine   threshold 75, top 3:          Detector.match_refine per frame  vs  Detector.match_refine_batch
  detect   threshold 65, every survivor: Detector.detect per frame        vs  Detector.detect_batch

A batch fills the GPU with the survivors of all its frames at once; one frame's pose stage keeps only a few SMs busy.  The
two paths alternate in blocks after warm-up; frames/s is a host clock around whole calls, each ending in a synchronise.
Reads the card's name and power limit, and exits non-zero unless every frame's output of the batch equals the single-frame
call's.

  python tools/batch_probe.py [--frames 96] [--sizes 1,8,32] [--out FILE]
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

SHIFTS = [(0, 0), (-68, -19), (-180, 57), (3, -2), (-2, 4)]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    if q.returncode != 0:
        raise RuntimeError("nvidia-smi failed: %s" % q.stderr.strip())
    name, power, clock = [s.strip() for s in q.stdout.strip().split(",")]
    return dict(name=name, power_limit=power, max_sm_clock=clock)


def objects(pairs):
    def arr(a):
        return None if a is None else a.tobytes()
    return [(m.x, m.y, m.similarity, m.class_id, m.template_id, arr(p.getR()), arr(p.getT()), p.getResidual()) for m, p in pairs]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=96, help="frames per path and batch size (rounded up to whole batches)")
    ap.add_argument("--sizes", default="1,8,32")
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
    sK = g["rf0_sceneK"].astype(np.float32)
    frame = [g["rgb"], g["depth"]]
    cid = "06_template"

    bank = bk.TemplateBank()
    bank.classes[cid] = bk.PackedPyramids(tmeta, feats, 2)
    with tempfile.TemporaryDirectory() as tmp:
        bank.write_packed(cid, os.path.join(tmp, cid + ".lmb"), 2)
        det = pkg.Detector(int(g["num_features"]), b["T"].tolist())
        det.readClasses([cid], os.path.join(tmp, "%s.lmb"))
    det.setTemplateRenders({cid: ((renders[k] for k in which), K, R, t)})

    workloads = [
        ("refine", 75.0, lambda fr: [det.match_refine(f, 75.0, [cid], sK, top_k=3) for f in fr],
         lambda fr: det.match_refine_batch(fr, 75.0, [cid], sK, top_k=3)),
        ("detect", 65.0, lambda fr: [det.detect(f, 65.0, [cid], sK) for f in fr],
         lambda fr: det.detect_batch(fr, 65.0, [cid], sK)),
    ]
    results = dict(card=card(), frame="tests/golden/driver_trace.npz", bank="bank_allScales_full (%d templates)" % G, runs=[])
    ok = True
    for name, thr, single, batch in workloads:
        for n in [int(s) for s in args.sizes.split(",")]:
            frames = [frame] * n
            want = [objects(x) for x in single(frames)]
            got = [objects(x) for x in batch(frames)]
            identical = want == got
            ok &= identical
            paths = [("single", single), ("batch", batch)]
            for _, fn in paths:  # warm-up: buffers sized for this batch
                fn(frames)
            calls = max(1, -(-args.frames // n))
            elapsed = {p: 0.0 for p, _ in paths}
            block = max(1, calls // 4)
            done = 0
            while done < calls:
                blk = min(block, calls - done)
                for p, fn in paths:
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    for _ in range(blk):
                        fn(frames)
                    torch.cuda.synchronize()
                    elapsed[p] += time.perf_counter() - t0
                done += blk
            fps = {p: round(calls * n / elapsed[p], 1) for p, _ in paths}
            results["runs"].append(dict(workload=name, threshold=thr, n_frames=n, entries_per_frame=len(want[0]),
                                        frames_timed=calls * n, identical=identical, frames_per_s=fps,
                                        batch_over_single=round(fps["batch"] / fps["single"], 3)))
            print(json.dumps(results["runs"][-1]), flush=True)
    line = json.dumps(results)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")
    if not ok:
        raise SystemExit("a batch returned something else than the single-frame calls")


if __name__ == "__main__":
    main()
