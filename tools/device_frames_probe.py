#!/usr/bin/env python
"""Frame rate from host frames against frames already in device memory, on the recorded driver frame
(tests/golden/driver_trace.npz) against the allScales bank with the shifted per-template renders of
tests/test_gpu_detect_batch.py:

  host    numpy rgb / u16 depth: lm_upload_images copies the frame and synchronises before the match is enqueued
  device  CUDA tensors already resident: lm_bind_images_device orders k_fe_ingest on the caller's stream, no synchronise

for detect (every survivor, 40 mm pose NMS) at thresholds 75 and 65 and match at 75.  The two inputs alternate in
blocks after warm-up; frames/s is a host clock around whole frames, each ending in a synchronise.  Results of both inputs
must be identical (exit status 1 otherwise).  --profile instead runs torch.profiler over device frames (u16 and float32
depth) and reports k_fe_ingest's mean time.  Reads the card's name and power limit.

  python tools/device_frames_probe.py [--frames 300] [--warmup 20] [--block 20] [--profile] [--out FILE]
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

SHIFTS = [(0, 0), (-68, -19), (-180, 57), (3, -2), (-2, 4)]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    if q.returncode != 0:
        raise RuntimeError("nvidia-smi failed: %s" % q.stderr.strip())
    name, power = [x.strip() for x in q.stdout.strip().split(",")[:2]]
    return dict(name=name, power_limit=power)


def setup():
    lib = importlib.import_module("6dpose_b200._lib")
    gold = os.path.join(ROOT, "tests", "golden")
    g = np.load(os.path.join(gold, "driver_trace.npz"))
    b = np.load(os.path.join(gold, "bank_allScales_full.npz"))
    packed = dict(class_begin=b["class_begin"], tmeta=b["tmeta"].astype(np.int32), feats=b["feats"].astype(np.int32))
    G = packed["tmeta"].shape[0]
    renders = [np.ascontiguousarray(np.roll(np.roll(g["render"], dy, 0), dx, 1)) for dy, dx in SHIFTS]
    K = np.repeat(g["rf0_modelK"][None], G, 0).astype(np.float32)
    R = np.repeat(g["rf0_modelR"][None], G, 0).astype(np.float32)
    t = np.repeat(g["rf0_modelT"].reshape(1, 3), G, 0).astype(np.float32)
    t[:, 0] += (np.arange(G) % 7) - 3.0
    t[:, 2] += np.arange(G) % 11
    nat = lib.NativeDetector(b["T"].tolist(), 0)
    nat.load_bank(packed, 4)
    nat.select(None, 0, 1)
    nat.set_template_renders(0, [renders[k] for k in np.arange(G) % len(renders)], K, R, t)
    return lib, nat, g["rgb"], g["depth"], g["rf0_sceneK"].astype(np.float32)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=300, help="timed frames per input and workload")
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--block", type=int, default=20)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    lib, nat, rgb, depth, sK = setup()
    d_rgb = torch.from_numpy(rgb).cuda()
    d_depth = torch.from_numpy(depth.view(np.int16)).cuda().view(torch.uint16)
    d_f32 = d_depth.to(torch.float32)
    torch.cuda.synchronize()
    report = dict(card=card(), frame=list(depth.shape))

    if args.profile:
        from torch.profiler import ProfilerActivity, profile
        for _ in range(args.warmup):
            nat.detect(d_rgb, d_depth, None, 75.0, sK)
        n = max(args.frames // 3, 10)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for fmt in ("u16", "f32"):
                for _ in range(n):
                    nat.detect(d_rgb, d_depth if fmt == "u16" else d_f32, None, 75.0, sK)
            torch.cuda.synchronize()
        times = [e.device_time for e in prof.events() if "k_fe_ingest" in e.name]
        kernels = {}
        for e in prof.events():
            if e.device_time > 0 and e.name.startswith("k_"):
                kernels.setdefault(e.name.split("(")[0], []).append(e.device_time)
        report["profile"] = dict(ingest_launches=len(times), ingest_us_u16=float(np.mean(times[:n])), ingest_us_f32=float(np.mean(times[n:])),
                                 front_end_us={k: float(np.mean(v)) for k, v in kernels.items() if k.startswith("k_fe_")})
    else:
        work = {
            "detect_75": lambda src: nat.detect(*src, None, 75.0, sK),
            "detect_65": lambda src: nat.detect(*src, None, 65.0, sK),
            "match_75": lambda src: nat.match_images(*src, None, 75.0),
        }
        inputs = {"host": (rgb, depth), "device": (d_rgb, d_depth)}
        ok = True
        for name, fn in work.items():
            outs = {k: fn(src) for k, src in inputs.items()}
            if name.startswith("detect"):
                same = all(np.array_equal(a, b, equal_nan=a.dtype.kind == "f") for a, b in zip(outs["host"][:4], outs["device"][:4]))
                same = same and outs["host"][4] == outs["device"][4]
            else:
                same = np.array_equal(outs["host"], outs["device"])
            ok = ok and same
            for k, src in inputs.items():
                for _ in range(args.warmup):
                    fn(src)
            spent = {k: 0.0 for k in inputs}
            done = {k: 0 for k in inputs}
            while done["host"] < args.frames:
                for k, src in inputs.items():
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    for _ in range(args.block):
                        fn(src)
                    torch.cuda.synchronize()
                    spent[k] += time.perf_counter() - t0
                    done[k] += args.block
            report[name] = dict(identical=bool(same), **{k + "_fps": done[k] / spent[k] for k in inputs})
        report["identical"] = ok
    line = json.dumps(report)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")
    if not args.profile and not report["identical"]:
        sys.exit(1)


if __name__ == "__main__":
    main()
