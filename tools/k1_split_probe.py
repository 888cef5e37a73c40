#!/usr/bin/env python
"""Where K1's time goes on the bench workload: the device time of the lowest level's blocks, of level 0's blocks (H-planes
when the bit-sliced refinement takes the whole bank) and of the whole K1 launch, each launched on its own `--reps` times
after a few matched frames (lm_debug_time_k1, CUDA events).  Development probe: prints one JSON line.

  python tools/k1_split_probe.py [--templates 3115] [--reps 2000] [--threshold 75]
"""
import argparse
import importlib
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--templates", type=int, default=3115)
    ap.add_argument("--reps", type=int, default=2000)
    ap.add_argument("--threshold", type=float, default=75.0)
    ap.add_argument("--width", type=int, default=640)
    ap.add_argument("--height", type=int, default=480)
    args = ap.parse_args()
    lib = importlib.import_module("6dpose_b200._lib")
    synth = importlib.import_module("6dpose_b200.synth")
    T = [4, 8]
    bank = synth.synth_bank(args.templates, num_features=150, levels=2, seed=1234, variants=35)
    packed = bank.pack(bank.class_ids(), 4)
    frames = [synth.synth_frame(args.width, args.height, levels=2, seed=1000 + i, bank=bank, plant=8, T=T)[0] for i in range(4)]
    nat = lib.NativeDetector(T)
    nat.load_bank(packed, 4)
    for q in frames:
        nat.match_quantized(q, args.threshold)
    plan = nat.plan()
    out = {"plan": {k: plan[k] for k in ("k1_band", "planes_level", "pseg", "k1_smem") if k in plan}}
    if "k1_low_mode" in plan:
        out["plan"]["k1_low_mode"] = plan["k1_low_mode"]
    nat.time_k1_us(-1, 50)  # warm-up
    out["k1_us"] = {"lowest_level": round(nat.time_k1_us(len(T) - 1, args.reps), 2),
                    "level_0": round(nat.time_k1_us(0, args.reps), 2),
                    "all": round(nat.time_k1_us(-1, args.reps), 2)}
    print(json.dumps(out))
    nat.close()


if __name__ == "__main__":
    main()
