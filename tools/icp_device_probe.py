"""refine_matches from numpy depths (lm_icp_process_batch: the planes copied to the device) against the same call from
CUDA tensors (lm_icp_process_batch_device), on the recorded driver frame (tests/golden/driver_trace.npz) and its box-NMS
survivors against the allScales bank, with the shifted renders of tests/test_gpu_pose_stage.py.  For the first 3, 35 and
~390 survivors the two arms run in alternating blocks within this one process; per arm it prints the median wall time
per call, the median device time lm_icp_last_stats reports (from the input copy to the last ICP kernel, box read-back
included), whether the outputs are identical, and the card's power limit and SM clock.

    python tools/icp_device_probe.py [--blocks 6] [--calls 20]
"""
import argparse
import importlib
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
lib = importlib.import_module("6dpose_b200._lib")
pr = importlib.import_module("6dpose_b200.pose_refine")

SHIFTS = [(0, 0), (-68, -19), (-180, 57), (3, -2), (-2, 4)]


class Survivor:  # all refine_matches reads of a match
    def __init__(self, x, y):
        self.x, self.y = x, y


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=6)
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--threshold", type=float, default=50.0)
    a = ap.parse_args()
    g = np.load(os.path.join(ROOT, "tests", "golden", "driver_trace.npz"))
    b = np.load(os.path.join(ROOT, "tests", "golden", "bank_allScales_full.npz"))
    packed = dict(class_begin=b["class_begin"], tmeta=b["tmeta"].astype(np.int32), feats=b["feats"].astype(np.int32))
    G = packed["tmeta"].shape[0]
    renders = [np.ascontiguousarray(np.roll(np.roll(g["render"], dy, 0), dx, 1)) for dy, dx in SHIFTS]
    which = np.arange(G) % len(renders)
    K = np.repeat(g["rf0_modelK"][None], G, 0).astype(np.float32)
    R = np.repeat(g["rf0_modelR"][None], G, 0).astype(np.float32)
    t = np.repeat(g["rf0_modelT"].reshape(1, 3), G, 0).astype(np.float32)
    t[:, 0] += (np.arange(G) % 7) - 3.0
    t[:, 2] += np.arange(G) % 11
    sK = g["rf0_sceneK"].astype(np.float32)
    nat = lib.NativeDetector(b["T"].tolist(), 0)
    nat.load_bank(packed, 4)
    nat.select(None, 0, 1)
    nat.upload_images(g["rgb"], g["depth"], None)
    nat.enqueue(a.threshold)
    nat.enqueue_post(0.5, 0)
    surv = nat.complete_post()[0]
    ms = [Survivor(int(s["x"]), int(s["y"])) for s in surv]
    native = pr._native(0)
    scene_t = torch.from_numpy(g["depth"].view(np.int16)).cuda().view(torch.uint16)
    render_t = [torch.from_numpy(r.view(np.int16)).cuda().view(torch.uint16) for r in renders]
    torch.cuda.synchronize()
    out = dict(card=card(), survivors=len(surv), threshold=a.threshold, sizes=[])
    for n in (3, 35, 390):
        n = min(n, len(surv))
        tid = surv["template_id"][:n].astype(np.int64)
        args = (K[tid], R[tid], t[tid])
        host_in = (g["depth"], sK, ms[:n], [renders[k] for k in which[tid]])
        dev_in = (scene_t, sK, ms[:n], torch.stack([render_t[k] for k in which[tid]]))
        flat = lambda ps: [(p.getResidual(), None if p.getR() is None else (p.getR().tobytes(), p.getT().tobytes())) for p in ps]
        same = flat(pr.refine_matches(*host_in, *args)) == flat(pr.refine_matches(*dev_in, *args))
        wall, kern = {"numpy": [], "tensor": []}, {"numpy": [], "tensor": []}
        for _ in range(a.blocks):
            for name, inp in (("numpy", host_in), ("tensor", dev_in)):
                for _ in range(a.calls):
                    t0 = time.perf_counter()
                    pr.refine_matches(*inp, *args)
                    wall[name].append((time.perf_counter() - t0) * 1e6)
                    kern[name].append(native.last_stats()["kernel_us"])
        out["sizes"].append(dict(n=n, identical=bool(same), **{"%s_wall_us" % k: float(np.median(v)) for k, v in wall.items()},
                                 **{"%s_kernel_us" % k: float(np.median(v)) for k, v in kern.items()}))
    out["card_after"] = card()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
