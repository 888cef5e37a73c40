#!/usr/bin/env python
"""What the depth gate of the coarse scan (Detector.setDepthGate) saves on the reference's fixture frame (tests/golden/
driver_trace.npz, in the BGR order the reference's own test reads it) against the whole allScales bank (2989 templates,
distances from tests/golden/allScales_depths.npz) with the shifted per-template renders of tests/test_gpu_pose_nms.py.

At thresholds 65, 75 and 80, gate off against tolerance 0.15, alternating in blocks after warm-up:
  candidates        coarse candidates (gate on: before / after the gate)
  filter_exact_us   refinement filter + exact refinement (stage timing events: median of 8 means over 16 frames)
  survivors         box-NMS survivors (IoU 0.5, every survivor)
  detect_fps        Detector.detect frames/s (front-end, match, box NMS, ICP of every survivor, pose NMS); host clock
                    around whole frames, each ending in a synchronise
Then, in a run of its own under torch.profiler: mean device time of k_depth_cells and of the coarse scan, gate off / on.
Reads the card's name and power limit; exits non-zero unless the first gated match at 75 lies on the ground-truth box.

  python tools/depth_gate_probe.py [--frames 100] [--warmup 10] [--block 10] [--out FILE]
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
    ap.add_argument("--frames", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
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
    nat.set_timing(64)

    def gate(tau):
        det.setDepthGate(tau)

    def match_stage(thr):
        nat.upload_images(rgb, depth, None)
        nat.enqueue(thr)
        nat.enqueue_post(0.5, 0)
        surv, _ = nat.complete_post()
        return surv

    results = dict(card=card(), frame="tests/golden/driver_trace.npz (BGR)", bank="bank_allScales_full (%d templates)" % G,
                   tolerance=TAU, frames=args.frames, runs=[])
    ok = True
    for thr in (65.0, 75.0, 80.0):
        run = dict(threshold=thr)
        for name, tau in (("off", None), ("on", TAU)):
            gate(tau)
            nat.set_timing(64)
            surv = match_stage(thr)
            nat.upload_images(rgb, depth, None)
            nat.run(thr)
            c = nat.counters()
            st = nat.depth_gate_stats() if tau is not None else None
            filt = []
            for _ in range(8):
                nat.set_timing(64)
                for _ in range(16):
                    match_stage(thr)
                s = nat.stage_times_us()
                filt.append(s["refine_filter"] + s["refine_exact"])
            run[name] = dict(candidates=c["coarse_candidates"], before_gate=st["before"] if st else c["coarse_candidates"],
                             empty_cells=st["empty_cells"] if st else None, survivors=int(len(surv)),
                             filter_exact_us=round(float(np.median(filt)), 1))
            if tau is not None and thr == 75.0:
                m = det.match([rgb, depth], thr, [cid], masks=[])[0]
                w, h = int(tmeta[m.template_id, 0, 0]), int(tmeta[m.template_id, 0, 1])
                gx, gy, gw, gh = 331, 130, 65, 64
                iw = max(0, min(m.x + w, gx + gw) - max(m.x, gx))
                ih = max(0, min(m.y + h, gy + gh) - max(m.y, gy))
                iou = iw * ih / float(w * h + gw * gh - iw * ih)
                run[name]["first_match"] = dict(x=m.x, y=m.y, template_id=m.template_id, iou_with_ground_truth=round(iou, 3))
                ok &= iou >= 0.5
        # detect frames/s, gate off / on alternating in blocks
        for tau in (None, TAU):
            gate(tau)
            for _ in range(args.warmup):
                det.detect([rgb, depth], thr, [cid], sK)
        elapsed = {"off": 0.0, "on": 0.0}
        kept = {}
        done = 0
        while done < args.frames:
            blk = min(args.block, args.frames - done)
            for name, tau in (("off", None), ("on", TAU)):
                gate(tau)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for _ in range(blk):
                    kept[name] = len(det.detect([rgb, depth], thr, [cid], sK))
                elapsed[name] += time.perf_counter() - t0
            done += blk
        for name in ("off", "on"):
            run[name]["detect_fps"] = round(args.frames / elapsed[name], 1)
            run[name]["detect_kept"] = kept[name]
        results["runs"].append(run)

    # kernel times under the profiler (a run of its own)
    from torch.profiler import ProfilerActivity, profile
    kern = {}
    for name, tau in (("off", None), ("on", TAU)):
        gate(tau)
        for _ in range(5):
            match_stage(75.0)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(50):
                match_stage(75.0)
        acc = {}
        for e in prof.events():
            if e.device_type.name == "CUDA" and any(k in e.name for k in ("k_depth_cells", "k_coarse_packed", "k_coarse_bytes")):
                key = "k_depth_cells" if "k_depth_cells" in e.name else "coarse_scan"
                acc.setdefault(key, []).append(e.device_time if hasattr(e, "device_time") else e.cuda_time)
        kern[name] = {k: round(float(np.mean(v)), 2) for k, v in acc.items()}
    results["kernel_us_threshold_75"] = kern
    gate(None)
    line = json.dumps(results)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")
    if not ok:
        raise SystemExit("the first gated match at threshold 75 is not on the ground-truth box")


if __name__ == "__main__":
    main()
