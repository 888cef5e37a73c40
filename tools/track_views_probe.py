#!/usr/bin/env python
"""View following (include/linemod_b200.h, lm_set_track_views) on the device:
  sequence   the synthetic turning solid of tests/view_object.py (180 degrees in 60 frames of 3 degrees) tracked with
             lm_track from its first frame's template, view following off and on (turn 20 degrees): per frame the
             rotation and position error against the truth, the template, and the number of switches
  kernel     k_track_views's device time from torch.profiler (CUDA activities, a run of its own) for 1 and 1024 objects
             against one class of 2989 templates (the allScales bank's size) and one of 30000, turn 0 so that every
             object scans its class; tiny renders, since the kernel reads only R_b and t_b
Reads the card's name, power limit and max SM clock in the same run.

  python tools/track_views_probe.py [--reps 50] [--out FILE]
"""
import argparse
import importlib
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from detect_probe import card  # noqa: E402


def sequence(lib, vo, tvm):
    Rb, tb, Kb = vo.templates()
    renders = [vo.template_render(Rb[g], tb[g]) for g in range(len(Rb))]
    synth = importlib.import_module("6dpose_b200.synth")
    bank = synth.synth_bank(len(Rb), num_features=30, seed=1, variants=35)
    nat = lib.NativeDetector([4, 8], 0)
    nat.load_bank(bank.pack(bank.class_ids(), 4), 4)
    nat.set_template_renders(0, renders, Kb, Rb, tb)
    seq = vo.sequence(Rb[tvm.START].astype(np.float64), tvm.FRAMES, tvm.STEP_DEG)
    out = {}
    for views in (False, True):
        nat.set_track_views(views, tvm.TURN_DEG)
        g, T = tvm.START, vo.start_T(seq[0][1], seq[0][2], Rb[tvm.START], tb[tvm.START])
        rows, switches = [], 0
        for f, (scene, R, b) in enumerate(seq[1:], 1):
            status, T_out, *_ = nat.track(scene, vo.K.astype(np.float32), [(0, g, T)], 30, 4)
            j = int(nat.track_templates()[0])
            if status[0] != 0:
                rows.append(dict(frame=f, status=int(status[0])))
                break
            switches += j != g
            g, T = j, T_out[0]
            rot, pos = vo.errors(T, Rb[g], tb[g], R, b)
            rows.append(dict(frame=f, template=g, rot_deg=round(rot, 3), pos_mm=round(pos, 3)))
        done = [r for r in rows if "rot_deg" in r]
        out["on" if views else "off"] = dict(switches=switches, frames=rows, worst_rot_deg=max(r["rot_deg"] for r in done),
                                             worst_pos_mm=max(r["pos_mm"] for r in done))
        print("view following %s: %d switches, worst rotation %.2f deg, worst position %.2f mm" %
              ("on" if views else "off", switches, out["on" if views else "off"]["worst_rot_deg"], out["on" if views else "off"]["worst_pos_mm"]))
    return out


def kernel(lib, reps):
    import torch
    from torch.profiler import ProfilerActivity, profile
    synth = importlib.import_module("6dpose_b200.synth")
    rng = np.random.default_rng(1)
    render = np.zeros((64, 64), np.uint16)
    render[24:40, 24:40] = 500
    sK = np.array([[60, 0, 32], [0, 60, 32], [0, 0, 1]], np.float32)
    scene = np.full((64, 64), 500, np.uint16)
    out = {}
    for G in (2989, 30000):
        bank = synth.synth_bank(G, num_features=30, seed=1, variants=1000)
        nat = lib.NativeDetector([4, 8], 0)
        nat.load_bank(bank.pack(bank.class_ids(), 4), 4)
        q = rng.normal(size=(G, 3))
        Rb = np.stack([importlib.import_module("pso_scenes").rodrigues(v) for v in q]).astype(np.float32)
        nat.set_template_renders(0, [render] * G, np.repeat(sK[None], G, 0), Rb, np.tile(np.float32([0, 0, 500]), (G, 1)))
        nat.set_track_views(True, 0.0)
        for n in (1, 1024):
            objs = [(0, int(rng.integers(G)), np.eye(4)) for _ in range(n)]
            nat.track(scene, sK, objs, 1, 4)  # warm-up
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(reps):
                    nat.track(scene, sK, objs, 1, 4)
                torch.cuda.synchronize()
            times = [e.device_time for e in prof.events() if "k_track_views" in e.name]
            out["%d_templates_%d_objects_us" % (G, n)] = round(float(np.mean(times)), 2) if times else None
            print("k_track_views: %d templates, %d objects: %s us (%d launches)" % (G, n, out["%d_templates_%d_objects_us" % (G, n)], len(times)))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    lib = importlib.import_module("6dpose_b200._lib")
    vo = importlib.import_module("view_object")
    tvm = importlib.import_module("test_track_views_model")
    res = dict(card=card(), sequence=sequence(lib, vo, tvm), kernel=kernel(lib, a.reps))
    print(json.dumps(dict(card=res["card"], kernel=res["kernel"])))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
