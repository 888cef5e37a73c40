"""How many coarse candidates sit in runs of x-neighbours: the lengths k_refine_filter_w sees as one warp.

A run is a maximal set of consecutive passing cells of one template in one coarse row, cut every RUN_CAP cells.  On the
bench workload (T = [4, 8]) neighbouring cells are 4 columns apart at the filtered level, so a run of up to 5 candidates
has its 16-column patches inside one 32-column window.  Prints the fraction of candidates in runs of length 1..RUN_CAP.

    python tools/filter_runs.py [--templates 3115] [--frames 16] [--threshold 75]

CPU only: the pass masks come from the oracle's coarse similarity map (oracle/liblm_oracle.so, built by build()).
"""
import argparse
import importlib
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

RUN_CAP = 5


def cut_runs(mask, Wd, cap=RUN_CAP):
    """Row-major pass mask of one template -> (first cell index in the candidate list, length) per run.

    Runs are consecutive set bits, cut at row ends (cell % Wd == 0) and every `cap` cells."""
    cells = np.flatnonzero(np.asarray(mask).ravel())
    firsts, lens = [], []
    for k, j in enumerate(cells.tolist()):
        if lens and j == cells[k - 1] + 1 and j % Wd != 0 and lens[-1] < cap:
            lens[-1] += 1
        else:
            firsts.append(k)
            lens.append(1)
    return np.asarray(firsts, np.int64), np.asarray(lens, np.int64)


def pass_masks(q, T, packed, threshold):
    """Per template: the lowest level's coarse pass mask (score > threshold, LL.cpp:1836-1852), shape (Hd, Wd)."""
    from oracle import oracle
    L, M = len(T), len(q[0])
    low, Tl = q[-1], T[-1]
    tmeta, feats = packed["tmeta"], packed["feats"]
    thr = np.float32(threshold)
    out = []
    for g in range(tmeta.shape[0]):
        tm_low = tmeta[g, (L - 1) * M:L * M]
        nf_low = int(tm_low[:, 3].sum())
        cmap, _ = oracle.coarse_map(low, Tl, tm_low, feats)
        if nf_low == 0:
            out.append(np.zeros(cmap.shape, bool))
            continue
        s = np.float32(np.float32(cmap.astype(np.float32)) * np.float32(100.0)) / np.float32(4 * nf_low)
        out.append(s > thr)
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--templates", type=int, default=3115)
    ap.add_argument("--features", type=int, default=150)
    ap.add_argument("--objects", type=int, default=1)
    ap.add_argument("--width", type=int, default=640)
    ap.add_argument("--height", type=int, default=480)
    ap.add_argument("--threshold", type=float, default=75.0)
    ap.add_argument("--seed", type=int, default=1234)
    ap.add_argument("--frames", type=int, default=16)
    args = ap.parse_args()
    synth = importlib.import_module("6dpose_b200.synth")
    T = [4, 8]
    cids = tuple("%02d_template" % (k + 1) for k in range(max(args.objects, 1)))
    bank = synth.synth_bank(args.templates, num_features=args.features, levels=2, seed=args.seed, variants=35,
                            class_ids=cids)
    packed = bank.pack(bank.class_ids(), 2 * len(T))
    hist = np.zeros(RUN_CAP + 1, np.int64)  # candidates per run length
    for i in range(args.frames):
        q, _ = synth.synth_frame(args.width, args.height, levels=2, seed=1000 + i, bank=bank, plant=8, T=T)
        for m in pass_masks(q, T, packed, args.threshold):
            _, lens = cut_runs(m, m.shape[1])
            hist += np.bincount(lens, weights=lens, minlength=RUN_CAP + 1).astype(np.int64)
    n = int(hist.sum())
    frac = {str(k): round(float(hist[k]) / max(n, 1), 4) for k in range(1, RUN_CAP + 1)}
    print(json.dumps(dict(frames=args.frames, threshold=args.threshold, templates=args.templates,
                          candidates_per_frame=n / args.frames, fraction_by_run_length=frac,
                          fraction_in_runs_ge3=round(float(hist[3:].sum()) / max(n, 1), 4))))


if __name__ == "__main__":
    main()
