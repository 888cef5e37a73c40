"""The box NMS on the device (k_post_nms) against its model (tests/post_nms_model.py), bit for bit: x, y, similarity,
class, template, pick order and counts.  Real frames: the reference's fixture frames and banks, the model fed the
oracle's raw records.  Crafted record sets: a frame's result block, held by the caller, overwritten on the handle's
stream between lm_enqueue and lm_enqueue_post with a chosen count and records."""
import importlib
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import post_nms_model as pm  # noqa: E402
from test_post_nms_model import bank, frames, seeded_boxes  # noqa: E402

pytestmark = pytest.mark.gpu

lib = importlib.import_module("6dpose_b200._lib")
synth = importlib.import_module("6dpose_b200.synth")

TOP_KS = (1, 3, 16, 17, 0)   # 16 = the survivors fetched with the counts, 17 takes the second copy


def check(got, nrec, want, counts):
    assert pm.same(got, want)
    assert len(got) == counts[0] and nrec == counts[1]


@pytest.mark.parametrize("name,tag,thr", [("63", "full", 60.0), ("127", "half", 60.0), ("allScales", "half", 65.0),
                                          ("allScales", "full", 65.0), ("allScales", "full", 75.0),
                                          ("allScales_full", "full", 75.0), ("allScales_full", "full", 80.0)])
def test_fixture_frames_equal_the_model(oracle, name, tag, thr):
    fr = frames()
    packed, T = bank(name)
    cb = packed["class_begin"]
    pre = oracle.match(fr[tag], T, packed, thr, presort=True)
    G = packed["tmeta"].shape[0]
    nat = lib.NativeDetector(T, 0)
    nat.load_bank(packed, 4)
    # a fresh handle's first frame (grown and replayed if it overflows the first block), then the same frame again
    for _ in range(2):
        got, nrec = nat.match_top(fr[tag], thr, 0.5, 0)
        check(got, nrec, *pm.post_nms(pre, packed["tmeta"][:, 0, :2], cb, 0.5, 0))
    for boxes in ("template", 2, 5):
        wh = packed["tmeta"][:, 0, :2].copy() if boxes == "template" else seeded_boxes(G, boxes)
        nat.set_boxes(None if boxes == "template" else wh)
        for iou in (0.3, 0.5, 0.7, 0.9, 0.99, 1.0, 2.0):
            every, counts = pm.post_nms(pre, wh, cb, iou, 0)
            for top_k in TOP_KS:
                got, nrec = nat.match_top(fr[tag], thr, iou, top_k)
                k = top_k if top_k > 0 else 1024
                check(got, nrec, every[:k], [min(counts[0], k), counts[1]])
    # the staged calls
    nat.upload_quantized(fr[tag])
    nat.enqueue(thr)
    nat.enqueue_post(0.5, 17)
    got, nrec = nat.complete_post()
    check(got, nrec, *pm.post_nms(pre, wh, cb, 0.5, 17))


def test_seeded_boxes_where_the_raw_records_differ(oracle):
    """allScales, threshold 65, seeded caller boxes, IoU 0.5: the NMS on the raw records (the device before the
    canonical dedupe) differs from the drivers here (tests/test_post_nms_model.py); the device equals the drivers."""
    fr = frames()
    packed, T = bank("allScales")
    cb = packed["class_begin"]
    wh = seeded_boxes(packed["tmeta"].shape[0], 2)
    nat = lib.NativeDetector(T, 0)
    nat.load_bank(packed, 4)
    nat.set_boxes(wh)
    for tag in ("half", "full"):
        fin = oracle.match(fr[tag], T, packed, 65.0)
        got, _ = nat.match_top(fr[tag], 65.0, 0.5, 0)
        assert pm.same(got, pm.driver_nms(fin, wh, cb, 0.5)), tag


# ---- crafted record sets ----------------------------------------------------------------------------------------
CAP = 16384                 # records the caller's block holds: 9 000 records sort in the global scratch


@pytest.fixture(scope="module")
def crafted():
    import torch
    bk = synth.synth_bank(24, num_features=63, seed=5, class_ids=("01_template", "02_template", "03_template"))
    packed = bk.pack(bk.class_ids(), 4)
    nat = lib.NativeDetector([4, 8], 0)
    nat.load_bank(packed, 4)
    q, _ = synth.synth_frame(640, 480, seed=6, bank=bk, plant=0, T=[4, 8])
    block = torch.zeros(16 + 16 * CAP, dtype=torch.uint8, device="cuda")
    nat.set_result_buffer(block.data_ptr(), CAP)
    yield nat, packed, q, block
    nat.set_result_buffer(0, 0)
    nat.close()


def run_crafted(crafted, recs, wh, iou, top_k):
    """Device survivors and n_records for the records `recs` (RECORD_DTYPE, work = global template index)."""
    import torch
    nat, packed, q, block = crafted
    assert len(recs) <= CAP
    nat.set_boxes(wh)
    src = torch.from_numpy(np.concatenate([np.array([len(recs)], np.int32).view(np.uint8),
                                           np.ascontiguousarray(recs, lib.RECORD_DTYPE).view(np.uint8)])).cuda()
    torch.cuda.synchronize()
    nat.upload_quantized(q)
    nat.enqueue(99.0)                                 # the frame's own records, at most a few, and its candidates
    with torch.cuda.stream(torch.cuda.ExternalStream(nat.stream())):
        block[0:4].copy_(src[0:4])                    # the count; coarse_candidates stays the frame's own
        if len(recs):
            block[16:16 + 16 * len(recs)].copy_(src[4:])
    nat.enqueue_post(iou, top_k)
    return nat.complete_post()


def as_model(recs, cb):
    g = recs["work"].astype(np.int64)
    c = np.searchsorted(cb, g, side="right") - 1
    out = np.zeros(len(recs), lib.MATCH_DTYPE)
    out["x"], out["y"], out["similarity"] = recs["x"], recs["y"], recs["similarity"]
    out["class_index"], out["template_id"] = c, g - cb[c]
    return out


def crafted_equals_model(crafted, recs, wh, ious=(0.0, 0.3, 0.5, 1.0), top_ks=TOP_KS):
    cb = crafted[1]["class_begin"]
    for iou in ious:
        for top_k in top_ks:
            got, nrec = run_crafted(crafted, recs, wh, iou, top_k)
            want, counts = pm.post_nms(as_model(recs, cb), wh, cb, iou, top_k)
            assert pm.same(got, want), (len(recs), iou, top_k)
            assert len(got) == counts[0] and nrec == counts[1] == len(recs)


def tie_records(rng, n, G):
    """Ties at every level of the key: few similarities, templates, positions; exact twins and cross-template pairs."""
    r = np.zeros(n, lib.RECORD_DTYPE)
    r["similarity"] = rng.choice(np.array([70.0, 75.5, 80.25, 100.0], np.float32), n)
    r["work"] = rng.randint(0, G, n)
    r["x"] = rng.randint(0, 6, n) * 4
    r["y"] = rng.randint(0, 6, n) * 4
    r["seq"] = np.arange(n)
    twins = rng.randint(0, n, n // 8)
    r[-len(twins):] = r[twins]
    return r[rng.permutation(n)]


def test_crafted_ties_twins_and_runs(crafted):
    G = crafted[1]["tmeta"].shape[0]
    rng = np.random.RandomState(11)
    for seed in range(3):
        wh = np.random.RandomState(seed).randint(0, 30, size=(G, 2)).astype(np.int32)
        crafted_equals_model(crafted, tie_records(rng, 700, G), wh, ious=(0.0, 0.1, 0.3, 0.5, 0.9, 1.0, 1.5))


def test_crafted_run_boundaries(crafted):
    """A (template 1) and B (template 3) of class 0 at one (x, y, similarity), with and without a record between them
    in the canonical order; B's box overlaps A's little and C's much."""
    cb = crafted[1]["class_begin"]
    G = crafted[1]["tmeta"].shape[0]
    wh = np.full((G, 2), 9, np.int32)
    wh[cb[0] + 0] = 29
    wh[cb[0] + 3] = 49

    def rec(x, y, s, t, c=0):
        return (x, y, s, cb[c] + t, 0)

    A, B, C = rec(100, 100, 90.0, 1), rec(100, 100, 90.0, 3), rec(120, 120, 80.0, 0)
    extras = [[], [rec(300, 300, 90.0, 2)], [rec(101, 300, 90.0, 1)], [rec(99, 0, 90.0, 3)], [rec(99, 0, 90.0, 1)],
              [rec(101, 300, 90.0, 3)], [rec(300, 300, 85.0, 2)], [A], [B], [rec(100, 100, 90.0, 2, 1)]]
    for extra in extras:
        recs = np.array([A, B, C] + extra, lib.RECORD_DTYPE)
        for perm in (np.arange(len(recs)), np.arange(len(recs))[::-1]):
            crafted_equals_model(crafted, recs[perm], wh, ious=(0.1,), top_ks=(0, 2))


def test_crafted_iou_at_the_threshold(crafted):
    """ovr = 1/3, 1/2 and 1 exactly (integer boxes, "+1" convention), thresholds at ovr and the next double on either
    side; zero-size boxes are one pixel."""
    cb = crafted[1]["class_begin"]
    G = crafted[1]["tmeta"].shape[0]
    wh = np.zeros((G, 2), np.int32)
    wh[0] = (9, 9)
    wh[1] = (19, 9)
    cases = (([(0, 0, 90.0, 0, 0), (5, 0, 80.0, 0, 0)], 1.0 / 3.0),
             ([(0, 0, 90.0, 0, 0), (0, 0, 80.0, 1, 0)], 0.5),
             ([(7, 7, 90.0, 2, 0), (7, 7, 80.0, 2, 0)], 1.0),
             ([(7, 7, 90.0, 2, 0), (8, 7, 80.0, 2, 0)], 0.0))
    for recs, ovr in cases:
        recs = np.array(recs, lib.RECORD_DTYPE)
        ious = [t for t in (ovr, np.nextafter(ovr, 2.0), np.nextafter(ovr, -1.0)) if t >= 0]
        crafted_equals_model(crafted, recs, wh, ious=ious, top_ks=(0,))
        for thr in ious:
            got, _ = run_crafted(crafted, recs, wh, thr, 0)
            assert len(got) == (2 if thr >= ovr else 1)
    assert cb[1] > 2


@pytest.mark.parametrize("n", [0, 1, 1023, 1024, 1025, 4999, 9000])
def test_crafted_counts(crafted, n):
    G = crafted[1]["tmeta"].shape[0]
    rng = np.random.RandomState(n)
    r = np.zeros(n, lib.RECORD_DTYPE)
    r["similarity"] = (rng.randint(600, 1000, n) / 10.0).astype(np.float32)
    r["work"] = rng.randint(0, G, n)
    r["x"] = rng.randint(0, 160, n) * 4
    r["y"] = rng.randint(0, 120, n) * 4
    r["seq"] = np.arange(n)
    wh = np.random.RandomState(1).randint(0, 40, size=(G, 2)).astype(np.int32)
    crafted_equals_model(crafted, r, wh, ious=(0.3, 1.0), top_ks=(3, 17, 0))


def test_crafted_more_than_1024_survivors(crafted):
    """1 500 disjoint one-pixel boxes, every one a survivor: exactly the model's first 1 024 come back."""
    G = crafted[1]["tmeta"].shape[0]
    n = 1500
    rng = np.random.RandomState(3)
    r = np.zeros(n, lib.RECORD_DTYPE)
    cell = rng.permutation(50 * 40)[:n]
    r["x"], r["y"] = (cell % 50) * 3, (cell // 50) * 3
    r["similarity"] = rng.choice(np.array([80.0, 90.0], np.float32), n)
    r["work"] = rng.randint(0, G, n)
    r["seq"] = np.arange(n)
    wh = np.zeros((G, 2), np.int32)
    got, nrec = run_crafted(crafted, r, wh, 0.5, 0)
    want, counts = pm.post_nms(as_model(r, crafted[1]["class_begin"]), wh, crafted[1]["class_begin"], 0.5, 0)
    assert counts == [1024, n, n] and len(got) == 1024 and nrec == n
    assert pm.same(got, want)
