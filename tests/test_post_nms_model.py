"""The box NMS model (tests/post_nms_model.py) against the reference drivers' pipeline on the reference's fixture
frames: nms() on the FINISHED list (std::sort + std::unique, LL.cpp:1772-1774) == the model's canonical dedupe +
greedy NMS on the raw records, while the NMS on the raw records alone (what k_post_nms did before the dedupe)
is told apart.  No GPU: the oracle builds on a CPU."""
import importlib
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import post_nms_model as pm  # noqa: E402

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
IOUS = (0.3, 0.5, 0.7, 0.9, 0.99)
BOX_SEEDS = (2, 5)          # seeded caller boxes, 20..160 pixels a side
DIVERGE_SEED = 2            # with it, the raw-record NMS differs from the drivers on both allScales frames at 65 / 0.5


def frames():
    fr = np.load(os.path.join(GOLD, "frames_case1.npz"))
    return {tag: [[fr["%s_l%d_m%d" % (tag, l, m)] for m in range(2)] for l in range(2)] for tag in ("full", "half")}


def bank(name):
    b = np.load(os.path.join(GOLD, "bank_%s.npz" % name))
    return dict(class_begin=b["class_begin"], tmeta=b["tmeta"].astype(np.int32), feats=b["feats"].astype(np.int32)), \
        b["T"].tolist()


def seeded_boxes(G, seed):
    return np.random.RandomState(seed).randint(20, 161, size=(G, 2)).astype(np.int32)


def box_sets(packed):
    G = packed["tmeta"].shape[0]
    sets = {"template": packed["tmeta"][:, 0, :2].copy()}
    for s in BOX_SEEDS:
        sets["seed%d" % s] = seeded_boxes(G, s)
    return sets


def fixture_cases():
    exp = np.load(os.path.join(GOLD, "expected_case1.npz"))
    out = []
    for key in sorted(exp.files):
        name, tag, thr = key.rsplit("_", 2)
        if len(exp[key]):
            out.append((name, tag, float(thr)))
    return out + [("allScales_full", "full", 75.0), ("allScales_full", "full", 80.0)]


def lowest_tid_dedupe(records):
    """The rule that does NOT reproduce the drivers: keep the lowest template_id per (x, y, similarity, class)."""
    s = records[pm.canonical_order(records)]
    key = np.stack([s["x"], s["y"], s["similarity"].view(np.int32), s["class_idx"]], 1)
    _, first = np.unique(key, axis=0, return_index=True)
    return s[np.sort(first)]


def test_model_equals_the_drivers_on_the_fixture_frames(oracle):
    fr = frames()
    cases = fixture_cases()
    assert len(cases) == 12
    deduped_some = 0
    for name, tag, thr in cases:
        packed, T = bank(name)
        pre = oracle.match(fr[tag], T, packed, thr, presort=True)
        fin = oracle.match(fr[tag], T, packed, thr)
        assert len(fin) > 0 and len(pre) >= len(fin)
        deduped_some += len(pre) > len(pm.canonical_dedupe(pre))
        cb = packed["class_begin"]
        for bn, wh in box_sets(packed).items():
            for iou in IOUS:
                want = pm.driver_nms(fin, wh, cb, iou)
                for top_k in (0, 1, 3, 17):
                    got, counts = pm.post_nms(pre, wh, cb, iou, top_k)
                    n = min(top_k, 1024) if top_k > 0 else 1024
                    assert pm.same(got, want[:n]), (name, tag, thr, bn, iou, top_k)
                    assert counts == [min(len(want), n), len(pre), -1 if top_k > 0 else len(want)]
    assert deduped_some >= 6


def test_raw_record_nms_differs_from_the_drivers(oracle):
    """Without the dedupe (the device before it) the NMS keeps matches std::unique removed: the comparison above
    can tell the two apart."""
    fr = frames()
    packed, T = bank("allScales")
    cb = packed["class_begin"]
    wh = seeded_boxes(packed["tmeta"].shape[0], DIVERGE_SEED)
    for tag in ("half", "full"):
        pre = oracle.match(fr[tag], T, packed, 65.0, presort=True)
        fin = oracle.match(fr[tag], T, packed, 65.0)
        want = pm.driver_nms(fin, wh, cb, 0.5)
        raw = pm.raw_nms(pre, wh, cb, 0.5)
        assert not pm.same(raw, want), tag
        assert pm.same(pm.post_nms(pre, wh, cb, 0.5)[0], want)
        # and the lowest-template rule is not the drivers' either
        low = pm.driver_nms(lowest_tid_dedupe(pre), wh, cb, 0.99)
        assert not pm.same(low, pm.driver_nms(fin, wh, cb, 0.99)), tag


def test_a_run_between_twins_decides_what_unique_removes():
    """A = (x, y, s, c) of template 1 and B = the same of template 3, with a box B's that overlaps A's little.  When A
    is the last record of template 1's run at s and B the first of template 3's, B follows A in the canonical order
    and is removed.  A record of template 2 at s in between -- or one of template 1 after A, or one of template 3
    before B -- makes B a match of its own, and B then also suppresses C, which A leaves alone."""
    dt = [("x", "<i4"), ("y", "<i4"), ("similarity", "<f4"), ("class_idx", "<i4"), ("template_id", "<i4")]
    wh = np.array([[29, 29], [9, 9], [9, 9], [49, 49]], np.int32)
    cb = np.array([0, 4], np.int32)
    A = (100, 100, 90.0, 0, 1)   # 10 x 10 pixels
    B = (100, 100, 90.0, 0, 3)   # 50 x 50 pixels: IoU with A 100 / 2500
    C = (120, 120, 80.0, 0, 0)   # 30 x 30 pixels inside B's box (IoU 900 / 2500), apart from A's
    cases = {
        "adjacent": ([], False),
        "run of template 2 between": ([(300, 300, 90.0, 0, 2)], True),
        "template 1 after A": ([(101, 300, 90.0, 0, 1)], True),
        "template 3 before B": ([(99, 0, 90.0, 0, 3)], True),
        "template 1 before A": ([(99, 0, 90.0, 0, 1)], False),
        "template 3 after B": ([(101, 300, 90.0, 0, 3)], False),
        "template 2 at another similarity": ([(300, 300, 85.0, 0, 2)], False),
        "exact twin of A": ([A], False),
        "exact twin of B": ([B], False),
    }
    for name, (extra, b_kept) in cases.items():
        recs = np.array([A, B, C] + extra, dt)
        for perm in (np.arange(len(recs)), np.arange(len(recs))[::-1]):
            d = [tuple(r) for r in pm.canonical_dedupe(recs[perm]).tolist()]
            assert (B in d) == b_kept and d.count(A) == 1 and d.count(B) <= 1, name
            got, counts = pm.post_nms(recs[perm], wh, cb, 0.1)
            got = [tuple(r) for r in got.tolist()]
            assert A in got and (B in got) == b_kept and (C in got) == (not b_kept), name
            assert counts == [len(got), len(recs), len(got)]
            assert len(got) == len(d) - b_kept     # every other record is disjoint from the rest


def test_iou_exactly_at_the_threshold():
    """ovr == thr survives, the next double above it too, the next below suppresses; integer boxes ("+1": a width
    of 9 is 10 pixels) give ovr = 1/3, 1/2 and 1 exactly."""
    dt = [("x", "<i4"), ("y", "<i4"), ("similarity", "<f4"), ("class_idx", "<i4"), ("template_id", "<i4")]
    cb = np.array([0, 3], np.int32)
    wh = np.array([[9, 9], [19, 9], [0, 0]], np.int32)
    for recs, ovr in (([(0, 0, 90.0, 0, 0), (5, 0, 80.0, 0, 0)], 1.0 / 3.0),    # inter 50, union 150
                      ([(0, 0, 90.0, 0, 0), (0, 0, 80.0, 0, 1)], 0.5),          # 10 x 10 inside 20 x 10
                      ([(7, 7, 90.0, 0, 2), (7, 7, 80.0, 0, 2)], 1.0),          # zero-size boxes: one pixel each
                      ([(7, 7, 90.0, 0, 2), (8, 7, 80.0, 0, 2)], 0.0)):
        recs = np.array(recs, dt)
        for thr, n in ((ovr, 2), (np.nextafter(ovr, 2.0), 2), (np.nextafter(ovr, -1.0), 1)):
            if thr >= 0:
                assert len(pm.post_nms(recs, wh, cb, thr)[0]) == n, (ovr, thr)


def test_banks_beyond_the_key_widths_are_refused():
    """The device's pick key holds 12 bits of class and 20 of template: a bank of 4 097 classes is refused, 4 096 is
    taken.  Host-only handle: no GPU involved."""
    lib = importlib.import_module("6dpose_b200._lib")
    tm = np.zeros((4097, 4, 4), np.int32)
    tm[:, :, 0:2] = 8
    tm[:, :, 3] = 1
    tm[:, :, 2] = np.arange(4097)[:, None]
    feats = np.zeros((4097, 3), np.int32)
    nat = lib.NativeDetector([4, 8], device=-1)
    with pytest.raises(RuntimeError, match="4096"):
        nat.load_bank(dict(class_begin=np.arange(4098, dtype=np.int32), tmeta=tm, feats=feats), 4)
    nat.load_bank(dict(class_begin=np.arange(4097, dtype=np.int32), tmeta=tm[:4096], feats=feats[:4096]), 4)
