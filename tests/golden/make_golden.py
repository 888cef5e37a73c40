#!/usr/bin/env python
"""Regenerates tests/golden/*.npz from the reference's own fixtures (needs /root/reference mounted
and oracle/_ref built: `make -C oracle ref`).

Inputs : linemodLevelup/test/case1/0000_{rgb,dep}.png (+ _half), banks 63/, 127/, allScales/
         (reference: linemodLevelup/test.cpp:90-128, 174-181 -- the invocations the reference's own
         test driver makes: Detector(127,{5,8}) + thr 75, Detector() + allScales + thr 80).
Stored : the quantized label pyramids produced by 6dpose_b200/frontend.py (so the GPU box needs no
         reference checkout), the packed template banks, and the expected match lists computed by the
         REFERENCE'S OWN CODE (oracle/_ref = linemodLevelup.cpp compiled unmodified).
"""
import importlib
import os
import sys

import cv2
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
CASE = "/root/reference/linemodLevelup/test/case1/"
OUT = os.path.dirname(os.path.abspath(__file__))


def main():
    fe = importlib.import_module("6dpose_b200.frontend")
    bk = importlib.import_module("6dpose_b200.bank")
    from oracle import oracle, ref
    assert ref.build(), "oracle/_ref could not be built (is /root/reference mounted?)"

    frames = {}
    for tag, suffix in (("full", ""), ("half", "_half")):
        rgb = cv2.imread(CASE + "0000_rgb%s.png" % suffix)  # BGR, as cv::imread in test.cpp:90
        dep = cv2.imread(CASE + "0000_dep%s.png" % suffix, cv2.IMREAD_UNCHANGED)
        q = fe.quantize_pyramid([rgb, dep], 2)
        frames[tag] = q
    np.savez_compressed(os.path.join(OUT, "frames_case1.npz"),
                        **{"%s_l%d_m%d" % (tag, l, m): frames[tag][l][m] for tag in frames for l in range(2) for m in range(2)})

    cases = []
    for bank_name, limit, T, thresholds in (("127", None, [5, 8], (75.0, 60.0)), ("63", None, [5, 8], (75.0, 60.0)),
                                           ("allScales", 7, [5, 8], (75.0, 65.0))):
        b = bk.TemplateBank()
        b.read_class(CASE + bank_name + "/06_template.yaml", 2)
        if limit:  # every limit-th template of the 2989 (all radii 600..1800 mm stay represented)
            b.classes["06_template"] = b.classes["06_template"][::limit]
        packed = b.pack(b.class_ids(), 4)
        np.savez_compressed(os.path.join(OUT, "bank_%s.npz" % bank_name), class_begin=packed["class_begin"],
                            tmeta=packed["tmeta"], feats=packed["feats"].astype(np.int16), T=np.asarray(T, np.int32))
        for tag in frames:
            for thr in thresholds:
                want = ref.match(frames[tag], T, packed, thr)
                again = oracle.match(frames[tag], T, packed, thr)
                assert np.array_equal(want, again), "restatement and reference disagree"
                key = "%s_%s_%g" % (bank_name, tag, thr)
                cases.append((key, want))
                print(key, len(want), want[:2])
    np.savez_compressed(os.path.join(OUT, "expected_case1.npz"), **{k: v for k, v in cases})


def make_allscales_full():
    """bank_allScales_full.npz / expected_allScales_full.npz: the reference's own large-bank invocation
    (linemodLevelup/test.cpp:174-181: Detector() -> T = {5, 8}, 63 features, readClasses(allScales), match at 80) on
    the fixture frame with ALL 2989 templates, plus threshold 75 (the drivers' value, linemod_and_levelup_test.py:324;
    61 912 coarse candidates) and the half-occluded frame at 80.  Expected lists by oracle/_ref (the reference's code)."""
    fe = importlib.import_module("6dpose_b200.frontend")
    bk = importlib.import_module("6dpose_b200.bank")
    from oracle import oracle, ref
    assert ref.build()
    b = bk.TemplateBank()
    b.read_class(CASE + "allScales/06_template.yaml", 2)
    packed = b.pack(b.class_ids(), 4)
    T = [5, 8]
    np.savez_compressed(os.path.join(OUT, "bank_allScales_full.npz"), class_begin=packed["class_begin"],
                        tmeta=packed["tmeta"].astype(np.int32), feats=packed["feats"].astype(np.uint8), T=np.asarray(T, np.int32))
    assert packed["feats"].max() < 256 and packed["feats"].min() >= 0
    out = {}
    for tag, suffix, thresholds in (("full", "", (80.0, 75.0)), ("half", "_half", (80.0,))):
        rgb = cv2.imread(CASE + "0000_rgb%s.png" % suffix)
        dep = cv2.imread(CASE + "0000_dep%s.png" % suffix, cv2.IMREAD_UNCHANGED)
        q = fe.quantize_pyramid([rgb, dep], 2)
        for thr in thresholds:
            want, st = ref.match(q, T, packed, thr), None
            again, st = oracle.match(q, T, packed, thr, want_stats=True)
            assert np.array_equal(want, again), "restatement and reference disagree"
            out["%s_%g" % (tag, thr)] = want
            out["%s_%g_stats" % (tag, thr)] = np.asarray([int(st["coarse_candidates"]), int(st["coarse_byte_adds"]),
                                                           int(st["refine_byte_adds"])], np.int64)
            print("allScales full", tag, thr, len(want), want[:2], {k: int(v) for k, v in st.items()})
    np.savez_compressed(os.path.join(OUT, "expected_allScales_full.npz"), **out)


if __name__ == "__main__":
    main()
    make_allscales_full()


def make_train_golden():
    """train_case1.npz: the reference's training fixture (test.cpp:36-51 train_test: train_{rgb,dep,mask}.png
    -> Detector().addTemplate -> writeClasses/06_template.yaml, the reference's own recorded output)."""
    bk = importlib.import_module("6dpose_b200.bank")
    rgb = cv2.imread(CASE + "train_rgb.png")
    dep = cv2.imread(CASE + "train_dep.png", cv2.IMREAD_UNCHANGED)
    mask = cv2.cvtColor(cv2.imread(CASE + "train_mask.png"), cv2.COLOR_RGB2GRAY)
    ref = bk.TemplateBank()
    ref.read_class(CASE + "writeClasses/06_template.yaml", 2)
    p = ref.pack(["06_template"], 4)
    np.savez_compressed(os.path.join(OUT, "train_case1.npz"), rgb=rgb, dep=dep, mask=mask, tmeta=p["tmeta"],
                        feats=p["feats"].astype(np.int16))


REF_SYNTH_CASES = [([4, 8], 640, 480, 150, 70, 75.0), ([5, 8], 640, 480, 127, 50, 70.0), ([5, 8], 640, 480, 63, 50, 70.0),
                   ([8], 320, 240, 40, 35, 60.0), ([2, 4, 8], 640, 512, 96, 35, 70.0), ([4, 8], 320, 256, 32, 3, -1.0)]


def make_reference_checks():
    """reference_checks.npz: what the reference's own code and tables give for the checks that used to read the
    reference checkout directly -- SIMILARITY_LUT (compiled reference), normal_lut.i, the compiled reference's match
    lists on the synthetic cases of tests/test_golden_and_ref.py, and whether it asserts on the mixed-size bank.
    Plus two YAML fixtures of the reference: writeClasses/06_template.yaml (older dialect) and the first template
    pyramid of 127/06_template.yaml (header included)."""
    import re
    import shutil
    synth = importlib.import_module("6dpose_b200.synth")
    from oracle import ref
    assert ref.build()
    out = {"similarity_lut": ref.similarity_lut()}
    body = open(os.path.join(CASE, "..", "..", "normal_lut.i")).read()
    body = body[body.index("{"):]
    out["normal_lut"] = np.array([int(x) for x in re.findall(r"\d+", body)], np.uint8)[:8000].reshape(20, 20, 20)
    for i, (T, W, H, nf, n, thr) in enumerate(REF_SYNTH_CASES):
        bank = synth.synth_bank(n, num_features=nf, levels=len(T), seed=21, class_ids=("01_template", "02_template"))
        q, _ = synth.synth_frame(W, H, levels=len(T), seed=9, bank=bank, plant=6, T=T)
        out["synth_%d" % i] = ref.match(q, T, bank.pack(bank.class_ids(), 2 * len(T)), thr)
    bank = synth.synth_bank(4, num_features=150, levels=2, seed=8)
    bank.classes["01_template"][2][2].features = bank.classes["01_template"][2][2].features[:10]
    q, _ = synth.synth_frame(320, 256, levels=2, seed=6)
    try:
        ref.match(q, [4, 8], bank.pack(bank.class_ids(), 4), 80.0)
        out["mixed_size_bank_asserts"] = np.bool_(False)
    except RuntimeError:
        out["mixed_size_bank_asserts"] = np.bool_(True)
    np.savez_compressed(os.path.join(OUT, "reference_checks.npz"), **out)
    shutil.copyfile(CASE + "writeClasses/06_template.yaml", os.path.join(OUT, "writeClasses_06_template.yaml"))
    lines = open(CASE + "127/06_template.yaml").read().split("\n")
    second = lines.index("      template_id: 1") - 1   # the "   -" opening the second pyramid
    open(os.path.join(OUT, "bank_127_first_pyramid.yaml"), "w").write("\n".join(lines[:second]) + "\n")


def make_shape_checks():
    """shape_checks.npz: the compiled reference's match lists on SHAPE_CASES (tests/match_shapes.py) -- small frames at
    the pyramid steps T the other fixtures do not reach (every T of 1..16 at the lowest level, 1..8 at the refined
    ones, three and four levels), so that the oracle is pinned wherever tests/test_gpu_match_shapes.py holds the GPU to
    it.  Plus the case list itself, as JSON."""
    import json
    sys.path.insert(0, os.path.dirname(OUT))
    import match_shapes as ms
    synth = importlib.import_module("6dpose_b200.synth")
    from oracle import oracle, ref
    assert ref.build()
    out = {"cases": np.asarray(json.dumps(ms.SHAPE_CASES))}
    for i, (T, W, H, n, nf, size, thr) in enumerate(ms.SHAPE_CASES):
        ms.frame_shape(T, W, H)
        assert ms.reference_can_run(T, W), "the compiled reference faults at %s %dx%d" % (T, W, H)
        packed, q, planted = ms.shape_case_data(synth, T, W, H, n, nf, size, thr)
        assert not ms.reference_overreads(T, W, H, packed), "the compiled reference reads out of bounds at %s %dx%d" % (T, W, H)
        want = ref.match(q, T, packed, thr)
        assert len(planted) > 0 and len(want) > 0, (T, W, H)
        assert np.array_equal(want, oracle.match(q, T, packed, thr)), "restatement and reference disagree at %s %dx%d" % (T, W, H)
        out["case_%d" % i] = want
        print(T, W, H, len(want), want[:1])
    np.savez_compressed(os.path.join(OUT, "shape_checks.npz"), **out)


if __name__ == "__main__":
    make_train_golden()
    make_reference_checks()
    # frame_crop_case1.npz: a 400x320 window of the reference's fixture frame around the object (raw RGB-D,
    # for the GPU front-end test)
    rgb = cv2.imread(CASE + "0000_rgb.png")
    dep = cv2.imread(CASE + "0000_dep.png", cv2.IMREAD_UNCHANGED)
    np.savez_compressed(os.path.join(OUT, "frame_crop_case1.npz"), rgb=rgb[40:360, 200:600].copy(), dep=dep[40:360, 200:600].copy())
    make_shape_checks()
