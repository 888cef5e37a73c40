"""Pinning of the oracle against what the reference's own linemodLevelup.cpp, compiled unmodified (oracle/_ref),
produced: (1) on synthetic cases and its tables (tests/golden/reference_checks.npz), (2) on the reference's fixture
frame and template banks (the other golden vectors).  All stored by tests/golden/make_golden.py."""
import importlib
import os

import numpy as np
import pytest

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def load_golden():
    fr = np.load(os.path.join(GOLD, "frames_case1.npz"))
    frames = {tag: [[fr["%s_l%d_m%d" % (tag, l, m)] for m in range(2)] for l in range(2)] for tag in ("full", "half")}
    banks = {}
    for name in ("127", "63", "allScales"):
        b = np.load(os.path.join(GOLD, "bank_%s.npz" % name))
        banks[name] = (dict(class_begin=b["class_begin"], tmeta=b["tmeta"], feats=b["feats"].astype(np.int32)), b["T"].tolist())
    exp = np.load(os.path.join(GOLD, "expected_case1.npz"))
    cases = []
    for key in exp.files:
        bank, tag, thr = key.split("_")
        cases.append((bank, tag, float(thr), exp[key]))
    return frames, banks, cases


def test_oracle_reproduces_the_reference_golden_vectors(oracle):
    frames, banks, cases = load_golden()
    assert len(cases) == 12
    nonempty = 0
    for bank, tag, thr, want in cases:
        packed, T = banks[bank]
        got = oracle.match(frames[tag], T, packed, thr)
        assert np.array_equal(got, want), (bank, tag, thr)
        nonempty += len(want) > 0
    assert nonempty >= 9


def load_allscales_full():
    """The reference's own large-bank invocation (linemodLevelup/test.cpp:174-181): Detector() = 63 features, T = {5, 8},
    ALL 2989 templates of test/case1/allScales, threshold 80; plus threshold 75 (61 912 coarse candidates)."""
    b = np.load(os.path.join(GOLD, "bank_allScales_full.npz"))
    packed = dict(class_begin=b["class_begin"], tmeta=b["tmeta"].astype(np.int32), feats=b["feats"].astype(np.int32))
    exp = np.load(os.path.join(GOLD, "expected_allScales_full.npz"))
    cases = [(k.split("_")[0], float(k.split("_")[1]), exp[k], exp[k + "_stats"]) for k in exp.files if not k.endswith("_stats")]
    return packed, b["T"].tolist(), cases


def test_oracle_reproduces_the_full_allscales_golden_vectors(oracle):
    frames, _, _ = load_golden()
    packed, T, cases = load_allscales_full()
    assert int(packed["class_begin"][-1]) == 2989 and len(cases) == 3
    for tag, thr, want, stats in cases:
        got, st = oracle.match(frames[tag], T, packed, thr, want_stats=True)
        assert np.array_equal(got, want), (tag, thr)
        assert [int(st["coarse_candidates"]), int(st["coarse_byte_adds"]), int(st["refine_byte_adds"])] == stats.tolist()
    full75 = [c for c in cases if c[0] == "full" and c[1] == 75.0][0]
    assert len(full75[2]) == 157 and int(full75[3][0]) == 61912   # BASELINE.md section 2's candidate count


def test_golden_top_match_sits_on_the_ground_truth_box():
    # GT box of the object in the fixture frame: [331, 130, 65, 64] (linemodLevelup/test.cpp:86)
    _, _, cases = load_golden()
    top = [c for c in cases if c[0] == "127" and c[1] == "full" and c[2] == 75.0][0][3][0]
    assert abs(int(top["x"]) - 331) <= 4 and abs(int(top["y"]) - 130) <= 4


# What the compiled reference (oracle/_ref) returned on these cases is stored in reference_checks.npz
# (tests/golden/make_golden.py, make_reference_checks), so the comparison needs no reference checkout.
REF_CHECKS = os.path.join(GOLD, "reference_checks.npz")


REF_SYNTH_CASES = [
    ([4, 8], 640, 480, 150, 70, 75.0), ([5, 8], 640, 480, 127, 50, 70.0), ([5, 8], 640, 480, 63, 50, 70.0),
    ([8], 320, 240, 40, 35, 60.0), ([2, 4, 8], 640, 512, 96, 35, 70.0), ([4, 8], 320, 256, 32, 3, -1.0),
]   # the same list as make_golden.REF_SYNTH_CASES: entry i is stored as synth_<i>


@pytest.mark.parametrize("T,W,H,nf,n,thr", REF_SYNTH_CASES)
def test_oracle_equals_compiled_reference(oracle, synth, T, W, H, nf, n, thr):
    bank = synth.synth_bank(n, num_features=nf, levels=len(T), seed=21, class_ids=("01_template", "02_template"))
    q, _ = synth.synth_frame(W, H, levels=len(T), seed=9, bank=bank, plant=6, T=T)
    packed = bank.pack(bank.class_ids(), 2 * len(T))
    a = oracle.match(q, T, packed, thr)
    b = np.load(REF_CHECKS)["synth_%d" % REF_SYNTH_CASES.index((T, W, H, nf, n, thr))]
    assert len(b) > 0 and np.array_equal(a, b)


def test_similarity_lut_equals_the_compiled_reference_table(oracle):
    assert np.array_equal(oracle.similarity_lut(), np.load(REF_CHECKS)["similarity_lut"])


def test_reference_assertion_matches_oracle_error(oracle, synth):
    T = [4, 8]
    bank = synth.synth_bank(4, num_features=150, levels=2, seed=8)
    bank.classes["01_template"][2][2].features = bank.classes["01_template"][2][2].features[:10]
    q, _ = synth.synth_frame(320, 256, levels=2, seed=6)
    packed = bank.pack(bank.class_ids(), 4)
    assert bool(np.load(REF_CHECKS)["mixed_size_bank_asserts"])   # the compiled reference raised here
    with pytest.raises(RuntimeError):
        oracle.match(q, T, packed, 80.0)


@pytest.mark.gpu
def test_cuda_path_reproduces_the_reference_golden_vectors():
    lib = importlib.import_module("6dpose_b200._lib")
    frames, banks, cases = load_golden()
    for bank, tag, thr, want in cases:
        packed, T = banks[bank]
        nat = lib.NativeDetector(T)
        nat.load_bank(packed, 4)
        got = nat.match_quantized(frames[tag], thr)
        assert len(got) == len(want), (bank, tag, thr)
        for k in ("x", "y", "template_id", "similarity"):
            assert np.array_equal(got[k], want[k]), (bank, tag, thr, k)
        assert np.array_equal(got["class_index"], want["class_idx"])


@pytest.mark.gpu
def test_cuda_path_reproduces_the_full_allscales_golden_vectors():
    """All 2989 templates of the reference's allScales bank on its fixture frame, thresholds 80 (test.cpp:174-181) and
    75: match lists bit-identical to the compiled reference, candidate / algorithmic byte counters equal."""
    lib = importlib.import_module("6dpose_b200._lib")
    frames, _, _ = load_golden()
    packed, T, cases = load_allscales_full()
    nat = lib.NativeDetector(T)
    nat.load_bank(packed, 4)
    for tag, thr, want, stats in cases:
        got = nat.match_quantized(frames[tag], thr)
        assert len(got) == len(want), (tag, thr)
        for k in ("x", "y", "template_id", "similarity"):
            assert np.array_equal(got[k], want[k]), (tag, thr, k)
        c = nat.counters()
        assert [c["coarse_candidates"], c["scan_bytes"], c["refine_bytes"]] == stats.tolist(), (tag, thr)


def test_shape_checks_list_is_current():
    import match_shapes as ms
    assert ms.stored_shape_cases() == [(T, W, H, n, nf, size, thr) for T, W, H, n, nf, size, thr in ms.SHAPE_CASES]


def _shape_ids():
    import match_shapes as ms
    return ["%s-%dx%d" % ("_".join(map(str, c[0])), c[1], c[2]) for c in ms.SHAPE_CASES]


@pytest.mark.parametrize("i", range(len(_shape_ids())), ids=_shape_ids())
def test_oracle_equals_compiled_reference_at_new_shapes(oracle, synth, i):
    """tests/golden/shape_checks.npz: the compiled reference's lists at every pyramid step T the GPU shape matrix runs."""
    import match_shapes as ms
    T, W, H, n, nf, size, thr = ms.SHAPE_CASES[i]
    ms.frame_shape(T, W, H)
    packed, q, planted = ms.shape_case_data(synth, T, W, H, n, nf, size, thr)
    # the stored list is the reference's defined result only where it reads nothing past its linear memories
    assert ms.reference_can_run(T, W) and not ms.reference_overreads(T, W, H, packed)
    want = np.load(ms.SHAPE_CHECKS)["case_%d" % i]
    assert len(planted) > 0 and len(want) > 0
    assert np.array_equal(oracle.match(q, T, packed, thr), want)


def test_reference_overreads_at_t1_with_features_on_the_template_side(synth):
    """What shape_case_data avoids at T = 1: synth_bank puts a feature at x = width (cropTemplates' extent), and the
    reference's coarse scan then reads past the last grid of its linear memories."""
    import match_shapes as ms
    bank = synth.synth_bank(6, num_features=32, levels=1, seed=21, size_range=((8, 32), (8, 32)))
    over = ms.reference_overreads([1], 64, 64, bank.pack(bank.class_ids(), 2))
    assert over and max(o[3] for o in over) > 0
    assert not ms.reference_overreads([2], 64, 64, bank.pack(bank.class_ids(), 2))
