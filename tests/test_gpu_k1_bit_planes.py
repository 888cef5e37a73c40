"""K1's lowest level, built bit-planes first: every live word of the coarse scan's spread bit-planes is stored whole each
frame (no atomics, nothing clears them between frames), and the lowest level's byte linear memories are built only when
the byte-wise coarse scan has templates (or the debug getter asks for them).

The bit-planes are read back (lm_debug_bit_planes) and compared word for word, live and slack, with the oracle's
quantized frame spread and packed in numpy: bit i of label o's words is set where the oracle's linear memory at index
i = grid * plane + position responds 4 to orientation o."""
import importlib

import numpy as np
import pytest

from match_shapes import SHAPE_CASES, shape_case_data

pytestmark = pytest.mark.gpu


def _expected_words(q_low, T, lbw, oracle):
    lm = oracle.linear_memories(q_low, T)  # [8, T*T, plane]
    bits = (lm == 4).reshape(8, -1)
    assert bits.shape[1] <= 32 * lbw
    padded = np.zeros((8, 32 * lbw), bool)
    padded[:, :bits.shape[1]] = bits
    return np.packbits(padded, axis=1, bitorder="little").view("<u4")  # [8, lbw]


def _check_bit_planes(nat, q, T, oracle):
    words = nat.bit_planes()
    plan = nat.plan()
    assert plan["bit_planes"] == int(words.size > 0), plan
    if words.size == 0:
        return 0
    words = words.reshape(2, 8, -1)
    for m in range(2):
        want = _expected_words(q[-1][m], T[-1], words.shape[2], oracle)
        bad = np.nonzero(words[m] != want)
        assert bad[0].size == 0, ("modality", m, "label, word", bad[0][:4], bad[1][:4], words[m][bad][:4], want[bad][:4])
    return words.size


def _assert_same(got, want):
    assert len(got) == len(want), (len(got), len(want))
    for k in ("x", "y", "template_id"):
        assert np.array_equal(got[k], want[k]), k
    assert np.array_equal(got["similarity"], want["similarity"])


def _native(T, packed, n_lists):
    lib = importlib.import_module("6dpose_b200._lib")
    nat = lib.NativeDetector(T)
    nat.load_bank(packed, n_lists)
    return nat


def _low_mode(plan):
    return (1 if plan["bit_planes"] else 0) | (2 if plan["byte_templates"] > 0 else 0)


@pytest.mark.parametrize("case", SHAPE_CASES, ids=["T%s-%dx%d" % ("_".join(map(str, c[0])), c[1], c[2]) for c in SHAPE_CASES])
def test_bit_planes_shape_cases(synth, oracle, case):
    T, W, H, n, nf, size, thr = case
    packed, q, _ = shape_case_data(synth, T, W, H, n, nf, size, thr)
    nat = _native(T, packed, 2 * len(T))
    got = nat.match_quantized(q, thr)
    _check_bit_planes(nat, q, T, oracle)
    assert nat.plan()["k1_low_mode"] == _low_mode(nat.plan())
    _assert_same(got, oracle.match(q, T, packed, thr))
    nat.close()


# the bench frame size (a word straddles rows of positions, Wd = 40, and grids, plane = 1200), a lowest level whose plane
# is a multiple of 32 (512 x 512: Wd = Hd = 32), and 300 features (the byte-wise coarse scan: bits and bytes)
@pytest.mark.parametrize("T,W,H,nf,mode", [([4, 8], 640, 480, 150, 1), ([4, 8], 512, 512, 150, 1), ([4, 8], 640, 480, 300, 3),
                                           ([5, 8], 640, 480, 127, 1)])
def test_bit_planes_bench_sizes(synth, oracle, T, W, H, nf, mode):
    bank = synth.synth_bank(40, num_features=nf, levels=len(T), seed=31)
    packed = bank.pack(bank.class_ids(), 2 * len(T))
    q, _ = synth.synth_frame(W, H, levels=len(T), seed=32, bank=bank, plant=4, T=T)
    nat = _native(T, packed, 2 * len(T))
    got = nat.match_quantized(q, 75.0)
    assert _check_bit_planes(nat, q, T, oracle) > 0
    assert nat.plan()["k1_low_mode"] == mode, nat.plan()
    _assert_same(got, oracle.match(q, T, packed, 75.0))
    nat.close()


@pytest.mark.parametrize("nf,mode", [(150, 1), (300, 3)], ids=["bits", "bits_and_bytes"])
def test_two_frames_back_to_back(synth, oracle, nf, mode):
    """A frame whose every spread bit is set, then an ordinary one, on one handle: no bit of the first may survive into
    the second's planes or match list (nothing clears the planes between frames any more)."""
    T = [4, 8]
    bank = synth.synth_bank(40, num_features=nf, levels=2, seed=41)
    packed = bank.pack(bank.class_ids(), 4)
    full = [[np.full((480 >> l, 640 >> l), 0xFF, np.uint8) for _ in range(2)] for l in range(2)]
    q2, _ = synth.synth_frame(640, 480, levels=2, seed=42, bank=bank, plant=4, T=T)
    nat = _native(T, packed, 4)
    assert len(nat.match_quantized(full, 100.0)) == 0  # every score is 100: nothing exceeds the threshold
    assert _check_bit_planes(nat, full, T, oracle) > 0
    got = nat.match_quantized(q2, 75.0)
    assert nat.plan()["k1_low_mode"] == mode, nat.plan()
    _check_bit_planes(nat, q2, T, oracle)
    want = oracle.match(q2, T, packed, 75.0)
    assert len(want) > 0
    _assert_same(got, want)
    nat.close()


@pytest.mark.parametrize("nf,mode", [(150, 1), (300, 3)], ids=["bits", "bits_and_bytes"])
def test_lowest_linear_memories_on_both_routes(synth, oracle, nf, mode):
    """The debug getter returns the oracle's linear memories at every level, whether or not the run built the lowest
    level's bytes; building them afterwards leaves the bit-planes and the next run's results as they were."""
    T = [4, 8]
    bank = synth.synth_bank(40, num_features=nf, levels=2, seed=51)
    packed = bank.pack(bank.class_ids(), 4)
    q, _ = synth.synth_frame(640, 480, levels=2, seed=52, bank=bank, plant=4, T=T)
    nat = _native(T, packed, 4)
    got = nat.match_quantized(q, 75.0)
    assert nat.plan()["k1_low_mode"] == mode, nat.plan()
    for l in (1, 0):
        for m in range(2):
            want = oracle.linear_memories(q[l][m], T[l])
            assert np.array_equal(nat.linear_memories(l, m, want.shape), want), (l, m)
    _check_bit_planes(nat, q, T, oracle)
    want = oracle.match(q, T, packed, 75.0)
    _assert_same(got, want)
    _assert_same(nat.match_quantized(q, 75.0), want)
    nat.close()
