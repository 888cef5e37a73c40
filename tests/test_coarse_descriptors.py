"""The bit-sliced coarse scan's feature descriptors (lm_coarse_descriptors, host only): one word per lowest-level feature,
decoded here the way k_coarse_packed decodes it and compared with a restatement from the bank -- the byte offsets of the
feature's window in its label's bit-plane and in its two neighbour labels' planes, and the bit shift.  Features outside
the level and the padding to 32 decode to windows that read only the planes' zero slack, and a template whose word
offsets do not fit goes to the byte-wise scan."""
import importlib
import os

import numpy as np
import pytest

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture(scope="module")
def lib():
    return importlib.import_module("6dpose_b200._lib")


@pytest.fixture(scope="module")
def synth():
    return importlib.import_module("6dpose_b200.synth")


def geometry(T, rows, cols):
    """Words per label block (lbw), written words per block (data), rounds: the detector's bit-plane sizing."""
    Wd, Hd = cols // T, rows // T
    plane = Wd * Hd
    nwords = (plane + 31) // 32
    rounds = (nwords + 31) // 32
    data = (T * T * plane + 31) // 32
    return Wd, plane, (data + 32 * rounds + 4 + 3) & ~3, data, rounds


def decode(d, lbw):
    """k_coarse_packed's decode: byte offsets of the label's window and of the lower and upper neighbour labels'."""
    d = np.asarray(d, np.int64)
    L4 = 4 * lbw
    off = (d >> 5) & ~3
    om = off + np.where(d & 0x20, 7 * L4, -L4)
    op = off + np.where(d & 0x40, -7 * L4, L4)
    return off, om, op, d & 31


def check_bank(lib, feats, tmeta, M, slot_low, T, rows, cols):
    feats = np.asarray(feats, np.int64)
    tmeta = np.asarray(tmeta, np.int64)
    desc, info, fits, zero = lib.coarse_descriptors(feats, tmeta, M, slot_low, T, rows, cols)
    G = len(tmeta)
    Wd, plane, lbw, data, rounds = geometry(T, rows, cols)
    assert fits.all()
    # the zero descriptor: all three windows lie in the slack of a label block, far enough from its end for the reads
    # of every lane (words idx and idx + 1, idx < 32 * rounds)
    for o in decode([zero], lbw)[:3]:
        w = int(o[0]) // 4
        assert int(o[0]) % 4 == 0 and 0 <= w // lbw < M * 8
        assert data <= w % lbw and w % lbw + 32 * rounds + 1 <= lbw
    assert zero & 31 == 0
    n_out = 0
    end = 0
    for g in range(G):
        first, n = int(info[g, 0]), int(info[g, 1])
        assert first == end and first % 32 == 0  # end to end, every run 128-byte aligned
        assert n == int(tmeta[g, slot_low:slot_low + M, 3].sum())
        pad = (n + 31) // 32 * 32
        end = first + pad
        assert np.all(desc[first + n:end] == zero)
        want = []
        for m in range(M):
            _, _, b, c = tmeta[g, slot_low + m]
            for x, y, lab in feats[b:b + c]:
                if x >= cols or y >= rows:  # LL.cpp:1330
                    want.append(None)
                    continue
                inner = ((y % T) * T + (x % T)) * plane + (y // T) * Wd + (x // T)
                wi = inner >> 5
                want.append((4 * ((m * 8 + lab) * lbw + wi), 4 * ((m * 8 + (lab + 7) % 8) * lbw + wi),
                             4 * ((m * 8 + (lab + 1) % 8) * lbw + wi), inner & 31))
        got = list(zip(*[a.tolist() for a in decode(desc[first:first + n], lbw)]))
        for k, w in enumerate(want):
            if w is None:
                assert desc[first + k] == zero
                n_out += 1
            else:
                assert got[k] == w, (g, k)
    assert end == len(desc)
    return n_out


def lowest(packed, W, H, T, M):
    levels = len(T)
    return dict(M=M, slot_low=(levels - 1) * M, T=T[-1], rows=H >> (levels - 1), cols=W >> (levels - 1))


@pytest.mark.parametrize("W,H", [(640, 480), (1280, 960)])
def test_bench_bank(lib, synth, W, H):
    bank = synth.synth_bank(3115, num_features=150, levels=2, seed=1234, variants=35)
    packed = bank.pack(bank.class_ids(), 4)
    check_bank(lib, packed["feats"], packed["tmeta"], **lowest(packed, W, H, [4, 8], 2))


def test_allscales_bank(lib):
    """The reference's 2989-template allScales bank, T = [5, 8], at 640x480."""
    b = np.load(os.path.join(GOLD, "bank_allScales_full.npz"))
    T = b["T"].tolist()
    assert T == [5, 8]
    check_bank(lib, b["feats"].astype(np.int32), b["tmeta"].astype(np.int32), **lowest(None, 640, 480, T, 2))


def odd_bank(G, M, levels, cols, rows, seed):
    """G templates with M modalities and odd feature counts, some features outside a cols x rows level."""
    rng = np.random.default_rng(seed)
    S = levels * M
    tmeta = np.zeros((G, S, 4), np.int32)
    feats = []
    for g in range(G):
        for s in range(S):
            n = int(rng.integers(0, 40)) * 2 + 1
            tmeta[g, s] = (int(rng.integers(8, 60)), int(rng.integers(8, 60)), len(feats), n)
            for _ in range(n):
                feats.append((int(rng.integers(0, cols + 12)), int(rng.integers(0, rows + 12)), int(rng.integers(0, 8))))
    return np.asarray(feats, np.int32), tmeta


@pytest.mark.parametrize("T,rows,cols", [(8, 240, 320), (5, 96, 130), (4, 60, 84)])
def test_three_modalities_odd_counts(lib, T, rows, cols):
    feats, tmeta = odd_bank(97, 3, 2, cols, rows, seed=T)
    n_out = check_bank(lib, feats, tmeta, M=3, slot_low=3, T=T, rows=rows, cols=cols)
    assert n_out > 0  # features outside the level were exercised


def test_word_offsets_that_do_not_fit_go_to_the_byte_scan(lib):
    """At 8192 x 8192 with T = 8 a label block holds 2 129 924 words, so a window late in the last block (modality 1,
    label 7) has a word offset >= 2^25 and does not fit: its template gets no descriptors and fits = False; the others
    keep theirs, end to end, a window early in that block included."""
    T, rows, cols = 8, 8192, 8192
    _, _, lbw, _, _ = geometry(T, rows, cols)
    assert 15 * lbw < 2 ** 25 <= 16 * lbw
    tmeta = np.zeros((4, 2, 4), np.int32)
    feats = np.array([(3, 5, 2), (9, 1, 7),      # template 0: modality 0 only
                      (100, 200, 6), (8, 8, 7),  # template 1: modality 1, label 7 -> block 15 (fits)
                      (8000, 8000, 0),           # template 2: modality 0
                      (15, 15, 7)], np.int32)    # template 3: modality 1, label 7, grid offset 63 of 64
    tmeta[0] = [(10, 10, 0, 2), (10, 10, 2, 0)]
    tmeta[1] = [(10, 10, 2, 0), (10, 10, 2, 2)]
    tmeta[2] = [(10, 10, 4, 1), (10, 10, 5, 0)]
    tmeta[3] = [(10, 10, 5, 0), (10, 10, 5, 1)]
    desc, info, fits, zero = lib.coarse_descriptors(feats, tmeta, 2, 0, T, rows, cols)
    inner = ((15 % T) * T + 15 % T) * (cols // T) * (rows // T) + (15 // T) * (cols // T) + 15 // T
    assert (8 + 7) * lbw + (inner >> 5) >= 2 ** 25
    assert fits.tolist() == [True, True, True, False]
    assert info[3].tolist() == [96, 0] and len(desc) == 96
    check_bank(lib, feats, tmeta[:3], 2, 0, T, rows, cols)


def test_rejects_bad_input(lib):
    feats, tmeta = odd_bank(3, 2, 2, 320, 240, seed=1)
    with pytest.raises(RuntimeError):
        lib.coarse_descriptors(feats, tmeta, 3, 2, 8, 240, 320)  # slots 2..4 of 4
    with pytest.raises(RuntimeError):
        lib.coarse_descriptors(feats, tmeta, 2, 2, 0, 240, 320)
