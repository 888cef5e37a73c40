"""CPU model of the N-planes the exact bit-sliced refinement (k_refine_bits) reads next to the H-planes.

k_refine_prep writes, for every (modality, label, grid), an N-plane in the H-plane's column-major, overlapping layout,
from the byte linear memories or, after K1 in planes mode, word for word from K1's H-planes: bit = (response == 1), i.e.
a neighbouring label's spread bit without the label's own, with the label wrap of lm_response (labels (o + 1) & 7 and
(o + 7) & 7).  Both planes share one buffer:
[H-planes][zero tail][N-planes][zero tail], so a descriptor's N window is its H window + n_off words, and the padding
descriptors (the H tail) land in the N tail.  Checked here:

  1. the N-plane from the byte linear memories equals the one from the H-planes of the label and its two neighbours,
     wrap included;
  2. the exact pass's two windows per feature, at the same word index, give 4*CH + CN == similarityLocal at every cell.

No GPU: this is the layout, restated with numpy integers."""
import numpy as np
import pytest

from test_oracle_cpu import np_linear_memories
from test_refine_bitslice_model import h_planes


def n_planes_from_bytes(lm, Wd, Hd):
    """k_refine_prep's byte branch: the N bit is response == 1 (bit 0 of the response byte)."""
    return h_planes(np.where(lm == 1, 4, 0).astype(lm.dtype), Wd, Hd)[0]


def n_planes_from_h(hp):
    """k_refine_prep after K1 in planes mode: N = (H[(o + 1) & 7] | H[(o + 7) & 7]) & ~H[o], word for word."""
    return np.stack([(hp[(o + 1) & 7] | hp[(o + 7) & 7]) & ~hp[o] for o in range(8)])


def plane_buffer(hps, nps, Wd, nyb):
    """The device buffer: H-planes of every modality, zero tail, N-planes, zero tail; returns (buffer, words, n_off)."""
    words = sum(p.size for p in hps)
    tail = (nyb + 1) * Wd + 64
    buf = np.zeros(2 * (words + tail), np.uint32)
    buf[:words] = np.concatenate([p.ravel() for p in hps])
    buf[words + tail:2 * words + tail] = np.concatenate([p.ravel() for p in nps])
    return buf, words, words + tail


@pytest.mark.parametrize("T,W,H,nf", [([4, 8], 320, 256, 48), ([5, 8], 320, 240, 40), ([4, 8], 320, 232, 36)])
def test_n_planes_and_exact_pass_agree_with_similarity_local(synth, T, W, H, nf):
    bank = synth.synth_bank(6, num_features=nf, levels=2, seed=4)
    q, planted = synth.synth_frame(W, H, levels=2, seed=9, bank=bank, plant=3, T=T)
    T0 = T[0]
    rows, cols = q[0][0].shape
    Wd, Hd = cols // T0, rows // T0
    lms = [np_linear_memories(q[0][m], T0) for m in range(2)]
    hps, nps = [], []
    for m in range(2):
        hp, nyb = h_planes(lms[m], Wd, Hd)
        npl = n_planes_from_bytes(lms[m], Wd, Hd)
        assert np.array_equal(npl, n_planes_from_h(hp))                                  # claim 1, wrap included
        assert npl[0].any() and npl[7].any()
        hps.append(hp)
        nps.append(npl)
    buf, words, n_off = plane_buffer(hps, nps, Wd, nyb)
    T2 = T0 * T0
    rng = np.random.default_rng(2)
    border = 8 * T0
    checked = 0
    for tid, tp in enumerate(bank.classes["01_template"]):
        w, h = tp[0].width, tp[0].height
        feats = [(m, int(x), int(y), int(lab)) for m in range(2) for x, y, lab in tp[m].features.tolist()]
        # descriptors as prepare_bank builds them, padded to a multiple of 32 with the H tail
        desc = []
        for m, fx, fy, lab in feats:
            pb = (m * 8 + lab) * T2 + (fy % T0) * T0 + fx % T0
            desc.append((pb * nyb * Wd + fx // T0) | ((fy // T0) << 23))
        desc += [words] * (-len(desc) % 32)
        pos = [(x, y) for cid, t, x, y in planted if t == tid]
        pos += [(int(rng.integers(0, cols)), int(rng.integers(0, rows))) for _ in range(4)]
        for px, py in pos:
            x = min(max(px, border), cols - w - border)
            y = min(max(py, border), rows - h - border)
            cx, cy = x // T0 - 8, y // T0 - 8
            patch = np.zeros((16, 16), np.int64)
            for m, fx, fy, lab in feats:
                g = (fy % T0) * T0 + fx % T0
                px0, py0 = cx + fx // T0, cy + fy // T0
                patch += lms[m][lab][g].reshape(Hd, Wd)[py0:py0 + 16, px0:px0 + 16]
            CH = np.zeros((16, 16), np.int64)
            CN = np.zeros((16, 16), np.int64)
            for d in desc:                                                # the kernel's addressing, padding included
                py0 = cy + (d >> 23)
                idx = (d & 0x7FFFFF) + (py0 >> 4) * Wd + cx
                s = np.uint32(py0 & 15)

                def window(base):
                    col_bits = (buf[base:base + 16] >> s) & np.uint32(0xFFFF)
                    return ((col_bits[None, :] >> np.arange(16, dtype=np.uint32)[:, None]) & 1).astype(np.int64)

                CH += window(idx)
                CN += window(idx + n_off)
            assert np.array_equal(4 * CH + CN, patch)                                      # claim 2
            checked += 1
    assert checked >= 24


def test_padding_descriptors_read_zeros_in_both_tails():
    """The padding descriptor (word `words`, row 0) of any candidate reads the H tail, and + n_off the N tail, both zero
    and both inside the buffer for every row block and column a patch can reach."""
    T, Wd, Hd, M = 4, 160, 120, 2
    nyb = ((Hd - 16) >> 4) + 1
    words = M * 8 * T * T * nyb * Wd
    tail = (nyb + 1) * Wd + 64
    n_off = words + tail
    assert n_off % 4 == 0                                            # k_refine_prep's 128-bit N stores stay aligned
    assert words + tail <= 1 << 23
    for cy in (0, Hd - 16):
        for cx in (0, Wd - 16):
            lo = words + ((cy >> 4) * Wd) + cx
            hi = lo + 15
            assert words <= lo and hi < words + tail                                      # H tail
            assert n_off + words <= n_off + lo and n_off + hi < 2 * (words + tail)        # N tail
