"""Frames, banks and a model that put the coarse scan (K2: k_coarse_packed and k_coarse_bytes) on its bounds.

The model follows the reference, not the kernels: for every selected template, the oracle's coarse map of the lowest
level (LL.cpp:1284-1354, zeros at positions j >= P as LL.cpp:1314 leaves them), the pass set score(raw) > threshold
(LL.cpp:1836-1852, the two float32 operations of tight_frames.score) and the raw score at every passing cell.  The
device's pass masks and raw scores (lm_debug_coarse) are held to it bit for bit.

On a one-hot frame of label o every feature responds 4 (label o), 1 (o +- 1 mod 8) or 0, so a template with a hits and
b neighbours scores 4a + b at every cell below P.  The constructions:

  * threshold sweep: for nf in SWEEP_NF, one template per attainable raw 0 .. 4 nf; thresholds score(raw_min - 1) for
    every raw_min 0 .. 4 nf + 1 (the compare is strict at raw_min), score(raw_min) and one ulp either side of it;
  * counter saturation and carries: CH = 255 (raw 1020), CN = 255, and mixes through 127 -> 128 and 254 -> 255, each
    template one full round and one remainder word (lanes of templates with different nf share the remainder tasks),
    under the team splits S = 8, 4, 2, 1 (filler templates set the task count);
  * label wrap: label-0 features on a label-7 frame, label-7 features on a label-0 frame, and a frame of both;
  * position edges: P at every residue mod 32 and P = 1, planes that are not a multiple of 32, P <= 0 (a template
    larger than the level: the reference adds nothing, LL.cpp:1351), and a negative threshold (raw_min = 0);
  * features outside the level (LL.cpp:1330), in both kernels;
  * byte kernel: nf 256 and 257, per-modality counts at its 63-feature flush, tiles of 511 / 512 / 513 features, 8191
    hits (raw 32 764), modalities with unequal P, skipped features inside a tile;
  * staging: bit-planes in shared memory (640x624 at [4, 8]) and in global memory (640x640).
"""
import numpy as np

import match_shapes as ms
import tight_frames as tf

bank_mod = tf.bank_mod
score = tf.score
M = 2


def min_passing_raw(threshold, nf):
    """Smallest raw with score > threshold (LL.cpp:1842-1844); 4 nf + 1 when none."""
    lo, hi = 0, 4 * nf + 1
    thr = np.float32(threshold)
    while lo < hi:
        mid = (lo + hi) >> 1
        if score(mid, nf) > thr:
            hi = mid
        else:
            lo = mid + 1
    return lo


def ulp_down(v):
    return np.nextafter(np.float32(v), np.float32(-np.inf))


# ---- frames ------------------------------------------------------------------------------------------------------------

def onehot_frame(W, H, levels, label):
    """Every pixel of every level and modality carries the one label."""
    return [[np.full((H >> l, W >> l), 1 << label, np.uint8) for _ in range(M)] for l in range(levels)]


def pair_frame(W, H, levels, a, b):
    """Pixel columns alternate labels a and b: at T >= 2 every spread cell holds both."""
    out = []
    for l in range(levels):
        row = np.where(np.arange(W >> l) % 2 == 0, 1 << a, 1 << b).astype(np.uint8)
        out.append([np.tile(row, (H >> l, 1)) for _ in range(M)])
    return out


def random_frame(W, H, levels, seed):
    """One random label per pixel: spread cells hold several labels, neighbours next to hits."""
    rng = np.random.default_rng(seed)
    return [[(1 << rng.integers(0, 8, (H >> l, W >> l))).astype(np.uint8) for _ in range(M)] for l in range(levels)]


# ---- templates ---------------------------------------------------------------------------------------------------------

def labels(nf, a, b, o, rng):
    """nf labels against a one-hot frame of label o: a hits, b neighbours (o + 1 and o - 1 alternately), the rest o + 4
    (response 0), in a random order."""
    lab = np.full(nf, (o + 4) % 8)
    lab[:a] = o
    nb = np.where(np.arange(b) % 2 == 0, (o + 1) % 8, (o + 7) % 8)
    lab[a:a + b] = nb
    return lab[rng.permutation(nf)]


def pyramid(lab, counts, sizes, levels, seed, outside=0, level_shape=None):
    """Template pyramid whose lowest level carries the labels `lab` split `counts` over the modalities, in boxes `sizes`
    ((w, h) per modality); positions inside the smallest box (x < w, y < h of every modality: the reference never reads
    past its linear memories).
    `outside` features of every modality move beyond the lowest level (x >= cols or y >= rows of level_shape = (cols,
    rows)).  Levels above: 8 features of label lab[0] per modality, in a box twice as large per level."""
    rng = np.random.default_rng(seed)
    T_ = bank_mod.Template
    low, at = [], 0
    wmin, hmin = min(s[0] for s in sizes), min(s[1] for s in sizes)
    for m in range(M):
        w, h = sizes[m]
        n = counts[m]
        f = np.stack([rng.integers(0, wmin, n), rng.integers(0, hmin, n), lab[at:at + n]], 1).astype(np.int32)
        for k in range(min(outside, n)):
            cols, rows = level_shape
            if k % 2 == 0:
                f[k, 0] = cols + k
            else:
                f[k, 1] = rows + k
        low.append(T_(w, h, levels - 1, f))
        at += n
    tp = []
    for l in range(levels - 1):
        s = 1 << (levels - 1 - l)
        for m in range(M):
            w, h = sizes[m][0] * s, sizes[m][1] * s
            f = np.stack([rng.integers(0, w, 8), rng.integers(0, h, 8), np.full(8, lab[0])], 1).astype(np.int32)
            tp.append(T_(w, h, l, f))
    return tp + low


def pattern_template(nf, a, b, o, seed, size=(8, 8), levels=1, split=None):
    rng = np.random.default_rng(seed)
    counts = split if split is not None else tf.split_modalities(nf)
    return pyramid(labels(nf, a, b, o, rng), counts, [size, size], levels, seed)


# ---- the model ---------------------------------------------------------------------------------------------------------

def positions(T_low, Wd, Hd, w, h):
    """template_positions P of a w x h template on a Wd x Hd level of step T_low (LL.cpp:1299-1309)."""
    return (Hd - (ms._cdiv(h - 1, T_low) + 1)) * Wd + (Wd - (ms._cdiv(w - 1, T_low) + 1)) + 1


def pack_words(bits, nwords):
    """bool [G, plane] -> uint32 [G, nwords] (bit j & 31 of word j >> 5)."""
    G, plane = bits.shape
    pad = np.zeros((G, nwords * 32), bool)
    pad[:, :plane] = bits
    return np.packbits(pad, axis=1, bitorder="little").view("<u4").reshape(G, nwords)


class CoarseModel:
    """Expected coarse outputs of every template of a packed bank on one frame (oracle.coarse_map of the lowest level)."""

    def __init__(self, oracle, q, T, packed):
        self.T = list(T)
        L = len(T)
        tm = np.asarray(packed["tmeta"]).reshape(len(packed["tmeta"]), L * M, 4)
        feats = np.asarray(packed["feats"]).reshape(-1, 3)
        low = q[-1]
        rows, cols = low[0].shape
        self.Wd, self.Hd = cols // T[-1], rows // T[-1]
        self.plane = self.Wd * self.Hd
        self.nwords = (self.plane + 31) // 32
        self.G = tm.shape[0]
        s = (L - 1) * M
        tm_low = tm[:, s:s + M]
        self.nf = tm_low[:, :, 3].sum(1).astype(np.int64)
        self.P = np.zeros((self.G, M), np.int64)
        self.raw = np.zeros((self.G, self.plane), np.int64)
        cache = {}
        for g in range(self.G):
            key = (tm_low[g, :, :2].tobytes(), b"".join(feats[b:b + n].tobytes() for b, n in tm_low[g, :, 2:4]))
            if key not in cache:
                cmap, _ = oracle.coarse_map(low, T[-1], tm_low[g], feats)
                cache[key] = cmap.astype(np.int64).ravel()
            self.raw[g] = cache[key]
            for m in range(M):
                self.P[g, m] = positions(T[-1], self.Wd, self.Hd, int(tm_low[g, m, 0]), int(tm_low[g, m, 1]))

    def passes(self, threshold):
        """bool [G, plane]: score(raw) > threshold; nothing for a template without lowest-level features."""
        with np.errstate(invalid="ignore", divide="ignore"):
            s = score(self.raw, np.maximum(self.nf, 1)[:, None])
        return (s > np.float32(threshold)) & (self.nf > 0)[:, None]

    def expected(self, threshold):
        """(mask uint32 [G, nwords], raw uint16 [G, plane]) as lm_debug_coarse returns them."""
        p = self.passes(threshold)
        return pack_words(p, self.nwords), np.where(p, self.raw, 0).astype(np.uint16)


# ---- the cases ---------------------------------------------------------------------------------------------------------

SWEEP_NF = (1, 2, 7, 8, 9, 31, 32, 33, 63, 64, 65, 127, 128, 129, 254, 255)
SWEEP_SHAPE = ([8], 64, 64)   # 8 x 8 positions; 16 x 16 templates: P = 55


def attainable(nf):
    """{4a + b : a + b <= nf} -> one (a, b) per raw."""
    out = {}
    for a in range(nf + 1):
        for b in range(nf - a + 1):
            out.setdefault(4 * a + b, (a, b))
    return out


def sweep_bank(nf):
    """One template per attainable raw of nf features against a one-hot frame of label nf % 8 (the neighbour labels
    wrap for nf % 8 in {0, 7})."""
    o = nf % 8
    tps = [pattern_template(nf, a, b, o, seed=nf * 10007 + r, size=(16, 16))
           for r, (a, b) in sorted(attainable(nf).items())]
    return tf.make_bank(tps), onehot_frame(SWEEP_SHAPE[1], SWEEP_SHAPE[2], 1, o)


def sweep_thresholds(nf):
    """score(raw_min - 1) for raw_min 0 .. 4 nf + 1, score(raw_min) and one ulp either side (unique, ascending)."""
    t = set()
    for r in range(-1, 4 * nf + 2):
        s = score(r, nf)
        t.update([float(s), float(ulp_down(s)), float(tf.ulp_up(s))])
    return [np.float32(v) for v in sorted(t)]


# (nf, hits, neighbours): CH through 127 -> 128, 254 -> 255 and 255; CN likewise; different nf side by side
PATTERNS = [(255, 255, 0), (255, 0, 255), (255, 127, 128), (255, 128, 127), (255, 254, 1), (255, 1, 254),
            (255, 127, 127), (254, 254, 0), (254, 0, 254), (128, 128, 0), (127, 127, 0), (128, 0, 128), (127, 0, 127),
            (129, 64, 65)]
SAT_LABEL = 2
SAT_SHAPE = ([8], 264, 256)   # 33 x 32 positions; 8 x 8 templates: P = 1056, one full round and one remainder word
FILLER = (8, 0, 0)            # nf = 8, every feature label o + 4: raw 0, never passes a threshold >= 0


def saturation_templates(levels=1, o=SAT_LABEL):
    return [pattern_template(nf, a, b, o, seed=100 + i, levels=levels) for i, (nf, a, b) in enumerate(PATTERNS)]


def saturation_bank(fillers=0, levels=1, o=SAT_LABEL):
    tps = saturation_templates(levels, o)
    filler = pattern_template(*FILLER, o, seed=7, levels=levels)
    return tf.make_bank(tps + [filler] * fillers)


def ladder(patterns=PATTERNS):
    """Thresholds that put raw_min on every pattern's raw (strict at it) and one above it, plus 0."""
    t = {0.0}
    for nf, a, b in patterns:
        r = 4 * a + b
        t.update([float(score(r - 1, nf)), float(score(r, nf))])
    return [np.float32(v) for v in sorted(t)]


def filler_count(words_per_template, n_patterns, sm_count, plane_bytes, split):
    """Fewest filler templates (same position words as the patterns) whose task count gives k_coarse_packed team size
    `split` on a GPU with sm_count SMs."""
    import importlib
    lib = importlib.import_module("6dpose_b200._lib")
    k = 0
    while True:
        words = np.full(n_patterns + k, words_per_template, np.int32)
        s = lib.coarse_tasks(words, sm_count, plane_bytes)[3]["split"]
        if s == split:
            return k
        assert s > split, (k, s, split)
        k += max(1, k // 8)


# label wrap: (frame label, [(nf, {label: count})]); the neighbours of 0 are 1 and 7, those of 7 are 6 and 0
WRAP_SHAPE = ([8], 128, 64)


def wrap_bank(frame_label, seed=0):
    """Templates of the labels around the wrap: hits, both neighbours (one through the wrap) and non-responses, in
    both kernels (the last one has 300 features)."""
    o = frame_label
    other = 0 if o == 7 else 7   # the neighbour across the wrap
    near = (o + 7) % 8 if o == 7 else (o + 1) % 8
    rng = np.random.default_rng(seed)
    specs = [{other: 40}, {other: 255}, {other: 100, o: 50, near: 30, (o + 4) % 8: 20}, {o: 10, other: 10},
             {other: 150, near: 150}]
    tps = []
    for i, spec in enumerate(specs):
        lab = np.concatenate([np.full(n, l) for l, n in spec.items()])
        lab = lab[rng.permutation(len(lab))]
        tps.append(pyramid(lab, tf.split_modalities(len(lab)), [(8, 8), (8, 8)], 1, seed=300 + i))
    return tf.make_bank(tps)


# position edges: 33 x 31 positions (plane 1023, the last word has 31 valid bits); P = (31 - hf) * 33 + 34 - wf
EDGE_SHAPE = ([8], 264, 248)
TINY_SHAPE = ([8], 40, 24)     # 5 x 3 positions: one partial word


def edge_bank(W, H, T, seed=1):
    """Templates whose P takes every residue mod 32 (hf = 1, wf = 1 .. 32 where the level allows), P = 1 (the
    template as large as the level) and P <= 0 (one cell wider: P = 0; one cell wider and taller: P = -Wd), 24 features
    of random labels each."""
    Wd, Hd = W // T, H // T
    sizes = [(T * wf, T) for wf in range(1, min(Wd, 32) + 1)] + [(Wd * T, Hd * T), ((Wd + 1) * T, Hd * T),
                                                                 ((Wd + 1) * T, (Hd + 1) * T)]
    rng = np.random.default_rng(seed)
    tps = []
    for i, (w, h) in enumerate(sizes):
        lab = rng.integers(0, 8, 24)
        tps.append(pyramid(lab, (12, 12), [(w, h), (w, h)], 1, seed=500 + i))
    return tf.make_bank(tps), sizes


def outside_bank(W, H, seed=2):
    """Features beyond the lowest level's cols or rows: they count in nf and add nothing (LL.cpp:1330).  Bit-sliced
    (40 and 255 features) and byte-wise (300, and 700 with the skipped features inside its first 512-feature tile)."""
    rng = np.random.default_rng(seed)
    tps = []
    for i, (nf, out) in enumerate([(40, 5), (255, 20), (300, 9), (700, 30)]):
        lab = rng.integers(0, 8, nf)
        tps.append(pyramid(lab, tf.split_modalities(nf), [(16, 16), (16, 16)], 1, seed=600 + i, outside=out,
                           level_shape=(W, H)))
    return tf.make_bank(tps)


BYTE_LABEL = 5
# (per-modality counts, sizes per modality or None for 8 x 8 both): every feature a hit
BYTE_SPECS = [((128, 128), None), ((128, 129), None), ((64, 62), ((8, 8), (16, 16))), ((64, 63), ((8, 8), (16, 16))),
              ((64, 64), ((8, 8), (16, 16))), ((126, 127), ((16, 16), (8, 8))), ((189, 189), None), ((511, 512), None),
              ((513, 64), None), ((4096, 4095), None), ((62, 63), ((16, 16), (8, 8))), ((63, 63), ((8, 8), (24, 8)))]


def byte_bank(o=BYTE_LABEL, mixed=False, seed=3):
    """Byte-kernel templates, every feature a hit (raw = 4 nf; 32 764 for 8191 features).  mixed: hits, neighbours and
    non-responses instead (a third of each)."""
    rng = np.random.default_rng(seed)
    tps = []
    for i, (counts, sizes) in enumerate(BYTE_SPECS):
        nf = sum(counts)
        lab = np.full(nf, o) if not mixed else labels(nf, nf // 3, nf // 3, o, rng)
        tps.append(pyramid(lab, counts, sizes or [(8, 8), (8, 8)], 1, seed=700 + i))
    return tf.make_bank(tps)


STAGING = {"k2_shared": ([4, 8], 640, 624), "k2_global": ([4, 8], 640, 640)}
