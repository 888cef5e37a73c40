"""Frames and banks that put the refinement filter and the best-cell arg-max exactly on their bounds, and a numpy model of
the filter's decision.

The refinement filter (k_refine_filter_w) drops a coarse candidate unless some cell of its 16x16 patch
has CH >= need = ceil((raw_keep - nf) / 3), where CH counts the features whose label bit is set in the spread mask at that
cell.  The bound is raw <= 3*CH + nf.  The frames here make it an equality:

  * mosaic frames: every level is a mosaic of blocks (even corners, even sides) filled with the 2x2 tile [[1,3],[5,7]]
    or [[0,2],[4,6]] of one-hot labels.  Every TxT window with T >= 3 holds a whole aligned tile, so every response is 4
    or 1 and raw = 3*CH + nf at every cell of every clamped patch.  Thresholds taken from attained similarities put
    hundreds of kept candidates at CH == need;
  * staircase templates on a uniform frame (the odd tile everywhere): the last k descriptors of a template carry odd
    labels (response 4), the others even ones (response 1), so every cell of every patch has raw = 3k + nf, all 256 cells
    tie, and the running bound CH >= need - remaining holds with equality at every check point;
  * zero-score patches: level 0 blanked over the left half, so candidates whose patch lies there score 0 at every cell
    and the reference's arg-max leaves its best cell at (-1, -1).

The model follows the reference's matchClass (LL.cpp:1797-1940), not the kernels: coarse candidates from the oracle's
coarse map with the float rule, the clamped patch origin, and per-cell CH and raw maps built from the level's response
maps.  It gives the expected `filter_dropped_bytes` counter and, on two-level pyramids, the kept records.
"""
import importlib

import numpy as np

synth = importlib.import_module("6dpose_b200.synth")
bank_mod = importlib.import_module("6dpose_b200.bank")

ODD_TILE = np.array([[1, 3], [5, 7]])
EVEN_TILE = np.array([[0, 2], [4, 6]])


def _cuts(rng, n):
    cuts = [0]
    while cuts[-1] < n:
        cuts.append(cuts[-1] + 2 * int(rng.integers(2, 13)))  # even sides, 4 .. 24 px
    return cuts


def mosaic_labels(rng, H, W):
    """One-hot label image: blocks with even corners and even sides, each the odd or the even 2x2 tile."""
    ys, xs = _cuts(rng, H), _cuts(rng, W)
    odd = rng.random((len(ys), len(xs))) < 0.5
    lab = np.empty((H, W), np.int64)
    for by in range(len(ys) - 1):
        for bx in range(len(xs) - 1):
            y0, y1, x0, x1 = ys[by], min(ys[by + 1], H), xs[bx], min(xs[bx + 1], W)
            tile = ODD_TILE if odd[by, bx] else EVEN_TILE
            lab[y0:y1, x0:x1] = np.tile(tile, ((y1 - y0) // 2, (x1 - x0) // 2))
    return (1 << lab).astype(np.uint8)


def mosaic_frame(W, H, levels, seed):
    """Quantized pyramid [[colour, normals] per level], every level and modality an independent mosaic."""
    rng = np.random.default_rng(seed)
    return [[mosaic_labels(rng, H >> l, W >> l) for _ in range(2)] for l in range(levels)]


def uniform_frame(W, H, levels):
    """Every level and modality tiled with the odd tile: odd labels respond 4, even labels 1."""
    return [[(1 << np.tile(ODD_TILE, ((H >> l) // 2, (W >> l) // 2))).astype(np.uint8) for _ in range(2)]
            for l in range(levels)]


def zero_score_frame(W, H, levels, seed, bank, T):
    """synth_frame with level 0 blanked over the left half: patches there score 0 at every cell."""
    q, _ = synth.synth_frame(W, H, levels=levels, seed=seed, bank=bank, plant=1, T=T)
    for m in range(2):
        q[0][m][:, : W // 2] = 0
    return q


def zero_case(unsafe=False, T=(4, 8), W=320, H=256):
    """Two-level frame (320x256 by default) blanked over the left half of level 0, with a three-template bank.
    unsafe=True moves a feature of template 1 below its box: prepare_bank does not call it "safe", so the byte-wise
    refinement takes it."""
    T = list(T)
    bank = synth.synth_bank(3, num_features=32, levels=2, seed=5)
    if unsafe:
        tps = bank.classes["01_template"]
        tps[1][0].features[5, 1] = tps[1][0].height + 6  # below the box, still over the blank half
    q = zero_score_frame(W, H, 2, 6, bank, T)
    return T, bank, q, bank.pack(bank.class_ids(), 4)


def make_unsafe(tp):
    """Moves a level-0 feature of template pyramid `tp` beyond its box: prepare_bank does not call the template "safe",
    so the filter hands its candidates unfiltered to the byte-wise refinement (k_refine<true>)."""
    tp[0].features[5, 0] = tp[0].width + 6


def split_modalities(nf):
    """Features per modality: a first modality with < 64 features would force the second below 64 too (LL.cpp:1813)."""
    a = nf // 2
    if a < 64 and nf - a >= 64:
        a = 64
    return a, nf - a


def staircase_template(nf, k, seed, w=64, h=64, nf_low=(20, 20), odd_all=False):
    """Template pyramid (two levels) whose level-0 descriptors, in prepare_bank order (modality 0, then modality 1),
    carry even labels on the first nf - k features and odd labels on the last k.  Level-1 features are all odd."""
    rng = np.random.default_rng(seed)
    a, b = split_modalities(nf) if not isinstance(nf, tuple) else nf
    n = a + b
    odd = np.arange(n) >= n - k
    if odd_all:
        odd[:] = True
    labs = np.where(odd, 2 * rng.integers(0, 4, n) + 1, 2 * rng.integers(0, 4, n))
    x = rng.integers(0, w + 1, n)
    y = rng.integers(0, h + 1, n)
    x[0], y[1], x[2], y[3] = 0, 0, w, h  # cropTemplates extents
    T_ = bank_mod.Template
    tp = [T_(w, h, 0, np.stack([x[:a], y[:a], labs[:a]], 1).astype(np.int32)),
          T_(w, h, 0, np.stack([x[a:], y[a:], labs[a:]], 1).astype(np.int32))]
    for m in range(2):
        nl = nf_low[m]
        f = np.stack([rng.integers(0, w // 2 + 1, nl), rng.integers(0, h // 2 + 1, nl),
                      2 * rng.integers(0, 4, nl) + 1], 1).astype(np.int32)
        tp.append(T_(w // 2, h // 2, 1, f))
    return tp


def make_bank(template_lists, class_id="01_template"):
    bank = bank_mod.TemplateBank()
    bank.classes[class_id] = list(template_lists)
    return bank


def score(raw, nf):
    """The reference's similarity: the same two IEEE single-precision operations."""
    return np.float32(np.float32(raw) * np.float32(100.0)) / np.float32(4 * nf)


def min_kept_raw(threshold, nf):
    """Smallest raw with !(score < threshold) (LL.cpp:1935-1937)."""
    lo, hi = 0, 4 * nf + 1
    thr = np.float32(threshold)
    while lo < hi:
        mid = (lo + hi) >> 1
        if not (score(mid, nf) < thr):
            hi = mid
        else:
            lo = mid + 1
    return lo


def need_of(threshold, nf):
    over = min_kept_raw(threshold, nf) - nf
    return -(-over // 3) if over > 0 else 0


def response_maps(oracle, q, T):
    """[levels][modality] -> u8 [8, rows, cols] responses (0, 1 or 4) of the reference's spread + LUT."""
    return [[oracle.response_maps(oracle.spread(q[l][m], T[l])) for m in range(len(q[l]))] for l in range(len(q))]


def reachable_responses(resp, T):
    """Responses outside the last T rows and columns (where the clipped spread window can leave a label out)."""
    return resp[:, : resp.shape[1] - T, : resp.shape[2] - T]


class Model:
    """The reference's decision for every (template, coarse candidate) of a frame, at the filtered level L - 2."""

    def __init__(self, oracle, q, T, packed):
        self.q, self.T, self.packed = q, list(T), packed
        self.L = len(T)
        self.M = len(q[0])
        self.tmeta, self.feats = packed["tmeta"], packed["feats"]
        self.G = self.tmeta.shape[0]
        lr = self.L - 2
        self.lr = lr
        rows, cols = q[lr][0].shape
        Tr = self.T[lr]
        self.rows, self.cols, self.Tr = rows, cols, Tr
        self.Wd, self.Hd = cols // Tr, rows // Tr
        resp = [oracle.response_maps(oracle.spread(q[lr][m], Tr)) for m in range(self.M)]
        self.resp = resp  # [modality] -> u8 [8, rows, cols] responses of the filtered level
        Tl = self.T[-1]
        low = q[-1]
        self.low_Wd = low[0].shape[1] // Tl
        self.low_off = Tl // 2 + (Tl % 2 - 1)
        off = Tr // 2 + (Tr % 2 - 1)
        self.off = off
        self.t = []
        for g in range(self.G):
            # coarse candidates: the lowest level's total similarity map, score > threshold (LL.cpp:1836-1852)
            tm_low = self.tmeta[g, (self.L - 1) * self.M:(self.L) * self.M]
            cmap, _ = oracle.coarse_map(low, Tl, tm_low, self.feats)
            nf_low = int(tm_low[:, 3].sum())
            w0, h0 = int(self.tmeta[g, lr * self.M, 0]), int(self.tmeta[g, lr * self.M, 1])
            fr = [self.feats[int(b):int(b) + int(n)] for (_, _, b, n) in self.tmeta[g, lr * self.M:(lr + 1) * self.M]]
            nf = sum(len(f) for f in fr)
            # "safe" (prepare_bank): at every refined level the clamp range is regular and every feature lies in the box
            safe = True
            for l in range(self.L - 1):
                wl, hl = int(self.tmeta[g, l * self.M, 0]), int(self.tmeta[g, l * self.M, 1])
                rl, cl = q[l][0].shape
                border = 8 * self.T[l]
                safe = safe and cl - wl - border >= border and rl - hl - border >= border
                for b, n in self.tmeta[g, l * self.M:(l + 1) * self.M, 2:4].tolist():
                    f = self.feats[b:b + n]
                    safe = safe and int(f[:, 0].max(initial=0)) <= wl and int(f[:, 1].max(initial=0)) <= hl
            ch = np.zeros((self.Hd, self.Wd), np.int32)
            raw = np.zeros((self.Hd, self.Wd), np.int32)
            if safe:
                for m, f in enumerate(fr):
                    for fx, fy, lab in f.tolist():
                        a = resp[m][lab][fy::Tr, fx::Tr][: self.Hd, : self.Wd]
                        raw[: a.shape[0], : a.shape[1]] += a
                        ch[: a.shape[0], : a.shape[1]] += a == 4
            self.t.append(dict(cmap=cmap.astype(np.int64), nf_low=nf_low, w=w0, h=h0, nf=nf, safe=safe, ch=ch, raw=raw))

    def filter_ok(self):
        """prepare_bank's frame limits for the filter's H-planes."""
        Wd, Hd, T = self.Wd, self.Hd, self.Tr
        nyb = ((Hd - 16) >> 4) + 1 if Hd >= 16 else 0
        words = self.M * 8 * T * T * nyb * Wd
        return Wd % 4 == 0 and Wd >= 16 and Hd >= 16 and Hd <= 512 and words > 0 and \
            words + (nyb + 1) * Wd + 64 <= 1 << 23

    def eligible(self, g):
        t = self.t[g]
        return self.filter_ok() and t["safe"] and 1 <= t["nf"] <= 511

    def candidates(self, g, threshold):
        """Coarse cells (row-major, the reference's push order) whose float score beats the threshold."""
        t = self.t[g]
        if t["nf_low"] == 0:
            return np.zeros(0, np.int64)
        s = score(t["cmap"].ravel(), t["nf_low"])
        return np.flatnonzero(s > np.float32(threshold))

    def patches(self, g, cells):
        """Clamped patch origins (LL.cpp:1871-1880, max before min) and the 16x16 CH / raw windows of the cells."""
        t = self.t[g]
        Tr, border = self.Tr, 8 * self.Tr
        Tl = self.T[-1]
        x = (cells % self.low_Wd) * Tl + self.low_off
        y = (cells // self.low_Wd) * Tl + self.low_off
        x = np.minimum(np.maximum(x * 2 + 1, border), self.cols - t["w"] - border)
        y = np.minimum(np.maximum(y * 2 + 1, border), self.rows - t["h"] - border)
        cx, cy = x // Tr - 8, y // Tr - 8
        win = np.lib.stride_tricks.sliding_window_view
        ch = win(t["ch"], (16, 16))[cy, cx]
        raw = win(t["raw"], (16, 16))[cy, cx]
        return x, y, ch, raw

    def decisions(self, g, threshold):
        """Per coarse candidate of template g: need, max CH, best raw, first-maximum cell (-1 when every cell is 0)."""
        t = self.t[g]
        cells = self.candidates(g, threshold)
        x, y, ch, raw = self.patches(g, cells)
        flat = raw.reshape(len(cells), 256)
        best = flat.max(axis=1, initial=0)
        first = np.where(best > 0, np.argmax(flat == best[:, None], axis=1), -1)
        return dict(cells=cells, x=x, y=y, need=need_of(threshold, t["nf"]), max_ch=ch.reshape(len(cells), 256).max(axis=1, initial=0),
                    best=best, first=first, ch=ch, raw=raw)

    def dropped_bytes(self, threshold):
        """The expected filter_dropped_bytes: 256 * nf for every candidate of an eligible template that cannot be kept."""
        total = 0
        for g in range(self.G):
            if not self.eligible(g):
                continue
            d = self.decisions(g, threshold)
            nf, need = self.t[g]["nf"], d["need"]
            if need > nf:
                total += 256 * nf * len(d["cells"])
            elif need > 0:
                total += 256 * nf * int((d["max_ch"] < need).sum())
        return total

    def kept(self, threshold, class_idx=0):
        """Kept records of a two-level pyramid in the reference's pre-sort order (safe templates only)."""
        assert self.L == 2
        out = []
        for g in range(self.G):
            t = self.t[g]
            assert t["safe"]
            d = self.decisions(g, threshold)
            first = d["first"]
            br = np.where(first >= 0, first // 16, -1)
            bc = np.where(first >= 0, first % 16, -1)
            sim = score(d["best"], t["nf"])
            xs = (d["x"] // self.Tr - 8 + bc) * self.Tr + self.off
            ys = (d["y"] // self.Tr - 8 + br) * self.Tr + self.off
            for i in np.flatnonzero(~(sim < np.float32(threshold))):
                out.append((int(xs[i]), int(ys[i]), float(sim[i]), class_idx, g))
        return out


def records(arr):
    """Oracle / C-ABI structured records -> sorted list of (x, y, similarity, class, template) tuples."""
    cls = "class_idx" if "class_idx" in arr.dtype.names else "class_index"
    return sorted(zip(arr["x"].tolist(), arr["y"].tolist(), [float(v) for v in arr["similarity"]],
                      arr[cls].tolist(), arr["template_id"].tolist()))


# ---- the cases the tests run --------------------------------------------------------------------------------------------

MOSAIC_BANK = dict(n=40, nf=150, seed=21, variants=40)


def mosaic_case(T, W, H, seed=0, unsafe=False):
    """Synthetic bank and mosaic frame.  With more than two levels the levels below the filtered one (L - 2) carry every
    label bit at every pixel: every cell there scores 100 %, so the filtered level alone decides what is kept.
    unsafe=True makes every third template unsafe (make_unsafe)."""
    bank = synth.synth_bank(MOSAIC_BANK["n"], num_features=MOSAIC_BANK["nf"], levels=len(T), seed=MOSAIC_BANK["seed"],
                            variants=MOSAIC_BANK["variants"])
    if unsafe:
        for tp in bank.classes["01_template"][::3]:
            make_unsafe(tp)
    q = mosaic_frame(W, H, len(T), seed)
    for l in range(len(T) - 2):
        q[l] = [np.full_like(a, 0xFF) for a in q[l]]
    return bank, q


def tight_thresholds(oracle, q, T, packed, percentiles=(50, 90, 99), n_threads=1):
    """Similarities of kept matches at threshold 40 (the oracle's own scores), at the given percentiles.  Each is a
    similarity some candidate attains, so raw_keep = 3 * need + nf on a mosaic frame."""
    want = oracle.match(q, T, packed, 40.0, n_threads=n_threads)
    sims = np.sort(want["similarity"])
    return [np.float32(sims[min(len(sims) - 1, int(len(sims) * p / 100))]) for p in percentiles]


_MOSAIC = {}


def mosaic_setup(oracle, T, W, H, percentiles=(50, 90, 99), n_threads=1, unsafe=False):
    """Bank, frame, packed bank, model and tight thresholds of a mosaic case (built once per process)."""
    key = (tuple(T), W, H, tuple(percentiles), unsafe)
    if key not in _MOSAIC:
        bank, q = mosaic_case(T, W, H, unsafe=unsafe)
        packed = bank.pack(bank.class_ids(), len(T) * 2)
        model = Model(oracle, q, T, packed)
        if len(T) == 2:
            thrs = tight_thresholds(oracle, q, T, packed, percentiles, n_threads)
        else:  # the filtered level is not the last one: take the similarities the model gives at that level
            sims = []
            for g in range(model.G):
                s = score(model.decisions(g, 40.0)["best"], model.t[g]["nf"])
                sims.extend(s[~(s < np.float32(40.0))].tolist())
            sims = np.sort(np.asarray(sims, np.float32))
            thrs = [np.float32(sims[min(len(sims) - 1, int(len(sims) * p / 100))]) for p in percentiles]
        _MOSAIC[key] = dict(bank=bank, q=q, packed=packed, model=model, thresholds=thrs)
    return _MOSAIC[key]


def ulp_up(thr):
    return np.nextafter(np.float32(thr), np.float32(np.inf))


# staircase: feature counts and the first hit index s = nf - k just before, at and just after a multiple of 64
STAIR_NF = (33, 64, 65, 96, 127, 128, 129, 255, 256, 257, 320, 511)


def stair_ks(nf):
    """Hit counts k whose first hit (descriptor nf - k) lies just before, at and just after the last multiple of 64 below
    nf; for 511 also k = nf (every feature a hit: CH = 511 fills all nine counter bits, raw = 2044)."""
    m = max(64 * ((nf - 1) // 64), 64) if nf > 64 else 0
    ks = {nf - s for s in (m - 1, m, m + 1) if 0 <= s < nf}
    if nf == 511:
        ks.add(nf)
    return sorted(ks)


def stair_cases():
    """(nf, k, threshold, need) for every staircase template: need = k (everything kept) and k + 1 (nothing kept).
    With k = nf the similarity is 100 %, and the coarse scan keeps only scores above the threshold: the threshold is one
    ulp below 100, which still gives need = nf, and there is no need = k + 1 case."""
    out = []
    for nf in STAIR_NF:
        for k in stair_ks(nf):
            thr = score(3 * k + nf, nf)
            if k == nf:
                out.append((nf, k, np.nextafter(thr, np.float32(-np.inf)), k))
                continue
            out.append((nf, k, thr, k))
            out.append((nf, k, ulp_up(thr), k + 1))
    return out


def stair_bank(nf, k, unsafe=False):
    """One staircase template; the 511-feature one (255 + 256, all odd) shares its bank with a 512-feature one
    (256 + 256), which the filter does not take.  unsafe=True appends an unsafe copy of the staircase template (the
    last template of the bank)."""
    tps = [staircase_template(nf, k, seed=1000 + nf * 7 + k)]
    if nf == 511:
        tps.append(staircase_template((256, 256), 512, seed=5, odd_all=True))
    if unsafe:
        tps.append(staircase_template(nf, k, seed=1000 + nf * 7 + k))
        make_unsafe(tps[-1])
    return make_bank(tps)
