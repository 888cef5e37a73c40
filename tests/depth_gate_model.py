"""Numpy model of the coarse scan's depth gate (include/linemod_b200.h, lm_set_depth_gate) and a match restatement that
takes the gate's per-(template, coarse cell) mask.

  gate_mask            the mask from depth, tmeta, distances and tolerance, vectorised as the header states it
  gate_mask_brute      the same definition restated pixel by pixel and candidate by candidate (checks gate_mask)
  GatedOracle          Detector::matchClass (LL.cpp:1797-1940) in numpy over the oracle's linear memories, with the
                       lowest-level candidates limited to the mask; the reference's std::sort + std::unique is the host
                       finisher lm_finish, which the suite pins against oracle/lm_oracle.cpp on every match list
"""
import importlib

import numpy as np

U16_MAX = 65535


def coarse_grid(rows, cols, T):
    """(Wd, Hd, B): the lowest level's coarse grid of a rows x cols frame and the full-resolution block side s * T_L."""
    L = len(T)
    lr, lc = rows, cols
    for _ in range(L - 1):
        lr, lc = lr // 2, lc // 2
    return lc // T[-1], lr // T[-1], T[-1] << (L - 1)


def cell_summary(depth, T):
    """lo, hi (int64 [Hd, Wd]) of the non-zero depths of each cell's block, and the empty cells (bool)."""
    depth = np.asarray(depth, np.uint16)
    rows, cols = depth.shape
    Wd, Hd, B = coarse_grid(rows, cols, T)
    lo = np.full((Hd, Wd), U16_MAX + 1, np.int64)
    hi = np.zeros((Hd, Wd), np.int64)
    d = depth[:min(rows, Hd * B), :min(cols, Wd * B)].astype(np.int64)
    pr, pc = Hd * B - d.shape[0], Wd * B - d.shape[1]
    d = np.pad(d, ((0, pr), (0, pc)))   # pixels beyond the image read as holes
    blocks = d.reshape(Hd, B, Wd, B).transpose(0, 2, 1, 3).reshape(Hd, Wd, B * B)
    nz = blocks > 0
    lo = np.where(nz, blocks, U16_MAX + 1).min(2)
    hi = np.where(nz, blocks, 0).max(2)
    empty = ~nz.any(2)
    return lo, hi, empty


def bands(z_mm, tau):
    """(zlo, zhi, has): the band of every template, float64 ceil / floor clamped to [0, 65535]; has = z > 0."""
    z = np.asarray(z_mm, np.float64)
    has = z > 0
    with np.errstate(invalid="ignore"):
        zlo = np.clip(np.ceil(np.where(has, z, 0.0) * (1.0 - tau)), 0, U16_MAX).astype(np.int64)
        zhi = np.clip(np.floor(np.where(has, z, 0.0) * (1.0 + tau)), 0, U16_MAX).astype(np.int64)
    return zlo, zhi, has


def sample_offsets(tmeta, T):
    """(ox, oy) per template: floor(floor(w / 2) / T_L) of Template::width / height at the lowest level, modality 0."""
    tm = np.asarray(tmeta).reshape(len(tmeta), -1, 4)
    s = (len(T) - 1) * 2
    return (tm[:, s, 0] // 2) // T[-1], (tm[:, s, 1] // 2) // T[-1]


def gate_mask(depth, tmeta, T, z_mm, tau):
    """bool [G, Hd, Wd]: candidate (cx, cy) of template g passes the gate."""
    lo, hi, empty = cell_summary(depth, T)
    Hd, Wd = lo.shape
    zlo, zhi, has = bands(z_mm, tau)
    ox, oy = sample_offsets(tmeta, T)
    cy, cx = np.meshgrid(np.arange(Hd), np.arange(Wd), indexing="ij")
    sx = cx[None] + ox[:, None, None]
    sy = cy[None] + oy[:, None, None]
    off = (sx >= Wd) | (sy >= Hd)
    sxc, syc = np.minimum(sx, Wd - 1), np.minimum(sy, Hd - 1)
    clo, chi, cem = lo[syc, sxc], hi[syc, sxc], empty[syc, sxc]
    inside = (clo <= zhi[:, None, None]) & (chi >= zlo[:, None, None])
    return off | cem | ~has[:, None, None] | inside


def gate_mask_brute(depth, tmeta, T, z_mm, tau):
    """gate_mask restated candidate by candidate, reading the block's pixels one at a time (small inputs only)."""
    import math
    depth = np.asarray(depth)
    rows, cols = depth.shape
    Wd, Hd, B = coarse_grid(rows, cols, T)
    tm = np.asarray(tmeta).reshape(len(tmeta), -1, 4)
    slot = (len(T) - 1) * 2
    out = np.zeros((len(tm), Hd, Wd), bool)
    for g in range(len(tm)):
        z = float(z_mm[g])
        w, h = int(tm[g, slot, 0]), int(tm[g, slot, 1])
        for cy in range(Hd):
            for cx in range(Wd):
                sx, sy = cx + (w // 2) // T[-1], cy + (h // 2) // T[-1]
                if sx >= Wd or sy >= Hd or not z > 0:
                    out[g, cy, cx] = True
                    continue
                vals = [int(depth[y, x]) for y in range(sy * B, min((sy + 1) * B, rows))
                        for x in range(sx * B, min((sx + 1) * B, cols)) if depth[y, x] != 0]
                if not vals:
                    out[g, cy, cx] = True
                    continue
                zlo = min(max(math.ceil(z * (1 - tau)), 0), U16_MAX)
                zhi = min(max(math.floor(z * (1 + tau)), 0), U16_MAX)
                out[g, cy, cx] = min(vals) <= zhi and max(vals) >= zlo
    return out


def gate_stats(mask, coarse_pass, depth, T, z_mm):
    """lm_depth_gate_stats for one unsharded frame: candidates before / after, empty cells, templates with a distance."""
    _, _, empty = cell_summary(depth, T)
    return dict(before=int(coarse_pass.sum()), after=int((coarse_pass & mask).sum()), empty_cells=int(empty.sum()),
                with_distance=int((np.asarray(z_mm, np.float64) > 0).sum()))


def _tdiv(a, b):
    """C++ integer division (truncates toward zero)."""
    a = np.asarray(a, np.int64)
    return np.sign(a) * (np.abs(a) // b)


def _score(raw, n):
    """(raw * 100.f) / (4 * n): two correctly rounded float32 operations (NaN for n = 0)."""
    with np.errstate(invalid="ignore", divide="ignore"):
        return (np.asarray(raw, np.float32) * np.float32(100)) / np.float32(4 * n)


class GatedOracle:
    """matchClass over one frame.  The linear memories and the coarse scores are computed once; match() then takes a
    threshold and an optional mask [G, Hd, Wd] that limits the lowest-level candidates."""

    def __init__(self, quantized, T, packed):
        from oracle import oracle
        self.T = [int(t) for t in T]
        self.L, self.M = len(T), 2
        self.packed = packed
        self.tmeta = np.asarray(packed["tmeta"], np.int64).reshape(len(packed["tmeta"]), self.L * self.M, 4)
        self.feats = np.asarray(packed["feats"], np.int64)
        self.G = self.tmeta.shape[0]
        self.lv = []
        for l in range(self.L):
            rows, cols = quantized[l][0].shape
            Tl = self.T[l]
            W, H = cols // Tl, rows // Tl
            labs = []
            for m in range(self.M):
                lm = oracle.linear_memories(quantized[l][m], Tl).reshape(8, -1).astype(np.int64)
                labs.append(np.pad(lm, ((0, 0), (0, W * H + 16 * W + 256))))  # reads past a plane see zeros
            self.lv.append(dict(rows=rows, cols=cols, T=Tl, W=W, H=H, plane=W * H, lab=labs))
        low = self.lv[-1]
        self.Wd, self.Hd = low["W"], low["H"]
        self.raw = np.zeros((self.G, low["H"] * low["W"]), np.int64)
        self.nfeat = np.zeros(self.G, np.int64)
        for g in range(self.G):
            self.raw[g], self.nfeat[g] = self._coarse(g)

    def _fe(self, g, slot):
        w, h, fb, fc = self.tmeta[g, slot]
        return w, h, self.feats[fb:fb + fc]

    def _base(self, lv, f):
        T, W = lv["T"], lv["W"]
        return lv["plane"] * ((f[:, 1] % T) * T + f[:, 0] % T) + (f[:, 1] // T) * W + f[:, 0] // T

    def _coarse(self, g):
        lv = self.lv[-1]
        T, W, H = lv["T"], lv["W"], lv["H"]
        total = np.zeros(W * H, np.int64)
        nfeat = 0
        for m in range(self.M):
            w, h, f = self._fe(g, (self.L - 1) * self.M + m)
            nfeat += len(f)
            wf, hf = int(_tdiv(w - 1, T)) + 1, int(_tdiv(h - 1, T)) + 1
            P = (H - hf) * W + (W - wf) + 1   # LL.cpp:1299-1309
            f = f[(f[:, 0] >= 0) & (f[:, 0] < lv["cols"]) & (f[:, 1] >= 0) & (f[:, 1] < lv["rows"])]
            if P <= 0 or len(f) == 0:
                continue
            idx = self._base(lv, f)[:, None] + np.arange(P)[None, :]
            total[:P] += lv["lab"][m][f[:, 2][:, None], idx].sum(0)
        return total, nfeat

    def coarse_pass(self, threshold):
        """bool [G, Hd, Wd]: the lowest-level candidates of the ungated scan."""
        sc = np.stack([_score(self.raw[g], self.nfeat[g]) for g in range(self.G)])
        return (sc > np.float32(threshold)).reshape(self.G, self.Hd, self.Wd)

    def _refine(self, g, x, y, l):
        lv = self.lv[l]
        T, W, cols, rows = lv["T"], lv["W"], lv["cols"], lv["rows"]
        border = 8 * T
        off = T // 2 + (T % 2 - 1)
        w0, h0, _ = self._fe(g, l * self.M)
        x = np.minimum(np.maximum(x * 2 + 1, border), cols - w0 - border)
        y = np.minimum(np.maximum(y * 2 + 1, border), rows - h0 - border)
        ox, oy = (_tdiv(x, T) - 8) * T, (_tdiv(y, T) - 8) * T
        tot = np.zeros((len(x), 256), np.int64)
        nf2 = 0
        rc = (np.arange(16)[:, None] * W + np.arange(16)[None, :]).reshape(-1)
        for m in range(self.M):
            _, _, f = self._fe(g, l * self.M + m)
            nf2 += len(f)
            if len(f) == 0:
                continue
            fx = f[None, :, 0] + ox[:, None]
            fy = f[None, :, 1] + oy[:, None]
            ok = (fx >= 0) & (fy >= 0) & (fx < cols) & (fy < rows)
            fxc, fyc = np.where(ok, fx, 0), np.where(ok, fy, 0)
            base = lv["plane"] * ((fyc % T) * T + fxc % T) + (fyc // T) * W + fxc // T
            vals = lv["lab"][m][np.broadcast_to(f[None, :, 2, None], base.shape + (1,)), base[..., None] + rc]
            tot += (vals * ok[..., None]).sum(1)
        sc = _score(tot, nf2)
        best = np.zeros(len(x), np.float32)
        br = np.full(len(x), -1)
        bc = np.full(len(x), -1)
        if nf2 > 0 and len(x):
            a = sc.argmax(1)
            mx = sc[np.arange(len(x)), a]
            pos = mx > 0
            best = np.where(pos, mx, np.float32(0)).astype(np.float32)
            br, bc = np.where(pos, a // 16, -1), np.where(pos, a % 16, -1)
        return (_tdiv(x, T) - 8 + bc) * T + off, (_tdiv(y, T) - 8 + br) * T + off, best

    def presort(self, threshold, mask=None):
        """Kept matches before sort / unique, in the reference's order (template, then coarse cell): structured array with
        the coarse cell (cx, cy) each came from."""
        thr = np.float32(threshold)
        cand = self.coarse_pass(threshold)
        if mask is not None:
            cand = cand & mask
        lowT = self.T[-1]
        off = lowT // 2 + (lowT % 2 - 1)
        out = []
        for g in range(self.G):
            cy, cx = np.nonzero(cand[g])
            if len(cx) == 0:
                continue
            x, y = cx * lowT + off, cy * lowT + off
            sim = _score(self.raw[g].reshape(self.Hd, self.Wd)[cy, cx], self.nfeat[g])
            for l in range(self.L - 2, -1, -1):
                for c0 in range(0, len(x), 128):
                    sl = slice(c0, c0 + 128)
                    x[sl], y[sl], sim[sl] = self._refine(g, x[sl], y[sl], l)
                keep = ~(sim < thr)
                x, y, sim, cx, cy = x[keep], y[keep], sim[keep], cx[keep], cy[keep]
            rec = np.zeros(len(x), PRESORT_DTYPE)
            rec["x"], rec["y"], rec["similarity"], rec["template"], rec["cx"], rec["cy"] = x, y, sim, g, cx, cy
            out.append(rec)
        return np.concatenate(out) if out else np.zeros(0, PRESORT_DTYPE)

    def finish(self, pre):
        """std::sort + std::unique of LL.cpp:1772-1774 over presort records (every class selected)."""
        lib = importlib.import_module("6dpose_b200._lib")
        nat = lib.NativeDetector(self.T, device=-1)
        nat.load_bank(self.packed, self.L * self.M)
        rec = np.zeros(len(pre), lib.RECORD_DTYPE)
        rec["x"], rec["y"], rec["similarity"], rec["work"] = pre["x"], pre["y"], pre["similarity"], pre["template"]
        rec["seq"] = np.arange(len(pre))
        out = nat.finish(rec)
        nat.close()
        return out

    def match(self, threshold, mask=None):
        return self.finish(self.presort(threshold, mask))


PRESORT_DTYPE = np.dtype([("x", "<i4"), ("y", "<i4"), ("similarity", "<f4"), ("template", "<i4"), ("cx", "<i4"), ("cy", "<i4")])


def as_oracle_dtype(matches):
    """MATCH_DTYPE -> the oracle's REC_DTYPE field names (class_idx), for comparisons with oracle.match."""
    from oracle import oracle
    out = np.zeros(len(matches), oracle.REC_DTYPE)
    for k in ("x", "y", "similarity", "template_id"):
        out[k] = matches[k]
    out["class_idx"] = matches["class_index"]
    return out
