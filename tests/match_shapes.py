"""Frame-size arithmetic of the match pipeline's kernel routes (include/linemod_b200.h, lm_debug_plan), restated from the
legality rules and the host plan of 6dpose_b200/csrc/linemod_b200.cu, and the shape cases whose match lists the compiled
reference fixed in tests/golden/shape_checks.npz (tests/golden/make_golden.py, make_shape_checks)."""
import os

import numpy as np

M = 2
MAX_ROUNDS = 5                 # LM_MAX_ROUNDS: spread bit-planes of the lowest level up to 5 rounds of 32 x 32 positions
BITS_SMEM_LIMIT = 200 * 1024   # LM_BITS_SMEM_LIMIT: k_coarse_packed stages bit-planes up to this size in shared memory
BAND_SMEM_LIMIT = 160 * 1024   # LM_BAND_SMEM_LIMIT: k_linear_memories_band's shared memory
FILTER_WORDS = 1 << 23         # the filter descriptor's 23-bit plane-offset field

SHAPE_CHECKS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "shape_checks.npz")


def _k1_need(T, Wd, planes):
    """Shared memory of one level in k_linear_memories_band (plan_k1); planes: the level is built as H-planes only."""
    nseg = 1
    if Wd % 4 == 0:
        for j in range(1, min(16, Wd // 4) + 1):
            if (Wd // 4) % j == 0 and (T * T * (Wd // 4)) // j >= 128:
                nseg = j
    if not planes:
        return ((Wd // nseg * T + T + 3 + 4) & ~3) * (2 * (2 * T - 1) + T), 0
    pseg = 4
    for c in (32, 16, 8):
        if Wd % c == 0 and T * T * c <= 128:
            pseg = c
            break
    return ((pseg * T + T + 3 + 4) & ~3) * (2 * (16 * T + T - 1) + 16 * T), pseg


def frame_shape(T, W, H):
    """Asserts that a W x H frame is legal at the pyramid steps T (each level's sides divisible by its T, rows * cols a
    multiple of 16, at most 65 536 lowest-level positions) and returns the numbers that route it."""
    L = len(T)
    lv = []
    for l, t in enumerate(T):
        rows, cols = H >> l, W >> l
        assert (rows << l) == H and (cols << l) == W, "level %d of %dx%d is not a plain halving" % (l, W, H)
        assert rows % t == 0 and cols % t == 0, "level %d: %dx%d not a multiple of T=%d" % (l, cols, rows, t)
        assert rows * cols % 16 == 0, "level %d: rows*cols not a multiple of 16" % l
        lv.append(dict(T=t, rows=rows, cols=cols, Wd=cols // t, Hd=rows // t, plane=(cols // t) * (rows // t)))
    low = lv[-1]
    assert low["plane"] <= 65536, "more than 65536 lowest-level positions"
    nwords = (low["plane"] + 31) // 32
    rounds = (nwords + 31) // 32
    lbw = (((low["T"] ** 2 * low["plane"] + 31) // 32 + 32 * rounds + 4 + 3) & ~3)
    out = dict(levels=lv, Wd=low["Wd"], Hd=low["Hd"], plane=low["plane"], words=nwords, rounds=rounds,
               bit_planes=rounds <= MAX_ROUNDS)
    out["plane_bytes"] = (M * 8 * lbw * 4 + 15) & ~15 if out["bit_planes"] else 0
    out["k2_smem"] = out["bit_planes"] and out["plane_bytes"] <= BITS_SMEM_LIMIT
    out["filter_ok"], out["filter_words"] = False, 0
    if L >= 2:
        r = lv[L - 2]
        nyb = ((r["Hd"] - 16) >> 4) + 1 if r["Hd"] >= 16 else 0
        words = M * 8 * r["T"] ** 2 * nyb * r["Wd"]
        out["filter_words"] = words + (nyb + 1) * r["Wd"] + 64
        out["filter_ok"] = (r["Wd"] % 4 == 0 and r["Wd"] >= 16 and 16 <= r["Hd"] <= 512 and words > 0
                            and out["filter_words"] <= FILTER_WORDS)
    aligned = all(v["cols"] % 4 == 0 and v["Wd"] % 4 == 0 and v["plane"] % 4 == 0 for v in lv)
    # K1 with and without the first refined level in planes mode
    for key, pl in (("k1", -1), ("k1_planes", L - 2 if L >= 2 else -1)):
        need = [_k1_need(v["T"], v["Wd"], l == pl) for l, v in enumerate(lv)]
        smem = max(n for n, _ in need)
        out[key] = dict(band=aligned and smem <= BAND_SMEM_LIMIT, smem=smem, pseg=need[pl][1] if pl >= 0 else 0)
    return out


# Shape cases pinned to the compiled reference: (T, W, H, templates per class, features, template size range, threshold).
# Small frames at every pyramid step T the suite had not run, synth_bank(seed 21, two classes), synth_frame(seed 9,
# four plants, border 0).
SHAPE_CASES = [
    ([1, 2], 160, 128, 6, 64, ((12, 40), (12, 40)), 70.0),
    ([2, 4], 288, 256, 6, 64, ((16, 60), (16, 60)), 70.0),
    ([2, 5], 320, 240, 6, 64, ((16, 60), (16, 60)), 70.0),
    ([2, 9], 288, 288, 6, 64, ((16, 60), (16, 60)), 70.0),
    ([3, 3], 192, 192, 6, 64, ((16, 48), (16, 48)), 70.0),
    ([3, 6], 384, 288, 6, 64, ((16, 60), (16, 60)), 70.0),
    ([4, 11], 352, 352, 6, 64, ((16, 60), (16, 60)), 70.0),
    ([5, 10], 320, 240, 6, 64, ((16, 60), (16, 60)), 70.0),
    ([5, 15], 480, 480, 6, 64, ((16, 90), (16, 90)), 70.0),
    ([6, 8], 672, 480, 6, 64, ((16, 60), (16, 60)), 70.0),
    ([6, 8], 384, 384, 6, 64, ((16, 60), (16, 60)), 70.0),
    ([6, 12], 384, 384, 6, 64, ((16, 60), (16, 60)), 70.0),
    ([7, 7], 448, 336, 6, 64, ((16, 60), (16, 60)), 70.0),
    ([7, 14], 448, 336, 6, 64, ((16, 60), (16, 60)), 70.0),
    ([8, 13], 416, 416, 6, 64, ((16, 60), (16, 60)), 70.0),
    ([8, 16], 384, 384, 6, 64, ((16, 60), (16, 60)), 70.0),
    ([16, 16], 512, 512, 6, 64, ((16, 120), (16, 120)), 70.0),
    ([1], 64, 64, 6, 32, ((8, 32), (8, 32)), 70.0),
    ([16], 512, 320, 6, 64, ((16, 120), (16, 120)), 70.0),
    ([2, 3, 6], 384, 288, 6, 64, ((16, 60), (16, 60)), 70.0),
    ([1, 3, 2, 4], 384, 384, 6, 64, ((16, 80), (16, 80)), 70.0),
]
# The compiled reference ORs spread rows with aligned 16-byte accesses (orUnaligned8u: the destination row is
# dereferenced as __m128i), so it faults unless every level's cols is a multiple of 16; every case above keeps to that
# (DESIGN.md §5).  The oracle and the GPU have no such limit, and the GPU shape matrix also runs sizes beyond it.


def reference_can_run(T, W):
    return all((W >> l) % 16 == 0 for l in range(len(T)))


def _cdiv(a, b):
    """C++ integer division (truncates toward zero)."""
    return -((-a) // b) if a < 0 else a // b


def reference_overreads(T, W, H, packed):
    """Reads of the compiled reference past the end of a label's linear memories ([T*T][Wd*Hd] bytes, one allocation
    per label) for this bank at this frame size: [(level, template, feature, bytes past the end)], empty if none.

    Coarse scan (similarity / similarity_64, LL.cpp:1284-1354): a feature reads template_positions bytes from its
    (y / T) * Wd + x / T in grid (y % T, x % T).  A feature at x = width at T = 1, or at a template side divisible by T
    in the last grid, reads past the last grid's end.  Refinement (similarityLocal, LL.cpp:1366-1420): 16 rows of 16
    bytes from the feature moved by the patch offset; the largest offset is that of the clamped centre max_x, max_y
    (LL.cpp:1861-1880), and a feature is only read while it lies inside the level."""
    L = len(T)
    tm = np.asarray(packed["tmeta"]).reshape(len(packed["tmeta"]), L * M, 4)
    ft = np.asarray(packed["feats"]).reshape(-1, 3)
    out = []
    for l, t in enumerate(T):
        rows, cols = H >> l, W >> l
        Wd, Hd = cols // t, rows // t
        end = t * t * Wd * Hd
        for g in range(tm.shape[0]):
            w0, h0 = int(tm[g, l * M, 0]), int(tm[g, l * M, 1])
            if l == L - 1:
                wf, hf = _cdiv(w0 - 1, t) + 1, _cdiv(h0 - 1, t) + 1
                n_read = (Hd - hf) * Wd + (Wd - wf) + 1
                ox = oy = 0
                if n_read <= 0:
                    continue
            else:
                border = 8 * t
                ox = (_cdiv(cols - w0 - border, t) - 8) * t
                oy = (_cdiv(rows - h0 - border, t) - 8) * t
            for m in range(M):
                first, count = int(tm[g, l * M + m, 2]), int(tm[g, l * M + m, 3])
                for k in range(first, first + count):
                    x, y = int(ft[k, 0]), int(ft[k, 1])
                    grid = (y % t) * t + x % t
                    if l == L - 1:
                        if x >= cols or y >= rows:
                            continue   # LL.cpp:1330
                        last = grid * Wd * Hd + (y // t) * Wd + x // t + n_read - 1
                    else:
                        if x + ox < 0 or y + oy < 0:
                            continue   # skipped at every offset (LL.cpp:1394)
                        lx, ly = min((x + ox) // t, Wd - 1), min((y + oy) // t, Hd - 1)
                        last = grid * Wd * Hd + (ly + 15) * Wd + lx + 15
                    if last >= end:
                        out.append((l, g, k, last - end + 1))
    return out


def shape_case_data(synth, T, W, H, n, nf, size, thr, plant=4):
    """Bank (packed) and quantized frame of one shape case.  At T = 1 on the lowest level, a feature on the template's
    right or bottom side (x = width or y = height, where cropTemplates puts the extreme ones) makes the reference's
    coarse scan read past its linear memories (reference_overreads); there the lowest level's features are moved one
    pixel inside, so that the reference's list is defined."""
    bank = synth.synth_bank(n, num_features=nf, levels=len(T), seed=21, class_ids=("01_template", "02_template"),
                            size_range=size)
    if T[-1] == 1:
        for tps in bank.classes.values():
            for tp in tps:
                for t in tp[2 * (len(T) - 1):]:
                    t.features[:, 0] = np.minimum(t.features[:, 0], t.width - 1)
                    t.features[:, 1] = np.minimum(t.features[:, 1], t.height - 1)
    q, planted = synth.synth_frame(W, H, levels=len(T), seed=9, bank=bank, plant=plant, T=T, border=0)
    return bank.pack(bank.class_ids(), 2 * len(T)), q, planted


def stored_shape_cases():
    """The case list shape_checks.npz was made from (same tuples as SHAPE_CASES)."""
    import json
    raw = json.loads(str(np.load(SHAPE_CHECKS)["cases"]))
    return [(c[0], c[1], c[2], c[3], c[4], tuple(tuple(r) for r in c[5]), c[6]) for c in raw]
