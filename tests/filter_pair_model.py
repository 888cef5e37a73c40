"""Lane-level numpy model of the refinement filter k_refine_filter_w (csrc/lm_kernels.cuh), candidate by candidate, and a
classifier of the pairs its warps take.

A warp takes candidates c and c + 1 of the ordered list (work items in shard order, each one's coarse cells row-major) and
runs their step chains side by side until one dies or runs out of features; the other goes on alone from the step it
has reached.  What the filter does with a candidate -- where it dies, which plane words it reads, whether it is kept --
depends on that candidate alone, so the model runs each one on its own and sums:

  * triage (filter_triage): 0 = pass on uncounted (a template the filter does not take, or need <= 0), 1 = drop uncounted
    (need > nf), 2 = count.  Triage 1 needs a threshold above 100 and so never meets a coarse candidate, and need <= 0
    holds for every template at once (threshold <= 25) or for none, so a counted candidate is never paired with a need <= 0
    one (need_facts);
  * a counted candidate is a chain of nfp = nf rounded up to 32 features, 32 per step, in descriptor order (modality 0,
    then modality 1).  After `done` features a check happens when thr = need - max(nf - done, 0) > 0 and done is a
    multiple of LM_FILTER_CHECK or the end.  Patch column k (lanes k and k + 16) stays alive while some row of the column
    has CH >= thr; the candidate dies when no column is alive.  A step reads 32 words per column alive before it (16
    lanes-worth per half-warp);
  * filter_bytes_read = 4 x (words + the 32 x nfp plane words k_refine_bits reads per survivor it finishes: the
    counter is shared by both kernels), filter_dropped_bytes = 256 x nf per dropped candidate, and lm_debug_plan entries
    16 (list length), 17 (survivors for k_refine_bits) and 18 (survivors for k_refine<true>).
"""
import numpy as np

import tight_frames as tf

CHECK = 64   # LM_FILTER_CHECK: features between two bound checks
STEP = 32    # features per step of a chain

COUNTED, SURV2, NEED0 = "counted", "surv2", "need0"


def need_facts(nfs=range(1, 512)):
    """need > nf (triage 1) exactly when the threshold is above 100, which no coarse score (<= 100) beats; need <= 0 exactly
    when the threshold is <= 25, whatever nf.  Returns the two boundary thresholds after checking them for every nf."""
    hi, lo = np.float32(100.0), np.float32(25.0)
    for nf in nfs:
        assert tf.need_of(hi, nf) == nf and tf.need_of(tf.ulp_up(hi), nf) == nf + 1
        assert tf.need_of(lo, nf) <= 0 and tf.need_of(tf.ulp_up(lo), nf) == 1
    return hi, lo


def check_points(nf):
    nfp = (nf + STEP - 1) // STEP * STEP
    return [d for d in range(STEP, nfp + 1, STEP) if d >= nf or d % CHECK == 0]


def prefix_ch(model, g, points):
    """Prefix CH maps [Hd, Wd] of template g after the first `done` features (descriptor order) for each done in points."""
    lr, Tr, Hd, Wd = model.lr, model.Tr, model.Hd, model.Wd
    feats = []
    for m, (_, _, b, n) in enumerate(model.tmeta[g, lr * model.M:(lr + 1) * model.M].tolist()):
        feats += [(m, fx, fy, lab) for fx, fy, lab in model.feats[b:b + n].tolist()]
    ch = np.zeros((Hd, Wd), np.int32)
    out, k = {}, 0
    for done in sorted(points):
        for m, fx, fy, lab in feats[k:min(done, len(feats))]:
            a = model.resp[m][lab][fy::Tr, fx::Tr][:Hd, :Wd]
            ch[:a.shape[0], :a.shape[1]] += a == 4
        k = max(k, min(done, len(feats)))
        out[done] = ch.copy()
    return out


def run_counted(snaps, nf, need, cx, cy):
    """Chains of the counted candidates of one template (patch origins cx, cy in cells).  Per candidate: dead, the step
    it ended at (death or nfp), plane words read, a partial column death survived at some check, died at the last check."""
    n = len(cx)
    nfp = (nf + STEP - 1) // STEP * STEP
    alive = np.ones((n, 16), bool)
    running = np.ones(n, bool)
    dead = np.zeros(n, bool)
    partial = np.zeros(n, bool)
    end = np.full(n, nfp, np.int64)
    words = np.zeros(n, np.int64)
    win = np.lib.stride_tricks.sliding_window_view
    for done in range(STEP, nfp + 1, STEP):
        words[running] += 32 * alive[running].sum(axis=1)
        thr = need - max(nf - done, 0)
        if thr > 0 and (done >= nf or done % CHECK == 0):
            cols = (win(snaps[done], (16, 16))[cy, cx] >= thr).any(axis=1)   # [n, 16]: column k has a row >= thr
            alive[running] = cols[running]
            died = running & ~alive.any(axis=1)
            dead |= died
            end[died] = done
            running &= ~died
            partial |= running & (alive.sum(axis=1) < 16)
    return dict(dead=dead, end=end, words=words, partial=partial, last=dead & (end == nfp))


class FilterModel:
    """The filter's list and outcome for one call: `model` (tight_frames.Model of the frame and bank), the threshold and
    the work items of the shard (template ids in shard order; default: every template)."""

    def __init__(self, model, threshold, items=None):
        self.model, self.threshold = model, np.float32(threshold)
        self.items = list(range(model.G)) if items is None else list(items)
        self.bits = model.L == 2          # k_refine_bits takes the survivors, unsafe ones go to a second list
        cols = {k: [] for k in ("item", "cell", "kind", "nf", "dead", "end", "words", "partial", "last")}
        for w, g in enumerate(self.items):
            cells = model.candidates(g, threshold)
            n = len(cells)
            if n == 0:
                continue
            nf = model.t[g]["nf"]
            need = tf.need_of(self.threshold, nf)
            assert need <= nf   # triage 1 is unreachable (need_facts)
            kind = SURV2 if not model.eligible(g) else (NEED0 if need <= 0 else COUNTED)
            cols["item"] += [w] * n
            cols["cell"] += cells.tolist()
            cols["kind"] += [kind] * n
            cols["nf"] += [nf] * n
            if kind == COUNTED:
                x, y, _, _ = model.patches(g, cells)
                r = run_counted(prefix_ch(model, g, check_points(nf)), nf, need, x // model.Tr - 8, y // model.Tr - 8)
                for k in ("dead", "end", "words", "partial", "last"):
                    cols[k] += r[k].tolist()
            else:
                cols["dead"] += [False] * n
                cols["end"] += [0] * n
                cols["words"] += [0] * n
                cols["partial"] += [False] * n
                cols["last"] += [False] * n
        self.c = {k: np.asarray(v) for k, v in cols.items()}
        self.n = len(self.c["item"])
        self.all_eligible = all(model.eligible(g) for g in self.items)

    def words(self):
        return int(self.c["words"].sum()) if self.n else 0

    def bits_words(self):
        """Plane words k_refine_bits reads for the survivors it finishes: an H and an N window (16 words each) per feature
        of the padded descriptor list, 32 * nfp per survivor."""
        if not self.bits or not self.n:
            return 0
        surv = ~self.c["dead"] & (self.c["kind"] != SURV2)
        return int((32 * ((self.c["nf"][surv] + STEP - 1) // STEP * STEP)).sum())

    def bytes_read(self):
        """lm_counters' filter_bytes_read: the plane bytes of the filter and of the bit-sliced exact pass behind it."""
        return 4 * (self.words() + self.bits_words())

    def dropped_bytes(self):
        return 256 * int(self.c["nf"][self.c["dead"]].sum()) if self.n else 0

    def kept(self):
        """The number of candidates that go on to the exact passes."""
        return self.n - int(self.c["dead"].sum()) if self.n else 0

    def plan(self):
        """lm_debug_plan entries 16, 17 and 18 of the call (-1: that kernel does not run)."""
        surv2 = int((self.c["kind"] == SURV2).sum()) if self.n else 0
        surv = self.kept() - surv2 if self.bits else self.kept()
        if self.bits:
            return [self.n, surv, -1 if self.all_eligible else surv2]
        return [self.n, -1, surv]

    def pair_classes(self):
        """Counts of the pair classes this list gives the filter's warps (pairs (2m, 2m + 1))."""
        out = {}

        def add(k):
            out[k] = out.get(k, 0) + 1

        add("list_len_%d" % min(self.n, 3))
        c = self.c
        for a in range(0, self.n, 2):
            b = a + 1
            for i, who in ((a, "A"), (b, "B")):
                if i < self.n and c["kind"][i] == COUNTED:
                    if c["partial"][i]:
                        add("partial_%s_%s" % (who, "dropped" if c["dead"][i] else "kept"))
                    if c["last"][i] and c["nf"][i] % 32:
                        add("last_check_death_nf_not_32")
                    if c["last"][i] and c["nf"][i] % 32 == 0 and c["nf"][i] % 64:
                        add("last_check_death_nf_32_not_64")
            if b >= self.n:
                add("unpaired_" + c["kind"][a])
                continue
            ka, kb = c["kind"][a], c["kind"][b]
            if ka != COUNTED or kb != COUNTED:
                add("pair_%s_%s" % (ka, kb))
                continue
            if c["item"][a] != c["item"][b]:
                add("two_templates")
                if c["nf"][a] != c["nf"][b]:
                    add("two_nf")
            da, db, ea, eb = c["dead"][a], c["dead"][b], c["end"][a], c["end"][b]
            if ea == eb:
                add("both_die_same_check" if da and db else "both_finish_same_step" if not (da or db) else
                    "one_dies_at_the_end_the_other_finishes")
            elif ea < eb:
                add("A_dies_first" if da else "A_finishes_B_goes_on_" + ("dropped" if db else "kept"))
            else:
                add("B_dies_first" if db else "B_finishes_A_goes_on_" + ("dropped" if da else "kept"))
        return out


def device_list(mask):
    """(work item, cell) of every entry of the device's ordered list, from lm_debug_coarse pass masks [n_work, nwords]:
    work items in shard order, each one's cells ascending (k_refine_prep)."""
    bits = np.unpackbits(np.ascontiguousarray(mask, "<u4").view(np.uint8), bitorder="little").reshape(mask.shape[0], -1)
    return np.nonzero(bits)


# ---- the pair-coverage frames (two levels, T = [4, 8], 320 x 256) -----------------------------------------------------

PAIR_T, PAIR_W, PAIR_H = [4, 8], 320, 256

# the "pairs" bank in list order: (features at level 0, kind).  Every template of it has 257 coarse candidates (odd), so
# template t starts at an odd list index for odd t and its first candidate shares a warp with template t - 1's last one:
# counted | surv2 (1), surv2 | counted (3), and counted pairs of a shorter and a longer chain in both orders (5 .. 13).
# 15 templates: the list ends on an unpaired counted candidate.
PAIR_BANK = [(96, "c"), (150, "unsafe"), (512, "big"), (150, "c"), (64, "c"), (200, "c"), (255, "c"), (100, "c"),
             (33, "c"), (160, "c"), (320, "c"), (127, "c"), (511, "c"), (96, "c"), (129, "c")]


def _pair_template(nf, kind, seed):
    if kind == "big":  # 256 + 256 features: more than the filter's 9-bit counters hold, so k_refine<true> takes it
        return tf.staircase_template((256, 256), 512, seed=seed, odd_all=True)
    tp = tf.staircase_template(nf, int(nf * 0.4), seed=seed)
    if kind == "unsafe":
        tf.make_unsafe(tp)
    return tp


def pairs_case(oracle, seed=3):
    """Mosaic level 0 (cell-to-cell variation: candidates of one template die at different checks, columns die one by
    one) under a uniform odd level 1: every template's level-1 features are odd labels, so every coarse cell scores 100 %
    and each template's candidate count is fixed by the frame size alone.  Thresholds: 25 (need = 0 everywhere) and one
    ulp above (need = 1), and the similarities of the oracle's 50th, 90th and 99th percentile kept match and one ulp above."""
    rng = np.random.default_rng(seed)
    q = [[tf.mosaic_labels(rng, PAIR_H, PAIR_W) for _ in range(2)], tf.uniform_frame(PAIR_W, PAIR_H, 2)[1]]
    bank = tf.make_bank([_pair_template(nf, kind, 100 + i) for i, (nf, kind) in enumerate(PAIR_BANK)])
    packed = bank.pack(bank.class_ids(), 4)
    thrs = [np.float32(25.0)] + tf.tight_thresholds(oracle, q, PAIR_T, packed, (50, 90, 99))
    return dict(q=q, bank=bank, packed=packed, thresholds=[t for thr in thrs for t in (thr, tf.ulp_up(thr))])


def sparse_case(spots, kinds, threshold=50.0, seed=7):
    """Level 1 the even tile with an odd 2 x 2 tile at each spot (cell (x, y) of the coarse grid); each template has one
    odd level-1 feature per modality at (0, 0), so it scores 100 % at the spot cells and 25 % elsewhere: at threshold 50
    (threshold 25 .. 100) its candidates are exactly the spots.  kinds as in PAIR_BANK, in list order."""
    rng = np.random.default_rng(seed)
    bank_mod = tf.bank_mod
    lab = np.tile(tf.EVEN_TILE, (PAIR_H // 4, PAIR_W // 4))
    for cx, cy in spots:
        lab[8 * cy + 2:8 * cy + 4, 8 * cx + 2:8 * cx + 4] = tf.ODD_TILE
    low = (1 << lab).astype(np.uint8)
    q = [[tf.mosaic_labels(rng, PAIR_H, PAIR_W) for _ in range(2)], [low, low.copy()]]
    tps = []
    for i, (nf, kind) in enumerate(kinds):
        tp = _pair_template(nf, kind, 300 + i)
        for m in (2, 3):
            tp[m] = bank_mod.Template(tp[m].width, tp[m].height, 1, np.array([[0, 0, 1]], np.int32))
        tps.append(tp)
    bank = tf.make_bank(tps)
    return dict(q=q, bank=bank, packed=bank.pack(bank.class_ids(), 4), thresholds=[np.float32(threshold)])


SPARSE_CASES = {
    "empty": ([], [(96, "c")]),                                     # no candidate: the filter runs on a list of 0
    "one": ([(10, 8)], [(127, "c")]),                               # a list of 1: one unpaired counted candidate
    "two": ([(10, 8), (5, 12)], [(96, "c")]),                       # a list of 2: one pair
    "three": ([(10, 8)], [(64, "c"), (200, "c"), (150, "unsafe")]),  # two counted, then an unpaired surv2 candidate
    # 511 | 33 features in one warp at 85 %: the short one finishes kept, the long one goes on and is dropped
    "long_short": ([(10, 8), (6, 5), (12, 10)], [(511, "c"), (33, "c")], 85.0),
}


def coverage_cases(oracle):
    """name -> dict(q, bank, packed, thresholds) of every frame the pair coverage counts: the pairs frame, the sparse
    frames and the zero-score frames of tight_frames (need <= 0 at thresholds 0 and -1, with and without an unsafe
    template)."""
    out = {"pairs": pairs_case(oracle)}
    for name, args in SPARSE_CASES.items():
        out["sparse_" + name] = sparse_case(*args)
    for unsafe in (False, True):
        T, bank, q, packed = tf.zero_case(unsafe)
        out["zero_unsafe" if unsafe else "zero"] = dict(q=q, bank=bank, packed=packed,
                                                         thresholds=[np.float32(0.0), np.float32(-1.0)])
    return out


REQUIRED = [  # (class, how many times the coverage frames must give it at least)
    ("A_dies_first", 5), ("B_dies_first", 5), ("both_die_same_check", 5),
    ("both_finish_same_step", 5),
    ("A_finishes_B_goes_on_kept", 1), ("A_finishes_B_goes_on_dropped", 1),
    ("B_finishes_A_goes_on_kept", 1), ("B_finishes_A_goes_on_dropped", 1),
    ("two_templates", 3), ("two_nf", 3),
    ("partial_A_kept", 5), ("partial_A_dropped", 5), ("partial_B_kept", 5), ("partial_B_dropped", 5),
    ("pair_counted_surv2", 1), ("pair_surv2_counted", 1),
    ("pair_need0_need0", 5), ("pair_need0_surv2", 1), ("pair_surv2_need0", 1),
    ("unpaired_counted", 1), ("unpaired_surv2", 1), ("unpaired_need0", 1),
    ("list_len_0", 1), ("list_len_1", 1), ("list_len_2", 1),
    ("last_check_death_nf_not_32", 5), ("last_check_death_nf_32_not_64", 5),
]
