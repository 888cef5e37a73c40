"""A seeded call program for one long-lived detector handle (tests/test_gpu_handle_sequences.py).

The handle (include/linemod_b200.h, lm_detector) keeps state between calls, each piece behind its own invalidation: the
bank prepared for the frame size, the shard's work list, the filter's per-threshold `need`, the box NMS's template info,
the depth gate's table, the template renders, the estimation / search / verification settings, and a result block and
candidate list that grow and never shrink.  A missing invalidation shows only on a handle that has seen an earlier call,
so the program walks one handle through every such transition, and the GPU test holds each call to the oracle and to a
fresh handle that was given only the state the call depends on.

program(seed) is a list of steps, each a dict with "op" and its arguments:
  state changes  load_bank, select, set_boxes, set_template_depths, set_depth_gate, set_template_renders,
                 set_pose_estimation, set_pose_search, set_pose_verify
  calls          match_quantized, bind_run, shard_run, match_images, match_top, detect, detect_batch, track, track_batch
Every call step carries "state", a snapshot of everything a fresh handle needs to make the same call.  The spine of
transitions (frame sizes, thresholds, banks, pose state) is the same for every seed; the seed picks the frames, the
thresholds inside their bands, the class subset, the shard layouts, the search settings and extra calls between spine
steps.  Everything here is numpy: the CPU test checks the coverage without a GPU."""
import functools
import importlib

import numpy as np

import tight_frames as tf

synth = importlib.import_module("6dpose_b200.synth")
pose_refine = importlib.import_module("6dpose_b200.pose_refine")

T = [4, 4]
SLOTS = 4
SEEDS = (0, 1)
NEG = -1.0            # every coarse position passes and every candidate is kept
CAND_LIST = 4 << 20   # candidate-list entries allocated up front (LM_CAND_DEFAULT)
RESULT_BLOCK = 1 << 16  # records of the initial internal result block

# Frame sizes of the spine, in order.  At T = [4, 4]: 648 x 480 has 162 level-0 columns per row of cells, not a multiple
# of 4, so the refinement filter is off; 704 x 480 has 88 x 60 lowest-level positions, 6 rounds of 32 x 32 (above
# LM_MAX_ROUNDS = 5), so no bit-planes are built.
SIZES = [(640, 480), (320, 240), (640, 480), (512, 512), (648, 480), (704, 480), (640, 480)]
FILTER_OFF = (648, 480)
NO_BIT_PLANES = (704, 480)
POSE_SIZE = (640, 480)

# Banks: A (two classes) and B (three, a different template count), W (class 01: 2 x 300 features at level 0, above the
# filter's 511; class 02: 2 x 100), S (1000 small templates of 8 features: at a negative threshold a 640 x 480 frame
# passes 1000 x 4800 coarse candidates, beyond the candidate list).
BANKS = dict(
    A=[dict(n=40, nf=120, seed=7, classes=("01_template", "02_template"))],
    B=[dict(n=25, nf=100, seed=8, classes=("01_template", "02_template", "03_template"))],
    W=[dict(n=12, nf=300, seed=9, classes=("01_template",)), dict(n=20, nf=100, seed=10, classes=("02_template",))],
    S=[dict(n=1000, nf=8, seed=5, classes=("01_template",), size_range=((16, 24), (16, 24)))],
)


@functools.lru_cache(maxsize=None)
def bank(name):
    """TemplateBank of a bank name (the parts' classes merged, in class order)."""
    out = None
    for part in BANKS[name]:
        b = synth.synth_bank(part["n"], num_features=part["nf"], levels=len(T), seed=part["seed"], class_ids=part["classes"],
                             variants=35, **({"size_range": part["size_range"]} if "size_range" in part else {}))
        if out is None:
            out = b
        else:
            out.classes.update(b.classes)
    return out


@functools.lru_cache(maxsize=None)
def packed(name):
    b = bank(name)
    return b.pack(b.class_ids(), SLOTS)


def n_templates(name):
    return int(packed(name)["class_begin"][-1])


def n_classes(name):
    return len(packed(name)["class_begin"]) - 1


def filter_features(name):
    """Level-0 feature count of every template (what the filter's `need` is computed from)."""
    tm = packed(name)["tmeta"].reshape(-1, SLOTS, 4)
    return tm[:, 0, 3] + tm[:, 1, 3]


@functools.lru_cache(maxsize=None)
def quantized(W, H, seed, bank_name):
    """Quantized pyramid of a synthetic frame with templates of the bank planted (synth.synth_frame)."""
    q, _ = synth.synth_frame(W, H, levels=len(T), seed=seed, bank=bank(bank_name), plant=6, T=T)
    return q


@functools.lru_cache(maxsize=None)
def rgbd(W, H, seed):
    return synth.synth_rgbd(W, H, seed)


def scene_k(W, H):
    return np.array([[572.0, 0, W / 2], [0, 572.0, H / 2], [0, 0, 1]], np.float32)


BOX_SEED = 3


def boxes(name, seed):
    """Box sizes of every template of the bank, seeded: 4 to 60 pixels a side, so that templates matched at one corner
    have boxes of different sizes and the NMS keeps more of them than with the templates' own sizes."""
    return np.random.RandomState(seed).randint(4, 61, size=(n_templates(name), 2)).astype(np.int32)


def template_depths(name, lo, hi):
    """Training distance (mm) per template: evenly from lo to hi, every fifth template without one (NaN)."""
    z = np.linspace(lo, hi, n_templates(name)).astype(np.float32)
    z[::5] = np.nan
    return z


RENDER_BASE = dict(R=np.eye(3, dtype=np.float32), t=np.array([0.0, 0.0, 800.0], np.float32))


def renders(name, variant):
    """(depths, K, R, t) for every template of the bank: one render per variant, a box of model depth."""
    W, H = POSE_SIZE
    r = np.zeros((H, W), np.uint16)
    x0, y0, s = 260 + 20 * variant, 190 + 10 * variant, 80 + 16 * variant
    r[y0:y0 + s, x0:x0 + s] = 800 + 40 * variant
    G = n_templates(name)
    K = np.repeat(scene_k(W, H)[None], G, 0)
    R = np.repeat(RENDER_BASE["R"][None], G, 0)
    t = np.repeat(RENDER_BASE["t"][None], G, 0)
    t[:, 2] += np.arange(G) % 5
    return [r] * G, K, R, t


def track_objects(name, rng, n):
    """(class_index, template_id, T) starts near the renders' pose, some of them far off the frame."""
    cb = packed(name)["class_begin"]
    out = []
    for k in range(n):
        c = int(rng.integers(0, len(cb) - 1))
        tid = int(rng.integers(0, cb[c + 1] - cb[c]))
        dx, dy, dz = rng.uniform(-30, 30), rng.uniform(-30, 30), rng.uniform(-40, 40)
        if k % 4 == 3:
            dx += 2000.0  # outside the frame
        T_ = pose_refine.pose_to_transform(np.eye(3), [dx, dy, 800.0 + dz], RENDER_BASE["R"], RENDER_BASE["t"])
        out.append((c, tid, T_))
    return out


def ulp_pair(name, thr_near):
    """(lo, hi = nextafter(lo, +inf)): a threshold pair near thr_near where the filter's need differs for some template of
    the bank (tight_frames.need_of): lo = score(3k + nf, nf) for the template's nf."""
    nf = int(filter_features(name)[0])
    k = int(round((thr_near / 100.0 * 4 * nf - nf) / 3))
    lo = np.float32(tf.score(3 * k + nf, nf))
    return float(lo), float(tf.ulp_up(lo))


DEFAULT_STATE = dict(bank=None, sel=(None, 0, 1, 0), boxes=None, depths=None, gate=None, renders=None,
                     est="point_to_plane", search=(64, 40, 40.0, 30.0, 20.0, 0), verify=(False, 10.0))
ESTIMATIONS = ("point_to_plane", "point_to_point", "pso")


class Builder:
    """Appends steps and keeps the state snapshot and the frame size every call step carries."""

    def __init__(self, seed):
        self.rng = np.random.default_rng(seed)
        self.steps = []
        self.state = dict(DEFAULT_STATE)
        self.size = SIZES[0]
        self.fseed = 0
        self.last_change = None

    def change(self, op, **kw):
        s = dict(op=op, **kw)
        if op == "load_bank":
            # the bank takes boxes, distances, renders and the selection with it; settings stay
            self.state.update(bank=kw["bank"], sel=(None, 0, 1, 0), boxes=None, depths=None, renders=None)
        elif op == "select":
            self.state["sel"] = (kw["classes"], kw["shard"], kw["count"], kw["layout"])
        elif op == "set_boxes":
            self.state["boxes"] = kw["seed"]
        elif op == "set_template_depths":
            self.state["depths"] = kw["range"]
        elif op == "set_depth_gate":
            self.state["gate"] = kw["tolerance"]
        elif op == "set_template_renders":
            self.state["renders"] = kw["variant"]
        elif op == "set_pose_estimation":
            self.state["est"] = kw["estimation"]
        elif op == "set_pose_search":
            self.state["search"] = kw["search"]
        elif op == "set_pose_verify":
            self.state["verify"] = kw["verify"]
        self.steps.append(s)
        self.last_change = len(self.steps) - 1

    def call(self, op, thr=None, size=None, fseed=None, **kw):
        if size is not None:
            self.size = size
        if fseed is None:
            self.fseed += 1
            fseed = self.fseed
        s = dict(op=op, state=dict(self.state), size=self.size, fseed=int(fseed), last_change=self.last_change, **kw)
        if thr is not None:
            s["thr"] = float(thr)
        self.steps.append(s)

    def thr(self, lo, hi):
        return float(np.float32(self.rng.uniform(lo, hi)))

    def extra(self, n=1):
        """n seeded extra match calls at the current size and state, thresholds in the ordinary band."""
        for _ in range(n):
            op = ("match_quantized", "bind_run", "match_top")[int(self.rng.integers(0, 3))]
            self.call(op, self.thr(65.0, 90.0))


def program(seed):
    b = Builder(seed)
    rng = b.rng
    # ---- bank A, frame sizes and thresholds ----
    b.change("load_bank", bank="A")
    b.call("match_quantized", 85.0, size=SIZES[0])
    b.call("match_quantized", 80.0, fseed=b.fseed)        # descending, same frame
    b.call("match_quantized", 70.0, fseed=b.fseed)
    b.call("bind_run", 70.0, fseed=b.fseed)               # repeated
    b.call("match_quantized", 90.0, fseed=b.fseed)        # ascending
    lo, hi = ulp_pair("A", b.thr(72.0, 82.0))
    b.call("match_quantized", hi, fseed=b.fseed, ulp="hi")  # the ulp pair downward ...
    b.call("match_quantized", lo, fseed=b.fseed, ulp="lo")
    b.call("bind_run", hi, fseed=b.fseed, ulp="hi")         # ... and upward
    for size in SIZES[1:]:
        b.call(("match_quantized", "bind_run")[int(rng.integers(0, 2))], b.thr(70.0, 85.0), size=size)
        b.extra(1)
    b.call("match_quantized", 100.0)
    b.call("match_top", 100.0, fseed=b.fseed)
    b.call("match_quantized", NEG, grows="result")        # result block grows
    b.call("match_quantized", b.thr(70.0, 85.0))          # the next ordinary frame
    # ---- selection ----
    # class 02 alone, then every class with 02 first: both move the templates of the box NMS's table
    b.change("select", classes=(1,), shard=0, count=1, layout=0)
    b.call("match_quantized", b.thr(65.0, 80.0))
    b.call("match_top", b.thr(65.0, 80.0), fseed=b.fseed)
    b.change("select", classes=(1, 0), shard=0, count=1, layout=0)
    b.call(("match_top", "match_quantized")[int(rng.integers(0, 2))], b.thr(65.0, 80.0), fseed=b.fseed)
    b.call("match_top", b.thr(65.0, 80.0))
    b.change("select", classes=None, shard=0, count=1, layout=0)
    b.call("match_quantized", b.thr(65.0, 80.0), fseed=b.fseed)
    n = int(rng.integers(2, 4))
    for layout in ((0, 1) if rng.integers(0, 2) else (1, 0)):
        for i in range(n):
            b.change("select", classes=None, shard=i, count=n, layout=layout)
            if i == 0:
                b.call("shard_run", b.thr(65.0, 80.0))
            else:
                b.call("shard_run", b.steps[-2]["thr"], fseed=b.fseed)
        b.change("select", classes=None, shard=0, count=1, layout=0)
        b.call("match_top", b.thr(65.0, 80.0))
    # ---- boxes ----
    # every survivor of the box NMS (top_k 0), with and without boxes at one frame and threshold: the survivors differ
    # (tests/test_handle_program.py)
    b.change("set_boxes", seed=BOX_SEED)
    b.call("match_top", b.thr(60.0, 75.0), top_k=0)
    b.change("set_boxes", seed=None)
    b.call("match_top", b.steps[-2]["thr"], fseed=b.fseed, top_k=0)
    # ---- banks: S (candidate list grows), B (another template count), W (filter eligibility toggles), A again ----
    b.change("load_bank", bank="S")
    b.call("match_quantized", NEG, grows="candidates")
    b.call("match_quantized", b.thr(75.0, 90.0))
    b.change("load_bank", bank="B")
    b.call("match_quantized", b.thr(65.0, 80.0), other_bank="A")
    b.extra(1)
    b.change("load_bank", bank="W")
    b.call("match_quantized", b.thr(65.0, 80.0))
    b.change("select", classes=(1,), shard=0, count=1, layout=0)   # class 02 only: every template eligible
    b.call("match_quantized", b.thr(65.0, 80.0), fseed=b.fseed)
    b.change("select", classes=None, shard=0, count=1, layout=0)
    b.call("bind_run", b.thr(65.0, 80.0), fseed=b.fseed)
    b.change("load_bank", bank="A")
    b.call("match_quantized", b.thr(70.0, 85.0))
    b.change("set_boxes", seed=BOX_SEED)
    b.call("match_top", b.thr(60.0, 75.0), top_k=0)
    b.change("load_bank", bank="A")                       # the same bank again: the boxes are gone
    b.call("match_top", b.steps[-2]["thr"], fseed=b.fseed, top_k=0)
    # ---- front-end ----
    for size in ((640, 480), (320, 240), (640, 480)):
        b.call("match_images", b.thr(55.0, 70.0), size=size)
    # ---- depth gate ----
    b.change("set_template_depths", range=(900.0, 1600.0))
    tol = [0.1, 0.3] if rng.integers(0, 2) else [0.3, 0.1]
    b.change("set_depth_gate", tolerance=tol[0])
    b.call("match_images", b.thr(40.0, 48.0))           # low enough that every gate change moves the passing candidates
    b.change("set_depth_gate", tolerance=tol[1])
    b.call("match_images", b.steps[-2]["thr"], fseed=b.fseed)
    b.change("set_template_depths", range=(600.0, 1300.0))
    b.call("match_images", b.steps[-2]["thr"], fseed=b.fseed)
    # ---- pose stage ----
    b.call("detect", b.thr(55.0, 65.0))                    # gated, no renders yet
    b.change("set_template_renders", variant=0)
    b.call("detect", b.steps[-2]["thr"], fseed=b.fseed)
    b.change("set_depth_gate", tolerance=None)
    b.call("detect", b.thr(55.0, 65.0))
    b.change("set_pose_verify", verify=(True, float(rng.choice([8.0, 12.0]))))
    b.call("detect", b.thr(55.0, 65.0), fseed=b.fseed)
    b.call("track", objects=track_objects("A", rng, 5))
    b.change("set_pose_estimation", estimation="point_to_point")
    b.call("detect_batch", b.thr(55.0, 65.0), frames=3)
    b.call("track_batch", objects=[track_objects("A", rng, 3) for _ in range(2)])
    b.change("set_pose_verify", verify=(True, 20.0))
    b.call("track", objects=track_objects("A", rng, 4))
    b.change("set_pose_estimation", estimation="pso")
    parts = int(rng.choice([16, 32]))
    b.change("set_pose_search", search=(parts, 12, 40.0, 30.0, 20.0, int(rng.integers(0, 100))))
    b.call("detect", b.thr(55.0, 65.0))
    b.change("set_pose_search", search=(parts, 16, 40.0, 30.0, 20.0, int(rng.integers(100, 200))))
    b.call("detect", b.steps[-2]["thr"], fseed=b.fseed)
    b.change("set_pose_verify", verify=(False, 10.0))
    b.change("set_pose_estimation", estimation="point_to_plane")
    b.call("track_batch", objects=[track_objects("A", rng, 2) for _ in range(3)])
    b.change("load_bank", bank="B")                       # renders of A are gone: "no renders"
    b.call("detect", b.thr(55.0, 65.0))
    b.change("set_template_renders", variant=1)
    b.call("detect", b.steps[-2]["thr"], fseed=b.fseed)
    b.change("load_bank", bank="A")
    b.call("detect", b.thr(55.0, 65.0))                   # "no renders" again
    b.change("set_template_renders", variant=2)
    b.call("detect", b.steps[-2]["thr"], fseed=b.fseed)
    b.call("match_quantized", b.thr(70.0, 85.0))
    return b.steps


def is_call(step):
    return "state" in step


TRANSITIONS = ("size", "threshold_down", "threshold_up", "threshold_repeat", "ulp_down", "ulp_up", "threshold_100",
               "threshold_negative_result", "threshold_negative_candidates", "after_growth", "filter_off", "no_bit_planes",
               "bank_count", "bank_wide", "bank_first_again", "select_subset", "select_all", "select_shard_contiguous",
               "select_shard_interleaved", "boxes", "boxes_none", "gate_tolerance", "gate_off", "template_depths",
               "renders_none", "renders_changed", "estimation", "search", "verify")


def transitions(steps):
    """How many times each transition of TRANSITIONS occurs between consecutive calls (and their state)."""
    out = dict.fromkeys(TRANSITIONS, 0)
    prev = None
    grown = False
    for s in steps:
        if not is_call(s):
            continue
        st = s["state"]
        if s.get("grows"):
            out["threshold_negative_" + s["grows"]] += 1
            grown = True
        elif grown and s["op"] != "shard_run":
            out["after_growth"] += 1
            grown = False
        if tuple(s["size"]) == FILTER_OFF:
            out["filter_off"] += 1
        if tuple(s["size"]) == NO_BIT_PLANES:
            out["no_bit_planes"] += 1
        if s.get("thr") == 100.0:
            out["threshold_100"] += 1
        if prev is not None:
            ps = prev["state"]
            if tuple(s["size"]) != tuple(prev["size"]):
                out["size"] += 1
            if "thr" in s and "thr" in prev and s["state"]["bank"] == ps["bank"]:
                d = np.float32(s["thr"]) - np.float32(prev["thr"])
                key = "threshold_down" if d < 0 else "threshold_up" if d > 0 else "threshold_repeat"
                out[key] += 1
                if s.get("ulp") and prev.get("ulp") and s["ulp"] != prev["ulp"]:
                    out["ulp_down" if d < 0 else "ulp_up"] += 1
            if st["bank"] != ps["bank"]:
                out["bank_count"] += n_templates(st["bank"]) != n_templates(ps["bank"])
                out["bank_wide"] += st["bank"] == "W"
                out["bank_first_again"] += st["bank"] == "A"
            elif s["last_change"] != prev["last_change"] and steps[s["last_change"]]["op"] == "load_bank":
                out["bank_first_again"] += st["bank"] == "A"
            if st["sel"] != ps["sel"]:
                cls, i, n, layout = st["sel"]
                if n > 1:
                    out["select_shard_interleaved" if layout else "select_shard_contiguous"] += 1
                elif cls is not None:
                    out["select_subset"] += 1
                else:
                    out["select_all"] += 1
            if st["boxes"] != ps["boxes"] and st["bank"] == ps["bank"]:
                out["boxes" if st["boxes"] else "boxes_none"] += 1
            if st["gate"] != ps["gate"]:
                out["gate_tolerance" if st["gate"] is not None and ps["gate"] is not None else "gate_off"] += 1
            if st["depths"] != ps["depths"] and st["depths"] is not None and ps["depths"] is not None:
                out["template_depths"] += 1
            if st["renders"] != ps["renders"]:
                out["renders_none" if st["renders"] is None else "renders_changed"] += 1
            for key in ("est", "search", "verify"):
                if st[key] != ps[key]:
                    out[dict(est="estimation").get(key, key)] += 1
        prev = s
    return out
