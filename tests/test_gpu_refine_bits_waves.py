"""k_refine_bits at survivor counts on both sides of each of its launch decisions: 0 and 1 survivor, one under and one over
every team-size boundary (a team of 8, 4, 2 or 1 warps per survivor, the largest that gives every survivor a team of the
resident CTAs in one round), and several rounds of single-warp teams.  Each count is held to the oracle (match list,
kept records, counters) and to lm_debug_plan, with K1 in planes mode (H-planes from K1, N-planes derived from them by
k_refine_prep) and without it (a bank with one unsafe template: both planes from the byte linear memories).

The counts are built exactly: the lowest level of the frame is dark except one lit pixel (every label bit) per chosen
cell, and every template's lowest-level features sit at (0, 0), so a template has one coarse candidate per lit cell of
its position range.  Level 0 is the uniform frame of tests/tight_frames.py and the templates are staircase templates:
every candidate survives the filter at need = k, none at need = k + 1."""
import os

import numpy as np
import pytest

import tight_frames as tf
from test_gpu_match_parity import _assert_same, _native

pytestmark = pytest.mark.gpu

THREADS = os.cpu_count() or 1
T = [4, 8]
W, H = 320, 256
NF, K = 150, 100                # five 32-feature steps per survivor
POSITIONS = 257                 # template positions of a 64 x 64 template at the lowest level of 320 x 256 (T = 8)


def _frame(n_lit):
    q = tf.uniform_frame(W, H, 2)
    Tl = T[-1]
    Wl = (W >> 1) // Tl
    for m in range(2):
        low = np.zeros_like(q[1][m])
        for j in range(n_lit):
            low[(j // Wl) * Tl, (j % Wl) * Tl] = 0xFF
        q[1][m] = low
    return q


def _bank(n_templates, unsafe):
    tps = []
    for g in range(n_templates + (1 if unsafe else 0)):
        tp = tf.staircase_template(NF, K, seed=300 + g)
        for m in (2, 3):
            tp[m].features[:, :2] = 0
        tps.append(tp)
    if unsafe:
        tf.make_unsafe(tps[-1])
    return tf.make_bank(tps)


def _run(oracle, n_templates, n_lit, unsafe, drop=False):
    """One frame; returns (plan, number of survivors the model expects)."""
    bank = _bank(n_templates, unsafe)
    q = _frame(n_lit)
    thr = tf.score(3 * K + NF, NF)
    if drop:
        thr = tf.ulp_up(thr)
    nat, packed = _native(T, bank)
    mdl = tf.Model(oracle, q, T, packed)
    surv = 0
    for g in range(mdl.G):
        if mdl.eligible(g):
            d = mdl.decisions(g, thr)
            surv += int((d["max_ch"] >= d["need"]).sum()) if d["need"] <= mdl.t[g]["nf"] else 0
    assert [g for g in range(mdl.G) if not mdl.eligible(g)] == ([mdl.G - 1] if unsafe else [])
    want, st = oracle.match(q, T, packed, thr, n_threads=THREADS, want_stats=True)
    got = nat.match_quantized(q, thr)
    _assert_same(got, want)
    c = nat.counters()
    assert c["coarse_candidates"] == int(st["coarse_candidates"])
    assert c["scan_bytes"] == int(st["coarse_byte_adds"])
    assert c["refine_bytes"] == int(st["refine_byte_adds"])
    assert c["kept"] == int(st["pre_unique"])
    assert c["filter_dropped_bytes"] == mdl.dropped_bytes(thr)
    plan = nat.plan()
    nat.close()
    assert plan["use_bits"] == 1 and plan["planes_level"] == (-1 if unsafe else 0), plan
    assert plan["filter_items"] == c["coarse_candidates"]
    assert plan["refine_bits_items"] == surv, (plan, surv)
    assert plan["refine_bits_ctas"] > 0
    return plan, surv


_GRID = {}


def _grid(oracle):
    """CTAs of k_refine_bits on this device (the resident ones), from a one-survivor frame."""
    if "ctas" not in _GRID:
        plan, surv = _run(oracle, 1, 1, False)
        assert surv == 1
        _GRID["ctas"] = plan["refine_bits_ctas"]
    return _GRID["ctas"]


def _shape(n, step):
    """(templates, lit cells per template, count): the count nearest n in the direction of step (-1 or 1) that a few
    more templates than n / 257 build exactly."""
    while True:
        g0 = max(1, -(-n // POSITIONS))
        for g in range(g0, g0 + 8):
            if n % g == 0 and n // g <= POSITIONS:
                return g, n // g, n
        n += step


CASES = ["zero", "one"] + ["%s_%d" % (side, ts) for ts in (8, 4, 2, 1) for side in ("under", "over")] + ["rounds"]


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("unsafe", [False, True], ids=["k1_planes", "prep_planes"])
def test_survivor_counts_around_team_and_wave_boundaries(oracle, case, unsafe):
    warps = 8 * _grid(oracle)
    if case == "zero":
        _, surv = _run(oracle, 2, 40, unsafe, drop=True)
        assert surv == 0
        return
    if case == "one":
        target = 1
    elif case == "rounds":
        target = 3 * warps + 1
    else:
        side, ts = case.split("_")
        bound = warps // int(ts)   # largest count a team of ts warps per survivor takes in one round
        target = bound if side == "under" else bound + 1
    step = -1 if case.startswith("under") else 1
    g, lit, n = _shape(target, step)
    _, surv = _run(oracle, g, lit, unsafe)
    assert surv == n
    if case.startswith("under"):   # inside the band of this team size
        ts = int(case.split("_")[1])
        assert n <= warps // ts and (ts == 8 or n > warps // (2 * ts)), (n, warps)
    elif case.startswith("over"):
        assert n > warps // int(case.split("_")[1]), (n, warps)
    elif case == "rounds":
        assert n > 3 * warps
