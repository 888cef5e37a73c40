"""The refinement filter and the best-cell arg-max on frames that put them exactly on their bounds (tests/tight_frames.py):
the C-ABI result equals the oracle's, and the filter's counter equals the numpy model's.

A filter that is too strict drops a candidate the reference keeps (the result changes); one that is too loose passes a
candidate it could have dropped (filter_dropped_bytes changes).  Every refinement route meets these frames through the
input that selects it: the filter in front of k_refine_bits (two levels) or k_refine<true> (three), banks with "unsafe"
templates (the filter hands their candidates to k_refine<true>), and frames the filter does not take (the filtered
level's Wd is not a multiple of 4, or it has more than 512 cell rows), where k_refine<false> refines every candidate."""
import os

import pytest

import tight_frames as tf
from test_gpu_match_parity import _assert_same, _native

pytestmark = pytest.mark.gpu

THREADS = os.cpu_count() or 1
_ORACLE = {}


def _want(oracle, key, q, T, packed, thr):
    """The oracle's result and stats, once per process."""
    k = key + (float(thr),)
    if k not in _ORACLE:
        _ORACLE[k] = oracle.match(q, T, packed, thr, n_threads=THREADS, want_stats=True)
    return _ORACLE[k]


def _check(nat, q, thr, want, st, mdl, dropped):
    got = nat.match_quantized(q, thr)
    _assert_same(got, want)
    c = nat.counters()
    assert c["coarse_candidates"] == int(st["coarse_candidates"])
    assert c["scan_bytes"] == int(st["coarse_byte_adds"])
    assert c["refine_bytes"] == int(st["refine_byte_adds"])
    assert c["kept"] == int(st["pre_unique"])
    assert c["filter_dropped_bytes"] == dropped, thr
    # the route: only the filter reads H-planes, only the byte-wise k_refine reads byte linear memories.  Two levels
    # refine the filter's eligible templates bit-sliced and the others byte-wise; deeper pyramids refine every survivor
    # byte-wise.
    if not mdl.filter_ok():
        assert c["filter_bytes_read"] == 0
    bytewise = [g for g in range(mdl.G) if mdl.L > 2 or not mdl.eligible(g)]
    assert (c["refine_bytes_read"] > 0) == any(len(mdl.candidates(g, thr)) > 0 for g in bytewise), thr


def _unsafe_templates(mdl):
    return [g for g in range(mdl.G) if not mdl.t[g]["safe"]]


@pytest.mark.parametrize("unsafe", [False, True], ids=["default", "unsafe"])
@pytest.mark.parametrize("T,W,H,pct", [
    ([4, 8], 640, 480, (50, 90, 99)),
    ([4, 8], 640, 512, (90,)),
    ([4, 8], 640, 464, (90,)),       # Hd = 116: the last row block of the H-planes is partial
    ([5, 8], 640, 480, (90,)),       # T not a power of two
    ([2, 4, 8], 640, 480, (50,)),    # filtered level 1, then level 0 byte-wise
    ([4, 4], 648, 480, (50, 90, 99)),  # Wd = 162 at level 0: no filter, k_refine<false> feature by feature
    ([4, 8], 640, 2064, (90,)),      # Hd = 516 at level 0: no filter, k_refine<false> with its row-wise early exit
])
def test_mosaic_frames_at_tight_thresholds(oracle, T, W, H, pct, unsafe):
    """Thresholds at similarities the frame attains (raw_keep = 3 * need + nf) and one ulp above them: hundreds of kept
    candidates have no filter slack at all.  unsafe: every third template has a feature outside its box, and at least
    one of them has a coarse candidate."""
    s = tf.mosaic_setup(oracle, T, W, H, percentiles=pct, n_threads=THREADS, unsafe=unsafe)
    nat, packed = _native(T, s["bank"])
    mdl = s["model"]
    for thr in s["thresholds"]:
        for t in (thr, tf.ulp_up(thr)):
            want, st = _want(oracle, ("mosaic", tuple(T), W, H, unsafe), s["q"], T, packed, t)
            assert len(want) > 0
            if unsafe:
                assert any(len(mdl.candidates(g, t)) > 0 for g in _unsafe_templates(mdl))
            _check(nat, s["q"], t, want, st, mdl, mdl.dropped_bytes(t))
    nat.close()


@pytest.mark.parametrize("T,W,H,unsafe", [
    ([4, 8], 640, 480, False),
    ([4, 8], 640, 480, True),     # an unsafe copy of the template next to it
    ([4, 4], 648, 480, False),    # Wd = 162 at level 0: no filter
    ([4, 8], 640, 2064, False),   # Hd = 516 at level 0: no filter, k_refine<false> with its row-wise early exit
], ids=["default", "unsafe", "no_filter_t44", "no_filter_tall"])
def test_staircase_templates_tie_every_cell(oracle, T, W, H, unsafe):
    """Every cell of every patch scores 3k + nf: the arg-max must return the first cell, and the filter's running bound
    holds with equality at every check point.  need = k keeps every candidate, need = k + 1 none; 12 feature counts from
    33 to 511 (CH = 511 and raw = 2044 in the last) and a 512-feature template on the byte-wise path next to it."""
    q = tf.uniform_frame(W, H, 2)
    cases = {}
    for nf, k, thr, need in tf.stair_cases():
        cases.setdefault((nf, k), []).append((thr, need))
    for (nf, k), thrs in cases.items():
        bank = tf.stair_bank(nf, k, unsafe)
        nat, packed = _native(T, bank)
        mdl = tf.Model(oracle, q, T, packed)
        assert _unsafe_templates(mdl) == ([mdl.G - 1] if unsafe else [])
        for thr, need in thrs:
            want, st = _want(oracle, ("stair", nf, k, tuple(T), W, H, unsafe), q, T, packed, thr)
            n0 = int((want["template_id"] == 0).sum())
            assert (n0 > 0) == (need == k), (nf, k, need)
            if unsafe:
                assert len(mdl.candidates(mdl.G - 1, thr)) > 0
            dropped = 0
            if need > k:
                dropped = mdl.dropped_bytes(thr)
                if mdl.filter_ok():
                    assert dropped == 256 * nf * len(mdl.candidates(0, thr)) > 0
            _check(nat, q, thr, want, st, mdl, dropped)
        nat.close()


ZERO_CASES = {
    "bits": ([4, 8], 320, 256, False),
    "unsafe_template": ([4, 8], 320, 256, True),
    "no_filter_t44": ([4, 4], 328, 256, False),     # Wd = 82 at level 0
    "no_filter_tall": ([4, 8], 320, 2064, False),   # Hd = 516 at level 0
}


@pytest.mark.parametrize("case", list(ZERO_CASES))
@pytest.mark.parametrize("thr", [0.0, -1.0])
def test_zero_score_patches(oracle, case, thr):
    """Candidates whose patch scores 0 at every cell are kept at thresholds <= 0 with the best cell at (-1, -1): the
    bit-sliced arg-max (k_refine_bits), the byte-wise one (k_refine) and a bank with an unsafe template (byte-wise next
    to bit-sliced) all place them at (x / T - 9) * T + offset."""
    T, W, H, unsafe = ZERO_CASES[case]
    T, bank, q, _ = tf.zero_case(unsafe, T, W, H)
    nat, packed = _native(T, bank)
    mdl = tf.Model(oracle, q, T, packed)
    want, st = oracle.match(q, T, packed, thr, want_stats=True)
    assert int((want["similarity"] == 0).sum()) >= 50
    if unsafe:  # before std::unique, which merges equal (x, y, similarity) records of different templates
        pre = oracle.match(q, T, packed, thr, presort=True)
        assert int(((pre["similarity"] == 0) & (pre["template_id"] == 1)).sum()) > 0
    _check(nat, q, thr, want, st, mdl, 0)
    nat.close()
