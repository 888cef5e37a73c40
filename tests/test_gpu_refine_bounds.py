"""The refinement filter and the best-cell arg-max on frames that put them exactly on their bounds (tests/tight_frames.py):
the C-ABI result equals the oracle's, and the filter's counter equals the numpy model's.

A filter that is too strict drops a candidate the reference keeps (the result changes); one that is too loose passes a
candidate it could have dropped (filter_dropped_bytes changes).  Every case runs under the default path and the
switchable ones; the switches are read when the handle is created."""
import os

import pytest

import tight_frames as tf
from test_gpu_match_parity import _assert_same, _native

pytestmark = pytest.mark.gpu

ENVS = [
    {},                                       # k_refine_filter_w + k_refine_bits (two levels) / k_refine (three)
    {"LINEMOD_B200_FILTER_VARIANT": "1"},     # 8-lane filter, survivors refined byte-wise
    {"LINEMOD_B200_BITS_EXACT": "0"},         # warp filter, survivors refined byte-wise
    {"LINEMOD_B200_FILTER": "0"},             # no filter: k_refine's row-wise early exit on every candidate
]
ENV_IDS = ["default", "filter8", "bytes_exact", "no_filter"]

THREADS = os.cpu_count() or 1
_ORACLE = {}


def _want(oracle, key, q, T, packed, thr):
    """The oracle's result and stats, once per process: they do not depend on the kernel path."""
    k = key + (float(thr),)
    if k not in _ORACLE:
        _ORACLE[k] = oracle.match(q, T, packed, thr, n_threads=THREADS, want_stats=True)
    return _ORACLE[k]


def _check(nat, q, thr, want, st, dropped, env):
    got = nat.match_quantized(q, thr)
    _assert_same(got, want)
    c = nat.counters()
    assert c["coarse_candidates"] == int(st["coarse_candidates"])
    assert c["scan_bytes"] == int(st["coarse_byte_adds"])
    assert c["refine_bytes"] == int(st["refine_byte_adds"])
    assert c["kept"] == int(st["pre_unique"])
    assert c["filter_dropped_bytes"] == (0 if env.get("LINEMOD_B200_FILTER") == "0" else dropped), thr


def _setenv(monkeypatch, env):
    for k, v in env.items():
        monkeypatch.setenv(k, v)


@pytest.mark.parametrize("env", ENVS, ids=ENV_IDS)
@pytest.mark.parametrize("T,W,H,pct", [
    ([4, 8], 640, 480, (50, 90, 99)),
    ([4, 8], 640, 512, (90,)),
    ([4, 8], 640, 464, (90,)),       # Hd = 116: the last row block of the H-planes is partial
    ([5, 8], 640, 480, (90,)),       # T not a power of two
    ([2, 4, 8], 640, 480, (50,)),    # filtered level 1, then level 0 byte-wise
])
def test_mosaic_frames_at_tight_thresholds(oracle, monkeypatch, env, T, W, H, pct):
    """Thresholds at similarities the frame attains (raw_keep = 3 * need + nf) and one ulp above them: hundreds of kept
    candidates have no filter slack at all."""
    _setenv(monkeypatch, env)
    s = tf.mosaic_setup(oracle, T, W, H, percentiles=pct, n_threads=THREADS)
    nat, packed = _native(T, s["bank"])
    for thr in s["thresholds"]:
        for t in (thr, tf.ulp_up(thr)):
            want, st = _want(oracle, ("mosaic", tuple(T), W, H), s["q"], T, packed, t)
            assert len(want) > 0
            _check(nat, s["q"], t, want, st, s["model"].dropped_bytes(t), env)
    nat.close()


@pytest.mark.parametrize("env", ENVS, ids=ENV_IDS)
def test_staircase_templates_tie_every_cell(oracle, monkeypatch, env):
    """Every cell of every patch scores 3k + nf: the arg-max must return the first cell, and the filter's running bound
    holds with equality at every check point.  need = k keeps every candidate, need = k + 1 none; 12 feature counts from
    33 to 511 (CH = 511 and raw = 2044 in the last) and a 512-feature template on the byte-wise path next to it."""
    _setenv(monkeypatch, env)
    T = [4, 8]
    q = tf.uniform_frame(640, 480, 2)
    cases = {}
    for nf, k, thr, need in tf.stair_cases():
        cases.setdefault((nf, k), []).append((thr, need))
    for (nf, k), thrs in cases.items():
        bank = tf.stair_bank(nf, k)
        nat, packed = _native(T, bank)
        mdl = None
        for thr, need in thrs:
            want, st = _want(oracle, ("stair", nf, k), q, T, packed, thr)
            n0 = int((want["template_id"] == 0).sum())
            assert (n0 > 0) == (need == k), (nf, k, need)
            dropped = 0
            if need > k:
                mdl = mdl or tf.Model(oracle, q, T, packed)
                dropped = mdl.dropped_bytes(thr)
                assert dropped == 256 * nf * len(mdl.candidates(0, thr)) > 0
            _check(nat, q, thr, want, st, dropped, env)
        nat.close()


@pytest.mark.parametrize("env,unsafe", [({}, False), ({"LINEMOD_B200_BITS_EXACT": "0"}, False), ({}, True),
                                        ({"LINEMOD_B200_FILTER": "0"}, False)],
                         ids=["bits", "bytes_exact", "unsafe_template", "no_filter"])
@pytest.mark.parametrize("thr", [0.0, -1.0])
def test_zero_score_patches(oracle, monkeypatch, env, unsafe, thr):
    """Candidates whose patch scores 0 at every cell are kept at thresholds <= 0 with the best cell at (-1, -1): the
    bit-sliced arg-max (k_refine_bits), the byte-wise one (k_refine) and a bank with an unsafe template (byte-wise next
    to bit-sliced) all place them at (x / T - 9) * T + offset."""
    _setenv(monkeypatch, env)
    T, bank, q, _ = tf.zero_case(unsafe)
    nat, packed = _native(T, bank)
    want, st = oracle.match(q, T, packed, thr, want_stats=True)
    assert int((want["similarity"] == 0).sum()) >= 50
    if unsafe:  # before std::unique, which merges equal (x, y, similarity) records of different templates
        pre = oracle.match(q, T, packed, thr, presort=True)
        assert int(((pre["similarity"] == 0) & (pre["template_id"] == 1)).sum()) > 0
    _check(nat, q, thr, want, st, 0, env)
    nat.close()
