"""The paired refinement filter (k_refine_filter_w: two candidates per warp) against its lane-level model
(tests/filter_pair_model.py): records equal to the oracle's, and exactly the model's filter_bytes_read,
filter_dropped_bytes, kept count and lm_debug_plan entries 16-18.  The list the model pairs is checked against the
device's (lm_debug_coarse pass masks, in shard order).

A filter that is too loose changes nothing but counters; the plane words it reads depend on each candidate alone (its
check schedule and which patch columns are still alive), so any pairing slip -- a survivor restarted, handed on uncounted
or counted with its partner's columns -- changes filter_bytes_read.  Frames: the pair-coverage frames (every kind of
pair), every tight_frames setup the filter runs on, the reference's 2989-template bank on its fixture frame, and the
peer exchange at worlds 2 and 3, where each rank filters its own shard."""
import importlib
import os

import numpy as np
import pytest

import filter_pair_model as fpm
import tight_frames as tf
from test_gpu_match_parity import _assert_same, _native

pytestmark = pytest.mark.gpu

THREADS = os.cpu_count() or 1


def _expect(nat, fm):
    """The filter's counters and plan entries and the device's candidate list equal the model's."""
    c = nat.counters()
    assert c["filter_bytes_read"] == fm.bytes_read()
    assert c["filter_dropped_bytes"] == fm.dropped_bytes()
    p = nat.plan()
    assert [p["filter_items"], p["refine_bits_items"], p["refine_filtered_items"]] == fm.plan(), (p, fm.plan())
    mask, _ = nat.coarse()
    w, j = fpm.device_list(mask)
    assert len(w) == fm.n and np.array_equal(w, fm.c["item"]) and np.array_equal(j, fm.c["cell"])
    return c


def _run(nat, oracle, q, T, packed, thr, mdl):
    got = nat.match_quantized(q, thr)
    want, st = oracle.match(q, T, packed, thr, n_threads=THREADS, want_stats=True)
    _assert_same(got, want)
    fm = fpm.FilterModel(mdl, thr)
    c = _expect(nat, fm)
    assert c["kept"] == int(st["pre_unique"])
    return fm


@pytest.fixture(scope="module")
def coverage(oracle):
    return fpm.coverage_cases(oracle)


@pytest.mark.parametrize("case", ["pairs", "sparse_empty", "sparse_one", "sparse_two", "sparse_three", "sparse_long_short",
                                  "zero", "zero_unsafe"])
def test_pair_coverage_frames(oracle, coverage, case):
    c = coverage[case]
    nat, packed = _native(fpm.PAIR_T, c["bank"])
    mdl = tf.Model(oracle, c["q"], fpm.PAIR_T, packed)
    for thr in c["thresholds"]:
        _run(nat, oracle, c["q"], fpm.PAIR_T, packed, thr, mdl)
    nat.close()


@pytest.mark.parametrize("unsafe", [False, True], ids=["default", "unsafe"])
@pytest.mark.parametrize("T,W,H,pct", [
    ([4, 8], 640, 480, (50, 90, 99)),
    ([4, 8], 640, 464, (90,)),       # Hd = 116: the last row block of the H-planes is partial
    ([5, 8], 640, 480, (90,)),
    ([2, 4, 8], 640, 480, (50,)),    # the filter in front of k_refine<true>
])
def test_mosaic_frames(oracle, T, W, H, pct, unsafe):
    s = tf.mosaic_setup(oracle, T, W, H, percentiles=pct, n_threads=THREADS, unsafe=unsafe)
    nat, packed = _native(T, s["bank"])
    for thr in s["thresholds"]:
        for t in (thr, tf.ulp_up(thr)):
            assert _run(nat, oracle, s["q"], T, packed, t, s["model"]).dropped_bytes() > 0
    nat.close()


def test_staircase_templates(oracle):
    """Every cell ties and the running bound holds with equality at every check: 12 feature counts from 33 to 511."""
    T = [4, 8]
    q = tf.uniform_frame(640, 480, 2)
    cases = {}
    for nf, k, thr, need in tf.stair_cases():
        cases.setdefault((nf, k), []).append(thr)
    for (nf, k), thrs in cases.items():
        bank = tf.stair_bank(nf, k)
        nat, packed = _native(T, bank)
        mdl = tf.Model(oracle, q, T, packed)
        for thr in thrs:
            _run(nat, oracle, q, T, packed, thr, mdl)
        nat.close()


def test_reference_bank_on_its_fixture_frame(oracle):
    """All 2989 templates of the reference's allScales bank (T = {5, 8}) on the full fixture frame at 80 and 75 (61 912
    coarse candidates): tens of thousands of pairs of real templates."""
    from test_golden_and_ref import load_allscales_full, load_golden
    lib = importlib.import_module("6dpose_b200._lib")
    frames, _, _ = load_golden()
    packed, T, cases = load_allscales_full()
    q = frames["full"]
    mdl = tf.Model(oracle, q, T, packed)
    nat = lib.NativeDetector(T)
    nat.load_bank(packed, 4)
    ran = 0
    for tag, thr, want, stats in cases:
        if tag != "full":
            continue
        got = nat.match_quantized(q, thr)
        assert len(got) == len(want)
        for k in ("x", "y", "template_id", "similarity"):
            assert np.array_equal(got[k], want[k]), (thr, k)
        fm = fpm.FilterModel(mdl, thr)
        assert fm.n == int(stats[0])
        _expect(nat, fm)
        ran += 1
    assert ran == 2
    nat.close()


def _peer_case(oracle, name):
    if name == "pairs":
        c = fpm.coverage_cases(oracle)["pairs"]
        return fpm.PAIR_T, c["bank"], c["q"], c["thresholds"][2:]
    s = tf.mosaic_setup(oracle, [4, 8], 640, 480, n_threads=THREADS, unsafe=True)
    return [4, 8], s["bank"], s["q"], s["thresholds"]


@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("name", ["pairs", "mosaic_unsafe"])
def test_peer_exchange_shards(oracle, world, name):
    """Handles over contiguous shards of one device, connected by the fused record exchange: every rank's filter counters
    and plan entries 16-18 cover its own shard (lm_counters' filter entries come from the rank's own device counters, the
    plan's from its own list and queue) and equal the model of that shard; they add up to the unsharded model.  Every
    rank's records equal the unsharded handle's."""
    lib = importlib.import_module("6dpose_b200._lib")
    T, bank, q, thrs = _peer_case(oracle, name)
    single, packed = _native(T, bank)
    mdl = tf.Model(oracle, q, T, packed)
    dets = []
    for r in range(world):
        d = lib.NativeDetector(T, 0)
        d.load_bank(packed, len(T) * 2)
        d.select(None, r, world)
        d.peer_export(world, 1 << 15)
        dets.append(d)
    bases = [d.peer_base() for d in dets]
    for r, d in enumerate(dets):
        d.peer_connect_local(r, world, bases)
    try:
        items = []
        for d in dets:
            b, n = d.shard_range()
            items.append(list(range(b, b + n)))
        assert sum(items, []) == list(range(mdl.G))
        for thr in thrs:
            single.upload_quantized(q)
            single.run(thr)
            want = single.fetch_records()
            whole = fpm.FilterModel(mdl, thr)
            _expect(single, whole)
            for d in dets:
                d.upload_quantized(q)
            for d in dets:
                d.enqueue(thr)
            for d in dets:
                d.complete()
            parts = [fpm.FilterModel(mdl, thr, it) for it in items]
            for d, fm in zip(dets, parts):
                got = d.fetch_records()
                for f in ("x", "y", "similarity", "work"):
                    assert np.array_equal(got[f], want[f]), f
                _expect(d, fm)
            assert sum(fm.bytes_read() for fm in parts) == whole.bytes_read()
            assert sum(fm.dropped_bytes() for fm in parts) == whole.dropped_bytes()
            assert sum(fm.plan()[0] for fm in parts) == whole.n
    finally:
        for d in dets:
            d.peer_disconnect()
        for d in dets:
            d.close()
        single.close()
