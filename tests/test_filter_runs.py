"""tools/filter_runs.py: the run-length count behind the refinement filter's decision not to share loads between
x-neighbouring candidates.  Its run-cutting rule against a vectorised numpy restatement, and its coarse pass masks
against the oracle's own candidate count."""
import importlib
import importlib.util
import os

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def fr():
    spec = importlib.util.spec_from_file_location("filter_runs", os.path.join(ROOT, "tools", "filter_runs.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def runs_numpy(mask, Wd, cap):
    """Runs of consecutive set cells, cut at row starts and every `cap` cells: (first candidate index, length)."""
    cells = np.flatnonzero(np.asarray(mask).ravel())
    if cells.size == 0:
        return np.zeros(0, np.int64), np.zeros(0, np.int64)
    cont = np.zeros(cells.size, bool)
    cont[1:] = (np.diff(cells) == 1) & (cells[1:] % Wd != 0)
    start = np.flatnonzero(~cont)                                   # maximal runs
    run_of = np.cumsum(~cont) - 1
    pos = np.arange(cells.size) - start[run_of]                     # position inside the maximal run
    firsts = np.flatnonzero(pos % cap == 0)
    lens = np.diff(np.append(firsts, cells.size))
    return firsts.astype(np.int64), lens.astype(np.int64)


def test_cut_runs_cases(fr):
    Wd = 8
    m = np.zeros((3, Wd), bool)
    m[0, 6:8] = True   # ends a row ...
    m[1, 0:7] = True   # ... and the next row starts with 7 cells: cut at the row start, then after 5
    m[2, 3] = True
    f, n = fr.cut_runs(m, Wd)
    assert n.tolist() == [2, 5, 2, 1]
    assert f.tolist() == [0, 2, 7, 9]
    f, n = fr.cut_runs(np.zeros((2, Wd), bool), Wd)
    assert f.size == 0 and n.size == 0


@pytest.mark.parametrize("Wd", [1, 5, 40, 37])
def test_cut_runs_matches_numpy(fr, Wd):
    rng = np.random.default_rng(Wd)
    for density in (0.05, 0.4, 0.8, 1.0):
        m = rng.random((11, Wd)) < density
        f, n = fr.cut_runs(m, Wd)
        g, k = runs_numpy(m, Wd, fr.RUN_CAP)
        assert f.tolist() == g.tolist() and n.tolist() == k.tolist(), density
        assert int(n.sum()) == int(m.sum()) and int(n.max(initial=1)) <= fr.RUN_CAP


def test_pass_masks_count_the_oracles_candidates(fr):
    from oracle import oracle
    synth = importlib.import_module("6dpose_b200.synth")
    T = [4, 8]
    bank = synth.synth_bank(40, num_features=150, seed=7, variants=35)
    q, _ = synth.synth_frame(640, 480, seed=11, bank=bank, plant=4, T=T)
    packed = bank.pack(bank.class_ids(), 4)
    for thr in (70.0, 75.0, 90.0):
        masks = fr.pass_masks(q, T, packed, thr)
        _, st = oracle.match(q, T, packed, thr, want_stats=True)
        assert sum(int(m.sum()) for m in masks) == int(st["coarse_candidates"]), thr
