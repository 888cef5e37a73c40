"""The bit-sliced coarse scan's task table and launch shape (lm_coarse_tasks, host only): every position word of a shard is
in exactly one task, full tasks are 32 words of one template, remainders pack in order, and a shard with no more tasks
than the GPU has warp slots runs in one round with no CTA holding more tasks than it has warps (or teams)."""
import importlib

import numpy as np
import pytest

SM = 132  # H100 SXM


@pytest.fixture(scope="module")
def lib():
    return importlib.import_module("6dpose_b200._lib")


@pytest.fixture(scope="module")
def synth():
    return importlib.import_module("6dpose_b200.synth")


def level_words(packed, W, H, T_low=8, levels=2, M=2):
    """Position words per template at the lowest level: ceil(P / 32) clamped to 1..nwords, P = template_positions
    (LL.cpp:1309) of the template's first modality there."""
    tm = np.asarray(packed["tmeta"]).reshape(len(packed["tmeta"]), -1, 4)
    cols, rows = W >> (levels - 1), H >> (levels - 1)
    Wd, Hd = cols // T_low, rows // T_low
    nwords = (Wd * Hd + 31) // 32
    s = (levels - 1) * M
    wf = (tm[:, s, 0] - 1) // T_low + 1
    hf = (tm[:, s, 1] - 1) // T_low + 1
    P = (Hd - hf) * Wd + (Wd - wf) + 1
    return np.minimum(np.maximum((P + 31) // 32, 1), nwords).astype(np.int32), nwords


def plane_bytes(W, H, T_low=8, levels=2, M=2):
    """Bit-plane bytes of the lowest level, zero words included (the detector's sizing)."""
    plane = (W >> (levels - 1)) // T_low * ((H >> (levels - 1)) // T_low)
    nwords = (plane + 31) // 32
    rounds = (nwords + 31) // 32
    lbw = ((T_low * T_low * plane + 31) // 32 + 32 * rounds + 4 + 3) & ~3
    zero = (nwords + 32 * rounds + 8 + 3) & ~3
    return ((M * 8 * lbw + zero) * 4 + 15) & ~15


def check_table(words, table, n_full, n_rem, shape):
    n = len(words)
    # full tasks: (item, round) for every round of every item, items in order
    want_full = [(i, r) for i in range(n) for r in range(int(words[i]) >> 5)]
    assert n_full == len(want_full)
    assert [tuple(t) for t in table[:n_full]] == want_full
    # remainders: (item, word) behind the item's full rounds, items in order, packed 32 to a task, the last one padded
    want_rem = [(i, k) for i in range(n) for k in range(int(words[i]) & ~31, int(words[i]))]
    assert n_rem == len(want_rem)
    rem = table[n_full:]
    assert len(rem) % 32 == 0 and len(rem) - n_rem < 32
    assert [tuple(t) for t in rem[:n_rem]] == want_rem
    assert np.all(rem[n_rem:] == rem[n_rem - 1]) if n_rem else len(rem) == 0
    # every (item, word < words) exactly once
    covered = np.zeros(int(words.sum()), np.int32)
    start = np.concatenate([[0], np.cumsum(words)[:-1]])
    for it, r in table[:n_full]:
        covered[start[it] + 32 * r: start[it] + 32 * r + 32] += 1
    for it, k in rem[:n_rem]:
        covered[start[it] + k] += 1
    assert np.all(covered == 1)
    tasks = n_full + (n_rem + 31) // 32
    assert shape["tasks"] == tasks
    return tasks


def slices(tasks, grid):
    # CTA b takes tasks b, b + grid, b + 2 grid, ...
    return [(tasks - b + grid - 1) // grid for b in range(grid)]


@pytest.mark.parametrize("W,H,n,objects", [
    (640, 480, 3115, 1),    # bench workload: one round
    (640, 480, 3115, 6),    # six objects: several rounds
    (1280, 960, 300, 1),    # 150 words a template: several full rounds each
])
def test_task_table_covers_every_word_once(lib, synth, W, H, n, objects):
    cids = tuple("%02d_template" % (k + 1) for k in range(objects))
    bank = synth.synth_bank(n, num_features=150, levels=2, seed=1234, variants=35, class_ids=cids)
    words, nwords = level_words(bank.pack(bank.class_ids(), 4), W, H)
    assert words.min() >= 1 and words.max() <= nwords
    table, n_full, n_rem, shape = lib.coarse_tasks(words, SM, plane_bytes(W, H))
    tasks = check_table(words, table, n_full, n_rem, shape)
    teams = shape["warps_per_cta"] // shape["split"]
    assert shape["grid"] <= SM and shape["warps_per_cta"] <= 24
    if tasks <= SM * 24:
        assert max(slices(tasks, shape["grid"])) <= teams
    else:
        assert shape["grid"] == SM and shape["warps_per_cta"] == 24 and shape["split"] == 1


def test_bench_bank_runs_in_one_round(lib, synth):
    """3115 templates at 640x480: 2100 full tasks + the 33 425 remainder words in 1045 tasks = 3145 tasks for the
    132 x 24 warp slots of an H100, so no CTA takes a second task per warp."""
    bank = synth.synth_bank(3115, num_features=150, levels=2, seed=1234, variants=35)
    words, _ = level_words(bank.pack(bank.class_ids(), 4), 640, 480)
    table, n_full, n_rem, shape = lib.coarse_tasks(words, SM, plane_bytes(640, 480))
    assert (n_full, n_rem, shape["tasks"]) == (2100, 33425, 3145)
    assert shape == dict(tasks=3145, split=1, warps_per_cta=24, grid=132)
    assert max(slices(3145, 132)) == 24


@pytest.mark.parametrize("n,split", [(70, 8), (600, 4), (1200, 2)])
def test_small_shard_team_mode(lib, synth, n, split):
    """Small shards share each task among a team of 2 / 4 / 8 warps; every CTA's share still fits its teams."""
    bank = synth.synth_bank(n, num_features=150, levels=2, seed=7, variants=35)
    words, _ = level_words(bank.pack(bank.class_ids(), 4), 640, 480)
    table, n_full, n_rem, shape = lib.coarse_tasks(words, SM, plane_bytes(640, 480))
    tasks = check_table(words, table, n_full, n_rem, shape)
    assert shape["split"] == split
    assert max(slices(tasks, shape["grid"])) <= shape["warps_per_cta"] // split


@pytest.mark.parametrize("tasks", [SM * 24 - 1, SM * 24, SM * 24 + 1])
def test_one_round_boundary(lib, tasks):
    """Exactly at, just below and just above one task per warp slot (one full round per item)."""
    words = np.full(tasks, 32, np.int32)
    table, n_full, n_rem, shape = lib.coarse_tasks(words, SM, plane_bytes(640, 480))
    assert (n_full, n_rem, shape["tasks"]) == (tasks, 0, tasks)
    assert shape["grid"] == SM and shape["warps_per_cta"] == 24 and shape["split"] == 1
    assert max(slices(tasks, SM)) == (24 if tasks <= SM * 24 else 25)


def test_rejects_bad_input(lib):
    with pytest.raises(RuntimeError):
        lib.coarse_tasks(np.array([3, 0, 5], np.int32), SM, plane_bytes(640, 480))
