"""The bit-sliced coarse scan at the edge of one round: shards whose exact task count fills the GPU's warp slots
(one task per warp, every CTA's slice as long as its warps) and one task more (a CTA's last warp takes a second
task), bit-exact against the CPU oracle."""
import importlib
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

T = [4, 8]
W, H = 640, 480


def _tasks(lib, words):
    return lib.coarse_tasks(words, 1, 0)[3]["tasks"]


def _words(packed):
    # position words per template at the lowest level (T = 8, 320 x 240: 40 x 30 positions, 38 words)
    tm = np.asarray(packed["tmeta"]).reshape(len(packed["tmeta"]), -1, 4)
    Wd, Hd = (W // 2) // 8, (H // 2) // 8
    wf = (tm[:, 2, 0] - 1) // 8 + 1
    hf = (tm[:, 2, 1] - 1) // 8 + 1
    P = (Hd - hf) * Wd + (Wd - wf) + 1
    return np.minimum(np.maximum((P + 31) // 32, 1), (Wd * Hd + 31) // 32).astype(np.int32)


@pytest.mark.parametrize("side", ["fills", "one_more"])
def test_one_round_edge_bit_exact(synth, oracle, side):
    import torch
    lib = importlib.import_module("6dpose_b200._lib")
    slots = torch.cuda.get_device_properties(0).multi_processor_count * 24
    # synth_bank(k) is the first k templates of synth_bank(n): pick k from the words of a larger bank
    big = synth.synth_bank(slots + 200, num_features=150, levels=2, seed=5)
    words = _words(big.pack(big.class_ids(), 4))
    full = np.cumsum(words >> 5)
    rem = np.cumsum(words & 31)
    tasks = full + (rem + 31) // 32           # tasks of the first k + 1 templates
    k = int(np.searchsorted(tasks, slots, side="right"))  # templates whose tasks still fit
    k = k if side == "fills" else k + 1
    bank = synth.synth_bank(k, num_features=150, levels=2, seed=5)
    packed = bank.pack(bank.class_ids(), 4)
    n_tasks = _tasks(lib, _words(packed))
    assert (n_tasks <= slots) if side == "fills" else (n_tasks > slots), (n_tasks, slots)
    assert n_tasks >= slots - 2
    q, _ = synth.synth_frame(W, H, levels=2, seed=13, bank=bank, plant=6, T=T)
    nat = lib.NativeDetector(T)
    nat.load_bank(packed, 4)
    got = nat.match_quantized(q, 75.0)
    want, st = oracle.match(q, T, packed, 75.0, n_threads=os.cpu_count() or 1, want_stats=True)
    assert len(want) > 0 and len(got) == len(want)
    for f in ("x", "y", "template_id"):
        assert np.array_equal(got[f], want[f]), f
    assert np.array_equal(got["similarity"], want["similarity"])
    assert nat.counters()["coarse_candidates"] == int(st["coarse_candidates"])
    nat.close()
