"""CPU checks of the sharded batch's surface: lm_peer_detect_batch is declared, exported and bound, a host-only handle
refuses it, and dist.detect_batch_sharded / match_refine_batch_sharded refuse a detector without a connected exchange
for this rank and world and check their frames, sceneK and masks before any device work (gloo, no native handle)."""
import importlib
import os
import re
import socket

import numpy as np
import pytest
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
lib = importlib.import_module("6dpose_b200._lib")


def frame(h=48, w=64):
    return [np.zeros((h, w, 3), np.uint8), np.zeros((h, w), np.uint16)]


K = np.eye(3, dtype=np.float32)


def test_symbol_declared_and_bound():
    text = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "linemod_b200.h")).read(), flags=re.S)
    decl = re.search(r"int lm_peer_detect_batch\(([^;]*)\);", text)
    want = re.search(r"int lm_detect_batch\(([^;]*)\);", text)
    assert decl and want
    assert re.sub(r"\s+", " ", decl.group(1)) == re.sub(r"\s+", " ", want.group(1))  # the arguments of lm_detect_batch
    L = lib.load()
    assert "lm_peer_detect_batch" in lib.SYMBOLS and hasattr(L, "lm_peer_detect_batch")
    assert L.lm_peer_detect_batch.argtypes == L.lm_detect_batch.argtypes
    assert callable(lib.NativeDetector.peer_detect_batch)


def test_host_only_handle():
    nat = lib.NativeDetector([4, 8], -1)
    f = frame()
    for pose_nms in (False, True):
        with pytest.raises(lib.LinemodLibraryError, match="error %d" % lib.LM_E_STATE):
            nat.peer_detect_batch(f[0][None], f[1][None], None, 75.0, K[None], pose_nms=pose_nms)
    with pytest.raises(ValueError, match="sceneK"):                 # the binding's own checks come first
        nat.peer_detect_batch(f[0][None], f[1][None], None, 75.0, np.zeros((2, 3, 3), np.float32))


def test_capacity_retry_only_for_the_outputs():
    """The binding calls again only when the call reported a total beyond the capacity it passed; an LM_E_CAPACITY
    without one (records beyond the exchange or the result block) raises instead of looping."""
    nat = lib.NativeDetector([4, 8], -1)
    f = frame()
    calls = []

    def records_overflow(*a):
        calls.append(a[19])                                        # cap
        return lib.LM_E_CAPACITY                                   # *n_out not written

    with pytest.raises(lib.LinemodLibraryError, match="error %d" % lib.LM_E_CAPACITY):
        nat._batch(records_overflow, f[0][None], f[1][None], None, 75.0, K[None], 0.5, 0, 30, False, True, 40.0, None)
    assert calls == [1024]

    calls.clear()

    def outputs_too_small(*a):
        calls.append(a[19])
        if a[19] < 7:
            a[20]._obj.value = 7                                   # byref(total): the entries the batch needs
            return lib.LM_E_CAPACITY
        a[20]._obj.value = 0
        return lib.LM_OK

    got = nat._batch(outputs_too_small, f[0][None], f[1][None], None, 75.0, K[None], 0.5, 0, 30, False, True, 40.0, 2)
    assert calls == [2, 7] and len(got) == 1


def sharded_worker(rank, world, port):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        pkg = importlib.import_module("6dpose_b200")
        dmod = importlib.import_module("6dpose_b200.dist")
        fns = (dmod.detect_batch_sharded, dmod.match_refine_batch_sharded)
        det = pkg.Detector()
        for fn in fns:
            for peers in (None, (rank, world + 1), ((rank + 1) % world, world)):  # not connected, or for another group
                det._peers = peers
                with pytest.raises(RuntimeError, match="connected"):
                    fn(det, [frame()], 75.0, [], K)
        det._peers = (rank, world)                                            # a stand-in for connect_peers
        for fn in fns:
            with pytest.raises(ValueError, match="no frames"):
                fn(det, [], 75.0, [], K)
            with pytest.raises(ValueError, match="one size"):
                fn(det, [frame(), frame(48, 80)], 75.0, [], K)
            with pytest.raises(RuntimeError, match="modalities"):
                fn(det, [frame()[:1]], 75.0, [], K)
            with pytest.raises(TypeError, match="uint16"):
                fn(det, [[frame()[0], frame()[1].astype(np.float32)]], 75.0, [], K)
            for bad in (np.eye(4, dtype=np.float32), np.zeros((3, 3, 3), np.float32)):
                with pytest.raises(ValueError, match="sceneK"):
                    fn(det, [frame(), frame()], 75.0, [], bad)
            with pytest.raises(TypeError, match="float32"):
                fn(det, [frame()], 75.0, [], np.eye(3))
            with pytest.raises(ValueError, match="masks"):
                fn(det, [frame(), frame()], 75.0, [], K, masks=[[]])
            with pytest.raises(TypeError):
                fn(det, [frame()], 75.0, [], K, masks=None)
            with pytest.raises(RuntimeError, match="modalities"):
                fn(det, [frame()], 75.0, [], K, masks=[[np.zeros((48, 64), np.uint8)]])
        assert det._native is None
    finally:
        dist.destroy_process_group()


def free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def test_sharded_batch_checks_before_any_device_work():
    mp.spawn(sharded_worker, args=(2, free_port()), nprocs=2, join=True)
