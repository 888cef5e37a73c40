"""CPU checks of the shared pose stage's surface: lm_peer_share_pose / lm_pose_stats are declared, exported and bound,
NativeDetector.peer_share_pose / pose_stats handle their arguments, and dist.connect_peers(share_pose=...) turns the
share on every rank after the connect barrier (gloo, a stand-in for the native handle)."""
import importlib
import os
import re
import socket

import numpy as np
import pytest
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
lib = importlib.import_module("6dpose_b200._lib")


def test_symbols_declared_and_bound():
    text = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "linemod_b200.h")).read(), flags=re.S)
    assert "int lm_peer_share_pose(lm_detector* d, int on);" in text
    assert "int lm_pose_stats(lm_detector* d, int64_t* out4);" in text
    L = lib.load()
    for name in ("lm_peer_share_pose", "lm_pose_stats"):
        assert name in lib.SYMBOLS and hasattr(L, name)
    assert callable(lib.NativeDetector.peer_share_pose) and callable(lib.NativeDetector.pose_stats)


def test_host_only_handle():
    nat = lib.NativeDetector([4, 8], -1)                   # host-only: no exchange can be connected
    with pytest.raises(lib.LinemodLibraryError, match="error %d" % lib.LM_E_STATE):
        nat.peer_share_pose(True)
    with pytest.raises(lib.LinemodLibraryError, match="error %d" % lib.LM_E_STATE):
        nat.peer_share_pose(np.bool_(False))
    assert nat.pose_stats() == [0, 0, 0, 0]
    for bad in ("yes", None, 1.0):
        with pytest.raises(TypeError):
            nat.peer_share_pose(bad)


def test_connect_peers_rejects_a_non_bool_share():
    dmod = importlib.import_module("6dpose_b200.dist")
    with pytest.raises(TypeError):
        dmod.connect_peers(object(), share_pose="on")


class FakeNative:
    def __init__(self, rank):
        self.rank, self.calls = rank, []

    def peer_export(self, world, capacity):
        self.calls.append(("export", world, capacity))
        return bytes([self.rank]) * lib.PEER_HANDLE_BYTES

    def peer_connect(self, rank, world, handles):
        self.calls.append(("connect", rank, world, [h[0] for h in handles]))

    def peer_share_pose(self, on):
        self.calls.append(("share", on))


class FakeDetector:
    def __init__(self, rank):
        self.native = FakeNative(rank)
        self.shard = (0, 1)

    def _select(self, class_ids):
        return self.native


def worker(rank, world, port, out_dir, share):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    dmod = importlib.import_module("6dpose_b200.dist")
    det = FakeDetector(rank)
    kw = {} if share is None else dict(share_pose=share)
    dmod.connect_peers(det, capacity_records=64, **kw)
    np.save(os.path.join(out_dir, "calls_%d.npy" % rank), np.asarray(repr(det.native.calls)))
    dist.destroy_process_group()


def free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


@pytest.mark.parametrize("share", [None, False, True])
def test_connect_peers_sets_the_share_on_every_rank(tmp_path, share):
    mp.spawn(worker, args=(2, free_port(), str(tmp_path), share), nprocs=2, join=True)
    for r in range(2):
        calls = eval(str(np.load(str(tmp_path / ("calls_%d.npy" % r)))))
        assert calls == [("export", 2, 64), ("connect", r, 2, [0, 1]), ("share", bool(share))], calls
