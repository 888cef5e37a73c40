"""The depth gate over the ranks of the peer exchange (lm_peer_detect_batch, what dist.detect_batch_sharded runs): each rank
gates its own shard on its own copy of the frames, and every rank returns what one unconnected handle over the whole bank
returns from lm_detect_batch with the same gate.  Data, frames and helpers of tests/test_gpu_peer_batch.py."""
import os

import numpy as np
import pytest

from test_gpu_peer_batch import (CAPACITY, FRAMES, WARM, batch_args, close, data, frame, handle, peer_batch, same,  # noqa: F401
                                 scene_ks)

pytestmark = pytest.mark.gpu
Z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "allScales_depths.npz"))["z_mm"]
TAU = 0.15


def gated(nat):
    nat.set_template_depths(0, Z)
    nat.set_depth_gate(TAU)
    return nat


@pytest.mark.parametrize("world", [2, 3])
def test_sharded_gated_batch_equals_the_single_gpu_one(data, world):
    ref = gated(handle(data))
    dets = [gated(handle(data, 0, (r, world))) for r in range(world)]
    try:
        # as test_gpu_peer_batch.connected: an unconnected batch of the largest shape first, then the exchange
        for d in dets:
            d.detect_batch(*batch_args(data, FRAMES[:WARM], scene_ks(data, WARM), 62.0, 0, True, True))
        for d in dets:
            d.peer_export(world, CAPACITY)
        bases = [d.peer_base() for d in dets]
        for r, d in enumerate(dets):
            d.peer_connect_local(r, world, bases)
        for d in dets:
            d.prepare()
        frame(dets, data, 75.0, 0, False, False)
        for share in (False, True):
            for d in dets:
                d.peer_share_pose(share)
            for pose_nms in (False, True):
                args = batch_args(data, FRAMES, scene_ks(data, len(FRAMES)), 75.0, 0, False, pose_nms)
                want = (ref.detect_batch(*args), ref.batch_counts.copy())
                for got in peer_batch(dets, args):
                    same(got, want)
        st = [d.depth_gate_stats() for d in dets]
        full = ref.depth_gate_stats()
        assert sum(s["before"] for s in st) == full["before"] and sum(s["after"] for s in st) == full["after"]
        assert sum(s["with_distance"] for s in st) == full["with_distance"] == 2989
        assert full["after"] < full["before"]
    finally:
        close(dets)
        ref.close()
