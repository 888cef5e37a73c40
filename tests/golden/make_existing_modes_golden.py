#!/usr/bin/env python
"""Records the poses of the two ICP estimations (point-to-plane, the default, and point-to-point; with and without
use_scene_cloud) as the build that preceded LM_POSE_PSO computed them, for tests/test_gpu_pose_pso.py, which holds
every later build to them bit for bit:

  existing_modes_poses.npz   per mode: lm_icp_process_batch's R, t, residual on every case of tests/icp_clouds.py, and
                             the pose stage's (lm_enqueue_pose + lm_complete_pose) survivors, R, t, residual on the
                             recorded driver frame (tests/golden/driver_trace.npz, the allScales bank and the shifted
                             renders of tests/test_gpu_peer_batch.py) at thresholds 75 and 65, every survivor

Run it from the root of the build to record, on a GPU:  python <this repository>/tests/golden/make_existing_modes_golden.py
--out FILE.  The package and library are imported from the current directory; the cases come from this file's tests/.
"""
import argparse
import importlib
import os
import sys

import numpy as np

TESTS = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, TESTS)
sys.path.insert(0, os.getcwd())

MODES = [(e, s) for e in ("point_to_plane", "point_to_point") for s in (False, True)]


def record():
    import icp_clouds
    import test_gpu_peer_batch as pb
    lib = importlib.import_module("6dpose_b200._lib")
    out = {}
    cases = icp_clouds.all_cases()
    data = pb.load_data()
    g = data["g"]
    for est, scene in MODES:
        key = "%s_%d" % (est, scene)
        icp = lib.NativeIcp()
        icp.set_use_scene_cloud(scene)
        R, t, r = [], [], []
        for c in cases:
            Ro, to, res = icp.process_batch(c.scene, [c.model], c.K, c.K[None], c.R[None], c.t[None], [c.xy], 30, est)
            R.append(Ro[0]); t.append(to[0]); r.append(res[0])
        out["icp_%s_R" % key], out["icp_%s_t" % key], out["icp_%s_res" % key] = np.array(R), np.array(t), np.array(r, np.float32)
        nat = pb.handle(data)
        for thr in (75, 65):
            surv, Ro, to, res, _ = nat.match_pose(g["rgb"], g["depth"], None, float(thr), data["sK"], 0.5, 0, 30, scene, est)
            k = "frame_%s_%d" % (key, thr)
            out[k + "_surv"], out[k + "_R"], out[k + "_t"], out[k + "_res"] = surv, Ro, to, res
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(os.path.dirname(os.path.abspath(__file__)), "existing_modes_poses.npz"))
    args = ap.parse_args()
    np.savez_compressed(args.out, **record())


if __name__ == "__main__":
    main()
