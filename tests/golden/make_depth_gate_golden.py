#!/usr/bin/env python
"""Regenerates the depth gate's fixtures from the reference's own files (needs /root/reference mounted):

  allScales_depths.npz   the training distance of each of the 2989 allScales templates, cam_t_w2c[2] of
                         linemodLevelup/test/case1/allScales/06_info.yaml (mm; 337 views at each of 600 ... 1800 mm)
  frame_half_case1.npz   the half-occluded fixture frame (0000_{rgb,dep}_half.png) as the pixels where it differs from
                         the full one (driver_trace.npz holds the full frame, in RGB order): flat pixel index, BGR colour
                         and depth there
"""
import os
import re

import cv2
import numpy as np

CASE = "/root/reference/linemodLevelup/test/case1/"
OUT = os.path.dirname(os.path.abspath(__file__))


def main():
    txt = open(CASE + "allScales/06_info.yaml").read()
    ids = [int(k) for k in re.findall(r"^(\d+):", txt, re.M)]
    z = [float(v.split(",")[2]) for v in re.findall(r"cam_t_w2c: \[([^\]]*)\]", txt)]
    assert ids == list(range(2989)) and len(z) == 2989
    np.savez_compressed(os.path.join(OUT, "allScales_depths.npz"), z_mm=np.asarray(z, np.float32))
    rgb, dep = cv2.imread(CASE + "0000_rgb.png"), cv2.imread(CASE + "0000_dep.png", cv2.IMREAD_UNCHANGED)
    rgbh, deph = cv2.imread(CASE + "0000_rgb_half.png"), cv2.imread(CASE + "0000_dep_half.png", cv2.IMREAD_UNCHANGED)
    idx = np.flatnonzero((rgbh != rgb).any(2) | (deph != dep))
    np.savez_compressed(os.path.join(OUT, "frame_half_case1.npz"), index=idx.astype(np.int32),
                        bgr=rgbh.reshape(-1, 3)[idx], depth=deph.reshape(-1)[idx])


if __name__ == "__main__":
    main()
