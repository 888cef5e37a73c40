"""The premise of lm_set_template_renders: poseRefine needs from the full model render only the 9x9-dilated box of its
non-zero pixels (LL.cpp:43-50), the render inside that box, and the anchor depth render[rows/2][cols/2] (LL.cpp:73).
So the crop, put back into a zero image with the anchor pixel restored, gives exactly the result of the full render --
checked with the ICP oracle (CPU), for renders inside the image and clipped at its border."""
import os

import numpy as np
import pytest

from oracle import icp_oracle

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "driver_trace.npz")


def from_crop(render):
    """What registration keeps, turned back into a full image."""
    bx, by, bw, bh = icp_oracle.model_bbox(render)
    out = np.zeros_like(render)
    out[by:by + bh, bx:bx + bw] = render[by:by + bh, bx:bx + bw]
    H, W = render.shape
    out[H // 2, W // 2] = render[H // 2, W // 2]
    return out


def same(a, b):
    if a is None or b is None:
        return a is None and b is None
    return np.array_equal(np.asarray(a), np.asarray(b), equal_nan=True)


def cases():
    g = np.load(GOLD)
    r = g["render"]
    ys, xs = np.nonzero(r)
    obj = r[ys.min():ys.max() + 1, xs.min():xs.max() + 1]
    h, w = obj.shape
    H, W = r.shape
    corner = np.zeros_like(r)                        # clipped at the top-left border
    corner[0:h - 7, 0:w - 5] = obj[7:, 5:]
    right = np.zeros_like(r)                         # clipped at the bottom-right border
    right[H - h + 6:H, W - w + 3:W] = obj[:h - 6, :w - 3]
    off_centre = np.roll(np.roll(r, -180, 0), 57, 1)  # anchor pixel 0: no scene centroid, NaN initial guess
    blob = np.zeros_like(r)
    yy, xx = np.mgrid[0:H, 0:W]
    inside = ((yy - 230) / 60.0) ** 2 + ((xx - 330) / 80.0) ** 2 < 1
    blob[inside] = (1000 + 20 * np.sin(xx[inside] / 9.0)).astype(np.uint16)
    return g, [("recorded", r, 273, 153), ("aligned", np.roll(np.roll(r, -68, 0), -19, 1), 273, 153), ("corner", corner, 329, 125),
               ("bottom_right", right, 40, 30), ("off_centre", off_centre, 309, 117), ("blob", blob, 200, 120)]


@pytest.mark.parametrize("use_scene", [False, True])
def test_crop_with_anchor_gives_the_full_render_result(use_scene):
    g, cs = cases()
    scene, sK, mK = g["depth"], g["rf0_sceneK"], g["rf0_modelK"]
    R, t = g["rf0_modelR"], g["rf0_modelT"].reshape(3)
    finite = 0
    for name, render, x, y in cs:
        crop = from_crop(render)
        # the clouds and centroids poseRefine builds (LL.cpp:43-104), NaN centroids included
        box = icp_oracle.model_bbox(render)
        assert icp_oracle.model_bbox(crop) == box, name
        for a, b in zip(icp_oracle.build_clouds(scene, render, sK, mK, x, y, box), icp_oracle.build_clouds(scene, crop, sK, mK, x, y, box)):
            assert same(a, b), name
        _, cm, cs_, _ = icp_oracle.build_clouds(scene, render, sK, mK, x, y, box)
        if not np.all(np.isfinite(cs_ - cm)):
            continue  # the oracle's KD-tree refuses a NaN initial guess; the clouds above are what both runs would use
        finite += 1
        want = icp_oracle.pose_refine(scene, render, sK, mK, R, t, x, y, max_iter=8, use_scene_cloud=use_scene)
        got = icp_oracle.pose_refine(scene, crop, sK, mK, R, t, x, y, max_iter=8, use_scene_cloud=use_scene)
        assert same(got["R"], want["R"]) and same(got["t"], want["t"]), name
        assert same(got["residual"], want["residual"]), name
        assert got.get("n_points") == want.get("n_points"), name
    assert 2 <= finite < len(cs)
    # the cases cover both sides of the premise
    boxes = [icp_oracle.model_bbox(r) for _, r, _, _ in cs]
    assert any(b[0] == 0 and b[1] == 0 for b in boxes) and any(b[0] + b[2] == 640 and b[1] + b[3] == 480 for b in boxes)
    assert any(r[240, 320] == 0 for _, r, _, _ in cs) and any(r[240, 320] > 0 for _, r, _, _ in cs)
