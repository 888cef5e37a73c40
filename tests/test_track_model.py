"""tests/track_model.py on hand-built cases: a flat square render seen by a camera with the render's own intrinsics, so that
T = identity projects every model point to its own pixel and a translation of k z / f metres moves it k pixels.  The
cases: an object straddling each frame edge, one entirely behind the camera, a zero-depth window, a window one pixel
over the cap and margin 0; and the pose -> T conversion against the package's and against T * init_base."""
import importlib

import numpy as np
import pytest

import track_model as tm

pr = importlib.import_module("6dpose_b200.pose_refine")

ROWS, COLS, Z = 48, 64, 500
K = np.array([[100.0, 0, 32.0], [0, 100.0, 24.0], [0, 0, 1]], np.float32)
RENDER = np.zeros((ROWS, COLS), np.uint16)
RENDER[16:28, 26:40] = Z          # box: x 26..39, y 16..27
BOX = (26, 16, 14, 12)
SCENE = np.full((ROWS, COLS), 600, np.uint16)


def moved(dx_px=0, dy_px=0, dz=0.0):
    T = np.eye(4)
    T[0, 3], T[1, 3], T[2, 3] = dx_px * (Z / 1000.0) / 100.0, dy_px * (Z / 1000.0) / 100.0, dz
    return T


def run(T, margin=4, cap=10 ** 6, scene=SCENE):
    return tm.track(scene, K, RENDER, K, T, margin, cap)


def test_identity_projects_to_the_render_box():
    out = run(np.eye(4))
    assert out["status"] == tm.TRACKED and out["box"] == BOX
    assert out["window"] == (22, 12, 22, 20)
    assert out["raw_model"].shape == (14 * 12, 3) and out["raw_scene"].shape == (22 * 20, 3)
    assert (out["raw_scene"][:, 2] == 0.6).all() and out["init"].tobytes() == np.eye(4).tobytes()
    assert out["source"].shape[0] > 0 and out["target"].shape[0] > 0


@pytest.mark.parametrize("dx, dy, box, window", [
    (-30, 0, (0, 16, 10, 12), (0, 12, 14, 20)),      # left edge
    (30, 0, (56, 16, 8, 12), (52, 12, 12, 20)),      # right edge
    (0, -20, (26, 0, 14, 8), (22, 0, 22, 12)),       # top edge
    (0, 30, (26, 46, 14, 2), (22, 42, 22, 6)),       # bottom edge
])
def test_an_object_straddling_each_edge(dx, dy, box, window):
    out = run(moved(dx, dy))
    assert out["status"] == tm.TRACKED
    assert out["box"] == box and out["window"] == window
    x, y, w, h = out["window"]
    assert x >= 0 and y >= 0 and x + w <= COLS and y + h <= ROWS


def test_entirely_outside_or_behind_the_camera():
    for T in (moved(200, 0), moved(0, 0, -1.0)):
        out = run(T)
        assert out["status"] == tm.OUTSIDE and out["window"] == (0, 0, 0, 0) and out["box"] == (0, 0, 0, 0)


def test_a_zero_depth_window():
    scene = SCENE.copy()
    scene[12:32, 22:44] = 0
    assert run(np.eye(4), scene=scene)["status"] == tm.NO_DEPTH
    scene[12, 43] = 1  # one pixel of depth in the window's corner
    out = run(np.eye(4), scene=scene)
    assert out["status"] == tm.TRACKED and out["raw_scene"].shape == (1, 3)


def test_a_window_one_pixel_over_the_cap():
    area = 22 * 20
    assert run(np.eye(4), cap=area)["status"] == tm.TRACKED
    assert run(np.eye(4), cap=area - 1)["status"] == tm.WINDOW


def test_margin_zero_is_the_box():
    out = run(np.eye(4), margin=0)
    assert out["window"] == out["box"] == BOX
    assert out["raw_scene"].shape == (14 * 12, 3)


def test_pose_to_transform():
    rng = np.random.default_rng(0)
    for _ in range(20):
        w = rng.normal(size=3)
        th = np.linalg.norm(w)
        k = w / th
        Kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
        Rb = (np.eye(3) + np.sin(th) * Kx + (1 - np.cos(th)) * Kx @ Kx).astype(np.float32)
        tb = rng.uniform(-100, 100, 3).astype(np.float32)
        tb[2] = rng.uniform(300, 1200)
        R = Rb.astype(np.float64) @ np.array([[np.cos(0.1), -np.sin(0.1), 0], [np.sin(0.1), np.cos(0.1), 0], [0, 0, 1]])
        t = rng.uniform(-200, 200, 3) + [0, 0, 800]
        T = tm.pose_to_transform(R, t, Rb, tb)
        assert T.tobytes() == pr.pose_to_transform(R, t, Rb, tb).tobytes()
        R2, t2 = tm.compose(T, Rb, tb)
        assert np.abs(R2 - R).max() < 1e-6 and np.abs(t2 - t).max() < 1e-3


def test_brought_close_along_its_line_of_sight():
    # the render's centroid moved to a quarter of its distance on the same ray: four times its size about the same pixel
    raw = tm.model_cloud(RENDER, K)
    c = raw.mean(0)
    T = np.eye(4)
    T[:3, 3] = -0.75 * c
    status, win, box = tm.window(raw, T, ROWS, COLS, K, 0, 10 ** 6)
    assert status == tm.TRACKED and win[2] * win[3] > 4 * BOX[2] * BOX[3]
    assert tm.window(raw, T, ROWS, COLS, K, 0, 4 * BOX[2] * BOX[3])[0] == tm.WINDOW
