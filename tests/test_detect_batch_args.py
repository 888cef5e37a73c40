"""Detector.match_refine_batch / detect_batch check their frames, sceneK and masks before any device work: these run
without a GPU."""
import importlib

import numpy as np
import pytest

pkg = importlib.import_module("6dpose_b200")


def frame(h=48, w=64):
    return [np.zeros((h, w, 3), np.uint8), np.zeros((h, w), np.uint16)]


K = np.eye(3, dtype=np.float32)


@pytest.mark.parametrize("method", ["match_refine_batch", "detect_batch"])
def test_frames_of_different_sizes(method):
    det = pkg.Detector()
    with pytest.raises(ValueError, match="one size"):
        getattr(det, method)([frame(), frame(48, 80)], 75.0, [], K)
    with pytest.raises(ValueError, match="one size"):
        getattr(det, method)([frame(), [np.zeros((48, 64, 3), np.uint8), np.zeros((40, 64), np.uint16)]], 75.0, [], K)
    assert det._native is None


@pytest.mark.parametrize("method", ["match_refine_batch", "detect_batch"])
def test_scene_matrix_shape(method):
    det = pkg.Detector()
    for bad in (np.eye(4, dtype=np.float32), np.zeros((2, 3, 3), np.float32), np.zeros((3, 9), np.float32)):
        with pytest.raises(ValueError, match="sceneK"):
            getattr(det, method)([frame(), frame(), frame()], 75.0, [], bad)
    with pytest.raises(TypeError, match="float32"):
        getattr(det, method)([frame(), frame()], 75.0, [], np.eye(3))
    assert det._native is None


def test_frames_masks_and_sources():
    det = pkg.Detector()
    with pytest.raises(ValueError, match="no frames"):
        det.detect_batch([], 75.0, [], K)
    with pytest.raises(ValueError, match="masks"):
        det.detect_batch([frame(), frame()], 75.0, [], K, masks=[[]])
    with pytest.raises(TypeError):
        det.detect_batch([frame()], 75.0, [], K, masks=None)
    with pytest.raises(RuntimeError, match="modalities"):
        det.detect_batch([frame()[:1]], 75.0, [], K)
    with pytest.raises(TypeError, match="uint16"):
        det.detect_batch([[frame()[0], frame()[1].astype(np.float32)]], 75.0, [], K)
    assert det._native is None
