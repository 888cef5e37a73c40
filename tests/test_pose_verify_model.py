"""The numpy model of the pose verification (tests/pose_verify_model.py) on hand-built cases at every boundary of
include/linemod_b200.h's steps 3-5: |d| equal to delta and one ulp either side, u and v at x.5, q_z equal to 0, -0 and
negative, each edge of the frame, a zero scene depth, a NaN pose and an empty cloud.  No GPU: test_gpu_pose_verify.py
holds the device to the same model."""
import numpy as np
import pytest

import icp_clouds
import pose_verify_model as pvm

CASES = pvm.boundary_cases()


@pytest.mark.parametrize("name", sorted(CASES))
def test_boundary_case_classes(name):
    pts, T, scene, sK, delta, want = CASES[name]
    got = pvm.classify(pts, T, scene, sK, delta)
    assert got.tolist() == want.tolist(), [pvm.NAMES[k] for k in got]
    score, counts = pvm.verify(pts, T, scene, sK, delta)
    assert counts[0] == len(pts) and counts[1:].sum() == len(pts)
    assert counts[1:].tolist() == [int((want == k).sum()) for k in range(5)]
    den = counts[1 + pvm.INLIER] + counts[1 + pvm.OCCLUDED] + counts[1 + pvm.VIOLATION]
    assert score.dtype == np.float32 and score == (np.float32(counts[1 + pvm.INLIER]) / np.float32(den) if den else 0.0)


def test_every_case_covers_its_boundary():
    names = set(CASES)
    for need in ("d_eq_delta_behind", "d_eq_delta_front", "u_half", "v_half", "qz_zero", "qz_negative_zero", "qz_negative",
                 "edges", "scene_zero", "nan_pose", "empty"):
        assert need in names
    # q_z really is -0.0 in that case, and the ulp cases really are one ulp from delta
    pts, T, *_ = CASES["qz_negative_zero"]
    qz = ((T[2, 0] * pts[:, 0] + T[2, 1] * pts[:, 1]) + T[2, 2] * pts[:, 2]) + T[2, 3]
    assert qz[0] == 0.0 and np.signbit(qz[0])
    assert CASES["d_eq_delta_behind_delta_ulp_below"][4] == np.nextafter(10.0, 0.0)
    # the NaN pose scores 0, the empty cloud 0, with zero counts
    assert pvm.verify(*CASES["nan_pose"][:5])[0] == 0.0
    s, c = pvm.verify(*CASES["empty"][:5])
    assert s == 0.0 and not c.any()


def test_model_cloud_is_the_rendered_surface():
    c = icp_clouds.size_case(129)
    pts = pvm.model_cloud(c.model, c.K)
    assert pts.shape == (int((c.model > 0).sum()), 3)
    # row-major crop order, metres
    rr, cc = np.nonzero(c.model)
    assert np.array_equal(pts[:, 2], c.model[rr, cc] / 1000.0)
    # the identity pose against the render itself as the scene, same intrinsics: every point on its own pixel
    score, counts = pvm.verify(pts, np.eye(4), c.model, c.K, 0.0)
    assert score == 1.0 and counts[1 + pvm.INLIER] == len(pts)
    # 30 mm further back in the scene: every point is a violation at 10 mm, an inlier at 30 mm
    deeper = np.where(c.model > 0, c.model + 30, 0).astype(np.uint16)
    assert pvm.verify(pts, np.eye(4), deeper, c.K, 10.0)[1][1 + pvm.VIOLATION] == len(pts)
    assert pvm.verify(pts, np.eye(4), deeper, c.K, 30.0)[0] == 1.0
