"""View following on the CPU (include/linemod_b200.h, lm_set_track_views): self-checks of tests/track_views_model.py at
its decision boundaries, and the synthetic sequence of tests/view_object.py tracked through tests/track_model.py and
oracle/icp_oracle.py -- lost with view following off, held with it on -- so the sequence the GPU test runs is known to
show the effect."""
import math

import numpy as np
import pytest

import pso_scenes
import track_model as tm
import track_views_model as vm
import view_object as vo
from oracle import icp_oracle

TURN_DEG = 20.0
HELD_ROT_DEG, HELD_POS_MM = 8.0, 10.0  # the on-run measured 3.7 degrees and 4.4 mm at worst


def rot(axis, deg):
    return pso_scenes.rodrigues(np.asarray(axis, float) / np.linalg.norm(axis) * np.radians(deg))


def T_of(R, t=(0.01, -0.02, 0.6)):
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = R, t
    return T


def test_threshold_uses_libm_cos():
    assert vm.tau(0.0) == 3.0
    assert vm.tau(90.0) == 1.0 + 2.0 * math.cos(math.pi / 2)
    assert vm.tau(179.0) < -0.99


def test_ties_go_to_the_lowest_template():
    R = rot((0, 0, 1), 40.0).astype(np.float32)
    Rb = np.stack([np.eye(3, dtype=np.float32), R, R, R])  # three equal best scores
    t = np.zeros((4, 3), np.float32)
    j, T2, s, sk, _ = vm.choose(Rb, t, 0, T_of(R.astype(np.float64)), 10.0)
    assert s[1] == s[2] == s[3] and j == 1
    # a NaN score is no candidate, and a template without a render neither
    Rb[1, 0, 0] = np.nan
    assert vm.choose(Rb, t, 0, T_of(R.astype(np.float64)), 10.0)[0] == 2
    assert vm.choose(Rb, t, 0, T_of(R.astype(np.float64)), 10.0, has=[1, 1, 0, 1])[0] == 3


def test_s_k_on_either_side_of_tau():
    Rb = np.stack([np.eye(3), rot((1, 0, 0), 90.0)]).astype(np.float32)
    t = np.array([[0, 0, 600], [5, -3, 650]], np.float32)
    T = T_of(rot((1, 0, 0), 50.0))
    sk = vm.scores(vm.rotation(T, Rb[0]), Rb)[0]
    # near the turn where tau meets s_k, the object switches exactly when s_k < tau, and a kept T keeps its bits
    deg = math.degrees(math.acos((sk - 1.0) / 2.0))
    sides = set()
    for i in range(-60, 61):
        d = deg + i * 2e-14
        j, T2, *_ = vm.choose(Rb, t, 0, T, d)
        assert j == (1 if sk < vm.tau(d) else 0)
        assert j == 1 or np.array_equal(T2, T)
        sides.add(sk < vm.tau(d))
    assert sides == {True, False}
    j, T2, *_ = vm.choose(Rb, t, 0, T, deg * 0.9)
    assert j == 1
    # the object stays put: T' [R_1 | b_1] == T [R_0 | b_0] up to rounding
    P = [np.eye(4), np.eye(4)]
    for k in range(2):
        P[k][:3, :3], P[k][:3, 3] = Rb[k], t[k] / 1000.0
    assert np.allclose(T2 @ P[1], T @ P[0], atol=1e-12)


def test_zero_turn_single_template_and_best_already():
    Rb = np.stack([np.eye(3), rot((0, 1, 0), 30.0), rot((0, 1, 0), 60.0)]).astype(np.float32)
    t = np.zeros((3, 3), np.float32)
    T = T_of(rot((0, 1, 0), 28.0))
    assert vm.choose(Rb, t, 0, T, 0.0)[0] == 1        # tau = 3: every turn re-chooses
    assert vm.choose(Rb, t, 1, T_of(rot((0, 1, 0), 1.0)), 0.0)[0] == 1  # k itself is best: no switch
    assert vm.choose(Rb[:1], t[:1], 0, T, 0.0)[0] == 0  # a single template
    assert vm.choose(Rb, t, 0, T_of(np.eye(3)), 0.0)[0] == 0  # s_k == 3 == tau: kept


@pytest.fixture(scope="module")
def bank():
    Rb, tb, Kb = vo.templates()
    return Rb, tb, Kb, {}


def render(bank, g):
    Rb, tb, _, cache = bank
    if g not in cache:
        cache[g] = vo.template_render(Rb[g], tb[g])
    return cache[g]


START = 7                  # the template the sequence starts at (its view is the first frame's)
FRAMES, STEP_DEG = 60, 3.0  # 180 degrees in all


def run_cpu(bank, views):
    """The sequence on the CPU: per frame the rotation and position error, and the number of switches."""
    Rb, tb, Kb, _ = bank
    seq = vo.sequence(Rb[START].astype(np.float64), FRAMES, STEP_DEG)
    g, T, switches, errs = START, vo.start_T(seq[0][1], seq[0][2], Rb[START], tb[START]), 0, []
    for scene, R, b in seq[1:]:
        if views:
            j, T, *_ = vm.choose(Rb, tb, g, T, TURN_DEG)
            switches += j != g
            g = j
        out = tm.track(scene, vo.K.astype(np.float32), render(bank, g), Kb[g], T, 4, 1 << 40)
        if out["status"] != tm.TRACKED:
            errs.append((math.inf, math.inf))
            break
        T = icp_oracle.registration_icp_p2pl(out["source"], out["target"], icp_oracle.estimate_normals(out["target"]), icp_oracle.MAX_DIST,
                                             out["init"])[0]
        errs.append(vo.errors(T, Rb[g], tb[g], R, b))
    return np.array(errs), switches


def test_sequence_is_lost_without_views_and_held_with_them(bank):
    off, n_off = run_cpu(bank, False)
    on, n_on = run_cpu(bank, True)
    assert n_off == 0 and n_on >= 3
    assert off[:, 0].max() > HELD_ROT_DEG or off[:, 1].max() > HELD_POS_MM
    assert len(on) == FRAMES and on[:, 0].max() <= HELD_ROT_DEG and on[:, 1].max() <= HELD_POS_MM
