"""The float64 cloud model of tests/pose_cloud_model.py and the crafted pose-stage cases the device is held to
(tests/test_gpu_pose_clouds.py), on the CPU: the model equals the oracle's build_clouds / voxel_down_sample on every
case (clouds bit for bit, centroids up to summation order), and every case reaches the edge it is built for."""
from dataclasses import dataclass, field

import numpy as np
import pytest

import icp_clouds as ic
import pose_cloud_model as pcm
from oracle import icp_oracle

CLASSES, PER_CLASS = 3, 4
G = CLASSES * PER_CLASS            # the bank of the device cases: 3 classes of 4 templates
CLASS_BEGIN = np.arange(0, G + 1, PER_CLASS)


@dataclass
class Case:
    name: str
    scene: np.ndarray              # u16 mm, srows x scols
    sK: np.ndarray                 # 3 x 3 f32
    renders: dict                  # template g -> (render u16, mK 3 x 3 f32); every template has one
    surv: list                     # (x, y, g) per survivor, in pick order
    select: list = None            # classes selected (None: all)
    info: dict = field(default_factory=dict)


def K(fx, fy, cx, cy):
    return np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1]], np.float32)


SK = K(572.41, 573.57, 325.26, 242.05)
RK = K(610.25, 590.75, 318.25, 241.75)   # fx != fy, fractional centre, not the scene's


def blob(rows, cols, r0, r1, c0, c1, z=1000, seed=0):
    """A render with a rectangle of non-zero depth z + a small pattern, rows [r0, r1) x cols [c0, c1)."""
    r = np.zeros((rows, cols), np.uint16)
    rr, cc = np.mgrid[r0:r1, c0:c1]
    r[r0:r1, c0:c1] = z + (rr * 7 + cc * 3 + seed) % 13
    return r


def noisy_scene(rows, cols, lo, hi, seed, holes=0.1):
    rng = np.random.default_rng(seed)
    s = rng.integers(lo, hi, (rows, cols)).astype(np.uint16)
    s[rng.random((rows, cols)) < holes] = 0
    return s


def default_renders(renders=None):
    """Every template of the bank gets a small render unless given one."""
    out = {g: (blob(480, 640, 230, 250, 305 + g, 335 + g, 1000, g), RK) for g in range(G)}
    out.update(renders or {})
    return out


def box(render):
    return icp_oracle.model_bbox(render)


def edges_case():
    scene = noisy_scene(480, 640, 900, 1100, 1)
    r0, r5 = blob(480, 640, 230, 250, 305, 335), blob(480, 640, 236, 246, 315, 327, 1010, 5)
    renders = default_renders({0: (r0, RK), 5: (r5, K(500.0, 500.0, 320.0, 240.0))})
    surv = []
    for k, (x, y) in enumerate((x, y) for x in (0, 1, 3, 4, 5) for y in (0, 1, 3, 4, 5)):
        surv.append((x, y, 0 if k % 2 else 5))
    for g in (0, 5):
        _, _, bw, bh = box(renders[g][0])
        for d in (2, 1, 0):   # x + bw (y + bh) = cols - 2, cols - 1 (posed), cols (not posed)
            surv.append((640 - d - bw, 100, g))
            surv.append((100, 480 - d - bh, g))
            surv.append((640 - d - bw, 480 - d - bh, g))
    return Case("edges", scene, SK, renders, surv)


ANCHOR_XY = (100, 100)


def anchor_case():
    """Scene depths at the anchor (1000 mm) +- 400 mm and 1 mm either side under the box, the dilated ring's scene pixels
    non-zero, and a second survivor over an empty scene."""
    r = blob(480, 640, 230, 250, 305, 335)
    r[240, 320] = 1000
    scene = noisy_scene(480, 640, 900, 1100, 2)
    bx, by, bw, bh = box(r)
    x, y = ANCHOR_XY
    vals = np.array([600, 601, 1400, 1401, 599, 1000, 1399, 1402, 900], np.uint16)
    reg = scene[y - 4:y - 4 + bh, x - 4:x - 4 + bw]
    reg[...] = vals[np.arange(reg.size).reshape(reg.shape) % len(vals)]
    ex, ey = 300, 300
    scene[ey - 4:ey - 4 + bh, ex - 4:ex - 4 + bw] = 0
    return Case("anchor", scene, SK, default_renders({0: (r, RK)}), [(x, y, 0), (ex, ey, 0), (400, 20, 0)])


def renders_case(srows, scols):
    """Renders of 481 x 641, 240 x 320 and 480 x 640 (anchors at rows // 2, cols // 2, one where it differs from
    (rows - 1) // 2), one clipped at all four borders (a 240 x 320 box, more than 2^16 pixels), a one-pixel render (a
    9 x 9 box, zero anchor); render K unlike the scene's."""
    rng = np.random.default_rng(srows)
    scene = rng.integers(550, 1450, (srows, scols)).astype(np.uint16)
    scene[rng.random((srows, scols)) < 0.05] = 0
    big = np.zeros((481, 641), np.uint16)
    big[200:281, 280:361] = 1000 + (np.arange(81 * 81).reshape(81, 81) % 17)
    small = blob(240, 320, 100, 140, 140, 180, 990, 3)
    even = np.zeros((480, 640), np.uint16)
    rr, cc = np.mgrid[200:280, 280:360]
    even[200:280, 280:360] = 1000 + (rr * 5 + cc * 11) % 29   # render[240, 320] != render[239, 319]
    clipped = blob(240, 320, 0, 240, 0, 320, 1005, 4)
    clipped[60:180, 80:240] = 0                                # a frame of depth touching all four borders
    one = np.zeros((480, 640), np.uint16)
    one[100, 150] = 350
    Ks = [K(610.25, 590.75, 318.25, 241.75), K(305.5, 296.25, 160.5, 119.75), K(700.0, 650.0, 330.5, 230.25),
          K(300.0, 310.0, 161.25, 118.5), K(600.0, 600.0, 320.0, 240.0)]
    renders = default_renders({g: (r, k) for g, (r, k) in enumerate(zip((big, small, even, clipped, one), Ks))})
    surv = [(40, 30, 0), (200, 150, 0), (10, 300, 1), (300, 20, 2), (100, 100, 2), (5, 5, 3), (200, 100, 3), (0, 0, 4),
            (scols - 11, srows - 11, 4), (scols - 9, 7, 4)]
    return Case("renders_%dx%d" % (scols, srows), scene, SK, renders, surv)


def multiclass_case():
    """Three classes with distinct renders per class, classes 0 and 2 selected, survivors of both."""
    renders = {g: (blob(480, 640, 220 + 2 * g, 250 + g, 300 + 3 * g, 330 + 2 * g, 950 + 10 * g, g),
                   K(560.0 + g, 560.0 + 2 * g, 320.5, 240.5)) for g in range(G)}
    scene = noisy_scene(480, 640, 900, 1100, 3)
    surv = [(50, 60, 1), (150, 160, 3), (250, 60, 9), (350, 160, 10), (450, 260, 8), (50, 300, 0)]
    return Case("multiclass", scene, SK, renders, surv, select=[0, 2])


def voxel_case():
    """A 1.25 mm pitch plane across the principal point (points on voxel boundaries), a cloud wholly in one voxel whose
    sorted run covers indices 511 and 512, and a crop of more than 2^16 pixels."""
    plane = np.zeros((480, 640), np.uint16)
    plane[200:281, 260:381] = 250                               # f 200 at 0.25 m: 1.25 mm pitch, both sides of cx
    tiny = np.zeros((480, 640), np.uint16)
    tiny[220:253, 300:333] = 1000                               # 33 x 33 pixels of 0.02 mm: one voxel of 1089 points
    wide = blob(480, 640, 50, 330, 100, 400, 1000, 7)           # a 288 x 308 box: 88 704 pixels
    renders = default_renders({0: (plane, K(200.0, 200.0, 320.0, 240.0)), 1: (tiny, K(50000.0, 50000.0, 316.0, 236.0)),
                               2: (wide, RK)})
    scene = noisy_scene(480, 640, 240, 1100, 4, 0.0)
    scene[:, :320] = 250
    return Case("voxels", scene, SK, renders, [(100, 100, 0), (300, 300, 1), (10, 20, 2)])


def crafted_cases():
    return [edges_case(), anchor_case(), renders_case(480, 640), renders_case(720, 1280), multiclass_case(), voxel_case()]


def case_clouds(c, use_scene):
    """The model of every survivor of case c, in pick order."""
    return [pcm.clouds(c.scene, c.renders[g][0], c.sK, c.renders[g][1], x, y, use_scene) for x, y, g in c.surv]


# ---- the compaction limit -----------------------------------------------------------------------------------------
LIMIT_ROWS, LIMIT_COLS = 2359, 889          # 2359 * 889 = 2^21 - 1 (= 7^2 * 127 * 337)
LIMIT_FRAME = (2368, 912)                   # rows, cols


def limit_render():
    rr, cc = np.mgrid[0:LIMIT_ROWS, 0:LIMIT_COLS]
    return (1000 + (rr + cc) % 7).astype(np.uint16)


def limit_scene():
    rr, cc = np.mgrid[0:LIMIT_FRAME[0], 0:LIMIT_FRAME[1]]
    return (1000 + (3 * rr + cc) % 11).astype(np.uint16)


LIMIT_K = K(10000.0, 10000.0, 444.5, 1179.5)  # 0.1 mm pitch: ~600 pixels per voxel


# ---- the tests ----------------------------------------------------------------------------------------------------
def same_bits(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    if a.shape != b.shape:
        return False
    na, nb = np.isnan(a), np.isnan(b)
    return bool(np.array_equal(na, nb) and np.array_equal(a[~na].view(np.uint64), b[~nb].view(np.uint64)))


def against_oracle(scene, render, sK, mK, x, y):
    """The model against icp_oracle: clouds bit for bit, centroids up to summation order."""
    for use_scene in (False, True):
        m = pcm.clouds(scene, render, sK, mK, x, y, use_scene)
        if not m["posed"]:
            continue
        mp, cm, cs, sp = icp_oracle.build_clouds(scene, render, sK, mK, x, y, m["box"])
        assert same_bits(m["raw_model"], mp)
        assert same_bits(m["raw_scene"], sp if use_scene else np.zeros((0, 3)))
        with np.errstate(invalid="ignore"):
            want = cs - cm
        got = m["init"][:3, 3]
        assert np.array_equal(np.isnan(got), np.isnan(want))
        ok = ~np.isnan(want)
        assert np.all(np.abs(got[ok] - want[ok]) <= 1e-12 * (1 + np.abs(want[ok])))
        src = icp_oracle.voxel_down_sample(mp)
        assert m["source"].shape == src.shape and np.max(np.abs(m["source"] - src), initial=0) <= 1e-12
        if use_scene:
            assert m["target"].shape == icp_oracle.voxel_down_sample(sp).shape


CASES = {c.name: c for c in crafted_cases()}


@pytest.mark.parametrize("name", sorted(CASES))
def test_model_equals_the_oracle(name):
    c = CASES[name]
    for x, y, g in c.surv:
        against_oracle(c.scene, c.renders[g][0], c.sK, c.renders[g][1], x, y)


def test_model_equals_host_clouds_of_the_icp_cases():
    for c in ic.all_cases():
        m = pcm.clouds(c.scene, c.model, c.K, c.K, c.xy[0], c.xy[1], True)
        mp, _, _, sp = icp_oracle.build_clouds(c.scene, c.model, c.K, c.K, c.xy[0], c.xy[1], m["box"])
        assert same_bits(m["raw_model"], mp) and same_bits(m["raw_scene"], sp), c.name


def test_edges_reach_their_boundaries():
    c = CASES["edges"]
    posed = [m["posed"] for m in case_clouds(c, False)]
    xs = {x for x, _, _ in c.surv}
    assert {0, 1, 3, 4, 5} <= xs and {0, 1, 3, 4, 5} <= {y for _, y, _ in c.surv}
    reach = {}
    for (x, y, g), p in zip(c.surv, posed):
        _, _, bw, bh = box(c.renders[g][0])
        for v, ext in ((x + bw, 640), (y + bh, 480)):
            if v >= ext - 2:
                reach.setdefault(ext - v, set()).add(p)
    assert reach == {2: {True}, 1: {True}, 0: {False}}
    assert any(posed) and not all(posed)
    # survivors at x or y < 4 read the clamped scene column / row 0
    m = pcm.clouds(c.scene, c.renders[5][0], c.sK, c.renders[5][1], 0, 0, True)
    assert m["posed"] and m["raw_scene"].shape[0] > 0


def test_anchor_window_is_exact_at_both_ends():
    a = 1000 / 1000.0
    assert not abs(600 / 1000.0 - a) < 0.4 and abs(601 / 1000.0 - a) < 0.4     # 0.4 exactly: out
    assert abs(1400 / 1000.0 - a) < 0.4 and not abs(1401 / 1000.0 - a) < 0.4    # 0.3999...: in
    c = CASES["anchor"]
    ms = case_clouds(c, True)
    m = ms[0]
    assert m["anchor"] == 1.0
    z = np.rint(m["centroid_points"][:, 2] * 1000).astype(int)
    assert {601, 1000, 1399, 1400} <= set(z) and not {599, 600, 1401, 1402} & set(z)
    # ring pixels: scene points that are not centroid points, more of them than the out-of-window ones
    assert m["raw_scene"].shape[0] > m["raw_model"].shape[0] > m["centroid_points"].shape[0]
    # the empty scene: no scene point, NaN initial translation
    assert ms[1]["raw_scene"].shape[0] == 0 and np.all(np.isnan(ms[1]["init"][:3, 3]))


def test_renders_and_intrinsics():
    for name in ("renders_640x480", "renders_1280x720"):
        c = CASES[name]
        ms = case_clouds(c, False)
        assert all(m["posed"] for m in ms[:-1]) and not ms[-1]["posed"]
        shapes = {c.renders[g][0].shape for _, _, g in c.surv}
        assert {(481, 641), (240, 320), (480, 640)} <= shapes
        even = c.renders[2][0]
        assert even[240, 320] != even[239, 319]
        assert box(c.renders[3][0]) == (0, 0, 320, 240) and 320 * 240 > 1 << 16
        assert box(c.renders[4][0])[2:] == (9, 9) and c.renders[4][0][240, 320] == 0
        # the one-pixel render's anchor is 0: no scene depth lies within 0.4 m of it, the initial guess is NaN
        assert np.all(np.isnan(ms[7]["init"][:3, 3])) and ms[7]["raw_model"].shape[0] == 1


def test_multiclass_survivors_use_their_class_renders():
    c = CASES["multiclass"]
    classes = {g // PER_CLASS for _, _, g in c.surv}
    assert classes <= set(c.select) and len(classes) == 2
    # a lookup without class_begin would take another template's render
    for _, _, g in c.surv:
        t = g % PER_CLASS
        assert not np.array_equal(c.renders[g][0], c.renders[t][0]) or g == t


def test_voxel_edges():
    c = CASES["voxels"]
    plane, tiny, wide = case_clouds(c, False)
    raw = plane["raw_model"]
    assert (raw[:, 0] < 0).any() and (raw[:, 0] > 0).any()
    u = (raw[:, 0] - (raw[:, 0].min() - pcm.VOXEL / 2)) / pcm.VOXEL
    assert np.any(np.abs(u - np.rint(u)) < 1e-5)                  # points on voxel boundaries
    assert plane["source"].shape[0] < 0.6 * raw.shape[0]
    assert tiny["source"].shape[0] == 1 and tiny["raw_model"].shape[0] == 1089
    _, starts, counts = pcm.voxel_runs(tiny["raw_model"])
    assert np.any((starts <= 511) & (starts + counts > 512))       # a run straddles sorted index 511 / 512
    bx, by, bw, bh = box(c.renders[2][0])
    assert bw * bh > 1 << 16 and wide["posed"]


def test_compaction_limit_case():
    r = limit_render()
    bx, by, bw, bh = box(r)
    assert (bw, bh) == (LIMIT_COLS, LIMIT_ROWS) and bw * bh == (1 << 21) - 1
    scene = limit_scene()
    m = pcm.clouds(scene, r, SK, LIMIT_K, 10, 5, False)
    assert m["posed"] and m["raw_model"].shape[0] == m["centroid_points"].shape[0] == (1 << 21) - 1
    m = pcm.clouds(scene, r, SK, LIMIT_K, 10, 5, True)
    assert m["raw_scene"].shape[0] == (1 << 21) - 1 and m["source"].shape[0] < 20000
