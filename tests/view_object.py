"""A synthetic asymmetric rigid solid for view following (include/linemod_b200.h, lm_set_track_views): an L-shaped block
with a cylinder on one face, as a dense surface sample with outward normals.  A view renders the faces turned to the
camera (back-face culling) with a nearest-depth z-buffer splat, as tests/pso_scenes.py splats.  It provides template
renders on a view sphere with in-plane tilts (K, R_b, t_b each) and a sequence of scenes of the solid turning over a
table plane, with the true pose of every frame.  Poses map object coordinates (metres) into the camera: p = R x + b."""
import numpy as np

import pso_scenes

ROWS, COLS = 240, 320
K = np.array([[290.0, 0.0, 160.0], [0.0, 290.0, 120.0], [0.0, 0.0, 1.0]])
DIST_MM = 600.0
STEP_MM = 0.6  # surface sample spacing


def _box(lo, hi):
    """Surface samples and normals of an axis-aligned box [lo, hi] (mm)."""
    pts, nrm = [], []
    lo, hi = np.asarray(lo, float), np.asarray(hi, float)
    for ax in range(3):
        u, v = [a for a in range(3) if a != ax]
        gu = np.arange(lo[u], hi[u] + 1e-9, STEP_MM)
        gv = np.arange(lo[v], hi[v] + 1e-9, STEP_MM)
        U, V = np.meshgrid(gu, gv, indexing="ij")
        for side, val in ((-1.0, lo[ax]), (1.0, hi[ax])):
            p = np.zeros((U.size, 3))
            p[:, u], p[:, v], p[:, ax] = U.ravel(), V.ravel(), val
            n = np.zeros_like(p)
            n[:, ax] = side
            pts.append(p)
            nrm.append(n)
    return np.concatenate(pts), np.concatenate(nrm)


def _inside(p, lo, hi):
    return np.all((p > np.asarray(lo) + 1e-6) & (p < np.asarray(hi) - 1e-6), 1)


def solid():
    """(points [n,3] m, normals [n,3]) of the L-block (a 90 x 50 x 30 mm slab, a 30 x 50 x 40 mm upright at one end) with
    a cylinder (radius 10 mm, length 30 mm) standing out of the slab's -y face, centred near the origin."""
    A = ([-45, -25, -15], [45, 25, 15])
    B = ([15, -25, 15], [45, 25, 55])
    pa, na = _box(*A)
    pb, nb = _box(*B)
    keep_a = ~(_inside(pa, [B[0][0], B[0][1], B[0][2] - 1], B[1]) | ((pa[:, 2] == 15) & (pa[:, 0] > 15)))
    keep_b = ~((pb[:, 2] == 15))
    th = np.arange(0, 2 * np.pi, STEP_MM / 10.0)
    ys = np.arange(-55, -25 + 1e-9, STEP_MM)
    TH, Y = np.meshgrid(th, ys, indexing="ij")
    pc = np.stack([-20 + 10 * np.cos(TH.ravel()), Y.ravel(), 10 * np.sin(TH.ravel())], 1)
    nc = np.stack([np.cos(TH.ravel()), np.zeros(TH.size), np.sin(TH.ravel())], 1)
    r = np.arange(0, 10 + 1e-9, STEP_MM)
    R, TH2 = np.meshgrid(r, th, indexing="ij")
    cap = np.stack([-20 + R.ravel() * np.cos(TH2.ravel()), np.full(R.size, -55.0), R.ravel() * np.sin(TH2.ravel())], 1)
    keep_a &= ~(((pa[:, 0] + 20) ** 2 + pa[:, 2] ** 2 < 100) & (pa[:, 1] == -25))
    pts = np.concatenate([pa[keep_a], pb[keep_b], pc, cap])
    nrm = np.concatenate([na[keep_a], nb[keep_b], nc, np.tile([0.0, -1.0, 0.0], (len(cap), 1))])
    pts = pts - pts.mean(0)
    return pts / 1000.0, nrm


PTS, NRM = solid()


def visible(R, b):
    """The surface samples facing a camera that sees the object at pose (R, b): camera-frame points (m)."""
    p = PTS @ R.T + b
    n = NRM @ R.T
    return p[(n * p).sum(1) < 0]


def render(R, b, table=None):
    """u16 mm depth of the solid at pose (R, b) (b in m), over a table (mm per pixel; None: empty background)."""
    bg = np.full((ROWS, COLS), 65535.0) if table is None else table
    z = pso_scenes.splat(visible(R, b), K, ROWS, COLS, bg)
    return np.where(z == 65535, 0, z).astype(np.uint16)


def look(d):
    """A rotation whose camera looks at the object from direction d (object frame): R maps d onto -z."""
    d = np.asarray(d, float) / np.linalg.norm(d)
    up = np.array([0.0, 0.0, 1.0]) if abs(d[2]) < 0.9 else np.array([0.0, 1.0, 0.0])
    x = np.cross(up, d)
    x /= np.linalg.norm(x)
    y = np.cross(d, x)
    return np.stack([x, y, -d])  # rows: the camera axes in object coordinates


def templates(n_views=42, tilts=(-30.0, -15.0, 0.0, 15.0, 30.0)):
    """Template poses on a Fibonacci view sphere with in-plane tilts: R_b [G,3,3] f32, t_b [G,3] f32 (mm, on the optical
    axis at DIST_MM), K [G,3,3] f32."""
    i = np.arange(n_views) + 0.5
    phi = np.arccos(1 - 2 * i / n_views)
    th = np.pi * (1 + 5 ** 0.5) * i
    dirs = np.stack([np.cos(th) * np.sin(phi), np.sin(th) * np.sin(phi), np.cos(phi)], 1)
    R = []
    for d in dirs:
        for a in tilts:
            R.append(pso_scenes.rodrigues(np.radians([0, 0, a])) @ look(d))
    R = np.asarray(R, np.float32)
    G = len(R)
    return R, np.tile(np.array([0, 0, DIST_MM], np.float32), (G, 1)), np.repeat(K[None].astype(np.float32), G, 0)


def template_render(R_b, t_b):
    return render(np.asarray(R_b, np.float64), np.asarray(t_b, np.float64) / 1000.0)


TABLE = (DIST_MM + 70.0) + 0.15 * (np.mgrid[0:ROWS, 0:COLS][0] - ROWS / 2)


def sequence(R_start, frames=40, step_deg=2.5, axis=(0.3, 1.0, 0.2)):
    """Scenes of the solid turning by step_deg per frame about `axis` (camera frame) from R_start and drifting 0.3 mm
    per frame, over TABLE: [(scene u16, R_true, b_true m)] for frames 0..frames."""
    w = np.asarray(axis, float) / np.linalg.norm(axis)
    out = []
    for f in range(frames + 1):
        R = pso_scenes.rodrigues(w * np.radians(step_deg * f)) @ R_start
        b = np.array([0.3 * f, -0.2 * f, DIST_MM]) / 1000.0
        out.append((render(R, b, TABLE), R, b))
    return out


def start_T(R_true, b_true, R_b, t_b):
    """The T that maps the template's render cloud (R_b, t_b mm) onto the object at (R_true, b_true m)."""
    Rb = np.asarray(R_b, np.float64)
    bb = np.asarray(t_b, np.float64) / 1000.0
    T = np.eye(4)
    T[:3, :3] = R_true @ Rb.T
    T[:3, 3] = b_true - T[:3, :3] @ bb
    return T


def errors(T, R_b, t_b, R_true, b_true):
    """(rotation error deg, position error mm) of the object pose T [R_b | t_b / 1000] against the truth."""
    P = np.eye(4)
    P[:3, :3], P[:3, 3] = np.asarray(R_b, np.float64), np.asarray(t_b, np.float64) / 1000.0
    E = np.asarray(T, np.float64) @ P
    dR = E[:3, :3] @ R_true.T
    ang = np.degrees(np.arccos(np.clip((np.trace(dR) - 1) / 2, -1, 1)))
    return float(ang), float(np.linalg.norm(E[:3, 3] - b_true) * 1000.0)
