"""RGB-D frames that put the quantization front-end exactly on its decision rules, and certify that they do.

Every count here is measured with cv2 and numpy on the frame itself, through the OpenCV calls of
6dpose_b200/frontend.py or the reference's loops restated plainly (LL.cpp), never with the GPU.  edge_frame asserts
each count against FLOORS and asserts that the frame's labels are not trivial at every pyramid level, so an edit that
makes a frame miss its edges fails where the frame is built.

Colour (LL.cpp:350-505):
  * gradient gate mag > 100: a texture of ramps with slopes near 1.25 px/px puts many pixels at squared magnitude 100
    with a passing vote.  A Sobel pair of a 3x3 window has dx = dy (mod 2), so squared magnitudes are even and 101 and
    102 cannot occur: the values next to the gate are 98, 100 and 104, and all three are counted;
  * channel ties: 12x12 patches of integer ramps, which the 7x7 blur leaves unchanged in their interior (the Sobel of
    slope s is 8 s).  Slopes (2, 1), (1, 2) and (-1, 2) share the squared magnitude 320 but fall in bins 1, 3 and 5, so
    the pick order of LL.cpp:395-412 decides the label: one patch kind per pair 0=1, 0=2, 1=2 and one with all three;
  * saturated 0/255 steps, whose Sobel responses reach the largest values a blurred u8 image gives;
  * votes: the texture's bins give 3x3 windows whose winning bin has exactly 5 votes and exactly 4.
Depth (LL.cpp:729-819):
  * flat planes at 1999 and 2000 mm and a ramp through both (the gate d < 2000);
  * flat steps of 49 and 50 mm in x and in y, whose neighbours at distance 5 differ by +-49 and +-50 (|delta| < 50);
  * zero-depth holes, and a block where half the pixels are holes, so 5x5 median windows hold exactly 12 and 13
    zeros; planes reach the frame's sides, so the rim of the normals (x < W - 6, y < H - 6) cuts objects.
  No depth lies in 1..49 mm: next to a zero-depth centre the reference indexes past NORMAL_LUT there.
Masks: nonzero values 1, 7 and 255; one band nonzero only on even (y, x), one only on odd (y, x), one full, one
empty.  The colour and depth masks swap the two lattices, so each level's nearest-neighbour decimation keeps one band
whole and drops the other.

An "observable" count is the number of pixels whose final label changes when the rule moves by one step (the gate,
a threshold, the pick order, the median rank, the pyrDown border, the decimated row): a kernel with that change fails
on the frame.
"""
import importlib

import cv2
import numpy as np

fe = importlib.import_module("6dpose_b200.frontend")

TILE_X, TILE_Y = 32, 8       # k_fe_gradient's tile; the other 2-D front-end kernels use the same 32x8 grid
INGEST_PX = 256              # pixels of a row per k_fe_ingest CTA
PATCH, PATCH_STEP = 12, 15   # tie / step patches: side and spacing
MASK_VALUES = (1, 7, 255)

# (ch0, ch1, ch2) slopes (sx, sy) of each patch kind
TIE_PATCHES = {
    "tie01": ((2, 1), (1, 2), (1, 0)),
    "tie02": ((2, 1), (1, 0), (1, 2)),
    "tie12": ((0, 1), (2, 1), (1, 2)),
    "tie012": ((2, 1), (1, 2), (-1, 2)),
}
PATCH_KINDS = list(TIE_PATCHES) + ["saturated"]

# floors of every edge count, met by the frame of every size in SHAPES
FLOORS = dict(
    gate98=4, gate100=20, gate104=4, gate100_observable=5, gate104_observable=2,
    tie01=16, tie02=16, tie12=16, tie012=16, pick_observable=16,
    saturated=20, vote4=20, vote5=20,
    depth1999=30, depth2000=30, depth2000_observable=10,
    delta_p50=20, delta_m50=20, delta_p49=20, delta_m49=20, delta50_observable=10, delta49_observable=10,
    holes=100, median_zeros12=3, median_zeros13=3, median_rank_observable=3, rim_x=10, rim_y=10,
)
MASK_FLOORS = dict(value1=20, value7=20, value255=20, even_lattice=20, odd_lattice=20, decimation_observable=20)
COLOR_FRACTION, NORMAL_FRACTION = 0.02, 0.30   # labelled share of every level, as tests/test_gpu_frontend.py requires

# (H, W, T) of the frames run through the GPU front-end: every one passes lm_upload_images' size rules, and together
# they put partial CTAs in x and in y, odd sources of pyrDown and of the decimation, and partial k_fe_ingest rows.
SHAPES = [
    (45, 80, [5]), (55, 80, [5]),          # odd rows, partial tiles in y (and in x)
    (65, 80, [5, 8]),                      # pyrDown and decimation from 65 rows
    (66, 96, [1, 3, 2, 4]),                # four levels, level 1 has 33 rows
    (60, 80, [2, 5]), (60, 48, [3, 6]),    # partial tiles in both dimensions at level 0
    (480, 640, [5, 8]),                    # the production size
]


def level_dims(H, W, levels):
    """(rows, cols) of every level: Size(cols / 2, rows / 2) per pyrDown (LL.cpp:564, 866)."""
    out = [(H, W)]
    for _ in range(1, levels):
        out.append((out[-1][0] // 2, out[-1][1] // 2))
    return out


def cta_facts(H, W, levels):
    """Where the front-end's grids leave partial CTAs and odd sources, per level of an H x W frame."""
    dims = level_dims(H, W, levels)
    return [dict(rows=r, cols=c, partial_x=c % TILE_X != 0, partial_y=r % TILE_Y != 0,
                 odd_source=l > 0 and (dims[l - 1][0] % 2 == 1 or dims[l - 1][1] % 2 == 1),
                 ingest_partial=l == 0 and c % INGEST_PX != 0)
            for l, (r, c) in enumerate(dims)]


# ---- colour ------------------------------------------------------------------------------------------------------
def _texture(rng, H, W, cell=10, slope=1.2, noise=0.5):
    yy, xx = np.mgrid[0:H, 0:W].astype(np.float32)
    img = np.zeros((H, W, 3), np.float32)
    for y0 in range(0, H, cell):
        for x0 in range(0, W, cell):
            a = rng.uniform(0, 2 * np.pi, 3)
            s = slope * rng.uniform(0.8, 1.2, 3)
            ys, xs = yy[y0:y0 + cell, x0:x0 + cell] - y0 - cell / 2, xx[y0:y0 + cell, x0:x0 + cell] - x0 - cell / 2
            for c in range(3):
                img[y0:y0 + cell, x0:x0 + cell, c] = 128 + s[c] * (np.cos(a[c]) * xs + np.sin(a[c]) * ys)
    img += rng.normal(0, noise, img.shape)
    return np.clip(np.rint(img), 0, 255).astype(np.uint8)


def patch_origins(H, W):
    """(kind, y0, x0) of the patches: rows and columns PATCH_STEP apart, the kinds rotating so that a small frame holds
    every kind."""
    out = []
    for k, y0 in enumerate(range(2, H - PATCH - 1, 2 * PATCH_STEP)):
        for j, x0 in enumerate(range(2, W - PATCH - 1, PATCH_STEP)):
            out.append((PATCH_KINDS[(j + 3 * k) % len(PATCH_KINDS)], y0, x0))
    return out


def color_image(H, W, seed=0):
    img = _texture(np.random.default_rng(seed), H, W)
    yy, xx = np.mgrid[0:PATCH, 0:PATCH] - PATCH // 2
    for kind, y0, x0 in patch_origins(H, W):
        p = img[y0:y0 + PATCH, x0:x0 + PATCH]
        if kind == "saturated":
            p[..., 0] = np.where(xx < 0, 0, 255)
            p[..., 1] = np.where(yy < 0, 255, 0)
            p[..., 2] = np.where(xx + yy < 0, 0, 255)
        else:
            for c, (sx, sy) in enumerate(TIE_PATCHES[kind]):
                p[..., c] = 128 + sx * xx + sy * yy
    return img


def color_parts(src):
    """The first steps of frontend.quantize_color (the same cv2 calls): per-channel Sobel dx, dy of the blurred image
    and their squared magnitudes, int32 H x W x 3."""
    sm = cv2.GaussianBlur(src, (7, 7), 0, 0, borderType=cv2.BORDER_REPLICATE)
    dx3 = cv2.Sobel(sm, cv2.CV_16S, 1, 0, ksize=3, borderType=cv2.BORDER_REPLICATE).astype(np.int32)
    dy3 = cv2.Sobel(sm, cv2.CV_16S, 0, 1, ksize=3, borderType=cv2.BORDER_REPLICATE).astype(np.int32)
    mag3 = dx3 * dx3 + dy3 * dy3
    return dx3, dy3, mag3


def _pick(dx3, dy3, mag3, order):
    """The strongest channel, ties to the first of `order` (LL.cpp:395-412 is order (0, 1, 2))."""
    best = mag3.max(2)
    idx = np.full(best.shape, order[-1])
    for c in reversed(order):
        idx = np.where(mag3[..., c] == best, c, idx)
    i = idx[..., None]
    dx = np.take_along_axis(dx3, i, 2)[..., 0].astype(np.float32)
    dy = np.take_along_axis(dy3, i, 2)[..., 0].astype(np.float32)
    return np.take_along_axis(mag3, i, 2)[..., 0].astype(np.float32), cv2.phase(dx, dy, angleInDegrees=True)


def bins(angle):
    """The bin image hysteresisGradient votes over: LL.cpp:427-440 (frontend._hysteresis's q)."""
    q = np.clip(np.rint(angle.astype(np.float32) * np.float32(16.0 / 360.0)), 0, 255).astype(np.uint8)
    q[0, :] = q[-1, :] = 0
    q[:, 0] = q[:, -1] = 0
    q[1:-1, 1:-1] &= 7
    return q


def votes(q):
    """Winning vote count of each interior pixel's 3x3 window (LL.cpp:457-505's loop); 0 on the border."""
    H, W = q.shape
    best = np.zeros((H, W), np.int32)
    for b in range(8):
        e = (q == b).astype(np.int32)
        acc = sum(e[1 + dy:H - 1 + dy, 1 + dx:W - 1 + dx] for dy in (-1, 0, 1) for dx in (-1, 0, 1))
        best[1:-1, 1:-1] = np.maximum(best[1:-1, 1:-1], acc)
    return best


def color_classes(src):
    """Per-pixel maps of the colour edge classes of one level's image, and the labels (frontend.quantize_color)."""
    H, W = src.shape[:2]
    dx3, dy3, mag3 = color_parts(src)
    mag, angle = _pick(dx3, dy3, mag3, (0, 1, 2))
    labels = fe._hysteresis(mag, angle, np.float32(100.0))
    inner = np.zeros((H, W), bool)
    inner[1:-1, 1:-1] = True
    v = votes(bins(angle))
    strong = inner & (mag > 100)
    cls = {"gate%d" % g: inner & (mag == g) for g in (98, 100, 104)}
    cls["gate100_observable"] = fe._hysteresis(mag, angle, np.float32(99.0)) != labels      # mag >= 100
    cls["gate104_observable"] = fe._hysteresis(mag, angle, np.float32(104.0)) != labels     # mag > 104
    top = mag3.max(2)
    tie = [mag3[..., c] == top for c in range(3)]
    b3 = [bins(cv2.phase(dx3[..., c].astype(np.float32), dy3[..., c].astype(np.float32), angleInDegrees=True))
          for c in range(3)]
    differ = lambda a, b: b3[a] != b3[b]
    cls["tie01"] = inner & tie[0] & tie[1] & ~tie[2] & differ(0, 1)
    cls["tie02"] = inner & tie[0] & tie[2] & ~tie[1] & differ(0, 2)
    cls["tie12"] = inner & tie[1] & tie[2] & ~tie[0] & differ(1, 2)
    cls["tie012"] = inner & tie[0] & tie[1] & tie[2] & differ(0, 1) & differ(1, 2) & differ(0, 2)
    m1, a1 = _pick(dx3, dy3, mag3, (1, 0, 2))     # the first two branches of the pick swapped
    cls["pick_observable"] = fe._hysteresis(m1, a1, np.float32(100.0)) != labels
    cls["saturated"] = inner & (np.maximum(np.abs(dx3), np.abs(dy3)).max(2) >= 400)
    cls["vote4"] = strong & (v == 4)     # labelled by best >= 4
    cls["vote5"] = strong & (v == 5)     # labelled here, dropped by best > 5
    return cls, labels


# ---- depth -------------------------------------------------------------------------------------------------------
DEPTH_CELL = 16
DEPTH_KINDS = ["flat1999", "flat2000", "ramp2000", "step_x50", "step_y50", "step_x49", "step_y49", "half_holes", "plane"]


def depth_image(H, W, seed=0):
    """Cells of DEPTH_CELL px in raster order, each one kind of DEPTH_KINDS (rotating), on tilted planes; plus sparse
    holes.  Every value is 0 or >= 50."""
    rng = np.random.default_rng(seed + 1)
    d = np.zeros((H, W), np.int64)
    i = 0
    for y0 in range(0, H, DEPTH_CELL):
        for x0 in range(0, W, DEPTH_CELL):
            y1, x1 = min(y0 + DEPTH_CELL, H), min(x0 + DEPTH_CELL, W)
            yy, xx = np.mgrid[y0:y1, x0:x1]
            ly, lx = yy - y0, xx - x0
            kind = DEPTH_KINDS[i % len(DEPTH_KINDS)]
            i += 1
            base = int(rng.integers(600, 1600))
            if kind == "flat1999":
                c = np.full(yy.shape, 1999)
            elif kind == "flat2000":
                c = np.full(yy.shape, 2000)
            elif kind == "ramp2000":
                c = 1992 + lx                               # 1992 .. 2007 across the cell
            elif kind.startswith("step"):
                h = int(kind[-2:])
                c = base + h * ((lx if kind[5] == "x" else ly) >= DEPTH_CELL // 2)
            elif kind == "half_holes":
                c = np.where(rng.random(yy.shape) < 0.5, 0, base)
            else:
                gx, gy = rng.integers(-4, 5, 2)
                c = base + gx * lx + gy * ly
            d[y0:y1, x0:x1] = c
    d[rng.random((H, W)) < 0.04] = 0
    assert d.min() >= 0 and d.max() < 65536
    return d.astype(np.uint16)


def _windows(a, r):
    """(2r+1)^2 shifted copies of a with BORDER_REPLICATE, stacked on the last axis."""
    p = np.pad(a, r, mode="edge")
    H, W = a.shape
    return np.stack([p[dy:dy + H, dx:dx + W] for dy in range(2 * r + 1) for dx in range(2 * r + 1)], -1)


def median_rank(labels, k):
    """The k-th smallest (1-based) of each 5x5 BORDER_REPLICATE window: k = 13 is cv2.medianBlur(labels, 5)."""
    return np.sort(_windows(labels, 2), -1)[..., k - 1]


def depth_classes(depth):
    H, W = depth.shape
    d = depth.astype(np.int64)
    labels = fe.quantize_depth(depth)
    raw = fe.normals_before_median(depth)
    inner = np.zeros((H, W), bool)
    inner[5:H - 6, 5:W - 6] = True
    cls = {"depth1999": inner & (d == 1999), "depth2000": inner & (d == 2000)}
    cls["depth2000_observable"] = fe.quantize_depth(depth, 2001, 50) != labels       # d <= 2000
    p = np.pad(d, 5)
    for h in (50, 49):
        for s, name in ((1, "p"), (-1, "m")):
            hit = np.zeros((H, W), bool)
            for dy in (-5, 0, 5):
                for dx in (-5, 0, 5):
                    if dy or dx:
                        hit |= p[5 + dy:5 + dy + H, 5 + dx:5 + dx + W] - d == s * h
            cls["delta_%s%d" % (name, h)] = inner & (d > 0) & (d < 2000) & hit
    cls["delta50_observable"] = fe.quantize_depth(depth, 2000, 51) != labels          # |delta| <= 50
    cls["delta49_observable"] = fe.quantize_depth(depth, 2000, 49) != labels          # |delta| < 49
    cls["holes"] = d == 0
    zeros = (_windows(raw, 2) == 0).sum(-1)
    cls["median_zeros12"] = zeros == 12
    cls["median_zeros13"] = zeros == 13
    cls["median_rank_observable"] = median_rank(raw, 12) != labels                    # the 12th element
    valid = (d >= 50) & (d < 2000)
    rim_x = np.zeros((H, W), bool)
    rim_y = np.zeros((H, W), bool)
    if W > 6:
        rim_x[5:H - 6, W - 6] = True
    if H > 6:
        rim_y[H - 6, 5:W - 6] = True
    cls["rim_x"] = rim_x & valid
    cls["rim_y"] = rim_y & valid
    # out of scope: a zero-depth centre with a 1..49 mm neighbour at distance 5
    small = (d > 0) & (d < 50)
    assert not small.any(), "depths of 1..49 mm"
    return cls, labels


# ---- masks -------------------------------------------------------------------------------------------------------
def mask_image(H, W, even_first):
    """Four bands over x: nonzero only on even (y, x), only on odd (y, x) (swapped when not even_first), everywhere, and
    nowhere; nonzero values cycle through MASK_VALUES."""
    yy, xx = np.mgrid[0:H, 0:W]
    band = np.minimum(4 * xx // W, 3)
    even = (yy % 2 == 0) & (xx % 2 == 0)
    odd = (yy % 2 == 1) & (xx % 2 == 1)
    lattice = [even, odd] if even_first else [odd, even]
    on = np.where(band == 0, lattice[0], np.where(band == 1, lattice[1], band == 2))
    val = np.asarray(MASK_VALUES, np.uint8)[(xx // 2 + yy // 2 + xx + yy) % 3]
    return np.where(on, val, 0).astype(np.uint8)


MASK_KINDS = (None, "color", "depth", "both")


def masks_of(H, W, kind):
    """[mask_color, mask_depth] of a mask kind (None: no masks)."""
    if kind is None:
        return None
    m0 = mask_image(H, W, True) if kind in ("color", "both") else None
    m1 = mask_image(H, W, False) if kind in ("depth", "both") else None
    return [m0, m1]


def mask_counts(mask):
    H, W = mask.shape
    yy, xx = np.mgrid[0:H, 0:W]
    on = mask != 0
    out = {"value%d" % v: int((mask == v).sum()) for v in MASK_VALUES}
    out["even_lattice"] = int((on & (yy % 2 == 0) & (xx % 2 == 0) & (xx < W // 2)).sum())
    out["odd_lattice"] = int((on & (yy % 2 == 1) & (xx % 2 == 1) & (xx < W // 2)).sum())
    half = cv2.resize(mask, (W // 2, H // 2), interpolation=cv2.INTER_NEAREST)
    out["decimation_observable"] = int((half != mask[1::2, ::2][:H // 2, :W // 2]).sum())   # row 2y+1 read for 2y
    return out


# ---- frames ------------------------------------------------------------------------------------------------------
def level_sources(rgb, levels):
    """The colour image of every level (cv2.pyrDown, as ColorGradientPyramid::pyrDown)."""
    out = [rgb]
    for _ in range(1, levels):
        s = out[-1]
        out.append(cv2.pyrDown(s, dstsize=(s.shape[1] // 2, s.shape[0] // 2)))
    return out


def edge_counts(rgb, depth):
    cc, _ = color_classes(rgb)
    dc, _ = depth_classes(depth)
    return {k: int(v.sum()) for k, v in {**cc, **dc}.items()}


def pyramid_border_observable(rgb, levels):
    """Level-1 colour labels that change when pyrDown replicates the border instead of reflecting it (101)."""
    if levels < 2:
        return 0
    size = (rgb.shape[1] // 2, rgb.shape[0] // 2)
    a = fe.quantize_color(cv2.pyrDown(rgb, dstsize=size))[0]
    b = fe.quantize_color(cv2.pyrDown(rgb, dstsize=size, borderType=cv2.BORDER_REPLICATE))[0]
    return int((a != b).sum())


def certify(counts, floors):
    short = {k: (counts[k], f) for k, f in floors.items() if counts[k] < f}
    assert not short, "edge counts below their floors (count, floor): %s" % short


def edge_frame(H, W, levels, masks=None, seed=0):
    """(rgb, depth, masks, counts) of an H x W frame for a pyramid of `levels`; masks is one of MASK_KINDS.  Asserts
    every count of FLOORS (and MASK_FLOORS for each mask given) and that every level's labels are not trivial."""
    rgb, depth = color_image(H, W, seed), depth_image(H, W, seed)
    mk = masks_of(H, W, masks)
    counts = edge_counts(rgb, depth)
    certify(counts, FLOORS)
    if levels > 1:
        counts["pyrdown_border_observable"] = pyramid_border_observable(rgb, levels)
        certify(counts, {"pyrdown_border_observable": 5})
    for i, m in enumerate(mk or []):
        if m is not None:
            c = mask_counts(m)
            certify(c, MASK_FLOORS)
            counts.update({"mask%d_%s" % (i, k): v for k, v in c.items()})
    q = fe.quantize_pyramid([rgb, depth], levels)
    for l, (qc, qn) in enumerate(q):
        counts["level%d_color_fraction" % l] = float((qc > 0).mean())
        counts["level%d_normal_fraction" % l] = float((qn > 0).mean())
        assert (qc > 0).mean() > COLOR_FRACTION and (qn > 0).mean() > NORMAL_FRACTION, (l, counts)
    return rgb, depth, mk, counts


def pixel_classes(rgb, depth, masks, level, modality, y, x):
    """Names of the edge classes pixel (y, x) of `level` belongs to: colour classes of that level's image; depth
    classes of the level-0 pixel it is decimated from; mask values; a partial CTA of the level."""
    names = []
    if modality == 0:
        src = level_sources(rgb, level + 1)[level]
        cls, _ = color_classes(src)
        H, W = src.shape[:2]
        names += [k for k, v in cls.items() if v[y, x]]
        if level > 0:
            up = level_sources(rgb, level)[level - 1]
            size = (up.shape[1] // 2, up.shape[0] // 2)
            if fe.quantize_color(cv2.pyrDown(up, dstsize=size, borderType=cv2.BORDER_REPLICATE))[0][y, x] != \
                    fe.quantize_color(src)[0][y, x]:
                names.append("pyrdown_border_observable")
    else:
        cls, _ = depth_classes(depth)
        H, W = depth.shape[0] >> level, depth.shape[1] >> level
        names += [k for k, v in cls.items() if v[y << level, x << level]]
        if level > 0:
            up = fe.quantize_pyramid([rgb, depth], level)[level - 1][1]
            if up[2 * y, 2 * x] != up[2 * y + 1, 2 * x]:
                names.append("decimation_row_observable")
    if masks and masks[modality] is not None:
        names.append("mask=%d" % masks[modality][y << level, x << level])
    if x >= W // TILE_X * TILE_X or y >= H // TILE_Y * TILE_Y:
        names.append("partial_tile")
    if y < 5 or x < 5 or y >= H - 6 or x >= W - 6:
        names.append("within 6 px of a side")
    return names or ["none"]
