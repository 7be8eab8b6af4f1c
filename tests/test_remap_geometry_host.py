"""Rectified and registered pyramids where the input, depth and colour geometries differ, on the CPU.

The rectifier (k_rectify) reads frames of in_w x in_h and writes w x h; the depth registration (k_register_scatter,
k_register_finish) reads dw x dh depth and a (dw+1) x (dh+1) corner-ray table and writes w x h; the create stages all of
them in sections sized from each (stage_layout in csrc/capi.cu).  When every size is the same, a swap of two of them is
invisible.  GEOMETRIES below are the cases where they differ, each with a stated reason that assert_reason() checks from
the geometry (and, where the reason is about footprints or the map, from the model's numbers) before any test relies on it;
tests/test_gpu_remap_geometry.py holds the kernels to the float32 models at these geometries.  Here, without a GPU:

  reasons        every geometry's stated case holds
  rectified      the model's intensity against an fp64 bilinear of the same taps within its forward-error bound, its
                 depth exactly the nearest tap, its validity and four-tap mask from fp64 comparisons
  registered     the model's depth against an independent fp64 reprojection (as tests/test_registration_host.py) at the
                 new depth cameras and targets
  footprints     shadows, empty footprints and footprints over DVO_B200_REGISTRATION_MAX_FOOTPRINT occur where the
                 geometry says they must, and leave the colour pixels only they cover empty
"""
import dataclasses
import functools

import numpy as np
import pytest

import rectify_model as rm
import registration_model as rg
from launch_plan_model import COARSE_TILES, level_geometry
from test_gpu_geometry import SIZES, _assert_reason, _intrinsics
from tile_geometry import TILE_H, TILE_W, bands, level_shapes, strips

N = 3                      # frames per batch: a per-image stride mix-up cannot hide in image 0
DEPTH_SCALE = 1.0 / 5000.0
FR1 = (517.3, 516.5, 318.6, 255.3)
LENS = (0.09, -0.21, 0.0012, -0.0008, 0.11)               # a mild barrel lens of a 16:9 colour camera
KV2 = (365.5, 365.5, 257.0, 206.0)                        # a Kinect-v2-like 512 x 424 time-of-flight camera
KV2_DIST = (0.0905, -0.2688, 0.0, 0.0, 0.0938)


def _T(tx, ty=0.0, tz=0.0, rx=0.0, ry=0.0, rz=0.0):
    """T_color_depth as nested tuples, so that a Geometry hashes"""
    from dvo_slam_b200 import synth
    return tuple(map(tuple, synth.se3_exp(np.array([tx, ty, tz, rx, ry, rz]))))


@dataclasses.dataclass(frozen=True)
class Geometry:
    """One create's geometry.  Colour frames of in_size with intrinsics K_in and lens dist (None: pinhole); level 0 of
    size with intrinsics K and `levels` levels.  rect: the frames go through a rectifier whose map is
    rm.undistort_map(size, K_in, dist, K_new = K).  depth: None (depth comes with the colour frames) or (dw, dh, K_d,
    dist_d, T_color_depth) of a depth camera registered into level 0."""
    name: str
    in_size: tuple
    K_in: tuple
    dist: tuple | None
    size: tuple
    K: tuple
    levels: int
    rect: bool
    depth: tuple | None = None
    seed: int = 0

    @property
    def map(self):
        return _map(self)


def _sizes_geometry(w, h, levels):
    """level 0 of a test_gpu_geometry.SIZES size from colour frames 1.5 times larger, through a rectifier whose view is a
    little wider than the frames' (NaN borders)"""
    s = max(w, h)
    return Geometry(f"sizes-{w}x{h}", (w + w // 2 + 1, h + h // 2 + 1), _intrinsics(w + w // 2 + 1, h + h // 2 + 1), None, (w, h),
                    (0.78 * s, 0.78 * s + 0.5, 0.47 * w + 0.3, 0.52 * h - 0.2), levels, True, seed=w * 1000 + h)


DOWN = Geometry("down-1280x720-640x360", (1280, 720), (930.0, 929.0, 641.3, 358.2), LENS, (640, 360),
                (465.0, 464.5, 320.4, 179.6), 5, True, seed=1)
RECTIFIED = [
    DOWN,
    Geometry("up-320x240-640x480", (320, 240), tuple(v / 2 for v in FR1), None, (640, 480), FR1, 5, True, seed=2),
    Geometry("crop-661x493-641x481", (661, 493), (600.0, 601.0, 331.4, 245.9), (0.05, 0.02, 0.0005, 0.0003, 0.0), (641, 481),
             (600.0, 601.0, 310.9, 239.6), 5, True, seed=3),
    Geometry("tall-400x300-264x360", (400, 300), (330.0, 330.5, 199.2, 150.3), None, (264, 360),
             (330.0 / 0.86, 330.5 / 0.86, 131.6, 179.8), 4, True, seed=4),
] + [_sizes_geometry(*s) for s in SIZES]
REGISTERED = [
    Geometry("kinect-512x424-960x540", (960, 540), (700.0, 699.5, 481.2, 268.9), None, (960, 540), (700.0, 699.5, 481.2, 268.9), 5,
             False, (512, 424, KV2, KV2_DIST, _T(0.052, 0.002, -0.003, 0.003, -0.004, 0.002)), seed=6),
    Geometry("odd-203x157-161x50", (161, 50), _intrinsics(161, 50), None, (161, 50), _intrinsics(161, 50), 3, False,
             (203, 157, (150.0, 150.5, 101.3, 78.6), None, _T(0.02, 0.0, 0.0, 0.0, 0.004, 0.0)), seed=7),
    Geometry("odd-203x157-223x49", (223, 49), _intrinsics(223, 49), None, (223, 49), _intrinsics(223, 49), 3, False,
             (203, 157, (150.0, 150.5, 101.3, 78.6), None, _T(-0.02, 0.005, 0.0, 0.0, 0.0, 0.003)), seed=8),
    Geometry("coarse-80x60-640x480", (640, 480), FR1, None, (640, 480), FR1, 5, False,
             (80, 60, (63.4, 63.3, 39.5, 29.4), None, _T(0.01, 0.0, 0.0, 0.0, 0.002, 0.0)), seed=9),
    Geometry("rectified-1280x720-reg-424x240-640x360", DOWN.in_size, DOWN.K_in, DOWN.dist, DOWN.size, DOWN.K, 5, True,
             (424, 240, (310.0, 310.5, 211.7, 119.4), None, _T(0.03, 0.0, 0.001, 0.002, 0.0, -0.001)), seed=10),
]
GEOMETRIES = RECTIFIED + REGISTERED
BY_NAME = {g.name: g for g in GEOMETRIES}
IDS = [g.name for g in GEOMETRIES]


@functools.lru_cache(maxsize=None)
def _map(g):
    return rm.undistort_map(g.size[0], g.size[1], g.K_in, g.dist or (0, 0, 0, 0, 0), g.K)


@functools.lru_cache(maxsize=None)
def rays(g):
    dw, dh, K_d, dist_d, _ = g.depth
    return rg.depth_rays((dw, dh), K_d, dist_d)


def _scene_config(g, holes=True):
    from dvo_slam_b200 import synth
    dc = None
    if g.depth is not None:
        dw, dh, K_d, dist_d, T = g.depth
        dc = synth.DepthCamera(dw, dh, K_d, T, dist_d)
    return synth.SceneConfig(width=g.in_size[0], height=g.in_size[1], intrinsics=g.K_in, distortion=g.dist, depth_camera=dc,
                             hole_fraction=0.03 if holes else 0.0)


@functools.lru_cache(maxsize=None)
def frames(g, holes=True):
    """N frames (a reference, its current frame, another reference) of g's colour camera in every host representation, their
    depth (the colour camera's own, or the depth camera's, float metres and raw), a blob mask per frame in the colour
    frames' geometry, and the pose between the first two"""
    from dvo_slam_b200 import synth
    cfg = _scene_config(g, holes)
    p, q = synth.make_pair(100 + 2 * g.seed, cfg), synth.make_pair(101 + 2 * g.seed, cfg)
    I = np.stack([p["I_ref"].numpy(), p["I_cur"].numpy(), q["I_ref"].numpy()]).astype(np.float32)
    Z = np.stack([p["Z_ref"].numpy(), p["Z_cur"].numpy(), q["Z_ref"].numpy()]).astype(np.float32)
    n, h, w = I.shape
    rng = np.random.default_rng(g.seed)
    yy, xx = np.ogrid[:h, :w]
    M = np.ones((n, h, w), np.uint8)
    for i in range(n):
        for _ in range(8):
            cy, cx, r = rng.integers(0, h), rng.integers(0, w), rng.integers(2, max(3, min(w, h) // 6))
            M[i][(yy - cy) ** 2 + (xx - cx) ** 2 <= r * r] = 0
    return {"float": (I, Z), "grey": np.clip(I, 0, 255).astype(np.uint8),
            "raw": np.where(np.isnan(Z), 0, np.round(Z * 5000.0)).astype(np.uint16),
            "bgr": rng.integers(0, 256, (n, h, w, 3), dtype=np.uint8), "masks": M, "T": p["T_true"]}


def inputs(f, fmt):
    """(image, depth) host arrays of one input format"""
    image = {"float32": f["float"][0], "grey8_depth16": f["grey"], "bgr8_depth16": f["bgr"]}[fmt]
    depth = f["float"][1] if fmt == "float32" else f["raw"]
    return image, depth


def model_planes(g, fmt, masked):
    """the float32 level-0 planes (I, Z, M) the create builds from, by the models; M None without masks"""
    f = frames(g)
    image, depth = inputs(f, fmt)
    masks = f["masks"] if masked else None
    scale = None if fmt == "float32" else DEPTH_SCALE
    if g.depth is None:
        return rm.remap_batch(image, depth, *g.map, masks, scale)
    return rg.register_batch(image, depth, rays(g), g.depth[4], g.size, g.K, masks, scale, g.map if g.rect else None)


def stage_bytes(g, fmt, masked, device):
    """the create's staging bytes for N frames (restating stage_layout of csrc/capi.cu): the uploaded depth, image and
    masks (host forms), the grey of BGR, then the remapped level-0 planes"""
    up = lambda v: (v + 255) // 256 * 256
    f32, bgr = fmt == "float32", fmt == "bgr8_depth16"
    npx = g.in_size[0] * g.in_size[1] * N
    dnpx = g.depth[0] * g.depth[1] * N if g.depth else npx
    end = 0
    if not device:
        image = up(dnpx * (4 if f32 else 2))
        end = image + npx * (4 if f32 else 3 if bgr else 1) + 64
        if masked:
            end = up(end) + npx
    if bgr:
        end = up(end) + npx
    return up(end) + g.size[0] * g.size[1] * N * (8 + (1 if g.rect and masked else 0))


def footprint_extents(g, k=0):
    """(ok, x1 - x0, y1 - y0) of the depth pixels of frame k before the footprint limit"""
    ok, _, x0, x1, y0, y1 = rg.footprints(frames(g)["float"][1][k], rays(g), g.depth[4], g.K)
    return ok, x1 - x0, y1 - y0


def _valid(g):
    mx, my = g.map
    w, h = g.in_size
    with np.errstate(invalid="ignore"):
        return (mx >= 0) & (mx <= w - 1) & (my >= 0) & (my <= h - 1)


def assert_reason(g):
    """the case each geometry exists for, from the geometry (and the models' maps and footprints) alone"""
    w, h = g.size
    ls = level_shapes(w, h, g.levels)
    tiles0 = level_geometry(w, h, g.levels)[0][0] * level_geometry(w, h, g.levels)[0][1]
    assert ls[-1][0] >= 8 and ls[-1][1] >= 2
    if g.rect:
        assert g.in_size != g.size, g.name            # a rectifier whose input and output sizes differ
    if g.rect and g.depth is None:
        assert not _valid(g).all(), g.name            # NaN borders: the map leaves the frame somewhere
    if g.name.startswith("down"):                     # exactly half each way; 360 rows end in a strip of 3
        assert g.in_size == (2 * w, 2 * h) and h % TILE_H == 3 and strips(h)[-1] == 3
    elif g.name.startswith("up"):                     # twice each way: output pixels share their 2 x 2 tap cell
        mx, my = g.map
        v = _valid(g)
        cells = np.unique(np.floor(mx[v]).astype(np.int64) * 100000 + np.floor(my[v]).astype(np.int64))
        assert g.size == (2 * g.in_size[0], 2 * g.in_size[1]) and cells.size * 3 < v.sum()
        assert (np.modf(mx[v])[0] == 0.5).any()       # and ties of the nearest depth tap, ax == 0.5 exactly
    elif g.name.startswith("crop"):                   # an odd crop: a 1-column band, odd sizes, several CTAs at level 0
        assert bands(w) == [TILE_W] * 4 + [1] and w % 2 == 1 and h % 2 == 1 and tiles0 > COARSE_TILES
        assert g.in_size[0] > w and g.in_size[1] > h
        assert not _valid(g)[:, -1].all()             # NaN border inside the partial band
    elif g.name.startswith("tall"):                   # taller than its input, not 4:3: swapping in_w, in_h moves pixels
        mx, my = g.map
        v = _valid(g)
        in_w, in_h = g.in_size
        assert h > in_h and in_w != in_h and 3 * w != 4 * h and 4 * w != 3 * h
        assert (mx[v] > in_h - 1).any()               # valid only while the x bound is in_w - 1
        assert ((my > in_h - 1) & (my <= in_w - 1)).any()     # invalid only while the y bound is in_h - 1
    elif g.name.startswith("sizes"):
        _assert_reason(w, h, g.levels)
    elif g.name.startswith("kinect"):                 # 512 x 424 depth, 16:9 colour: no side or aspect in common
        dw, dh = g.depth[:2]
        assert dw * h != dh * w and dw != w and dh != h and h % TILE_H == 1 and bands(ls[2][0]) == [160, 80]
    elif g.name.startswith("odd"):                    # odd depth camera into an odd SIZES colour size
        dw, dh = g.depth[:2]
        assert dw % 2 == 1 and dh % 2 == 1 and w % 2 == 1 and (w, h, g.levels) in SIZES
        _assert_reason(w, h, g.levels)
    elif g.name.startswith("coarse"):                 # footprints on both sides of the limit of 8 colour pixels
        ok, ex, ey = footprint_extents(g)
        big = np.maximum(ex, ey)[ok]
        assert (big == rg.MAX_FOOTPRINT).sum() > 100 and (big == rg.MAX_FOOTPRINT + 1).sum() > 100, np.bincount(big)
        assert big.min() >= rg.MAX_FOOTPRINT - 1 and big.max() <= rg.MAX_FOOTPRINT + 1
    elif g.name.startswith("rectified"):              # registration through a rectifier of another input size
        assert g.rect and g.depth is not None and g.in_size != g.size and g.depth[:2] not in (g.in_size, g.size)
    else:
        raise AssertionError(f"no stated reason for {g.name}")


@pytest.mark.parametrize("g", GEOMETRIES, ids=IDS)
def test_geometry_reason(g):
    assert_reason(g)


def test_every_sizes_entry_is_a_rectifier_output():
    assert {g.size for g in RECTIFIED if g.name.startswith("sizes")} == {(w, h) for w, h, _ in SIZES}
    assert len(set(IDS)) == len(IDS)


# ---- rectified planes against fp64 --------------------------------------------------------------------------------------
U = 2.0 ** -24             # unit roundoff of float32


def _bilinear64(img, mx, my, w, h):
    """fp64 bilinear of the float32 map's taps: (value, bound, nearest tap (y, x), valid); bound: the forward error of the
    model's six float32 roundings (1 - a, two products and a sum per row, then the same across rows), 6u / (1 - 6u) of the
    sum of |weight * tap|, plus one rounding of each weight's own"""
    sx, sy = mx.astype(np.float64), my.astype(np.float64)
    valid = (sx >= 0) & (sx <= w - 1) & (sy >= 0) & (sy <= h - 1)
    sx, sy = np.where(valid, sx, 0), np.where(valid, sy, 0)
    x0 = np.minimum(np.floor(sx), w - 2).astype(np.int64)
    y0 = np.minimum(np.floor(sy), h - 2).astype(np.int64)
    ax, ay = sx - x0, sy - y0                       # exact: the float32 map value minus an integer
    I = img.astype(np.float64)
    taps = [(1 - ax) * (1 - ay), ax * (1 - ay), (1 - ax) * ay, ax * ay]
    vals = [I[y0, x0], I[y0, x0 + 1], I[y0 + 1, x0], I[y0 + 1, x0 + 1]]
    v = sum(t * q for t, q in zip(taps, vals))
    mag = sum(t * np.abs(q) for t, q in zip(taps, vals))
    g6 = 7 * U / (1 - 7 * U)
    near = (y0 + (ay >= 0.5), x0 + (ax >= 0.5))
    return v, g6 * mag, near, valid, (y0, x0)


@pytest.mark.parametrize("g", [g for g in GEOMETRIES if g.rect], ids=[g.name for g in GEOMETRIES if g.rect])
def test_rectified_planes_against_fp64(g):
    f = frames(g)
    mx, my = g.map
    w, h = g.in_size
    for k in range(N):
        fd, rd = f["float"][1][k], f["raw"][k]
        if g.depth is not None:          # the depth is the depth camera's: stand-ins of the colour size take the nearest tap
            fd, rd = f["float"][0][k] * np.float32(0.01), f["grey"][k].astype(np.uint16) * 37
        for img, depth, scale in ((f["float"][0][k], fd, None), (f["grey"][k], rd, DEPTH_SCALE)):
            I, Z, M = rm.remap(img, depth, mx, my, f["masks"][k], scale)
            v64, bound, (yn, xn), valid, (y0, x0) = _bilinear64(img, mx, my, w, h)
            assert np.array_equal(np.isnan(I), ~valid) and np.array_equal(np.isnan(Z) & valid, np.isnan(Z) & ~np.isnan(I))
            err = np.abs(I[valid].astype(np.float64) - v64[valid])
            assert (err <= bound[valid]).all(), (k, float((err / np.maximum(bound[valid], 1e-300)).max()))
            want_z = rg.depth_metres(depth, scale)[yn, xn]
            assert np.array_equal(Z[valid], want_z[valid], equal_nan=True), k
            m = f["masks"][k] != 0
            usable = valid & m[y0, x0] & m[y0, x0 + 1] & m[y0 + 1, x0] & m[y0 + 1, x0 + 1]
            assert np.array_equal(M.astype(bool), usable), k
            assert valid.any() and (~valid).any() and usable.any() and (valid & ~usable).any()


# ---- registered depth against fp64 --------------------------------------------------------------------------------------
def _rays64(g):
    """fp64 rays through the depth pixel centres and corners (tests/registration_model.py's Newton in float64, not rounded)"""
    dw, dh, K_d, dist_d, _ = g.depth
    fx, fy, cx, cy = K_d

    def r(u, v):
        xd, yd = np.broadcast_arrays((u - cx) / fx, (v - cy) / fy)
        return (xd.copy(), yd.copy()) if dist_d is None else rg._undistort(xd.copy(), yd.copy(), dist_d)
    c = r(np.arange(dw, dtype=np.float64)[None, :], np.arange(dh, dtype=np.float64)[:, None])
    k = r(np.arange(dw + 1, dtype=np.float64)[None, :] - 0.5, np.arange(dh + 1, dtype=np.float64)[:, None] - 0.5)
    return c, k


def _reproject64(g, depth):
    """float64 forward projection of every depth pixel: (ok, Zc, x-extent, y-extent) of its corner rays in the colour camera"""
    (crx, cry), (kx, ky) = _rays64(g)
    T, K = np.asarray(g.depth[4]), g.K
    dh, dw = depth.shape
    d = depth.astype(np.float64)
    ok = np.isfinite(d) & (d > 0)
    d = np.where(ok, d, 1.0)

    def proj(rx, ry):
        P = np.stack([rx * d, ry * d, d], -1) @ T[:3, :3].T + T[:3, 3]
        return K[0] * P[..., 0] / P[..., 2] + K[2], K[1] * P[..., 1] / P[..., 2] + K[3], P[..., 2]
    zc = proj(crx, cry)[2]
    corners = [proj(kx[a:a + dh, b:b + dw], ky[a:a + dh, b:b + dw]) for a in (0, 1) for b in (0, 1)]
    xs, ys = np.stack([c[0] for c in corners]), np.stack([c[1] for c in corners])
    return ok, zc, (xs.min(0), xs.max(0)), (ys.min(0), ys.max(0))


def _coverage64(g, depth, Z, eps=1e-3, rel=2e-6):
    """From the fp64 reprojection: per colour pixel the nearest depth whose footprint surely covers it (inf: none), whether
    the model's value is some loosely covering footprint's depth, and per colour pixel whether a footprint under the limit
    may cover it at all.  Footprints within rounding of the limit count as both."""
    w, h = g.size
    ok, zc, (x0, x1), (y0, y1) = _reproject64(g, depth)
    lim = rg.MAX_FOOTPRINT
    lo = np.full((h, w), np.inf)
    found = np.zeros((h, w), bool)
    maybe = np.zeros((h, w), bool)
    x0, y0 = np.where(ok, x0, 0), np.where(ok, y0, 0)
    x1, y1 = np.where(ok, x1, 0), np.where(ok, y1, 0)
    # the float32 footprint [ceil x0, ceil x1) lies between these integer extents
    sure_under = (np.ceil(x1 + eps) - np.ceil(x0 - eps) <= lim) & (np.ceil(y1 + eps) - np.ceil(y0 - eps) <= lim)
    may_under = (np.ceil(x1 - eps) - np.ceil(x0 + eps) <= lim) & (np.ceil(y1 - eps) - np.ceil(y0 + eps) <= lim)
    for oy in range(lim + 3):
        for ox in range(lim + 3):
            xx, yy = np.ceil(x0 - eps).astype(np.int64) + ox, np.ceil(y0 - eps).astype(np.int64) + oy
            inside = ok & (xx >= 0) & (xx < w) & (yy >= 0) & (yy < h)
            loose = inside & (xx < x1 + eps) & (yy < y1 + eps)
            tight = inside & sure_under & (xx >= x0 + eps) & (xx < x1 - eps) & (yy >= y0 + eps) & (yy < y1 - eps)
            np.minimum.at(lo, (yy[tight], xx[tight]), zc[tight])
            maybe[yy[loose & may_under], xx[loose & may_under]] = True
            zo = Z[yy[loose], xx[loose]]
            hit = np.abs(zo - zc[loose]) <= rel * zc[loose]
            found[yy[loose][hit], xx[loose][hit]] = True
    return lo, found, maybe


@pytest.mark.parametrize("g", REGISTERED, ids=[g.name for g in REGISTERED])
def test_registered_depth_against_fp64_reprojection(g):
    """Every finite registered depth is the fp64 Zc of a depth pixel whose footprint covers the colour pixel (to rounding);
    no footprint under the limit that surely covers it is nearer; every surely covered pixel holds a depth; and no pixel
    that only footprints over the limit could cover holds one"""
    f = frames(g, holes=False)
    for k in range(N):
        depth = f["float"][1][k]
        Z = rg.register(depth, rays(g), g.depth[4], g.size, g.K)
        lo, found, maybe = _coverage64(g, depth, Z)
        fin = np.isfinite(Z)
        assert fin.mean() > 0.5, (k, fin.mean())
        assert found[fin].all(), k
        assert (Z[fin] <= lo[fin] * (1 + 2e-6)).all(), k
        assert not np.isfinite(lo[~fin]).any(), k
        assert not fin[~maybe].any(), k


def _gaps(Z, reach=12):
    """NaN colour pixels with a finite pixel within `reach` to their left and to their right in the same row"""
    fin = np.isfinite(Z)
    left = np.zeros_like(fin)
    right = np.zeros_like(fin)
    for s in range(1, reach + 1):
        left[:, s:] |= fin[:, :-s]
        right[:, :-s] |= fin[:, s:]
    return ~fin & left & right


@pytest.mark.parametrize("g", REGISTERED, ids=[g.name for g in REGISTERED])
def test_shadows_empty_and_over_limit_footprints(g):
    """Without depth holes, the gaps inside the registered depth are what the geometry makes: occlusion shadows behind
    the box where the depth camera sits off the colour camera's axis, footprints that hold no colour pixel centre where
    the depth camera is finer than the colour camera, and footprints over the limit where it is 8 times coarser.  Each
    kind occurs where the geometry says, and the colour pixels only they cover stay empty."""
    f = frames(g, holes=False)
    depth = f["float"][1][0]
    Z = rg.register(depth, rays(g), g.depth[4], g.size, g.K)
    okf, _, x0, x1, y0, y1 = rg.footprints(depth, rays(g), g.depth[4], g.K)
    ex, ey = x1 - x0, y1 - y0
    empty = okf & ((ex == 0) | (ey == 0))
    over = okf & ((ex > rg.MAX_FOOTPRINT) | (ey > rg.MAX_FOOTPRINT))
    gaps = _gaps(Z)
    fx_ratio = g.K[0] / g.depth[2][0]
    if fx_ratio < 1:                                  # finer depth: some footprints cover no colour pixel centre
        assert empty.sum() > 0.05 * okf.sum(), (g.name, empty.sum(), okf.sum())
    else:
        assert not empty.any(), g.name
    if g.name.startswith("coarse"):
        assert over.sum() > 0.05 * okf.sum()
        # the colour pixels that only over-limit footprints cover are empty; every other covered one holds a depth
        w, h = g.size
        cov_over = np.zeros((h, w), bool)
        cov_under = np.zeros((h, w), bool)
        for oy in range(rg.MAX_FOOTPRINT + 1):
            for ox in range(rg.MAX_FOOTPRINT + 1):
                xx, yy = x0 + ox, y0 + oy
                inside = okf & (xx < x1) & (yy < y1) & (xx >= 0) & (xx < w) & (yy >= 0) & (yy < h)
                cov_over[yy[inside & over], xx[inside & over]] = True
                cov_under[yy[inside & ~over], xx[inside & ~over]] = True
        only = cov_over & ~cov_under
        assert only.sum() > 0.05 * h * w and np.isnan(Z[only]).all() and np.isfinite(Z[cov_under]).all()
    else:
        assert not over.any(), g.name
    if g.name.startswith(("kinect", "rectified")):   # a baseline of 3 to 5 cm at 1.1-2.5 m: shadows beside the box
        assert gaps.sum() > 50, (g.name, gaps.sum())
    if fx_ratio >= 1 and not g.name.startswith("coarse"):
        # no empty and no over-limit footprint: every gap is a shadow, a colour pixel no depth pixel reaches
        okf64, _, (ax0, ax1), (ay0, ay1) = _reproject64(g, depth)
        w, h = g.size
        reach = np.zeros((h, w), bool)
        for oy in range(rg.MAX_FOOTPRINT + 1):
            for ox in range(rg.MAX_FOOTPRINT + 1):
                xx, yy = np.ceil(ax0 - 1e-3).astype(np.int64) + ox, np.ceil(ay0 - 1e-3).astype(np.int64) + oy
                inside = okf64 & (xx < ax1 + 1e-3) & (yy < ay1 + 1e-3) & (xx >= 0) & (xx < w) & (yy >= 0) & (yy < h)
                reach[yy[inside], xx[inside]] = True
        assert not reach[gaps].any(), g.name
