"""Rectified and registered pyramids on the H100 where the input, depth and colour geometries differ.

The geometries are those of tests/test_remap_geometry_host.py (GEOMETRIES, each with a stated reason asserted before use):
rectifiers that downscale 1280 x 720 to 640 x 360, upscale 320 x 240 to 640 x 480, crop 661 x 493 to 641 x 481, make a
264 x 360 view taller than its 400 x 300 input, and give each size of test_gpu_geometry.SIZES from larger frames; depth
registration from a 512 x 424 camera into 960 x 540, from an odd 203 x 157 camera into two odd SIZES targets, from an
80 x 60 camera whose footprints straddle DVO_B200_REGISTRATION_MAX_FOOTPRINT, and through a 1280 x 720 -> 640 x 360
rectifier.  Per geometry, with N = 3 frames:
  builds         every format, mask roles None / reference / both (masks in the colour frames' geometry), the host path
                 and the device path from cropped planes whose pitch and stride are not the output's: every plane at every
                 level, the selection at two thresholds, S and level_info bit for bit against the float32 model's planes
                 through the plain create
  records        residual records and the intensity error image bit for bit against MIRROR (rectify_model.oracle_pyramid),
                 P / LL / A / b to 2e-6, both estimators, two poses, at the two finest levels with a partial band or a
                 partial last strip and NaN there
  alignments     batch = reversed batch = single alignments, bit for bit
  stage growth   every geometry built on one context in increasing staging size (each build reallocates), then in
                 decreasing size (each reuses a larger stage holding another geometry's bytes), equals its build on a
                 fresh context
  map edges      maps holding in_w - 1, in_h - 1, one ulp either side, the smallest negative float, -0.0, NaN, +-Inf and
                 nearest-tap ties in the partial band, the last strip and inside, against the model
"""
import collections
import functools

import numpy as np
import pytest
import torch

import rectify_model as rm
from test_corrected_estimator import corrected_mode
from test_gpu_device_input import _to_device
from test_gpu_geometry import _check_level, _edge_shift, _small_motion, corrected  # noqa: F401  (fixture)
from test_remap_geometry_host import (BY_NAME, DEPTH_SCALE, GEOMETRIES, IDS, N, assert_reason, frames, inputs, model_planes,
                                      rays, stage_bytes)
from tile_geometry import TILE_H, TILE_W, has_partial_band

pytestmark = pytest.mark.gpu

FORMATS = ["float32", "grey8_depth16", "bgr8_depth16"]
MASKS = [None, "reference", "both"]
SELECTIONS = [(0.0, 0.0), (6.0, 0.02)]
_reason = functools.lru_cache(maxsize=None)(assert_reason)


def _handles(eng, g, map_xy=None):
    """(rectifier or None, registration or None) of g on eng"""
    rect = eng.rectifier(g.in_size, *(map_xy or g.map), g.K) if g.rect else None
    reg = eng.depth_registration(g.depth[:2], rays(g), np.asarray(g.depth[4]), g.size, g.K) if g.depth else None
    return rect, reg


def _release(h):
    for x in h:
        if x is not None:
            x.release()


@pytest.fixture(scope="module")
def handles(engine):
    made = {}

    def get(g):
        if g.name not in made:
            made[g.name] = _handles(engine, g)
        return made[g.name]
    yield get
    for h in made.values():
        _release(h)


def _build(eng, h, g, fmt, mask, path, f=None):
    """the rectified or registered create of g's N frames"""
    rect, reg = h
    f = f or frames(g)
    image, depth = inputs(f, fmt)
    kw = {"depth_scale": None if fmt == "float32" else DEPTH_SCALE, "mask_roles": mask or "reference"}
    m = f["masks"] if mask else None
    if path == "device":
        fill_z = float("nan") if fmt == "float32" else 777
        image, depth = _to_device(image, "crop", fill=99), _to_device(depth, "crop", fill=fill_z)
        m = _to_device(m, "crop", torch.bool, fill=1) if mask else None
    if reg is None:
        return eng.pyramid_rectified_batch(rect, image, depth, g.levels, masks=m, **kw)
    return eng.pyramid_registered_batch(reg, image, depth, g.levels, masks=m, rectifier=rect, **kw)


@pytest.fixture(scope="module")
def model_build(engine):
    """(g, fmt, mask) -> the float32 pyramids of the models' planes by the plain (masked) create; the last few kept"""
    cache = collections.OrderedDict()

    def get(g, fmt, mask):
        key = (g.name, fmt, mask)
        if key not in cache:
            I, Z, M = model_planes(g, fmt, mask is not None)
            kw = {} if mask is None else {"masks": M, "mask_roles": mask}
            cache[key] = engine.pyramid_batch(I, Z, g.K, g.levels, **kw)
            while len(cache) > 6:
                cache.popitem(last=False)
        return cache[key]
    return get


def _outputs(P, levels):
    """everything a pyramid shows: per level its info, planes and the selection at SELECTIONS"""
    out = []
    for l in range(levels):
        out += [P.level_info(l), P.download(l)]
        for sel in SELECTIONS:
            out += list(P.select(l, *sel))
    return out


def _assert_same(a, b):
    assert len(a) == len(b)
    for k, (x, y) in enumerate(zip(a, b)):
        if isinstance(x, np.ndarray):
            assert x.dtype == y.dtype and x.shape == y.shape and np.array_equal(x.view(np.uint8), y.view(np.uint8)), k
        else:
            assert x == y, k


def _assert_same_pyramid(p, q, levels):
    """bit for bit, NaN payloads included; the selection's S and mask at both thresholds; level_info"""
    assert p.mask_roles == q.mask_roles
    _assert_same(_outputs(p, levels), _outputs(q, levels))


# ---- builds against the model build --------------------------------------------------------------------------------------
@pytest.mark.parametrize("path", ["host", "device"])
@pytest.mark.parametrize("mask", MASKS)
@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("g", GEOMETRIES, ids=IDS)
def test_build_equals_the_model_build(engine, handles, model_build, g, fmt, mask, path):
    _reason(g)
    R = _build(engine, handles(g), g, fmt, mask, path)
    H = model_build(g, fmt, mask)
    assert len(R) == N
    assert all(p.level_info(0) == (g.size[0], g.size[1], tuple(np.float32(g.K))) for p in R)
    for p, q in zip(R, H):
        _assert_same_pyramid(p, q, g.levels)


# ---- records against MIRROR ----------------------------------------------------------------------------------------------
def _record_levels(g, oref):
    """the two finest levels with a partial band or a partial last strip that holds NaN (intensity through a rectifier,
    depth otherwise)"""
    out = []
    for l in range(g.levels):
        lw, lh, _ = oref.level_info(l)
        edge = np.zeros((lh, lw), bool)
        if has_partial_band(lw):
            edge[:, (lw // TILE_W) * TILE_W:] = True
        if lh % TILE_H:
            edge[(lh // TILE_H) * TILE_H:, :] = True
        if edge.any() and np.isnan(oref.planes(l)[0 if g.rect else 1][edge]).any():
            out.append(l)
    return out[:2]


@pytest.mark.parametrize("estimator", ["reference", "corrected"])
@pytest.mark.parametrize("g", GEOMETRIES, ids=IDS)
def test_records_against_mirror(engine, corrected, oracle, handles, g, estimator):
    _reason(g)
    eng, mode = (engine, oracle.mode("mirror")) if estimator == "reference" else (corrected, corrected_mode(oracle))
    I, Z, _ = model_planes(g, "float32", False)
    oref, ocur = (rm.oracle_pyramid(oracle, I[k], Z[k], g.K, g.levels) for k in (0, 1))
    R = _build(engine, handles(g), g, "float32", None, "host")
    levels = _record_levels(g, oref)
    assert len(levels) == 2, (g.name, levels)
    checked = 0
    for lvl in levels:
        for T in (_small_motion(), _edge_shift(g.size[0], g.size[1], g.K, Z[0])):
            checked += _check_level(eng, mode, R[0], R[1], oref, ocur, lvl, T, (0.0, 0.0)) > 0
    assert checked >= 2, checked


# ---- whole alignments ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt,mask", [("float32", None), ("bgr8_depth16", "both")], ids=["float32", "bgr8-both"])
@pytest.mark.parametrize("g", GEOMETRIES, ids=IDS)
def test_batch_reversed_and_single_alignments(engine, handles, g, fmt, mask):
    from dvo_slam_b200.engine import Config
    _reason(g)
    R = _build(engine, handles(g), g, fmt, mask, "host")
    refs, curs = [R[0], R[2], R[1]], [R[1], R[0], R[0]]
    cfg = Config(first_level=g.levels - 1, last_level=0, max_iterations_per_level=50, precision=1e-4)
    batch = engine.match_batch(refs, curs, cfg, raw=True)
    rev = engine.match_batch(refs[::-1], curs[::-1], cfg, raw=True)
    for i in range(N):
        single = engine.match_batch([refs[i]], [curs[i]], cfg, raw=True)
        assert bytes(batch[i]) == bytes(single[0]) == bytes(rev[N - 1 - i]), i
    assert engine.match_batch(refs[:1], curs[:1], cfg)[0].levels[-1]["valid_pixels"] > 0


# ---- staging growth ------------------------------------------------------------------------------------------------------
def test_stage_growth_and_reuse():
    """BGR frames with masks from the host take every staging section.  In increasing staging size each create
    reallocates the stage; in decreasing size each reads a stage that still holds a larger geometry's frames and planes.
    Both give what a fresh context gives."""
    from dvo_slam_b200.engine import Engine
    fmt, mask = "bgr8_depth16", "both"
    order = sorted(GEOMETRIES, key=lambda g: stage_bytes(g, fmt, True, False))
    sizes = [stage_bytes(g, fmt, True, False) for g in order]
    assert all(a < b for a, b in zip(sizes, sizes[1:])), sizes

    def run(eng, g):
        h = _handles(eng, g)
        try:
            out = []
            for P in _build(eng, h, g, fmt, mask, "host"):
                out += _outputs(P, g.levels)
                P.release()
            return out
        finally:
            _release(h)
    want = {}
    for g in order:
        eng = Engine(device=0)
        try:
            want[g.name] = run(eng, g)
        finally:
            eng.close()
    eng = Engine(device=0)
    try:
        for g in order + order[::-1]:
            _reason(g)
            _assert_same(run(eng, g), want[g.name])
    finally:
        eng.close()


# ---- map edges -----------------------------------------------------------------------------------------------------------
F32 = np.float32


def _poked(g):
    """g's map with edge values written at rows and columns that include the partial band and the last strip"""
    mx, my = (a.copy() for a in g.map)
    h, w = mx.shape
    W, H = g.in_size
    up = lambda v: np.nextafter(F32(v), F32(np.inf))
    dn = lambda v: np.nextafter(F32(v), F32(-np.inf))
    cx, cy = F32(W / 2 + 0.37), F32(H / 2 + 0.61)
    inf, nan = F32(np.inf), F32(np.nan)
    values = [(W - 1, cy), (up(W - 1), cy), (dn(W - 1), cy), (cx, H - 1), (cx, up(H - 1)), (cx, dn(H - 1)), (W - 1, H - 1),
              (up(W - 1), H - 1), (W - 1, up(H - 1)), (F32(-0.0), cy), (cx, F32(-0.0)), (F32(-0.0), F32(-0.0)), (dn(0), cy),
              (cx, dn(0)), (0, 0), (nan, cy), (cx, nan), (inf, cy), (-inf, cy), (cx, inf), (cx, -inf), (W - 1.5, H - 1.5),
              (W - 1.5, cy), (cx, H - 1.5), (F32(0.5), F32(0.5)), (W - 2, H - 2), (H - 1, cy), (cx, W - 1)]
    for k, (vx, vy) in enumerate(values):
        y, x = (3 + 7 * k) % h, (5 + 11 * k) % w
        for yy, xx in ((y, w - 1), (h - 1, x), (y, x), (y, (w // TILE_W) * TILE_W + k % max(1, w % TILE_W))):
            mx[yy, min(xx, w - 1)], my[yy, min(xx, w - 1)] = F32(vx), F32(vy)
    return mx, my


EDGE_GEOMETRIES = ["crop-661x493-641x481", "tall-400x300-264x360", "down-1280x720-640x360", "up-320x240-640x480", "sizes-161x50",
                   "sizes-700x9"]


@pytest.mark.parametrize("mask", [None, "both"])
@pytest.mark.parametrize("fmt", ["float32", "grey8_depth16"])
@pytest.mark.parametrize("name", EDGE_GEOMETRIES)
def test_map_edges(engine, name, fmt, mask):
    g = BY_NAME[name]
    _reason(g)
    assert g.size != (640, 480) or g.in_size != (640, 480)
    mx, my = _poked(g)
    f = frames(g)
    image, depth = inputs(f, fmt)
    I, Z, M = rm.remap_batch(image, depth, mx, my, f["masks"] if mask else None, None if fmt == "float32" else DEPTH_SCALE)
    kw = {} if mask is None else {"masks": M, "mask_roles": mask}
    H = engine.pyramid_batch(I, Z, g.K, g.levels, **kw)
    h = _handles(engine, g, (mx, my))
    try:
        for path in ("host", "device"):
            R = _build(engine, h, g, fmt, mask, path)
            for p, q in zip(R, H):
                _assert_same_pyramid(p, q, g.levels)
    finally:
        _release(h)
