"""The pyramid and the level kernel across image sizes chosen for the tile edges, against the oracle.

The level kernel cuts every level into 160 x 7 tiles (tests/tile_geometry.py); the pyramid pads odd widths to an even pitch
and ends the selection mask on a partial word when w * h is not a multiple of 32.  Each size below reaches a case the
640 x 480 family never does (a partial band of 1, 33, 63, 128 or 159 columns, whole bands only, strips of 5 or 6 rows, odd
widths below an even level 0, one band per level, very tall or very wide levels, the smallest legal sizes), and each test
asserts that case from the geometry first, so that a later change of the sizes or of the tiles cannot make it vacuous.  Per size, level and selection: the pyramid bit for bit, the residual records
and the intensity error image bit for bit against MIRROR, P / LL / A / b to 2e-6, the same in the corrected estimator,
whole alignments, the three input paths, the argument bounds and a pyramid built into a recycled slab.
"""
import functools

import numpy as np
import pytest

from helpers import nan_equal, pose_delta
from test_corrected_estimator import corrected_mode
from test_gpu_generic_tiles import _rot_z, _shift_z
from tile_geometry import TILE_H, TILE_W, bands, in_partial_band, level_shapes, strips

pytestmark = pytest.mark.gpu

# (level-0 width, height, levels)
SIZES = [(161, 50, 3), (193, 55, 3), (223, 49, 3), (288, 62, 3), (319, 41, 3), (320, 96, 3), (250, 188, 4), (40, 300, 3),
         (700, 9, 3), (32, 8, 3)]
IDS = [f"{w}x{h}" for w, h, _ in SIZES]
SELECTIONS = [(0.0, 0.0), (4.0, 0.02)]      # the default thresholds, and one non-default (intensity, depth) pair
PP = np.array([[2000.0, -30.0], [-30.0, 9000.0]], dtype=np.float32)
DEPTH_SCALE = 1.0 / 5000.0


def _intrinsics(w, h):
    """focal lengths scale with the longer side (so a tall image is not a 150-degree view), principal point off-centre"""
    s = max(w, h)
    return (0.81 * s, 0.81 * s + 0.5, 0.47 * w + 0.3, 0.52 * h - 0.2)


def _assert_reason(w, h, levels):
    """the case each size exists for, from the geometry alone"""
    ls = level_shapes(w, h, levels)
    ws, hs = [s[0] for s in ls], [s[1] for s in ls]
    if (w, h) == (161, 50):        # a 1-column band; an odd width and a mask tail at level 0; a last strip of 1 and of 5 rows
        assert bands(w) == [160, 1] and h % TILE_H == 1 and w % 2 == 1 and (w * h) % 32 != 0 and hs[2] % TILE_H == 5
    elif (w, h) == (193, 55):      # a 33-column band: one round and one pixel; a last strip of 6 rows at every level
        assert bands(w) == [160, 33] and all(v % TILE_H == 6 for v in hs)
    elif (w, h) == (223, 49):      # a 63-column band: two rounds less one pixel; whole strips; odd widths below an even level 0
        assert bands(w) == [160, 63] and h % TILE_H == 0 and ws[0] % 2 == 1 and ws[1] % 2 == 1 and ws[2] % 2 == 1
    elif (w, h) == (288, 62):      # a partial band of whole rounds: the generic loop with no pixel masked off in its last round
        assert bands(w) == [160, 128] and bands(w)[-1] % 32 == 0 and h % TILE_H == 6
    elif (w, h) == (319, 41):      # a band one column short of full, then a level of one such band
        assert bands(w) == [160, 159] and bands(ws[1]) == [159] and h % TILE_H == 6
    elif (w, h) == (320, 96):      # whole bands only at levels 0 and 1, with a last strip of 5 rows
        assert bands(ws[0]) == [160, 160] and bands(ws[1]) == [160] and h % TILE_H == 5 and len(strips(h)) == 14
    elif (w, h) == (250, 188):
        assert ws == [250, 125, 62, 31] and [v % 2 for v in ws] == [0, 1, 0, 1]
    elif (w, h) == (40, 300):
        assert all(len(bands(v)) == 1 and v < TILE_W for v in ws) and len(strips(h)) == 43
    elif (w, h) == (700, 9):
        assert len(bands(w)) == 5 and bands(w)[-1] < TILE_W and len(strips(h)) == 2 and hs[-1] == 2
    elif (w, h) == (32, 8):
        assert ls == [(32, 8), (16, 4), (8, 2)]
    else:
        raise AssertionError(f"no stated reason for {w}x{h}")


def _cfg(first, last, sel=(0.0, 0.0)):
    from dvo_slam_b200.engine import Config
    return Config(first_level=first, last_level=last, max_iterations_per_level=50, precision=1e-4,
                  intensity_derivative_threshold=sel[0], depth_derivative_threshold=sel[1])


@functools.lru_cache(maxsize=None)
def _scene(w, h):
    from dvo_slam_b200 import synth
    p = synth.make_pair(1000 * w + h, synth.SceneConfig(width=w, height=h, intrinsics=_intrinsics(w, h)))
    a = {k: p[k].numpy() for k in ("I_ref", "Z_ref", "I_cur", "Z_cur")}
    a["K"] = p["intrinsics"]
    return a


@functools.lru_cache(maxsize=None)
def _oracle_pyramids(w, h, levels):
    from oracle import oracle_py as orc
    a = _scene(w, h)
    return orc.Pyramid(a["I_ref"], a["Z_ref"], a["K"], levels), orc.Pyramid(a["I_cur"], a["Z_cur"], a["K"], levels)


@pytest.fixture(scope="module")
def gpu_pyramids(engine):
    cache = {}

    def get(w, h, levels):
        if (w, h, levels) not in cache:
            a = _scene(w, h)
            cache[(w, h, levels)] = (engine.pyramid(a["I_ref"], a["Z_ref"], a["K"], levels),
                                     engine.pyramid(a["I_cur"], a["Z_cur"], a["K"], levels))
        return cache[(w, h, levels)]
    return get


@pytest.fixture(scope="module")
def corrected(engine):
    from dvo_slam_b200.engine import Engine
    eng = Engine(device=0, estimator="corrected")
    yield eng
    eng.close()


def _small_motion():
    T = _rot_z(0.8) @ _shift_z(0.01)
    T[0, 3] = 0.004
    return T


def _edge_shift(w, h, K, Z):
    """a translation that moves the last valid column / row of the reference (at its median depth) about an eighth of the
    level-0 size past the right / bottom edge, so that taps of the right and bottom tiles fall outside the image"""
    fx, fy, _, _ = K
    valid = ~np.isnan(Z)
    xl = int(np.flatnonzero(valid.any(axis=0))[-1])
    yl = int(np.flatnonzero(valid.any(axis=1))[-1])
    T = np.eye(4)
    T[0, 3] = (w - xl + max(2.0, 0.12 * w)) * float(np.nanmedian(Z[:, xl])) / fx
    T[1, 3] = (h - yl + max(2.0, 0.12 * h)) * float(np.nanmedian(Z[yl])) / fy
    return T


def _projected(op, lvl, T, mask):
    """(u', v') in float64 of the selected reference points of a level under T"""
    w, h, (fx, fy, ox, oy) = op.level_info(lvl)
    Z = op.plane(lvl, 1)
    ys, xs = np.nonzero(mask)
    z = Z[ys, xs].astype(np.float64)
    p = np.stack([(xs - ox) / fx * z, (ys - oy) / fy * z, z])
    q = T[:3, :3] @ p + T[:3, 3:4]
    return fx * q[0] / q[2] + ox, fy * q[1] / q[2] + oy


def _poses(w, h, lvl):
    a = _scene(w, h)
    out = [("small", _small_motion()), ("edge", _edge_shift(w, h, a["K"], a["Z_ref"]))]
    if lvl == 0:
        out.append(("roll20", _rot_z(20.0)))
    return out


def _unfused(mode):
    m = type(mode).from_buffer_copy(mode)
    m.fused_pixel_math = 0
    return m


def _check_linearisation(lg, lo, lo_unfused):
    """P / LL / A / b to 2e-6 of their largest element (LL: 2e-6 relative + 0.5); n exact; n = 0 only counts.  P, A, b: or
    to the oracle's own spread between fused and unfused pixel arithmetic where that is larger.  P inverts a 2 x 2 sum, and
    on a level with few, strongly correlated residuals that inverse is ill-conditioned; A and b are weighted by P.  At
    700 x 9, level 0, 20 degree roll (182 points) the condition number of P is 1.2e5: summation order alone moves P and A by
    4.1e-6 of their largest elements (GPU against MIRROR, weights on), and the oracle's fused and unfused arithmetic give P
    4.5e-5 apart."""
    assert lg["n"] == lo["n"]
    if lo["n"] == 0:
        return
    for k in ("precision", "A", "b"):
        big = np.abs(lo[k]).max()
        spread = np.abs(lo_unfused[k] - lo[k]).max() / big if big > 0 else 0.0
        assert np.allclose(lg[k], lo[k], rtol=0, atol=max(2e-6, spread) * big), (k, lg[k], lo[k], spread)
    assert abs(lg["ll"] - lo["ll"]) <= 2e-6 * abs(lo["ll"]) + 0.5, (lg["ll"], lo["ll"])


def _check_level(eng, mode, gref, gcur, oref, ocur, lvl, T, sel):
    """residual records and the intensity error image bit-exact, linearisations (weights off and on) to the bounds"""
    from oracle import oracle_py as orc
    cfg = _cfg(lvl, lvl, sel)
    n_g, img_g = eng.residual_image(gref, gcur, lvl, T, cfg)
    n_o, img_o = orc.residual_image(oref, ocur, lvl, T, mode, *sel)
    assert n_g == n_o and nan_equal(img_g, img_o), (lvl, n_g, n_o)
    ne_g, err_g = eng.intensity_error_image(gref, gcur, lvl, T, cfg)
    ne_o, err_o = orc.intensity_error_image(oref, ocur, lvl, T, mode, *sel)
    assert ne_g == ne_o and np.array_equal(err_g, err_o), (lvl, ne_g, ne_o)
    for uw in (False, True):
        lg = eng.linearize(gref, gcur, lvl, T, uw, PP, cfg)
        lo = orc.linearize(oref, ocur, lvl, T, mode, uw, PP, *sel)
        assert lg["n"] == n_o
        _check_linearisation(lg, lo, orc.linearize(oref, ocur, lvl, T, _unfused(mode), uw, PP, *sel))
    return n_o


def _check_pyramid(gp, op, levels):
    from oracle import oracle_py as orc
    for lvl in range(levels):
        got, want = gp.download(lvl), op.planes(lvl)
        want[1][np.isnan(want).any(axis=0)] = np.nan        # device depth is masked where any channel is NaN
        assert got.shape == want.shape
        for c in range(6):
            assert nan_equal(got[c], want[c]), (lvl, c)
        assert gp.level_info(lvl) == op.level_info(lvl)
    for sel in SELECTIONS + [SELECTIONS[0]]:                # back to the defaults: the selection cache switches both ways
        for lvl in range(levels):
            S, mask = gp.select(lvl, *sel)
            So, masko = orc.select(op, lvl, *sel)
            assert S == So and np.array_equal(mask, masko), (lvl, sel, S, So)


def _check_alignment(eng, gref, gcur, oref, ocur, levels, sel):
    """valid pixels per level as MIRROR; where the control flow is MIRROR's, the pose within 1e-4 of MIRROR, or within the
    oracle's own spread between fused and unfused pixel arithmetic where that is larger (the rule of the thresholded
    alignments in test_gpu_selection_thresholds.py).  On 700 x 9 with thresholds (516 points at level 0) that spread is
    what the GPU's 1.2e-4 m from MIRROR is measured against."""
    from oracle import oracle_py as orc
    r = eng.match(gref, gcur, _cfg(levels - 1, 0, sel))
    ocfg = orc.config(first_level=levels - 1, last_level=0, max_iterations_per_level=50, precision=1e-4,
                      intensity_derivative_threshold=sel[0], depth_derivative_threshold=sel[1])
    o = orc.match(oref, ocur, ocfg, orc.mode("mirror"))
    assert [l["valid_pixels"] for l in r.levels] == [l["valid_pixels"] for l in o["levels"]]
    same = ([l["termination"] for l in r.levels] == [l["termination"] for l in o["levels"]] and
            [l["num_iterations"] for l in r.levels] == [l["num_iterations"] for l in o["levels"]])
    if same:
        st, sr = pose_delta(o["T"], orc.match(oref, ocur, ocfg, _unfused(orc.mode("mirror")))["T"])
        dt, dr = pose_delta(o["T"], r.transformation)
        assert dt < max(1e-4, st) and dr < max(1e-4, sr), (dt, dr, st, sr)
    return r, same


# ---- 1. the pyramid ----
@pytest.mark.parametrize("w,h,levels", SIZES, ids=IDS)
def test_pyramid(gpu_pyramids, w, h, levels):
    _assert_reason(w, h, levels)
    gref, gcur = gpu_pyramids(w, h, levels)
    oref, ocur = _oracle_pyramids(w, h, levels)
    _check_pyramid(gref, oref, levels)
    _check_pyramid(gcur, ocur, levels)


def test_some_level_has_a_mask_tail_and_an_odd_pitch():
    tails = [(w, h, l) for w, h, n in SIZES for l, (lw, lh) in enumerate(level_shapes(w, h, n)) if (lw * lh) % 32]
    odd = [(w, h, l) for w, h, n in SIZES for l, (lw, _) in enumerate(level_shapes(w, h, n)) if lw % 2]
    assert any(l == 0 for _, _, l in tails) and len(tails) >= 8 and len(odd) >= 8, (tails, odd)


# ---- 2. / 3. the level kernel at fixed poses, both estimators ----
@pytest.mark.parametrize("estimator", ["reference", "corrected"])
@pytest.mark.parametrize("w,h,levels", SIZES, ids=IDS)
def test_level_kernel_at_fixed_poses(engine, corrected, oracle, gpu_pyramids, w, h, levels, estimator):
    _assert_reason(w, h, levels)
    eng, mode = (engine, oracle.mode("mirror")) if estimator == "reference" else (corrected, corrected_mode(oracle))
    gref, gcur = gpu_pyramids(w, h, levels)
    oref, ocur = _oracle_pyramids(w, h, levels)
    checked = 0
    for sel in SELECTIONS:
        for lvl in range(levels):
            lw, lh, _ = oref.level_info(lvl)
            S, mask = oracle.select(oref, lvl, *sel)
            for name, T in _poses(w, h, lvl):
                if name == "edge" and S > 0:
                    u, v = _projected(oref, lvl, T, mask)
                    assert (u > lw - 1).any() and (v > lh - 1).any(), (lvl, sel)      # taps past the right and bottom edges
                checked += _check_level(eng, mode, gref, gcur, oref, ocur, lvl, T, sel) > 0
    assert checked >= 2 * levels, checked          # most (level, pose, selection) cases have constraints to compare


def test_an_odd_selection_ends_in_a_partial_band_or_the_last_strip(oracle):
    """the corrected estimator's re-admitted odd last point is compared above in a partial band or the last strip"""
    hits = []
    for w, h, levels in SIZES:
        oref, _ = _oracle_pyramids(w, h, levels)
        for sel in SELECTIONS:
            for lvl in range(levels):
                lw, lh, _ = oref.level_info(lvl)
                S, mask = oracle.select(oref, lvl, *sel)
                if S % 2 == 0:
                    continue
                last = int(np.flatnonzero(mask.reshape(-1))[-1])
                y, x = divmod(last, lw)
                in_last_strip = y >= ((lh - 1) // TILE_H) * TILE_H
                if in_partial_band(x, lw) or in_last_strip:
                    hits.append((w, h, lvl, sel, S, x, y))
    assert hits
    print("odd selections ending in a partial band or the last strip:", hits)


# ---- 4. whole alignments ----
@pytest.mark.parametrize("sel", SELECTIONS, ids=["default", "thresholds"])
@pytest.mark.parametrize("w,h,levels", SIZES, ids=IDS)
def test_alignment(engine, oracle, gpu_pyramids, w, h, levels, sel):
    _assert_reason(w, h, levels)
    gref, gcur = gpu_pyramids(w, h, levels)
    oref, ocur = _oracle_pyramids(w, h, levels)
    r, same = _check_alignment(engine, gref, gcur, oref, ocur, levels, sel)
    print(f"{w}x{h} {sel}: levels {[(l['termination'], l['num_iterations'], l['valid_pixels']) for l in r.levels]} same={same}")


# ---- 5. input paths ----
ODD_W = [s for s in SIZES if s[0] % 2]


def test_input_path_sizes_cover_odd_strides():
    assert any(h % 2 for _, h, _ in ODD_W) and any(h % 2 == 0 for _, h, _ in ODD_W)
    assert any((w * h) % 2 for w, h, _ in ODD_W)      # the per-image stride of an n = 3 batch is odd


def _raw_inputs(w, h, n=3):
    """n BGR frames and u16 depth images derived from the scene (the depth quantum is the TUM one), with zero raw depth
    (invalid) where the scene has none"""
    a = _scene(w, h)
    rng = np.random.default_rng(w * 7 + h)
    bgr = np.empty((n, h, w, 3), np.uint8)
    raw = np.empty((n, h, w), np.uint16)
    for i in range(n):
        base = (a["I_ref"] if i % 2 == 0 else a["I_cur"]).astype(np.int32)
        for c in range(3):
            bgr[i, :, :, c] = np.clip(base + rng.integers(-20, 21, size=(h, w)), 0, 255)
        Z = a["Z_ref"] if i % 2 == 0 else a["Z_cur"]
        raw[i] = np.where(np.isnan(Z), 0, np.round(np.nan_to_num(Z) / DEPTH_SCALE)).astype(np.uint16)
    return bgr, raw


@pytest.mark.parametrize("w,h,levels", ODD_W, ids=[f"{w}x{h}" for w, h, _ in ODD_W])
def test_input_paths(engine, oracle, w, h, levels):
    """float input, 8-bit grey + u16 raw depth, and BGR + u16, each as one n = 3 batch, give the same pyramid.  With an odd
    width the 8-bit level-1 reduction takes its unaligned loads."""
    assert w % 2 == 1
    n = 3
    K = _intrinsics(w, h)
    bgr, raw = _raw_inputs(w, h, n)
    grey = np.stack([oracle.bgr_to_grey(bgr[i]) for i in range(n)])
    depth = np.stack([oracle.convert_raw_depth(raw[i], DEPTH_SCALE) for i in range(n)])
    grey_u8 = grey.astype(np.uint8)
    assert np.array_equal(grey_u8.astype(np.float32), grey)
    p_float = engine.pyramid_batch(grey, depth, K, levels)
    p_raw = engine.pyramid_raw_batch((grey_u8.ctypes.data, raw.ctypes.data, n, h, w), DEPTH_SCALE, K, levels)
    p_bgr = engine.pyramid_bgr_batch((bgr.ctypes.data, raw.ctypes.data, n, h, w), DEPTH_SCALE, K, levels)
    engine.synchronize()
    for i in range(n):
        op = oracle.Pyramid(grey[i], depth[i], K, levels)
        for lvl in range(levels):
            f = p_float[i].download(lvl)
            want = op.planes(lvl)
            want[1][np.isnan(want).any(axis=0)] = np.nan
            assert all(nan_equal(f[c], want[c]) for c in range(6)), (i, lvl)
            assert nan_equal(p_raw[i].download(lvl), f), (i, lvl, "raw")
            assert nan_equal(p_bgr[i].download(lvl), f), (i, lvl, "bgr")
            S, mask = p_float[i].select(lvl)
            for q in (p_raw[i], p_bgr[i]):
                Sq, maskq = q.select(lvl)
                assert Sq == S and np.array_equal(maskq, mask)


# ---- 6. argument bounds ----
def test_argument_bounds_are_status_codes(engine):
    def build(w, h, levels):
        rng = np.random.default_rng(0)
        I = rng.uniform(0, 255, (h, w)).astype(np.float32)
        Z = rng.uniform(0.5, 3.0, (h, w)).astype(np.float32)
        return engine.pyramid(I, Z, _intrinsics(w, h), levels)

    assert [s[0] for s in level_shapes(40, 300, 4)][-1] < 8 and [s[1] for s in level_shapes(700, 9, 4)][-1] < 2
    for w, h, levels in ((31, 8, 1), (32, 1, 1), (40, 300, 4), (700, 9, 4), (32, 8, 4)):
        with pytest.raises(RuntimeError):
            build(w, h, levels)
    for w, h, levels in ((40, 300, 3), (700, 9, 3), (32, 8, 3), (32, 2, 1)):     # the largest legal level counts
        p = build(w, h, levels)
        assert p.num_levels == levels and p.level_info(levels - 1)[:2] == level_shapes(w, h, levels)[-1]
        p.release()


# ---- 7. a recycled slab ----
def _garbage(w, h, kind, rng):
    """kind "selected": huge finite intensities and random depths, so every pixel with a full neighbourhood is selected;
    kind "nonfinite": +-inf, NaN and 1e30 intensities and random depths with holes"""
    if kind == "selected":
        I = (rng.uniform(-1e30, 1e30, (h, w)) * np.where((np.indices((h, w)).sum(0) % 2) == 0, 1, -1)).astype(np.float32)
        Z = rng.uniform(0.3, 9.0, (h, w)).astype(np.float32)
    else:
        I = rng.choice(np.array([np.inf, -np.inf, np.nan, 1e30], np.float32), size=(h, w))
        Z = rng.uniform(0.3, 9.0, (h, w)).astype(np.float32)
        Z[rng.random((h, w)) < 0.3] = np.nan
    return I, Z


def _everything(eng, gref, gcur, w, h, levels):
    """every output of points 1-4 for one pyramid pair, as raw arrays / values"""
    out = []
    for lvl in range(levels):
        out += [gref.download(lvl), gcur.download(lvl)]
    for sel in SELECTIONS + [SELECTIONS[0]]:
        for lvl in range(levels):
            out += list(gref.select(lvl, *sel))
        for lvl in range(levels):
            for _, T in _poses(w, h, lvl):
                cfg = _cfg(lvl, lvl, sel)
                out += list(eng.residual_image(gref, gcur, lvl, T, cfg)) + list(eng.intensity_error_image(gref, gcur, lvl, T, cfg))
                for uw in (False, True):
                    out += list(eng.linearize(gref, gcur, lvl, T, uw, PP, cfg).values())
        r = eng.match(gref, gcur, _cfg(levels - 1, 0, sel))
        out += [r.transformation, r.information, r.log_likelihood, repr(r.levels)]
    return out


def _identical(a, b):
    assert len(a) == len(b)
    for k, (x, y) in enumerate(zip(a, b)):
        if isinstance(x, np.ndarray):
            assert x.dtype == y.dtype and x.shape == y.shape and np.array_equal(x.view(np.uint8), y.view(np.uint8)), k
        elif isinstance(x, float) and np.isnan(x):
            assert np.isnan(y), k
        else:
            assert x == y, k


@pytest.mark.parametrize("w,h,levels", [(161, 50, 3), (40, 300, 3)], ids=["161x50", "40x300"])
def test_recycled_slab(oracle, w, h, levels):
    """Pyramid memory comes from a per-context pool keyed by byte size and is never cleared.  A pyramid built into a slab
    that held garbage of the same size must compute exactly what the same pyramid on a fresh context computes."""
    from dvo_slam_b200.engine import Engine
    _assert_reason(w, h, levels)
    ls = level_shapes(w, h, levels)
    assert any(lw % 2 for lw, _ in ls) or all(len(bands(lw)) == 1 and lw < TILE_W for lw, _ in ls)
    tails = [l for l, (lw, lh) in enumerate(ls) if (lw * lh) % 32]
    assert tails
    a = _scene(w, h)
    oref, ocur = _oracle_pyramids(w, h, levels)

    def tail(mask, l):
        lw, lh = ls[l]
        return mask.reshape(-1)[(lw * lh // 32) * 32:].copy()
    stale = {l: [] for l in tails}      # what the garbage leaves in the mask tail words
    fresh = Engine(device=0)
    try:
        fref = fresh.pyramid(a["I_ref"], a["Z_ref"], a["K"], levels)
        fcur = fresh.pyramid(a["I_cur"], a["Z_cur"], a["K"], levels)
        want = _everything(fresh, fref, fcur, w, h, levels)
    finally:
        fresh.close()
    rng = np.random.default_rng(5)
    for kind in ("selected", "nonfinite"):
        eng = Engine(device=0)
        try:
            garbage = [eng.pyramid(*_garbage(w, h, kind, rng), a["K"], levels) for _ in range(2)]
            for l in tails:
                m = [g.select(l)[1] for g in garbage]
                assert kind != "selected" or all(x.all() for x in m), (kind, l)
                stale[l] += [tail(x, l) for x in m]
            for g in garbage:
                g.release()
            gref = eng.pyramid(a["I_ref"], a["Z_ref"], a["K"], levels)
            gcur = eng.pyramid(a["I_cur"], a["Z_cur"], a["K"], levels)
            _check_pyramid(gref, oref, levels)
            _check_pyramid(gcur, ocur, levels)
            for sel in SELECTIONS:
                for lvl in range(levels):
                    for _, T in _poses(w, h, lvl):
                        _check_level(eng, oracle.mode("mirror"), gref, gcur, oref, ocur, lvl, T, sel)
                _check_alignment(eng, gref, gcur, oref, ocur, levels, sel)
            _identical(_everything(eng, gref, gcur, w, h, levels), want)
        finally:
            eng.close()
    # at every level with a mask tail, some garbage left a tail word that is not the real one: a stale word cannot pass
    for l in tails:
        real = tail(oracle.select(oref, l)[1], l)
        assert any(not np.array_equal(s, real) for s in stale[l]), l
