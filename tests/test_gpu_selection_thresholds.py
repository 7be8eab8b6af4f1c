"""Non-default point selection (DenseTracker::Config::Intensity/DepthDerivativeThreshold) through the level kernel, against
the oracle with the same thresholds.  The default thresholds (0, 0) select nearly every valid pixel; these select a subset,
which runs the re-selection on an already-built pyramid, tiles with few or no points, an odd last point elsewhere, and
levels with fewer than 50 points, where the reference's log-likelihood keeps no term at all (n_keep = 0).

Statements and tolerances are those of test_gpu_parity.py: residual records bit-exact, counts exact, P / LL / A / b to
2e-6 (use_weights 0 and 1), against MIRROR in reference mode and against corrected_mode(oracle) in corrected mode; whole
alignments within POSE_TOL_T / POSE_TOL_R of FAITHFUL.  Each threshold pair's purpose is asserted from the oracle's own
selection, so a case cannot silently stop covering what it is for.
"""
import os

import numpy as np
import pytest

from helpers import (GOLDEN_LEVELS, GOLDEN_SEEDS, POSE_TOL_R, POSE_TOL_T, golden_images, load_golden, nan_equal,
                     odd_point_margin, pose_delta)
from test_corrected_estimator import corrected_mode
from test_gpu_generic_tiles import _rot_z, _shift_z, partial_pair
from tile_geometry import WIN_ROWS, assert_partial_band, in_partial_band

pytestmark = pytest.mark.gpu

PP = np.array([[2000.0, -30.0], [-30.0, 9000.0]], dtype=np.float32)
THRESHOLDS = {
    "moderate": (4.0, 0.02),
    "intensity_only": (8.0, 0.0),
    "depth_only": (0.0, 0.1),
    "sparse": (60.0, 0.5),       # at 640x480 level 4 fewer than 50 points stay valid
}


def _pose():
    T = _rot_z(1.5) @ _shift_z(0.015)
    T[0, 3] = 0.01
    return T


def _cfg(ti, td, **kw):
    from dvo_slam_b200.engine import Config
    return Config(intensity_derivative_threshold=ti, depth_derivative_threshold=td, **kw)


def _planes(c, oracle, levels, engine):
    c["gref"] = engine.pyramid(c["I_ref"], c["Z_ref"], c["K"], levels)
    c["gcur"] = engine.pyramid(c["I_cur"], c["Z_cur"], c["K"], levels)
    c["oref"] = oracle.Pyramid(c["I_ref"], c["Z_ref"], c["K"], levels)
    c["ocur"] = oracle.Pyramid(c["I_cur"], c["Z_cur"], c["K"], levels)
    return c


def _synth(seed, scfg=None):
    from dvo_slam_b200 import synth
    p = synth.make_pair(seed, scfg)
    c = {k: p[k].numpy() for k in ("I_ref", "Z_ref", "I_cur", "Z_cur")}
    c["K"], c["xi"] = p["intrinsics"], p["xi"]
    return c


@pytest.fixture(scope="module")
def corrected(engine):
    from dvo_slam_b200.engine import Engine
    eng = Engine(device=0, estimator="corrected")
    yield eng
    eng.close()


@pytest.fixture(scope="module")
def full(engine, oracle):
    return _planes(_synth(0), oracle, 5, engine)


@pytest.fixture(scope="module")
def wide(engine, oracle):
    """the 720 x 540 scene of test_gpu_generic_tiles: every level to 2 has full bands and a partial one"""
    return _planes(partial_pair(0), oracle, 5, engine)


@pytest.fixture(scope="module")
def odd_size(engine, oracle):
    from dvo_slam_b200 import synth
    scfg = synth.SceneConfig(width=203, height=155, intrinsics=(164.0, 163.5, 101.3, 77.2))
    return _planes(_synth(77, scfg), oracle, 3, engine)


@pytest.fixture(scope="module")
def golden(engine, oracle):
    out = []
    for seed in GOLDEN_SEEDS:
        g = load_golden(seed)
        c = golden_images(g, oracle)
        c["K"], c["T"] = g["K"], g["kat_T"]
        out.append(_planes(c, oracle, GOLDEN_LEVELS, engine))
    return out


def _engines(engine, corrected, oracle):
    return {"reference": (engine, oracle.mode("mirror")), "corrected": (corrected, corrected_mode(oracle))}


def _check(eng, m, oracle, c, lvl, T, ti, td):
    """records bit-exact, counts exact, P / LL / A / b to 2e-6; returns (n, S)"""
    cfg = _cfg(ti, td)
    n_g, img_g = eng.residual_image(c["gref"], c["gcur"], lvl, T, cfg)
    n_o, img_o = oracle.residual_image(c["oref"], c["ocur"], lvl, T, m, ti, td)
    assert n_g == n_o and nan_equal(img_g, img_o), (lvl, ti, td, n_g, n_o)
    for uw in (False, True):
        lg = eng.linearize(c["gref"], c["gcur"], lvl, T, uw, PP, cfg)
        lo = oracle.linearize(c["oref"], c["ocur"], lvl, T, m, uw, PP, ti, td)
        assert lg["n"] == lo["n"] == n_o, (lvl, ti, td, uw)
        if n_o < 6:
            continue
        # relative to the matrix, as A and b: the off-diagonal of P is a cancelling sum, a few 1e-3 of the diagonal here, and
        # fp32 summation order alone moves it by a few 1e-6 of itself (seen: 17.313183 vs 17.313225 beside 4509 and 6611)
        assert np.allclose(lg["precision"], lo["precision"], rtol=0, atol=2e-6 * np.abs(lo["precision"]).max()), \
            (lvl, ti, td, uw, lg["precision"], lo["precision"])
        assert abs(lg["ll"] - lo["ll"]) <= 2e-6 * abs(lo["ll"]) + 0.5, (lvl, ti, td, uw, lg["ll"], lo["ll"])
        assert np.allclose(lg["A"], lo["A"], rtol=0, atol=2e-6 * np.abs(lo["A"]).max())
        assert np.allclose(lg["b"], lo["b"], rtol=0, atol=2e-6 * np.abs(lo["b"]).max())
    S, mask = oracle.select(c["oref"], lvl, ti, td)
    gS, gmask = c["gref"].select(lvl, ti, td)
    assert gS == S and np.array_equal(gmask, mask)
    return n_o, S


def _odd_thresholds(oracle, c, lvl, T, partial_band=False):
    """the first thresholds (1.0, 0.02), (1.25, 0.02), ... that select an odd number S of points at this level whose last
    point has a valid residual by itself (EXACT mode keeps the odd point): the point the reference's SSE loop never visits;
    partial_band: and that point lies in the level's partial band"""
    lw = c["oref"].level_info(lvl)[0]
    for ti in np.arange(1.0, 40.0, 0.25):
        S, mask = oracle.select(c["oref"], lvl, float(ti), 0.02)
        if S % 2 == 0 or S < 50:
            continue
        last = np.flatnonzero(mask.reshape(-1))[-1]
        if partial_band and not in_partial_band(int(last) % lw, lw):
            continue
        _, exact = oracle.residual_image(c["oref"], c["ocur"], lvl, T, oracle.mode("exact"), float(ti), 0.02)
        if not np.isnan(exact[0].reshape(-1)[last]):
            return float(ti), 0.02, last
    raise AssertionError("no threshold gave an odd selection with a valid last point")


@pytest.mark.parametrize("estimator", ["reference", "corrected"])
@pytest.mark.parametrize("lvl", [0, 1, 4])
@pytest.mark.parametrize("name", list(THRESHOLDS))
def test_full_resolution_levels(engine, corrected, oracle, full, name, lvl, estimator):
    eng, m = _engines(engine, corrected, oracle)[estimator]
    ti, td = THRESHOLDS[name]
    n, S = _check(eng, m, oracle, full, lvl, _pose(), ti, td)
    S0, _ = oracle.select(full["oref"], lvl, 0.0, 0.0)
    assert S < S0 or (lvl == 4 and S == S0), (name, lvl, S, S0)     # the thresholds take points away
    if name == "sparse" and lvl == 4:
        assert 6 <= n < 50, n                              # the whole log-likelihood is the dropped tail in reference mode


def test_thresholds_change_what_is_selected(oracle, full):
    """intensity-only and depth-only thresholds each remove points the other keeps, so the two are distinct cases"""
    si, mi = oracle.select(full["oref"], 0, *THRESHOLDS["intensity_only"])
    sd, md = oracle.select(full["oref"], 0, *THRESHOLDS["depth_only"])
    mi, md = mi.astype(bool), md.astype(bool)
    assert (mi & ~md).any() and (md & ~mi).any() and 0 < si and 0 < sd


@pytest.mark.parametrize("estimator", ["reference", "corrected"])
def test_odd_selection_with_a_valid_last_point(engine, corrected, oracle, wide, estimator):
    """An odd selection count S whose last point is valid: reference mode drops it (as MIRROR does), corrected mode keeps it.
    Level 1 of the 720 x 540 scene (bands of 160, 160 and 40 columns), with the last point in the partial band: the
    corrected kernel re-admits it in the generic loop of a partial-band tile."""
    eng, m = _engines(engine, corrected, oracle)[estimator]
    T = _pose()
    c = wide
    assert_partial_band(c["oref"].level_info(1)[0])
    ti, td, last = _odd_thresholds(oracle, c, 1, T, partial_band=True)
    n, S = _check(eng, m, oracle, c, 1, T, ti, td)
    assert S % 2 == 1 and S < oracle.select(c["oref"], 1)[0]
    _, img = eng.residual_image(c["gref"], c["gcur"], 1, T, _cfg(ti, td))
    assert np.isnan(img[0].reshape(-1)[last]) == (estimator == "reference")
    if estimator == "corrected":
        n_r, _ = engine.residual_image(c["gref"], c["gcur"], 1, T, _cfg(ti, td))
        assert n == n_r + 1
        ne, err = eng.intensity_error_image(c["gref"], c["gcur"], 1, T, _cfg(ti, td))
        ne_o, err_o = oracle.intensity_error_image(c["oref"], c["ocur"], 1, T, m, ti, td)
        assert ne == ne_o == n and np.array_equal(err, err_o) and err.reshape(-1)[last] > 0


@pytest.mark.parametrize("estimator", ["reference", "corrected"])
@pytest.mark.parametrize("name", list(THRESHOLDS))
def test_golden_frames(engine, corrected, oracle, golden, name, estimator):
    eng, m = _engines(engine, corrected, oracle)[estimator]
    ns = []
    for c in golden:
        for lvl in range(GOLDEN_LEVELS):
            ns.append(_check(eng, m, oracle, c, lvl, c["T"], *THRESHOLDS[name])[0])
    if name == "sparse":
        assert any(6 <= n < 50 for n in ns), ns


@pytest.mark.parametrize("estimator", ["reference", "corrected"])
@pytest.mark.parametrize("name", list(THRESHOLDS))
def test_odd_image_size(engine, corrected, oracle, odd_size, name, estimator):
    """203x155: partial bands, odd row counts, rounds of 32 pixels ending mid-row"""
    eng, m = _engines(engine, corrected, oracle)[estimator]
    for lvl in range(3):
        _check(eng, m, oracle, odd_size, lvl, _pose(), *THRESHOLDS[name])


@pytest.mark.parametrize("estimator", ["reference", "corrected"])
def test_generic_loop_with_thresholds(engine, corrected, oracle, full, estimator):
    """thresholds together with the poses that force the generic pixel loop (test_gpu_generic_tiles.py): a 20 degree roll
    (tile rows span more rows than the window holds) and a camera moved past the median depth (corners behind it)"""
    eng, m = _engines(engine, corrected, oracle)[estimator]
    assert WIN_ROWS < 160 * np.tan(np.deg2rad(20.0))          # a tile row spans more rows than the window holds
    dz = float(np.nanmedian(full["Z_ref"]))
    for T in (_rot_z(20.0), _shift_z(-dz)):
        n, _ = _check(eng, m, oracle, full, 0, T, *THRESHOLDS["moderate"])
        assert n > 0


def test_selection_cache_switches_thresholds(engine, oracle, full):
    """One reference pyramid through thresholds A, then the defaults, then A again (match and linearize), with select() calls
    for other thresholds in between: every result is bit-identical to the same call on a freshly built pyramid."""
    from dvo_slam_b200.engine import Config
    c = full
    A = THRESHOLDS["moderate"]
    T = _pose()

    def run(ref, th):
        cfg = Config(first_level=4, last_level=0, max_iterations_per_level=50, precision=1e-4,
                     intensity_derivative_threshold=th[0], depth_derivative_threshold=th[1])
        r = engine.match(ref, c["gcur"], cfg, with_iterations=True)
        lin = engine.linearize(ref, c["gcur"], 1, T, True, PP, cfg)
        return r, lin

    def same(a, b):
        (ra, la), (rb, lb) = a, b
        assert np.array_equal(ra.transformation, rb.transformation) and np.array_equal(ra.information, rb.information)
        assert ra.log_likelihood == rb.log_likelihood and ra.levels == rb.levels
        assert [(it["n"], it["nll"]) for it in ra.iterations] == [(it["n"], it["nll"]) for it in rb.iterations]
        for k in ("n", "ll"):
            assert la[k] == lb[k]
        for k in ("precision", "A", "b"):
            assert np.array_equal(la[k], lb[k])

    shared = engine.pyramid(c["I_ref"], c["Z_ref"], c["K"], 5)
    sequence = [A, (0.0, 0.0), A, (0.0, 0.0)]
    for k, th in enumerate(sequence):
        fresh = engine.pyramid(c["I_ref"], c["Z_ref"], c["K"], 5)
        same(run(shared, th), run(fresh, th))
        shared.select(0, *THRESHOLDS["sparse"])           # another selection on the same pyramid must not leak into the next call
        shared.select(3, *THRESHOLDS["intensity_only"])
    r_a, r_0 = run(shared, A)[0], run(shared, (0.0, 0.0))[0]
    assert [l["valid_pixels"] for l in r_a.levels] != [l["valid_pixels"] for l in r_0.levels]


def test_whole_alignments(engine, oracle):
    """640x480 pairs with thresholds: pose within the stated tolerance of FAITHFUL, the same selected-pixel counts, and where
    the iteration counts equal MIRROR's the pose agrees to 1e-4, or to the oracle's own spread where that is larger.  With
    ~40k points at level 0 instead of ~270k the fp32 summation order matters more: on seed 3 the oracle's MIRROR mode with
    and without fused pixel arithmetic ends 1.8e-3 m apart, and the GPU, with MIRROR's iteration counts, 2.7e-4 m from it."""
    from dvo_slam_b200.engine import Config
    compared = 0
    for seed, name in ((0, "moderate"), (1, "intensity_only"), (2, "depth_only"), (3, "moderate")):
        ti, td = THRESHOLDS[name]
        c = _planes(_synth(seed), oracle, 5, engine)
        kw = dict(first_level=4, last_level=0, max_iterations_per_level=50, precision=1e-4,
                  intensity_derivative_threshold=ti, depth_derivative_threshold=td)
        r = engine.match(c["gref"], c["gcur"], Config(**kw))
        fa = oracle.match(c["oref"], c["ocur"], oracle.config(**kw), oracle.mode("faithful"))
        mi = oracle.match(c["oref"], c["ocur"], oracle.config(**kw), oracle.mode("mirror"))
        dt, dr = pose_delta(fa["T"], r.transformation)
        assert dt < POSE_TOL_T and dr < POSE_TOL_R, (seed, name, dt, dr)
        assert [l["valid_pixels"] for l in r.levels] == [l["valid_pixels"] for l in fa["levels"]]
        assert r.levels[-1]["valid_pixels"] < oracle.select(c["oref"], 0)[0]
        if [l["num_iterations"] for l in r.levels] == [l["num_iterations"] for l in mi["levels"]]:
            compared += 1
            unfused = oracle.mode("mirror")
            unfused.fused_pixel_math = 0
            st, sr = pose_delta(mi["T"], oracle.match(c["oref"], c["ocur"], oracle.config(**kw), unfused)["T"])
            dt, dr = pose_delta(mi["T"], r.transformation)
            assert dt < max(1e-4, st) and dr < max(1e-4, sr), (seed, name, dt, dr, st, sr)
    assert compared >= 1


def test_fused_batch_with_thresholds(engine, oracle):
    """72 640x480 pairs (one fused launch for all levels) with thresholds, each reference pyramid appearing 18 times: every
    record bit-equal to a single alignment, and to the same batch run as one launch per level group"""
    from dvo_slam_b200.engine import Config
    cs = [_synth(s) for s in range(4)]
    K = cs[0]["K"]
    refs = [engine.pyramid(c["I_ref"], c["Z_ref"], K, 5) for c in cs]
    curs = [engine.pyramid(c["I_cur"], c["Z_cur"], K, 5) for c in cs]
    n = 72
    idx = [(i * 3) % 4 for i in range(n)]
    ti, td = THRESHOLDS["moderate"]
    cfg = Config(first_level=4, last_level=0, max_iterations_per_level=50, precision=1e-4,
                 intensity_derivative_threshold=ti, depth_derivative_threshold=td)
    b = [refs[k] for k in idx], [curs[k] for k in idx]
    first = engine.match_batch(*b, cfg)                   # re-selects the four pyramids for these thresholds
    l0 = engine.kernel_launches()
    batch = engine.match_batch(*b, cfg)                   # selections cached: launches are the alignment's only
    for x, y in zip(first, batch):
        assert np.array_equal(x.transformation, y.transformation)
    fused_launches = engine.kernel_launches() - l0
    os.environ["DVO_B200_NO_FUSE"] = "1"
    try:
        l0 = engine.kernel_launches()
        unfused = engine.match_batch(*b, cfg)
        assert engine.kernel_launches() - l0 == fused_launches + 1
    finally:
        del os.environ["DVO_B200_NO_FUSE"]
    single = [engine.match(refs[k], curs[k], cfg) for k in range(4)]
    for i in range(n):
        for other in (single[idx[i]], unfused[i]):
            assert np.array_equal(batch[i].transformation, other.transformation), i
            assert np.array_equal(batch[i].information, other.information), i
            assert batch[i].log_likelihood == other.log_likelihood and batch[i].levels == other.levels, i
    S0 = oracle.select(oracle.Pyramid(cs[0]["I_ref"], cs[0]["Z_ref"], K, 5), 0, ti, td)[0]
    assert batch[0].levels[-1]["valid_pixels"] == S0


@pytest.mark.parametrize("th", [(0.0, 0.0), THRESHOLDS["moderate"], THRESHOLDS["sparse"]])
def test_intensity_error_image_reference_mode(engine, oracle, golden, full, th):
    """computeIntensityErrorImage in reference mode against the oracle's MIRROR mode, at default and non-default thresholds"""
    m = oracle.mode("mirror")
    for c, lvls, T in [(g, range(GOLDEN_LEVELS), g["T"]) for g in golden] + [(full, (0, 4), _pose())]:
        for lvl in lvls:
            n_g, img_g = engine.intensity_error_image(c["gref"], c["gcur"], lvl, T, _cfg(*th))
            n_o, img_o = oracle.intensity_error_image(c["oref"], c["ocur"], lvl, T, m, *th)
            assert n_g == n_o and np.array_equal(img_g, img_o), (lvl, th, n_g, n_o)


def test_intensity_error_image_odd_point_stays_zero(engine, oracle):
    """the odd-selection case of tests/helpers.py in reference mode: the odd last point is never visited, so its entry is 0"""
    margin, im, oref, ocur = odd_point_margin(oracle)
    K = load_golden(GOLDEN_SEEDS[0])["K"]
    Z = im["Z_ref"].copy()
    Z[-margin:, :] = np.nan
    Z[:, -margin:] = np.nan
    gref = engine.pyramid(im["I_ref"], Z, K, 1)
    gcur = engine.pyramid(im["I_ref"], im["Z_ref"], K, 1)
    S, mask = gref.select(0)
    assert S % 2 == 1
    last = np.flatnonzero(mask.reshape(-1))[-1]
    n_g, img_g = engine.intensity_error_image(gref, gcur, 0, np.eye(4))
    n_o, img_o = oracle.intensity_error_image(oref, ocur, 0, np.eye(4), oracle.mode("mirror"))
    assert n_g == n_o and np.array_equal(img_g, img_o)
    _, exact = oracle.residual_image(oref, ocur, 0, np.eye(4), oracle.mode("exact"))
    assert img_g.reshape(-1)[last] == 0.0 and not np.isnan(exact[0].reshape(-1)[last])     # valid, but never visited
