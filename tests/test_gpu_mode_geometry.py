"""The photometric mode, motion priors, weight maps and the multi-hypothesis match at the tile-edge image sizes.

The sizes are test_gpu_geometry.SIZES (each with its stated reason) and two more whose partial band or odd width falls on a
level of more than COARSE_TILES tiles, which runs several CTAs per pair: 641 x 481 (bands 160, 160, 160, 160, 1; 69
strips) and 497 x 373 (bands 160, 160, 160, 17; 54 strips, the last of 2 rows).  Per size and estimator:
  records        residual_image(..., ab=) bit for bit against the oracle (MIRROR or the corrected mode), every level, two
                 poses, every (alpha, beta) of the ledger; linearize(..., ab=) against the ledger (tests/linearization_ledger.py)
  alignments     match_batch_photometric and match_batch(prior_information=) in the photometric, prior and photometric + prior
                 modes: batch = reversed batch = single alignments bit for bit, also under test_gpu_prior.PLANS; Lambda = mu I
                 is the mu path; the pose within 1e-4 of the oracle's where the iteration counts are the oracle's
  step replay    the photometric + prior log of one alignment per size (tests/step_replay.py)
  weight maps    every map entry against the fp64 warp (tests/warp64.py), in the four modes, last levels 0 and levels - 1,
                 a current-role mask on one pair, device and host outputs in padded buffers prefilled with a sentinel
  hypotheses     k = 4 with photometric, prior and maps, screened on a level with a partial band or an odd width: the
                 helpers of test_gpu_hypotheses_modes.py check continuation, screening, pick and maps
Each test asserts the case it needs from the geometry first.  At the module's end two lines give the ledger maxima of the
photometric mode at these sizes and the largest |kernel - fp64| / bound of the maps, with the tie band's share.
"""
import ctypes as C
import dataclasses
import json

import numpy as np
import pytest

import step_replay as sr
import warp64 as W
import weight_maps_model as wmm
from helpers import nan_equal, pose_delta
from launch_plan_model import COARSE_TILES, level_geometry
from test_corrected_estimator import corrected_mode
from test_gpu_geometry import SIZES, _assert_reason, _edge_shift, _intrinsics, _scene, _small_motion
from test_gpu_hypotheses import _cfg as _hcfg
from test_gpu_hypotheses_modes import _check_call, _inputs
from test_gpu_linearization_ledger import ABS, _check, engines, maxima  # noqa: F401  (fixtures: the ledger's line)
from test_gpu_prior import PLANS, _same
from test_gpu_step_replay import _gpu_log
from tile_geometry import TILE_H, TILE_W, bands, has_partial_band, level_shapes, strips

pytestmark = pytest.mark.gpu

NEW_SIZES = [(641, 481, 5), (497, 373, 4)]
ALL = SIZES + NEW_SIZES
IDS = [f"{w}x{h}" for w, h, _ in ALL]
EXPOSURE = (1.1, -7.5)
DELTA = np.array([4e-3, -3e-3, 2e-3, -2e-3, 3e-3, 1e-3])
PRIORS = (sr._spd(3, 1e9), sr._rank_one(1e12), sr.PRIOR_MU * np.eye(6))
MODES = ("photometric", "prior", "photometric+prior")
MAP_MODES = ("default", "photometric", "prior", "photometric+prior")      # test_gpu_weight_maps.MODES
MASK_WEIGHT = 0.3
ESTIMATORS = ("reference", "corrected")


def _assert_new_reason(w, h, levels):
    """a partial band or an odd width on a level of more than COARSE_TILES tiles"""
    tiles = [s * b for s, b, _ in level_geometry(w, h, levels)]
    if (w, h) == (641, 481):       # a 1-column band and an odd width on a 345-tile level 0
        assert bands(w) == [TILE_W] * 4 + [1] and len(strips(h)) == 69 and w % 2 == 1 and tiles[0] > COARSE_TILES
    elif (w, h) == (497, 373):     # a 17-column band, odd width and height, a 2-row last strip, on a 216-tile level 0
        assert len(bands(w)) == 4 and bands(w)[-1] == 17 and w % 2 == 1 and h % 2 == 1 and strips(h)[-1] == 2
        assert tiles[0] > COARSE_TILES
    else:
        raise AssertionError(f"no stated reason for {w}x{h}")


def _reason(w, h, levels):
    if (w, h, levels) in SIZES:
        _assert_reason(w, h, levels)
    else:
        _assert_new_reason(w, h, levels)


def test_new_sizes_reach_several_ctas_per_pair():
    """the new sizes are why SIZES is not enough: no SIZES level has more than COARSE_TILES tiles"""
    for w, h, levels in SIZES:
        assert max(s * b for s, b, _ in level_geometry(w, h, levels)) <= COARSE_TILES
    for w, h, levels in NEW_SIZES:
        _assert_new_reason(w, h, levels)


@pytest.fixture(scope="module")
def report(request):
    """the maps' largest |kernel - fp64| / bound and tie band, printed at the module's end past output capture"""
    rep = W.Report()
    yield rep
    line = "weight maps against the fp64 warp (|kernel - fp64| / bound): " + json.dumps(
        {**{k: float("%.3g" % v) for k, v in rep.maxima.items()}, "tie_band": rep.tie, "candidates": rep.candidates})
    cap = request.config.pluginmanager.getplugin("capturemanager")
    if cap is None:
        print("\n" + line)
    else:
        with cap.global_and_fixture_disabled():
            print("\n" + line)


def _mask(w, h):
    m = np.ones((h, w), np.uint8)
    m[h // 4:h // 2 + 1, w // 5:w // 2] = 0
    return m


@pytest.fixture(scope="module")
def pyramids(engine):
    """(w, h, levels, masked) -> (gpu ref, gpu cur, oracle ref, oracle cur); the current frame under EXPOSURE"""
    from dvo_slam_b200 import synth
    from oracle import oracle_py as orc
    cache = {}

    def get(w, h, levels, masked=False):
        key = (w, h, levels, masked)
        if key not in cache:
            a = _scene(w, h)
            Ic = synth.exposure(a["I_cur"], *EXPOSURE)
            kw = {"mask": _mask(w, h), "mask_roles": "both"} if masked else {}
            cache[key] = (engine.pyramid(a["I_ref"], a["Z_ref"], a["K"], levels, **kw), engine.pyramid(Ic, a["Z_cur"], a["K"], levels, **kw),
                          None if masked else orc.Pyramid(a["I_ref"], a["Z_ref"], a["K"], levels),
                          None if masked else orc.Pyramid(Ic, a["Z_cur"], a["K"], levels))
        return cache[key]
    return get


def _mode(oracle, estimator):
    return oracle.mode("mirror") if estimator == "reference" else corrected_mode(oracle)


def _cfg(levels, last=0, mu=0.0):
    from dvo_slam_b200.engine import Config
    return Config(first_level=levels - 1, last_level=last, max_iterations_per_level=50, precision=1e-4, mu=mu, use_initial_estimate=1)


# ---- records and linearisation -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("estimator", ESTIMATORS)
@pytest.mark.parametrize("w,h,levels", ALL, ids=IDS)
def test_photometric_records_and_linearisation(engine, engines, maxima, oracle, pyramids, w, h, levels, estimator):
    _reason(w, h, levels)
    gref, gcur, oref, ocur = pyramids(w, h, levels)
    a = _scene(w, h)
    mode = _mode(oracle, estimator)
    eng = engines[estimator]
    checked = 0
    for lvl in range(levels):
        for T in (_small_motion(), _edge_shift(w, h, a["K"], a["Z_ref"])):
            for ab in ABS:
                n_g, img_g = eng.residual_image(gref, gcur, lvl, T, None, ab)
                n_o, img_o = oracle.residual_image(oref, ocur, lvl, T, mode, ab=ab)
                assert n_g == n_o and nan_equal(img_g, img_o), (lvl, ab, n_g, n_o)
                checked += n_o > 0
        for ab in ABS:
            _check(engines, maxima, "photometric-sizes", estimator, gref, gcur, lvl, _small_motion(), a["K"], ab=ab)
    assert checked >= levels


# ---- whole alignments ----------------------------------------------------------------------------------------------------
def _run(eng, refs, curs, cfg, T0, photometric, prior, iters=True):
    if photometric:
        return eng.match_batch_photometric(refs, curs, cfg, T0, with_iterations=iters, prior_information=prior)
    return eng.match_batch(refs, curs, cfg, T0, with_iterations=iters, prior_information=prior), None


def _eq(a, b):
    return np.array_equal(np.asarray(a), np.asarray(b), equal_nan=True)


@pytest.mark.parametrize("estimator", ESTIMATORS)
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("w,h,levels", ALL, ids=IDS)
def test_alignments(engine, oracle, pyramids, w, h, levels, mode, estimator, monkeypatch):
    from dvo_slam_b200 import synth
    _reason(w, h, levels)
    gref, gcur, oref, ocur = pyramids(w, h, levels)
    photometric, use_prior = "photometric" in mode, "prior" in mode
    n = len(PRIORS)
    T0 = [synth.se3_exp(DELTA * (1 + 0.3 * k)) for k in range(n)]
    lam = np.stack(PRIORS) if use_prior else None
    refs, curs, cfg = [gref] * n, [gcur] * n, _cfg(levels)
    engine.set_estimator(estimator)
    try:
        single = [_run(engine, [gref], [gcur], cfg, [T0[i]], photometric, None if lam is None else lam[i:i + 1]) for i in range(n)]
        rb, abb = _run(engine, refs, curs, cfg, T0, photometric, lam)
        rr, abr = _run(engine, refs, curs, cfg, T0[::-1], photometric, None if lam is None else lam[::-1])
        for i in range(n):
            s, sab = single[i]
            assert _same(rb[i], s[0]) and _same(rr[n - 1 - i], s[0]), i
            assert sab is None or (_eq(abb[i], sab[0]) and _eq(abr[n - 1 - i], sab[0])), i
        big = 12
        for knob, value in PLANS:
            if knob:
                monkeypatch.setenv(knob, value)
            r, rab = _run(engine, refs * big, curs * big, cfg, T0 * big, photometric, None if lam is None else np.concatenate([lam] * big),
                          iters=False)
            if knob:
                monkeypatch.delenv(knob)
            for i in range(n * big):
                s, sab = single[i % n]
                assert _eq(r[i].transformation, s[0].transformation) and _eq(r[i].information, s[0].information), (knob, i)
                assert rab is None or _eq(rab[i], sab[0]), (knob, i)
        if use_prior:   # Lambda = mu I (the last prior) is the mu path (DESIGN §4.9)
            mu = float(PRIORS[-1][0, 0])
            want, wab = _run(engine, [gref], [gcur], _cfg(levels, mu=mu), [T0[-1]], photometric, None)
            assert _same(single[-1][0][0], want[0], ll_tol=1e-14)
            assert wab is None or _eq(single[-1][1][0], wab[0])
        same = 0
        ocfg = oracle.config(first_level=levels - 1, last_level=0, max_iterations_per_level=50, precision=1e-4, use_initial_estimate=1)
        m = _mode(oracle, estimator)
        for i in range(n):
            kw = dict(T_init=T0[i], prior=None if lam is None else lam[i], photometric=photometric)
            o = oracle.match(oref, ocur, ocfg, m, **kw)
            r = single[i][0][0]
            if [(l["termination"], l["num_iterations"]) for l in r.levels] != [(l["termination"], l["num_iterations"]) for l in o["levels"]]:
                continue
            same += 1
            unf = type(m).from_buffer_copy(m)
            unf.fused_pixel_math = 0
            st, sr_ = pose_delta(o["T"], oracle.match(oref, ocur, ocfg, unf, **kw)["T"])
            dt, dr = pose_delta(o["T"], r.transformation)
            assert dt < max(1e-4, st) and dr < max(1e-4, sr_), (i, dt, dr, st, sr_)
        print(f"{w}x{h} {mode} {estimator}: {same} of {n} alignments with the oracle's iteration counts")
    finally:
        engine.set_estimator("reference")


# ---- step replay ---------------------------------------------------------------------------------------------------------
# step_replay.PHOTOMETRIC, with the prior term held to 2e-11 instead of 2e-12 of its sensitivity scale.  The replay's pose
# agrees with the kernel's to the pose bound, 1e-14 absolute per entry; carried through li = log(initial) that moves
# li^T Lambda li by up to ~2 |Lambda li| 6e-14, which relative to the scale 2 |Lambda li| |li| is 6e-14 / |li|: 2e-11 for
# the |li| of a few 1e-3 these alignments start at (T_init = exp(DELTA)).  Measured at most 4.7e-12 (32 x 8) on an H100.
REPLAY_BOUNDS = dataclasses.replace(sr.PHOTOMETRIC, prior_rel=2e-11)
@pytest.mark.parametrize("w,h,levels", ALL, ids=IDS)
def test_step_replay(engine, oracle, w, h, levels):
    from dvo_slam_b200 import synth
    _reason(w, h, levels)
    a = _scene(w, h)
    c = sr._base(I_ref=a["I_ref"], Z_ref=a["Z_ref"], I_cur=synth.exposure(a["I_cur"], *EXPOSURE), Z_cur=a["Z_cur"], K=a["K"],
                 levels=levels, cfg=dict(first_level=levels - 1, last_level=0, max_iterations_per_level=50, precision=1e-4,
                                         use_initial_estimate=1),
                 T_init=synth.se3_exp(DELTA), photometric=True, prior=PRIORS[0])
    log = _gpu_log(engine, c)
    rep = sr.replay_case(c, log, REPLAY_BOUNDS)
    print(f"{w}x{h}: replay maxima {json.dumps({k: float('%.3g' % v) for k, v in rep.maxima.items()})}")
    assert not rep.failures, rep.failures[:5]


# ---- weight maps against the fp64 warp -----------------------------------------------------------------------------------
SENTINEL_F, SENTINEL_B = -12345.0, 9


def _padded_maps(n, w, h, w0, h0, device):
    """every output in buffers with a longer row and a larger image than the map, prefilled with a sentinel, and the
    dvo_b200_weight_maps that points at them (device: torch CUDA tensors, else numpy)"""
    import torch
    from dvo_slam_b200.engine import MAPS_MEMORY, MapPlane, WeightMaps
    if device:
        mk = lambda shape, dt, v: torch.full(shape, v, dtype=dt, device="cuda")
        ptr = lambda t: t.data_ptr()
        f32, u8, f64 = torch.float32, torch.uint8, torch.float64
    else:
        mk = lambda shape, dt, v: np.full(shape, v, dtype=dt)
        ptr = lambda t: t.ctypes.data
        f32, u8, f64 = np.float32, np.uint8, np.float64
    bufs = {k: mk((n, h + 1, w + 3), f32, SENTINEL_F) for k in ("weight", "residual_i", "residual_z")}
    bufs["mask"] = mk((n, h0 + 1, w0 + 5), u8, SENTINEL_B)
    bufs["estimate"] = mk((n, 4, 4), f64, 0.0)
    bufs["precision"] = mk((n, 2, 2), f32, 0.0)
    wm = WeightMaps()
    wm.memory = MAPS_MEMORY["device" if device else "host"]
    for k in ("weight", "residual_i", "residual_z"):
        setattr(wm, k, MapPlane(ptr(bufs[k]), 4 * (w + 3), 4 * (w + 3) * (h + 1)))
    wm.mask = MapPlane(ptr(bufs["mask"]), w0 + 5, (w0 + 5) * (h0 + 1))
    wm.mask_weight = MASK_WEIGHT
    wm.estimate = C.cast(ptr(bufs["estimate"]), C.POINTER(C.c_double))
    wm.precision = C.cast(ptr(bufs["precision"]), C.POINTER(C.c_float))
    if device:
        torch.cuda.synchronize()
    return bufs, wm


def _unpad(bufs, w, h, w0, h0):
    """the maps inside their extents; asserts that nothing outside them was written"""
    out = {}
    for k in ("weight", "residual_i", "residual_z"):
        a = np.asarray(bufs[k].cpu() if hasattr(bufs[k], "cpu") else bufs[k])
        assert (a[:, h:] == SENTINEL_F).all() and (a[:, :, w:] == SENTINEL_F).all(), k
        out[k] = a[:, :h, :w]
        assert not (out[k] == SENTINEL_F).any(), k             # every float inside written
    m = np.asarray(bufs["mask"].cpu() if hasattr(bufs["mask"], "cpu") else bufs["mask"])
    assert (m[:, h0:] == SENTINEL_B).all() and (m[:, :, w0:] == SENTINEL_B).all()
    out["mask"] = m[:, :h0, :w0]
    assert np.isin(out["mask"], (0, 1)).all()                   # every byte inside written
    for k in ("estimate", "precision"):
        out[k] = np.asarray(bufs[k].cpu() if hasattr(bufs[k], "cpu") else bufs[k])
    return out


@pytest.mark.parametrize("estimator", ESTIMATORS)
@pytest.mark.parametrize("mode", MAP_MODES)
@pytest.mark.parametrize("w,h,levels", ALL, ids=IDS)
def test_weight_maps_against_the_fp64_warp(engine, pyramids, report, w, h, levels, mode, estimator):
    """pair 0 plain, pair 1 with a mask in both roles (the kCurMask instances); last levels 0 and levels - 1"""
    from dvo_slam_b200 import synth
    _reason(w, h, levels)
    photometric, use_prior = "photometric" in mode, "prior" in mode
    plain, masked = pyramids(w, h, levels), pyramids(w, h, levels, True)
    refs, curs = [plain[0], masked[0]], [plain[1], masked[1]]
    T0 = [synth.se3_exp(DELTA), synth.se3_exp(-0.7 * DELTA)]
    lam = np.stack(PRIORS[:2]) if use_prior else None
    w0, h0 = w, h
    engine.set_estimator(estimator)
    try:
        for last in (0, levels - 1):
            lw, lh, _ = refs[0].level_info(last)
            # the stated case: the maps' level has an odd width, a partial band or a partial last strip
            assert lw % 2 == 1 or has_partial_band(lw) or lh % TILE_H != 0, (lw, lh, last)
            cfg = _cfg(levels, last)
            dev, wm = _padded_maps(2, lw, lh, w0, h0, True)
            res, ab = engine._match(refs, curs, cfg, T0, True, lam, photometric, None, wm)
            host, wmh = _padded_maps(2, lw, lh, w0, h0, False)
            res_h, ab_h = engine._match(refs, curs, cfg, T0, False, lam, photometric, None, wmh)
            d, hst = _unpad(dev, lw, lh, w0, h0), _unpad(host, lw, lh, w0, h0)
            for k in d:
                assert np.array_equal(d[k], hst[k], equal_nan=d[k].dtype.kind == "f"), (last, k)
            for i in range(2):
                assert _eq(res[i].transformation, res_h[i].transformation)
                wgt, e_i, e_z, P, T = d["weight"][i], d["residual_i"][i], d["residual_z"][i], d["precision"][i], d["estimate"][i]
                assert np.abs(np.linalg.inv(T) - res[i].transformation).max() < 1e-12
                if res[i].is_nan():
                    assert np.isnan(wgt).all() and (d["mask"][i] == 1).all()
                    continue
                ab_i = None if ab is None else ab[i]
                _, planes = engine.residual_image(refs[i], curs[i], last, T, cfg, ab=ab_i)
                assert nan_equal(e_i, planes[0]) and nan_equal(e_z, planes[1]), (last, i)
                fin = np.isfinite(wgt)
                ref64 = wmm.student_weights(e_i[fin], e_z[fin], P)
                assert (np.abs(wgt[fin].astype(np.float64) - ref64) <= 4 * np.spacing(np.abs(ref64).astype(np.float32))).all()
                sel = W.selection(refs[i].select(last)[1], estimator)
                want = W.warp64(refs[i].download(last), curs[i].download(last), sel, refs[i].level_info(last)[2],
                                curs[i].level_info(last)[2], T, P, ab_i)
                n_before = len(report.failures)
                W.compare(want, e_i, e_z, wgt, d["mask"][i], last, MASK_WEIGHT, report)
                assert len(report.failures) == n_before, (last, i, report.failures[n_before:][:4])
    finally:
        engine.set_estimator("reference")
    assert report.tie <= 0.01 * report.candidates, (report.tie, report.candidates)


def test_some_maps_size_writes_level0_pixels_past_the_last_level():
    """the footprint branch of k_weight_maps: some level-0 column or row has no level-L parent at a size and last level of
    the test above (odd level sizes)"""
    hits = [(w, h, L) for w, h, levels in ALL for L in (0, levels - 1)
            for lw, lh in [level_shapes(w, h, levels)[L]] if (lw << L) < w or (lh << L) < h]
    assert any((w, h) == (641, 481) for w, h, _ in hits) and len(hits) >= 4, hits


# ---- the multi-hypothesis match ------------------------------------------------------------------------------------------
def _screen_level(w, h, levels):
    """the finest level above 0 with a partial band or an odd width: the screening ends there"""
    shapes = level_shapes(w, h, levels)
    for s in range(1, levels):
        lw = shapes[s][0]
        if lw % 2 == 1 or has_partial_band(lw):
            return s
    raise AssertionError(f"{w}x{h}: no level above 0 with a partial band or an odd width")


def _truth(w, h):
    """the pose the scene of _scene(w, h) was made with"""
    from dvo_slam_b200 import synth
    return synth.make_pair(1000 * w + h, synth.SceneConfig(width=w, height=h, intrinsics=_intrinsics(w, h)))["T_true"]


@pytest.mark.parametrize("estimator", ESTIMATORS)
@pytest.mark.parametrize("w,h,levels", ALL, ids=IDS)
def test_hypotheses(engine, pyramids, w, h, levels, estimator):
    _reason(w, h, levels)
    s = _screen_level(w, h, levels)
    lw = level_shapes(w, h, levels)[s][0]
    assert lw % 2 == 1 or has_partial_band(lw)
    plain, masked = pyramids(w, h, levels), pyramids(w, h, levels, True)
    batch = [{"pair": {"T_true": _truth(w, h)}}] * 2
    H, lam, ab0 = _inputs(batch, 4, w + h, True, True)
    engine.set_estimator(estimator)
    try:
        _check_call(engine, [plain[0], masked[0]], [plain[1], masked[1]], H, s, 0.3, _hcfg(levels - 1, 0), lam, ab0, True, True)
    finally:
        engine.set_estimator("reference")
