"""Multi-hypothesis alignment in the photometric mode, with motion priors and with weight maps, on the GPU
(dvo_b200_match_batch_hypotheses_modes): k = 1 is the single-pair entry point of the mode; with k = 4 the continuation is the
single alignment from the chosen (H, Lambda, (alpha, beta)_0) and the screening runs are those alignments stopped at the screen
level, bit for bit, under both estimators, with masks, mixed intrinsics, every batch position and launch plan; the maps are
those of dvo_b200_match_batch_maps in device and host memory; under an exposure change the near start wins; refusals move no
counters; the old entry point is the new one with every mode argument NULL."""
import ctypes as C

import numpy as np
import pytest

import hypotheses_model as hm
from dvo_slam_b200 import synth
from dvo_slam_b200.engine import MAPS_MEMORY, CResult, Config, MapPlane, WeightMaps
from test_gpu_hypotheses import FIRST, LAST, NEAR, SCENE, TOL_R, TOL_T, WIDE, _cfg, _eq, _hypotheses, _mask, _pose_err, _same

pytestmark = pytest.mark.gpu
MASK_WEIGHT = 0.3
MODES = [dict(photometric=True), dict(prior=True), dict(photometric=True, prior=True)]


def _lam(rng, k):
    """k symmetric positive semi-definite 6 x 6 priors of the order of an alignment's normal equations; the first is 0"""
    out = [np.zeros((6, 6))]
    while len(out) < k:
        M = rng.normal(size=(6, 6)) * np.sqrt(np.r_[[2e3] * 3, [2e4] * 3])[:, None]
        L = M @ M.T
        out.append(0.5 * (L + L.T))
    return np.stack(out)


def _ab0(rng, k):
    return np.stack([[1.0, 0.0]] + [[rng.uniform(0.9, 1.1), rng.uniform(-5, 5)] for _ in range(k - 1)])


def _inputs(batch, k, seed, photometric, prior):
    rng = np.random.default_rng(seed)
    H = np.stack([_hypotheses(q["pair"], k, i) for i, q in enumerate(batch)])
    lam = np.stack([_lam(rng, k) for _ in batch]) if prior else None
    ab0 = np.stack([_ab0(rng, k) for _ in batch]) if photometric else None
    return H, lam, ab0


def _single(engine, refs, curs, cfg, T, lam=None, ab0=None, photometric=False, maps=False, iterations=True):
    """the single-pair entry point of the mode: (results, (alpha, beta) or None, maps or None)"""
    if maps:
        out = engine.match_batch_maps(refs, curs, cfg, T, prior_information=lam, photometric_init=ab0, photometric=photometric,
                                      mask_weight=MASK_WEIGHT, with_iterations=iterations)
        return out[0], (out[2] if photometric else None), out[1]
    if photometric:
        res, ab = engine.match_batch_photometric(refs, curs, cfg, T, ab0, with_iterations=iterations, prior_information=lam)
        return res, ab, None
    return engine.match_batch(refs, curs, cfg, T, with_iterations=iterations, prior_information=lam), None, None


def _call(engine, refs, curs, H, s, ratio, cfg, lam, ab0, photometric, maps, iterations=True, screen=True):
    """one modes call, unpacked: (results, best, scores, screen results, (alpha, beta), screen (alpha, beta), maps)"""
    out = list(engine.match_batch_hypotheses(refs, curs, H, s, ratio, cfg, with_iterations=iterations, screen_results=screen,
                                             prior_information=lam, photometric_init=ab0, photometric=photometric, maps=maps,
                                             mask_weight=MASK_WEIGHT if maps else None))
    res, best, scores = out[:3]
    rest = out[3:]
    scr = rest.pop(0) if screen else None
    ab = rest.pop(0) if photometric else None
    scr_ab = rest.pop(0) if photometric and screen else None
    mp = rest.pop(0) if maps else None
    assert not rest
    return res, best, scores, scr, ab, scr_ab, mp


def _same_maps(a, b):
    assert a.keys() == b.keys()
    for key in a:
        x, y = a[key].cpu().numpy(), b[key].cpu().numpy()
        assert np.array_equal(x, y, equal_nan=x.dtype.kind == "f"), key


def _check_call(engine, refs, curs, H, s, ratio, cfg, lam, ab0, photometric, maps):
    """one call against its definition: screening runs, scores, choice, continuation (with its log), (alpha, beta) and maps"""
    n, k = H.shape[:2]
    res, best, scores, scr, ab, scr_ab, mp = _call(engine, refs, curs, H, s, ratio, cfg, lam, ab0, photometric, maps)
    cfg_s = _cfg(cfg.first_level, s, mu=cfg.mu)
    rep = lambda xs: [x for x in xs for _ in range(k)]
    want, want_ab, _ = _single(engine, rep(refs), rep(curs), cfg_s, H.reshape(n * k, 4, 4),
                               None if lam is None else lam.reshape(n * k, 6, 6), None if ab0 is None else ab0.reshape(n * k, 2),
                               photometric, iterations=False)
    for p in range(n):
        want_scores = [hm.score(want[p * k + j].levels[-1], ratio) for j in range(k)]
        assert _eq(scores[p], want_scores), (p, scores[p], want_scores)
        assert best[p] == hm.pick(want_scores), p
        for j in range(k):
            assert _same(scr[p][j], want[p * k + j], iterations=False), (p, j)
            if photometric:
                assert np.array_equal(scr_ab[p, j], want_ab[p * k + j]), (p, j)
        b = best[p]
        one, one_ab, one_maps = _single(engine, [refs[p]], [curs[p]], cfg, H[p, b:b + 1], None if lam is None else lam[p, b:b + 1],
                                        None if ab0 is None else ab0[p, b:b + 1], photometric, maps)
        assert _same(res[p], one[0]), p
        assert res[p].iterations and len(res[p].levels) == cfg.first_level - cfg.last_level + 1
        if photometric:
            assert np.array_equal(ab[p], one_ab[0]), p
        if maps:
            _same_maps({key: v[p:p + 1] for key, v in mp.items()}, one_maps)
    return res, best


@pytest.fixture(scope="module")
def batch(engine):
    """four 320 x 240 pairs, 3 levels, the current frames under different exposures"""
    out = []
    for i, (g, b) in enumerate(((1.0, 0.0), (1.1, -6.0), (0.9, 8.0), (1.15, -12.0))):
        p = synth.make_pair(80 + i, SCENE)
        out.append({"ref": engine.pyramid(p["I_ref"].numpy(), p["Z_ref"].numpy(), SCENE.intrinsics, 3),
                    "cur": engine.pyramid(synth.exposure(p["I_cur"].numpy(), g, b), p["Z_cur"].numpy(), SCENE.intrinsics, 3),
                    "pair": p})
    return out


def _ids(m):
    return "+".join(sorted(m))


@pytest.mark.parametrize("estimator", ["reference", "corrected"])
@pytest.mark.parametrize("maps", [False, True])
@pytest.mark.parametrize("mode", MODES, ids=_ids)
def test_one_hypothesis_is_the_single_entry_point(engine, batch, estimator, maps, mode):
    refs, curs = [q["ref"] for q in batch], [q["cur"] for q in batch]
    photometric, prior = mode.get("photometric", False), mode.get("prior", False)
    H, lam, ab0 = _inputs(batch, 2, 1, photometric, prior)
    H, lam, ab0 = H[:, 1:], None if lam is None else lam[:, 1:], None if ab0 is None else ab0[:, 1:]
    engine.set_estimator(estimator)
    try:
        want, want_ab, want_maps = _single(engine, refs, curs, _cfg(), H[:, 0], None if lam is None else lam[:, 0],
                                           None if ab0 is None else ab0[:, 0], photometric, maps)
        for s in (FIRST, FIRST - 1, LAST):
            res, best, scores, _, ab, _, mp = _call(engine, refs, curs, H, s, 0.0, _cfg(), lam, ab0, photometric, maps, screen=False)
            assert np.array_equal(best, np.zeros(len(refs))) and scores.shape == (len(refs), 1)
            for p in range(len(refs)):
                assert _same(res[p], want[p]), (s, p)
            if photometric:
                assert np.array_equal(ab, want_ab), s
            if maps:
                _same_maps(mp, want_maps)
    finally:
        engine.set_estimator("reference")


@pytest.mark.parametrize("estimator", ["reference", "corrected"])
@pytest.mark.parametrize("s,ratio", [(FIRST, 0.0), (FIRST - 1, 0.5), (LAST, 0.6)])
def test_continuation_follows_the_chosen_triple(engine, batch, estimator, s, ratio):
    refs, curs = [q["ref"] for q in batch], [q["cur"] for q in batch]
    engine.set_estimator(estimator)
    try:
        for seed, mode in enumerate(MODES):
            photometric, prior = mode.get("photometric", False), mode.get("prior", False)
            H, lam, ab0 = _inputs(batch, 4, 10 + seed, photometric, prior)
            _check_call(engine, refs, curs, H, s, ratio, _cfg(), lam, ab0, photometric, maps=True)
        # the photometric mode with cfg->mu, and without maps
        H, _, ab0 = _inputs(batch, 4, 20, True, False)
        _check_call(engine, refs[:2], curs[:2], H[:2], s, ratio, _cfg(mu=0.05), None, ab0[:2], True, maps=False)
    finally:
        engine.set_estimator("reference")


@pytest.mark.parametrize("estimator", ["reference", "corrected"])
def test_masks_and_mixed_intrinsics(engine, estimator):
    other = synth.SceneConfig(width=320, height=240, intrinsics=(287.0, 291.5, 161.0, 118.5))
    pyr, pairs = [], []
    for i, (scene, kw) in enumerate(((SCENE, {}), (SCENE, {"mask": _mask(1), "mask_roles": "reference"}),
                                     (SCENE, {"mask": _mask(2), "mask_roles": "both"}), (other, {}),
                                     (other, {"mask": _mask(4), "mask_roles": "both"}))):
        p = synth.make_pair(90 + i, scene)
        pyr.append((engine.pyramid(p["I_ref"].numpy(), p["Z_ref"].numpy(), scene.intrinsics, 3, **kw),
                    engine.pyramid(synth.exposure(p["I_cur"].numpy(), 1.05, -4.0), p["Z_cur"].numpy(), scene.intrinsics, 3, **kw)))
        pairs.append({"pair": p})
    H, lam, ab0 = _inputs(pairs, 3, 30, True, True)
    engine.set_estimator(estimator)
    try:
        for s, ratio in ((FIRST - 1, 0.4), (LAST, 0.0)):
            _check_call(engine, [a for a, _ in pyr], [b for _, b in pyr], H, s, ratio, _cfg(), lam, ab0, True, maps=True)
    finally:
        engine.set_estimator("reference")


def test_plan_and_batch_position_change_nothing(engine, batch, monkeypatch):
    k, s = 8, FIRST - 1
    H, lam, ab0 = _inputs(batch, k, 40, True, True)
    single = [_call(engine, [q["ref"]], [q["cur"]], H[i:i + 1], s, 0.3, _cfg(), lam[i:i + 1], ab0[i:i + 1], True, False, screen=False)
              for i, q in enumerate(batch)]
    big = 512
    idx = [i % len(batch) for i in range(big)]
    idx[511] = 0
    refs, curs = [batch[i]["ref"] for i in idx], [batch[i]["cur"] for i in idx]
    for knob, value in ((None, None), ("DVO_B200_NO_WALK", "1"), ("DVO_B200_FINE_G", "2"), ("DVO_B200_NO_FUSE", "1")):
        if knob:
            monkeypatch.setenv(knob, value)
        for order in (1, -1):
            o = list(range(big))[::order]
            sel = [idx[i] for i in o]
            res, best, scores, _, ab, _, _ = _call(engine, [refs[i] for i in o], [curs[i] for i in o], H[sel], s, 0.3, _cfg(), lam[sel],
                                                   ab0[sel], True, False, iterations=(knob is None), screen=False)
            for pos, i in enumerate(o):
                r1, b1, s1, _, ab1, _, _ = single[idx[i]]
                assert best[pos] == b1[0] and _eq(scores[pos], s1[0]), (knob, order, i)
                assert _same(res[pos], r1[0], iterations=(knob is None)), (knob, order, i)
                assert np.array_equal(ab[pos], ab1[0]), (knob, order, i)
        if knob:
            monkeypatch.delenv(knob)


@pytest.mark.parametrize("estimator", ["reference", "corrected"])
def test_the_near_hypothesis_wins_under_an_exposure_change(engine, estimator):
    p = synth.make_pair(0, WIDE)
    T = p["T_true"]
    ref = engine.pyramid(p["I_ref"].numpy(), p["Z_ref"].numpy(), WIDE.intrinsics, 3)
    cur = engine.pyramid(synth.exposure(p["I_cur"].numpy(), 1.15, -10.0), p["Z_cur"].numpy(), WIDE.intrinsics, 3)
    decoys = [synth.se3_exp(np.array([0.0, 0.0, 0.0, 0.35, -0.3, 0.25])) @ T, np.linalg.inv(T)]
    H = np.stack([np.eye(4), synth.se3_exp(NEAR) @ T] + decoys)[None]
    engine.set_estimator(estimator)
    try:
        plain, _ = engine.match_batch_photometric([ref], [cur], _cfg(), [np.eye(4)])
        assert _pose_err(plain[0].transformation, T)[1] > 0.05, _pose_err(plain[0].transformation, T)
        for s in (FIRST, FIRST - 1):
            res, best, scores, _, ab, _, _ = _call(engine, [ref], [cur], H, s, 0.3, _cfg(), None, None, True, False, screen=False)
            assert best[0] == 1, scores
            dt, dr = _pose_err(res[0].transformation, T)
            assert dt < TOL_T and dr < TOL_R, (dt, dr)
            assert abs(ab[0, 0] - 1.15) < 0.1, ab
    finally:
        engine.set_estimator("reference")


def _host_maps(n, w, h, w0, h0):
    """host buffers of every output and the dvo_b200_weight_maps that points at them"""
    bufs = {key: np.zeros((n, h, w), np.float32) for key in ("weight", "residual_i", "residual_z")}
    bufs["mask"] = np.zeros((n, h0, w0), np.uint8)
    bufs["estimate"] = np.zeros((n, 4, 4), np.float64)
    bufs["precision"] = np.zeros((n, 2, 2), np.float32)
    wm = WeightMaps()
    wm.memory = MAPS_MEMORY["host"]
    for key in ("weight", "residual_i", "residual_z"):
        setattr(wm, key, MapPlane(bufs[key].ctypes.data, 4 * w, 4 * w * h))
    wm.mask = MapPlane(bufs["mask"].ctypes.data, w0, w0 * h0)
    wm.mask_weight = MASK_WEIGHT
    wm.estimate = bufs["estimate"].ctypes.data_as(C.POINTER(C.c_double))
    wm.precision = bufs["precision"].ctypes.data_as(C.POINTER(C.c_float))
    return bufs, wm


def _raw_call(engine, refs, curs, H, s, cfg, lam=None, ab0=None, ab=None, scr_ab=None, maps=None, old=False):
    """the C entry points themselves: (rc, results bytes, best, scores)"""
    n, k = H.shape[:2]
    dp = C.POINTER(C.c_double)
    P = lambda a: None if a is None else a.ctypes.data_as(dp)
    rh, ch = (C.c_void_p * n)(*[r.handle for r in refs]), (C.c_void_p * n)(*[c.handle for c in curs])
    res, scr = (CResult * n)(), (CResult * (n * k))()
    best = (C.c_int32 * n)()
    sc = np.zeros((n, k))
    Hc = np.ascontiguousarray(H, dtype=np.float64)
    if old:
        rc = engine.lib.dvo_b200_match_batch_hypotheses(engine.ctx, C.byref(cfg), n, rh, ch, k, P(Hc), s, 0.0, res, best, P(sc), scr, None, 0)
    else:
        rc = engine.lib.dvo_b200_match_batch_hypotheses_modes(engine.ctx, C.byref(cfg), n, rh, ch, k, P(Hc), s, 0.0, P(lam), P(ab0), P(ab),
                                                              P(scr_ab), res, best, P(sc), scr, None, 0,
                                                              None if maps is None else C.byref(maps))
    return rc, bytes(res) + bytes(scr), list(best), sc


@pytest.mark.parametrize("s", [FIRST - 1, LAST])
def test_host_maps_equal_device_maps(engine, batch, s):
    refs, curs = [q["ref"] for q in batch], [q["cur"] for q in batch]
    H, lam, ab0 = _inputs(batch, 4, 50, True, True)
    w, h = refs[0].level_info(LAST)[:2]
    w0, h0 = refs[0].level_info(0)[:2]
    bufs, wm = _host_maps(len(refs), w, h, w0, h0)
    ab, scr_ab = np.zeros((len(refs), 2)), np.zeros((len(refs), 4, 2))
    rc, _, best, _ = _raw_call(engine, refs, curs, H, s, _cfg(), np.ascontiguousarray(lam), np.ascontiguousarray(ab0), ab, scr_ab, wm)
    assert rc == 0, engine.lib.dvo_b200_last_error(engine.ctx)
    _, b2, _, _, ab2, scr_ab2, dev = _call(engine, refs, curs, H, s, 0.0, _cfg(), lam, ab0, True, True, iterations=False)
    assert list(b2) == best and np.array_equal(ab, ab2) and np.array_equal(scr_ab, scr_ab2)
    for key, v in dev.items():
        assert np.array_equal(bufs[key], v.cpu().numpy(), equal_nan=bufs[key].dtype.kind == "f"), key


def test_old_entry_point_is_the_modes_call_without_modes(engine, batch):
    refs, curs = [q["ref"] for q in batch], [q["cur"] for q in batch]
    H, _, _ = _inputs(batch, 4, 60, False, False)
    for s in (FIRST, LAST):
        old = _raw_call(engine, refs, curs, H, s, _cfg(), old=True)
        new = _raw_call(engine, refs, curs, H, s, _cfg())
        assert old[0] == new[0] == 0
        assert old[1] == new[1] and old[2] == new[2] and np.array_equal(old[3], new[3], equal_nan=True)


def test_refusals_move_no_counters(engine, batch):
    q = batch[0]
    engine.synchronize()
    L, ctx = engine.lib, engine.ctx
    h0, k0, d0 = engine.h2d_bytes(), engine.kernel_launches(), engine.d2h_bytes()
    k = 3
    H = np.tile(np.eye(4), (1, k, 1, 1))
    lam = np.zeros((1, k, 6, 6))
    ab0 = np.tile([1.0, 0.0], (1, k, 1))
    ab, scr_ab = np.zeros((1, 2)), np.zeros((1, k, 2))
    asym, neg, inf_ab = lam.copy(), lam.copy(), ab0.copy()
    asym[0, 2, 0, 1] = 1.0
    neg[0, 1, 3, 3] = -1.0
    inf_ab[0, 2, 1] = np.inf
    good_maps = engine._device_maps([q["ref"]], _cfg(), MASK_WEIGHT)
    bad_maps = WeightMaps()
    bad_maps.memory = 7
    bad_weight = WeightMaps()
    bad_weight.memory = MAPS_MEMORY["device"]
    bad_weight.mask = good_maps[1].mask
    bad_weight.mask_weight = float("nan")
    host_maps = _host_maps(1, 320, 240, 320, 240)
    host_maps[1].memory = MAPS_MEMORY["device"]
    cases = [
        (dict(H=np.tile(np.eye(4), (1, 65, 1, 1))), "k = 65"),
        (dict(ab0=ab0), "photometric_init without photometric"),
        (dict(scr_ab=scr_ab), "screen_photometric without photometric"),
        (dict(lam=lam, cfg=_cfg(mu=0.1)), "cfg->mu must be 0"),
        (dict(lam=asym), "prior_information of hypothesis 2 of pair 0 is not symmetric"),
        (dict(lam=neg), "prior_information of hypothesis 1 of pair 0 is not positive semi-definite"),
        (dict(ab0=inf_ab, ab=ab), "photometric_init of hypothesis 2 of pair 0 is not finite"),
        (dict(maps=bad_maps), "unknown memory 7"),
        (dict(maps=bad_weight), "mask_weight must be finite and > 0"),
        (dict(maps=host_maps[1]), "weight is not device or managed memory of device"),
        # the order: the hypotheses checks first, then the modes in the header's order
        (dict(H=np.tile(np.eye(4), (1, 65, 1, 1)), ab0=ab0, lam=asym), "k = 65"),
        (dict(ab0=inf_ab, lam=asym, cfg=_cfg(mu=0.1)), "photometric_init without photometric"),
        (dict(ab0=inf_ab, ab=ab, lam=asym, maps=bad_maps), "prior_information of hypothesis 2"),
        (dict(ab0=inf_ab, ab=ab, maps=bad_maps), "photometric_init of hypothesis 2"),
    ]
    for kw, want in cases:
        cfg = kw.pop("cfg", _cfg())
        Hk = kw.pop("H", H)
        args = {key: (np.ascontiguousarray(v) if isinstance(v, np.ndarray) else v) for key, v in kw.items()}
        rc = _raw_call(engine, [q["ref"]], [q["cur"]], Hk, 1, cfg, **args)[0]
        msg = L.dvo_b200_last_error(ctx).decode()
        assert rc == -1 and msg.startswith("match_batch_hypotheses: ") and want in msg, (want, msg)
    assert engine.h2d_bytes() == h0 and engine.kernel_launches() == k0 and engine.d2h_bytes() == d0
    rc = _raw_call(engine, [q["ref"]], [q["cur"]], H, 1, _cfg(), np.ascontiguousarray(lam), np.ascontiguousarray(ab0), ab, scr_ab,
                   good_maps[1])[0]
    assert rc == 0 and engine.kernel_launches() > k0
