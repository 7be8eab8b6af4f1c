"""The motion prior on the GPU (dvo_b200_match_batch_prior): Lambda = mu I against the mu path bit for bit under every
estimator, mask instance and launch plan, Lambda = 0 against mu = 0, batch invariance with a different Lambda per pair, the
oracle definition (orc_match_with's prior input, oracle/dvo_oracle.h), stiff priors and the refusals."""
import ctypes as C

import numpy as np
import pytest

from dvo_slam_b200 import synth
from dvo_slam_b200.engine import CResult, Config

pytestmark = pytest.mark.gpu
SCENE = synth.SceneConfig(width=320, height=240, intrinsics=tuple(v / 2 for v in synth.FR1_INTRINSICS))
# levels 0 and 1 of 400 x 300 have full 160-column bands and a partial one (160, 160, 80 and 160, 40 columns)
SCENE400 = synth.SceneConfig(width=400, height=300, intrinsics=tuple(v * 400 / 640 for v in synth.FR1_INTRINSICS))
MUS = (0.05, 1.0, 25.0)
DELTA = np.array([4e-3, -3e-3, 2e-3, -2e-3, 3e-3, 1e-3])
PLANS = ((None, None), ("DVO_B200_FINE_G", "2"), ("DVO_B200_FINE_G", "4"), ("DVO_B200_TAIL", "6,6"), ("DVO_B200_COARSE_TILES", "0"),
         ("DVO_B200_COARSE_TILES", "1000000"), ("DVO_B200_NO_FUSE", "1"), ("DVO_B200_NO_WALK", "1"), ("DVO_B200_CONTIGUOUS", "1"),
         ("DVO_B200_STRIPS_PER_CTA", "3"))
STIFF = 1e18   # A is ~1e11 on its diagonal at 320 x 240


def _cfg(mu=0.0):
    return Config(first_level=2, last_level=0, max_iterations_per_level=50, precision=1e-4, mu=mu, use_initial_estimate=1)


def _mask(k, h=240, w=320):
    m = np.ones((h, w), np.uint8)
    m[40 + 10 * k:110 + 10 * k, 60:150] = 0
    return m


def _batch(engine, scene, seed0):
    out = []
    for k in range(6):
        p = synth.make_pair(seed0 + k, scene)
        kw = {"mask": _mask(k, scene.height, scene.width), "mask_roles": "both"} if k in (1, 4) else {}
        out.append({"ref": engine.pyramid(p["I_ref"].numpy(), p["Z_ref"].numpy(), scene.intrinsics, 3, **kw),
                    "cur": engine.pyramid(p["I_cur"].numpy(), p["Z_cur"].numpy(), scene.intrinsics, 3, **kw),
                    "T0": synth.se3_exp(DELTA * (1 + 0.3 * k)) @ p["T_true"], "pair": p})
    return out


@pytest.fixture(scope="module")
def batch(engine):
    """six pairs with their initial estimates; pairs 1 and 4 have a mask in both roles (the kCurMask instances)"""
    return _batch(engine, SCENE, 60)


@pytest.fixture(scope="module")
def batch400(engine):
    """the same at 400 x 300: the prior instances' generic loop in partial bands, which no hook reaches"""
    from tile_geometry import assert_partial_band
    assert_partial_band(SCENE400.width)
    assert_partial_band(SCENE400.width // 2)
    return _batch(engine, SCENE400, 160)


def _spd(rng, scale):
    M = rng.standard_normal((6, 6))
    S = (M @ M.T + 0.5 * np.eye(6)) * scale
    return 0.5 * (S + S.T)


def _run(engine, refs, curs, cfg, T0, photometric, prior=None, iters=False):
    if photometric:
        return engine.match_batch_photometric(refs, curs, cfg, T0, with_iterations=iters, prior_information=prior)
    return engine.match_batch(refs, curs, cfg, T0, with_iterations=iters, prior_information=prior), None


def _eq(a, b):
    return np.array_equal(np.asarray(a), np.asarray(b), equal_nan=True)


def _same(r0, r1, ll_tol=None):
    """bits of everything; ll_tol: the prior log-likelihood and log_likelihood to that relative tolerance instead"""
    if not (_eq(r0.transformation, r1.transformation) and _eq(r0.information, r1.information)):
        return False
    if r0.num_iterations_total != r1.num_iterations_total or len(r0.levels) != len(r1.levels):
        return False
    for a, b in zip(r0.levels, r1.levels):
        if a.keys() != b.keys() or not all(a[k] == b[k] or (a[k] != a[k] and b[k] != b[k]) for k in a):
            return False
    close = (lambda x, y: abs(x - y) <= ll_tol * abs(y)) if ll_tol is not None else (lambda x, y: x == y or (x != x and y != y))
    if not close(r0.log_likelihood, r1.log_likelihood):
        return False
    for x, y in zip(r0.iterations, r1.iterations):
        for k in ("level", "id", "n", "nll", "precision", "x", "A"):
            if not _eq(x[k], y[k]):
                return False
        if not close(x["prior"], y["prior"]):
            return False
    return len(r0.iterations) == len(r1.iterations)


@pytest.mark.parametrize("photometric", [False, True])
@pytest.mark.parametrize("estimator", ["reference", "corrected"])
def test_scalar_prior_equals_the_mu_path_under_every_plan(engine, batch, batch400, estimator, photometric, monkeypatch):
    for b in (batch, batch400):
        _scalar_prior_equals_the_mu_path_under_every_plan(engine, b, estimator, photometric, monkeypatch)


def _scalar_prior_equals_the_mu_path_under_every_plan(engine, batch, estimator, photometric, monkeypatch):
    refs, curs, T0 = [q["ref"] for q in batch], [q["cur"] for q in batch], [q["T0"] for q in batch]
    n = len(refs)
    mus = [MUS[i % 3] for i in range(n)]
    lam = np.stack([mu * np.eye(6) for mu in mus])
    engine.set_estimator(estimator)
    try:
        want = {mu: _run(engine, refs, curs, _cfg(mu), T0, photometric, iters=True) for mu in MUS}
        got, ab = _run(engine, refs, curs, _cfg(), T0, photometric, lam, iters=True)
        for i in range(n):
            w, wab = want[mus[i]]
            assert any(it["prior"] != 0.0 for it in w[i].iterations)
            assert _same(got[i], w[i], ll_tol=1e-14), i
            assert ab is None or _eq(ab[i], wab[i])
        zero, zab = _run(engine, refs, curs, _cfg(), T0, photometric, np.zeros((n, 6, 6)), iters=True)
        ref0, rab = _run(engine, refs, curs, _cfg(0.0), T0, photometric, iters=True)
        for i in range(n):
            assert _same(zero[i], ref0[i]), i
            assert zab is None or _eq(zab[i], rab[i])
        big = 12
        for knob, value in PLANS:
            if knob:
                monkeypatch.setenv(knob, value)
            r, rab = _run(engine, refs * big, curs * big, _cfg(), T0 * big, photometric, np.concatenate([lam] * big))
            if knob:
                monkeypatch.delenv(knob)
            for i in range(n * big):
                w, wab = want[mus[i % n]]
                assert _eq(r[i].transformation, w[i % n].transformation) and _eq(r[i].information, w[i % n].information), (knob, i)
                assert rab is None or _eq(rab[i], wab[i % n]), (knob, i)
    finally:
        engine.set_estimator("reference")


@pytest.mark.parametrize("photometric", [False, True])
def test_full_priors_are_batch_invariant(engine, batch, photometric):
    refs, curs, T0 = [q["ref"] for q in batch], [q["cur"] for q in batch], [q["T0"] for q in batch]
    n = len(refs)
    rng = np.random.default_rng(11)
    lam = np.stack([_spd(rng, 10.0 ** rng.uniform(8, 11)) for _ in range(n)])
    single = [_run(engine, [refs[i]], [curs[i]], _cfg(), [T0[i]], photometric, lam[i:i + 1], iters=True) for i in range(n)]
    rb, abb = _run(engine, refs, curs, _cfg(), T0, photometric, lam, iters=True)
    rr, abr = _run(engine, refs[::-1], curs[::-1], _cfg(), T0[::-1], photometric, lam[::-1], iters=True)
    big = 512
    idx = [i % n for i in range(big)]
    rg, abg = _run(engine, [refs[i] for i in idx], [curs[i] for i in idx], _cfg(), [T0[i] for i in idx], photometric, lam[idx])
    for i in range(n):
        s, sab = single[i]
        assert _same(rb[i], s[0]) and _same(rr[n - 1 - i], s[0]), i
        assert sab is None or (_eq(abb[i], sab[0]) and _eq(abr[n - 1 - i], sab[0]))
    for k in range(big):
        s, sab = single[idx[k]]
        assert _eq(rg[k].transformation, s[0].transformation) and _eq(rg[k].information, s[0].information), k
        assert sab is None or _eq(abg[k], sab[0])


def _pose_err(T, T_true):
    """translation and rotation norms of the error of Result.transformation T, which estimates T_true^-1"""
    d = synth.se3_log(T_true @ T)
    return np.linalg.norm(d[:3]), np.linalg.norm(d[3:])


@pytest.mark.parametrize("photometric", [False, True])
def test_alignments_match_the_prior_oracle(engine, oracle, batch, photometric):
    rng = np.random.default_rng(3)
    ocfg = oracle.config(first_level=2, last_level=0, max_iterations_per_level=50, precision=1e-4, use_initial_estimate=1)
    for q in batch[:4]:
        if q is batch[1]:
            continue   # masked: the prior oracle has no masks
        p = q["pair"]
        lam = _spd(rng, 1e9)
        r, ab = _run(engine, [q["ref"]], [q["cur"]], _cfg(), [q["T0"]], photometric, lam[None])
        o = oracle.match(oracle.Pyramid(p["I_ref"].numpy(), p["Z_ref"].numpy(), SCENE.intrinsics, 3),
                         oracle.Pyramid(p["I_cur"].numpy(), p["Z_cur"].numpy(), SCENE.intrinsics, 3), ocfg, oracle.mode("mirror"),
                         q["T0"], prior=lam, photometric=photometric)
        dt, dr = _pose_err(r[0].transformation, np.linalg.inv(o["T"]))
        assert dt < 1e-4 and dr < 1e-4, (dt, dr)
        assert [(l["termination"], l["num_iterations"]) for l in r[0].levels] == \
            [(l["termination"], l["num_iterations"]) for l in o["levels"]]
        scale = np.abs(o["information"]).max()
        assert np.allclose(r[0].information, o["information"], rtol=2e-6, atol=2e-6 * scale)
        if photometric:
            assert np.allclose(ab[0], o["ab"], rtol=1e-3, atol=1e-2), (ab[0], o["ab"])


@pytest.mark.parametrize("photometric", [False, True])
def test_stiff_priors(engine, batch, photometric):
    q = batch[0]
    r, _ = _run(engine, [q["ref"]], [q["cur"]], _cfg(), [q["T0"]], photometric, STIFF * np.eye(6)[None])
    assert np.abs(synth.se3_log(q["T0"] @ r[0].transformation)).max() < 1e-8
    for k in (0, 4):
        e = np.zeros(6); e[k] = 1.0
        r, _ = _run(engine, [q["ref"]], [q["cur"]], _cfg(), [q["T0"]], photometric, STIFF * np.outer(e, e)[None])
        d = synth.se3_log(q["T0"] @ r[0].transformation)
        # the held quantity is log(initial), equal to log(T0 Result.T) to first order in the increments
        assert abs(d[k]) < 2e-4, d
        assert np.abs(np.delete(d, k)).max() > 2e-3, d


def test_refusals_move_no_counters(engine, batch):
    q = batch[0]
    engine.synchronize()
    L, ctx = engine.lib, engine.ctx
    h0, k0 = engine.h2d_bytes(), engine.kernel_launches()
    rh, ch = (C.c_void_p * 1)(q["ref"].handle), (C.c_void_p * 1)(q["cur"].handle)
    res = (CResult * 1)()
    dp = C.POINTER(C.c_double)
    good = np.eye(6)
    asym = np.eye(6); asym[0, 1] = 1e-300
    neg = np.diag([1, 1, 1, 1, 1, -1e-3])
    nan = np.eye(6); nan[3, 3] = np.nan
    ab0, ab = np.array([1.0, 0.0]), np.zeros(2)
    P = lambda a: np.ascontiguousarray(a, dtype=np.float64).ctypes.data_as(dp)
    cases = [(_cfg(), None, None, None), (_cfg(), asym, None, None), (_cfg(), neg, None, None), (_cfg(), nan, None, None),
             (_cfg(0.05), good, None, None), (_cfg(), good, ab0, None), (_cfg(), good, np.array([np.inf, 0.0]), ab)]
    for cfg, lam, a0, a in cases:
        rc = L.dvo_b200_match_batch_prior(ctx, C.byref(cfg), 1, rh, ch, None, None if lam is None else P(lam),
                                          None if a0 is None else P(a0), None if a is None else P(a), res, None, 0)
        assert rc != 0
    # and the batch checks of dvo_b200_match_batch
    bad = Config(first_level=0, last_level=1)
    assert L.dvo_b200_match_batch_prior(ctx, C.byref(bad), 1, rh, ch, None, P(good), None, None, res, None, 0) != 0
    assert engine.h2d_bytes() == h0 and engine.kernel_launches() == k0
    # an accepted call stages 288 bytes per pair more than dvo_b200_match_batch
    engine.match_batch([q["ref"]], [q["cur"]], _cfg(), [q["T0"]])
    h1 = engine.h2d_bytes()
    engine.match_batch([q["ref"]], [q["cur"]], _cfg(), [q["T0"]], prior_information=good[None])
    h2 = engine.h2d_bytes()
    assert h2 - h1 == (h1 - h0) + 288
