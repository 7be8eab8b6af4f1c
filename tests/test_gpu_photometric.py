"""The photometric mode on the GPU against its oracle definition (tests/photometric_oracle.py): residual records bit for
bit, the hooks at (1, 0) against the default hooks, whole alignments, batch invariance, accuracy and refusals."""
import ctypes as C

import numpy as np
import pytest

import photometric_oracle as pho
from dvo_slam_b200 import synth
from dvo_slam_b200.engine import CResult, Config

pytestmark = pytest.mark.gpu
SCENE = synth.SceneConfig(width=320, height=240, intrinsics=tuple(v / 2 for v in synth.FR1_INTRINSICS))
ABS = [(1.0, 0.0), (1.1, -7.5), (0.85, 12.0)]


@pytest.fixture(scope="module")
def pairs():
    return [synth.make_pair(s, SCENE) for s in range(4)]


def _gpu(engine, pair, Ic=None):
    Ic = pair["I_cur"].numpy() if Ic is None else Ic
    return (engine.pyramid(pair["I_ref"].numpy(), pair["Z_ref"].numpy(), SCENE.intrinsics, 3),
            engine.pyramid(Ic, pair["Z_cur"].numpy(), SCENE.intrinsics, 3))


@pytest.mark.parametrize("ab", ABS)
def test_records_match_the_oracle_mirror(engine, oracle, pairs, ab):
    pair = pairs[0]
    ref, cur = _gpu(engine, pair)
    pref = pho.Pyramid(pair["I_ref"].numpy(), pair["Z_ref"].numpy(), SCENE.intrinsics, 3)
    pcur = pho.Pyramid(pair["I_cur"].numpy(), pair["Z_cur"].numpy(), SCENE.intrinsics, 3)
    T = np.linalg.inv(pair["T_true"])
    m = oracle.mode("mirror")
    for level in (0, 2):
        n, img = engine.residual_image(ref, cur, level, T, ab=ab)
        no, imgo = pho.residual_image(pref, pcur, level, T, ab, m)
        assert n == no and np.array_equal(img, imgo, equal_nan=True)
        g = engine.linearize(ref, cur, level, T, ab=ab)
        o = pho.linearize(pref, pcur, level, T, ab, m)
        assert g["n"] == o["n"]
        assert np.allclose(g["precision"], o["precision"], rtol=2e-6)
        assert abs(g["ll"] - o["ll"]) <= 2e-6 * abs(o["ll"])
        scale = np.abs(o["A"]).max()
        assert np.allclose(g["A"], o["A"], rtol=2e-6, atol=2e-6 * scale)
        assert np.allclose(g["b"], o["b"], rtol=2e-6, atol=2e-6 * np.abs(o["b"]).max())


@pytest.mark.parametrize("estimator", ["reference", "corrected"])
def test_hooks_at_identity_equal_the_default_hooks(engine, pairs, estimator):
    pair = pairs[1]
    ref, cur = _gpu(engine, pair)
    T = np.linalg.inv(pair["T_true"])
    engine.set_estimator(estimator)
    try:
        for level in (0, 2):
            n, img = engine.residual_image(ref, cur, level, T)
            n2, img2 = engine.residual_image(ref, cur, level, T, ab=(1.0, 0.0))
            assert n == n2 and np.array_equal(img, img2, equal_nan=True)
            d = engine.linearize(ref, cur, level, T, use_weights=True, prev_precision=np.array([800.0, 5.0, 5.0, 300.0]))
            p = engine.linearize(ref, cur, level, T, use_weights=True, prev_precision=np.array([800.0, 5.0, 5.0, 300.0]), ab=(1.0, 0.0))
            assert d["n"] == p["n"] and d["ll"] == p["ll"] and np.array_equal(d["precision"], p["precision"])
            assert np.array_equal(d["A"], p["A"][:6, :6]) and np.array_equal(d["b"], p["b"][:6])
    finally:
        engine.set_estimator("reference")


def _pose_err(T_est, T_true):
    d = synth.se3_log(T_true @ T_est)
    return np.abs(d[:3]).max(), np.abs(d[3:]).max()


def test_alignments_match_the_oracle_and_are_batch_invariant(engine, oracle, pairs):
    cfg = Config(first_level=2, last_level=0, max_iterations_per_level=50, precision=1e-4)
    ocfg = oracle.config(first_level=2, last_level=0, max_iterations_per_level=50, precision=1e-4)
    exps = [(1.1, 0.0), (0.9, 5.0), (1.2, -15.0), (1.0, 0.0)]
    refs, curs, orcs = [], [], []
    for pair, (g, b) in zip(pairs, exps):
        Ic = synth.exposure(pair["I_cur"].numpy(), g, b)
        r, c = _gpu(engine, pair, Ic)
        refs.append(r); curs.append(c)
        orcs.append(pho.match(pho.Pyramid(pair["I_ref"].numpy(), pair["Z_ref"].numpy(), SCENE.intrinsics, 3),
                              pho.Pyramid(Ic, pair["Z_cur"].numpy(), SCENE.intrinsics, 3), ocfg, oracle.mode("mirror")))
    res, ab = engine.match_batch_photometric(refs, curs, cfg)
    for i, (r, o) in enumerate(zip(res, orcs)):
        dt, dr = _pose_err(r.transformation, np.linalg.inv(o["T"]))
        assert dt < 1e-4 and dr < 1e-4, (i, dt, dr)
        assert np.allclose(ab[i], o["ab"], rtol=1e-3, atol=1e-2), (i, ab[i], o["ab"])
    # identical bits: the batch, the reversed batch and single alignments, with each estimator
    for estimator in ("reference", "corrected"):
        engine.set_estimator(estimator)
        try:
            big = 512
            rb, ab_b = engine.match_batch_photometric([refs[i % 4] for i in range(big)], [curs[i % 4] for i in range(big)], cfg)
            rr, ab_r = engine.match_batch_photometric(refs[::-1], curs[::-1], cfg)
            for i in range(4):
                rs, ab_s = engine.match_batch_photometric([refs[i]], [curs[i]], cfg)
                assert np.array_equal(rs[0].transformation, rb[i].transformation) and np.array_equal(ab_s[0], ab_b[i])
                assert np.array_equal(rs[0].transformation, rr[3 - i].transformation) and np.array_equal(ab_s[0], ab_r[3 - i])
                assert np.array_equal(rb[i].transformation, rb[i + 4].transformation)
        finally:
            engine.set_estimator("reference")


def test_photometric_mode_is_more_accurate_on_exposure_pairs(engine):
    cfg = Config(first_level=2, last_level=0, max_iterations_per_level=50, precision=1e-4)
    rng = np.random.default_rng(5)
    refs, curs, truth = [], [], []
    for s in range(16):
        pair = synth.make_pair(100 + s, SCENE)
        g, b = rng.uniform(0.85, 1.15), rng.uniform(-15, 15)
        if abs(g - 1) < 0.05:
            g = 1.1
        r, c = _gpu(engine, pair, synth.exposure(pair["I_cur"].numpy(), g, b))
        refs.append(r); curs.append(c); truth.append(pair["T_true"])
    dflt = engine.match_batch(refs, curs, cfg)
    phot, _ = engine.match_batch_photometric(refs, curs, cfg)
    e_d = np.median([_pose_err(r.transformation, t)[0] for r, t in zip(dflt, truth)])
    e_p = np.median([_pose_err(r.transformation, t)[0] for r, t in zip(phot, truth)])
    assert e_p * 3 <= e_d, (e_d, e_p)


def test_refusals_move_no_counters(engine, pairs):
    ref, cur = _gpu(engine, pairs[0])
    engine.synchronize()
    cfg = Config()
    L, ctx = engine.lib, engine.ctx
    h0, k0 = engine.h2d_bytes(), engine.kernel_launches()
    rh, ch = (C.c_void_p * 1)(ref.handle), (C.c_void_p * 1)(cur.handle)
    res = (CResult * 1)()
    bad = np.array([np.nan, 0.0])
    out = np.zeros(2)
    dp = C.POINTER(C.c_double)
    assert L.dvo_b200_match_batch_photometric(ctx, C.byref(cfg), 1, rh, ch, None, None, res, None, None, 0) != 0
    assert L.dvo_b200_match_batch_photometric(ctx, C.byref(cfg), 1, rh, ch, None, bad.ctypes.data_as(dp), res, out.ctypes.data_as(dp),
                                              None, 0) != 0
    T = np.eye(4)
    img = np.zeros((7, 240, 320), np.float32)
    assert L.dvo_b200_residual_image_photometric(ctx, C.byref(cfg), ref.handle, cur.handle, 0, T.ctypes.data_as(dp), bad.ctypes.data_as(dp),
                                                 img.ctypes.data_as(C.POINTER(C.c_float)), None) != 0
    assert L.dvo_b200_linearize_photometric(ctx, C.byref(cfg), ref.handle, cur.handle, 0, T.ctypes.data_as(dp), bad.ctypes.data_as(dp), 0,
                                            None, None, None, None, None, None) != 0
    assert engine.h2d_bytes() == h0 and engine.kernel_launches() == k0


# ---- the generic pixel loops, current-role masks, both estimators, every launch plan ----------------------------------
from test_corrected_estimator import corrected_mode  # noqa: E402

PP = np.array([[2000.0, -30.0], [-30.0, 9000.0]], dtype=np.float32)
AB_FORCED = (1.08, -6.0)


def _rot_z(deg):
    a = np.deg2rad(deg)
    T = np.eye(4)
    T[:2, :2] = [[np.cos(a), -np.sin(a)], [np.sin(a), np.cos(a)]]
    return T


def _shift_z(dz):
    T = np.eye(4)
    T[2, 3] = dz
    return T


def _blobs(h, w, seed, n=8, rmax=40):
    rng = np.random.default_rng(seed)
    m = np.ones((h, w), np.uint8)
    yy, xx = np.ogrid[:h, :w]
    for _ in range(n):
        cy, cx, r = rng.integers(0, h), rng.integers(0, w), rng.integers(4, rmax)
        m[(yy - cy) ** 2 + (xx - cx) ** 2 <= r * r] = 0
    return m


@pytest.fixture(scope="module")
def pair0():
    p = synth.make_pair(0)
    a = {k: p[k].numpy() for k in ("I_ref", "Z_ref", "I_cur", "Z_cur")}
    a["K"] = p["intrinsics"]
    return a


def _check_records_both_estimators(engine, oracle, gref, gcur, pref, pcur, lvl, T, ab):
    for est, mode in (("reference", oracle.mode("mirror")), ("corrected", corrected_mode(oracle))):
        engine.set_estimator(est)
        try:
            n, img = engine.residual_image(gref, gcur, lvl, T, ab=ab)
            no, imgo = pho.residual_image(pref, pcur, lvl, T, ab, mode)
            assert n == no and n > 0 and np.array_equal(img, imgo, equal_nan=True), (est, lvl, n, no)
            for uw in (False, True):
                g = engine.linearize(gref, gcur, lvl, T, uw, PP, ab=ab)
                o = pho.linearize(pref, pcur, lvl, T, ab, mode, uw, PP)
                assert g["n"] == o["n"] == no, (est, lvl, uw)
                assert np.allclose(g["precision"], o["precision"], rtol=2e-6, atol=2e-6 * np.abs(o["precision"]).max()), (est, lvl, uw)
                assert abs(g["ll"] - o["ll"]) <= 2e-6 * abs(o["ll"]) + 0.5, (est, lvl, uw)
                assert np.allclose(g["A"], o["A"], rtol=0, atol=2e-6 * np.abs(o["A"]).max()), (est, lvl, uw)
                assert np.allclose(g["b"], o["b"], rtol=0, atol=2e-6 * np.abs(o["b"]).max()), (est, lvl, uw)
        finally:
            engine.set_estimator("reference")


@pytest.mark.parametrize("case", ["inexact", "no_window", "partial_band", "cur_mask_dirty", "cur_mask_inexact"])
def test_records_on_the_generic_loops(engine, oracle, pair0, case):
    """The cases of test_gpu_generic_tiles.py / test_gpu_mask_roles.py at (alpha, beta) != (1, 0): inexact = a 20 degree roll
    (no tile row fits the window), no_window = the camera past the median depth (tile corners behind it), partial_band =
    levels 1 and 2 of the 720 x 540 scene of test_gpu_generic_tiles (full 160-column bands and a partial one), cur_mask_* =
    a mask in the current role (the per-tap test of the masked stage-B loop), on exact-window tiles that touch it and on
    inexact ones."""
    from test_gpu_generic_tiles import partial_pair, partial_pose
    from tile_geometry import assert_partial_band
    a = partial_pair(0) if case == "partial_band" else pair0
    h, w = a["I_ref"].shape
    m, lvls = None, [0]
    if case == "inexact":
        T = _rot_z(20.0)
    elif case == "no_window":
        T = _shift_z(-float(np.nanmedian(a["Z_ref"])))
    elif case == "partial_band":
        T, lvls = partial_pose(), [1, 2]
        for lvl in lvls:
            assert_partial_band(w >> lvl)
    elif case == "cur_mask_dirty":
        m = np.ones((h, w), np.uint8)
        m[4::32, 4::32] = 0
        T = _rot_z(0.5) @ _shift_z(0.01)
    else:
        m, T = _blobs(h, w, 3), _rot_z(20.0)
    gref = engine.pyramid(a["I_ref"], a["Z_ref"], a["K"], 5)
    gcur = engine.pyramid(a["I_cur"], a["Z_cur"], a["K"], 5) if m is None else \
        engine.pyramid(a["I_cur"], a["Z_cur"], a["K"], 5, mask=m, mask_roles="both")
    pref = pho.Pyramid(a["I_ref"], a["Z_ref"], a["K"], 5)
    pcur = pho.Pyramid(a["I_cur"], a["Z_cur"], a["K"], 5, mask=m)
    for lvl in lvls:
        _check_records_both_estimators(engine, oracle, gref, gcur, pref, pcur, lvl, T, AB_FORCED)


def _same(r0, ab0, r1, ab1):
    return (np.array_equal(r0.transformation, r1.transformation) and np.array_equal(r0.information, r1.information, equal_nan=True)
            and (r0.log_likelihood == r1.log_likelihood or (np.isnan(r0.log_likelihood) and np.isnan(r1.log_likelihood)))
            and np.array_equal(ab0, ab1) and len(r0.levels) == len(r1.levels)
            and all(a.keys() == b.keys() and all(a[k] == b[k] or (a[k] != a[k] and b[k] != b[k]) for k in a)
                    for a, b in zip(r0.levels, r1.levels)))


@pytest.fixture(scope="module")
def masked_batch(engine):
    """six exposure pairs; pairs 1, 3 and 4 have a mask in both roles (the current role selects the kCurMask instances)"""
    exps = [(1.1, 0.0), (0.9, 5.0), (1.2, -15.0), (1.0, 0.0), (0.85, 10.0), (1.05, -8.0)]
    out = []
    for k, (g, b) in enumerate(exps):
        p = synth.make_pair(30 + k, SCENE)
        Ic = synth.exposure(p["I_cur"].numpy(), g, b)
        m = _blobs(240, 320, 50 + k, n=6, rmax=30) if k in (1, 3, 4) else None
        kw = {} if m is None else {"mask": m, "mask_roles": "both"}
        out.append({"gref": engine.pyramid(p["I_ref"].numpy(), p["Z_ref"].numpy(), SCENE.intrinsics, 3, **kw),
                    "gcur": engine.pyramid(Ic, p["Z_cur"].numpy(), SCENE.intrinsics, 3, **kw),
                    "pref": pho.Pyramid(p["I_ref"].numpy(), p["Z_ref"].numpy(), SCENE.intrinsics, 3, mask=m),
                    "pcur": pho.Pyramid(Ic, p["Z_cur"].numpy(), SCENE.intrinsics, 3, mask=m)})
    return out


@pytest.mark.parametrize("estimator", ["reference", "corrected"])
def test_masked_alignments_match_the_oracle_under_every_plan(engine, oracle, masked_batch, estimator, monkeypatch):
    """With current-role masks in the batch: each alignment within 1e-4 of the oracle's (MIRROR, or MIRROR with the three
    quirks off for the corrected estimator), and the batch, the reversed batch, single alignments and a 72-pair batch under
    every plan override return the same bits."""
    cfg = Config(first_level=2, last_level=0, max_iterations_per_level=50, precision=1e-4)
    ocfg = oracle.config(first_level=2, last_level=0, max_iterations_per_level=50, precision=1e-4)
    mode = oracle.mode("mirror") if estimator == "reference" else corrected_mode(oracle)
    refs, curs = [q["gref"] for q in masked_batch], [q["gcur"] for q in masked_batch]
    engine.set_estimator(estimator)
    try:
        single = [engine.match_batch_photometric([r], [c], cfg) for r, c in zip(refs, curs)]
        for (res, ab), q in zip(single, masked_batch):
            o = pho.match(q["pref"], q["pcur"], ocfg, mode)
            dt, dr = _pose_err(res[0].transformation, np.linalg.inv(o["T"]))
            assert dt < 1e-4 and dr < 1e-4, (dt, dr)
            assert np.allclose(ab[0], o["ab"], rtol=1e-3, atol=1e-2), (ab[0], o["ab"])
        batch, ab_b = engine.match_batch_photometric(refs, curs, cfg)
        rev, ab_r = engine.match_batch_photometric(refs[::-1], curs[::-1], cfg)
        n = len(refs)
        for i in range(n):
            assert _same(batch[i], ab_b[i], single[i][0][0], single[i][1][0]), i
            assert _same(rev[n - 1 - i], ab_r[n - 1 - i], single[i][0][0], single[i][1][0]), i
        big_r, big_c = refs * 12, curs * 12
        for knob, value in ((None, None), ("DVO_B200_FINE_G", "2"), ("DVO_B200_FINE_G", "4"), ("DVO_B200_TAIL", "6,6"),
                            ("DVO_B200_COARSE_TILES", "0"), ("DVO_B200_COARSE_TILES", "1000000"), ("DVO_B200_NO_FUSE", "1"),
                            ("DVO_B200_NO_WALK", "1"), ("DVO_B200_CONTIGUOUS", "1"), ("DVO_B200_STRIPS_PER_CTA", "3")):
            if knob:
                monkeypatch.setenv(knob, value)
            r, ab = engine.match_batch_photometric(big_r, big_c, cfg)
            if knob:
                monkeypatch.delenv(knob)
            for i in range(len(big_r)):
                s = single[i % n]
                assert _same(r[i], ab[i], s[0][0], s[1][0]), (knob, value, i)
    finally:
        engine.set_estimator("reference")
