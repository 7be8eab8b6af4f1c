"""The photometric mode without a GPU: the oracle's definition (the ab inputs of oracle/dvo_oracle.h) against the oracle's
default mode and finite differences, its accuracy under exposure changes, and the C ABI's bindings and refusals."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from dvo_slam_b200 import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MODES = ("faithful", "mirror", "exact")
ERR_INVALID_ARGUMENT = -1   # DVO_B200_ERR_INVALID_ARGUMENT


@pytest.fixture(scope="module")
def pair_small(small_scene):
    return synth.make_pair(3, small_scene)


def _pyrs(oracle, pair, scene, levels=3):
    return (oracle.Pyramid(pair["I_ref"].numpy(), pair["Z_ref"].numpy(), scene.intrinsics, levels),
            oracle.Pyramid(pair["I_cur"].numpy(), pair["Z_cur"].numpy(), scene.intrinsics, levels))


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("use_weights", [False, True])
def test_identity_brightness_equals_the_default_linearisation(oracle, pair_small, small_scene, mode, use_weights):
    """At (alpha, beta) = (1, 0): count, P, LL, the pose block of A and b[0..5] equal orc_linearize bit for bit."""
    oref, ocur = _pyrs(oracle, pair_small, small_scene)
    T = np.linalg.inv(pair_small["T_true"]) @ synth.se3_exp(np.array([2e-3, -1e-3, 1e-3, 1e-3, 2e-3, -1e-3]))
    T = np.linalg.inv(T)
    pp = np.array([[900.0, 10.0], [10.0, 400.0]], dtype=np.float32)
    m = oracle.mode(mode)
    for level in (0, 1):
        d = oracle.linearize(oref, ocur, level, T, m, use_weights, pp)
        p = oracle.linearize(oref, ocur, level, T, m, use_weights, pp, ab=[1.0, 0.0])
        assert p["n"] == d["n"] and p["ll"] == d["ll"]
        assert np.array_equal(p["precision"], d["precision"])
        assert np.array_equal(p["A"][:6, :6], d["A"]) and np.array_equal(p["b"][:6], d["b"])
        n, img = oracle.residual_image(oref, ocur, level, T, m)
        n2, img2 = oracle.residual_image(oref, ocur, level, T, m, ab=[1.0, 0.0])
        assert n == n2 and np.array_equal(img, img2, equal_nan=True)


def _objective(oracle, pref, pcur, T, ab, m, P, level):
    """sum w (r^T P r) / 2 with fixed P and unit weights, in float64 from the residual image (EXACT mode)"""
    _, img = oracle.residual_image(pref, pcur, level, T, m, ab=ab)
    ei, ez = img[0].astype(np.float64), img[1].astype(np.float64)
    ok = ~np.isnan(ei)
    r = np.stack([ei[ok], ez[ok]])
    return 0.5 * np.einsum("in,ij,jn->", r, P.astype(np.float64), r)


def test_brightness_columns_match_finite_differences(oracle, pair_small, small_scene):
    """b[6], b[7] = -d/d(alpha, beta) of the EXACT objective with unit weights; A[6:, 6:] its Gauss-Newton Hessian."""
    pref, pcur = _pyrs(oracle, pair_small, small_scene)
    T = np.linalg.inv(pair_small["T_true"])
    m = oracle.mode("exact")
    ab = np.array([1.05, -3.0])
    lin = oracle.linearize(pref, pcur, 1, T, m, ab=ab)
    P = lin["precision"]
    f = lambda x: _objective(oracle, pref, pcur, T, x, m, P, 1)
    for k, h in ((0, 1e-3), (1, 0.25)):
        e = np.zeros(2); e[k] = h
        g = (f(ab + e) - f(ab - e)) / (2 * h)
        assert abs(-g - lin["b"][6 + k]) <= 1e-3 * max(1.0, abs(g)), (k, g, lin["b"][6 + k])
    # the Hessian block: the objective is quadratic in (alpha, beta) at fixed points
    a0 = f(ab)
    for k, h in ((0, 1e-2), (1, 1.0)):
        e = np.zeros(2); e[k] = h
        hh = (f(ab + e) - 2 * a0 + f(ab - e)) / h ** 2
        assert abs(hh - lin["A"][6 + k, 6 + k]) <= 1e-3 * abs(hh), (k, hh, lin["A"][6 + k, 6 + k])


def test_ldlt8_and_schur(oracle):
    rng = np.random.default_rng(1)
    M = rng.standard_normal((8, 8))
    A = M @ M.T + 8 * np.eye(8)
    b = rng.standard_normal(8)
    x = oracle.ldlt_solve(A, b)
    assert np.allclose(x, np.linalg.solve(A, b), rtol=1e-12, atol=1e-12)
    S = oracle.schur_pose(A)
    want = A[:6, :6] - A[:6, 6:] @ np.linalg.solve(A[6:, 6:], A[6:, :6])
    assert np.allclose(S, want, rtol=1e-12, atol=1e-10)


EXPOSURES = [(1.0, 0.0), (1.1, 0.0), (0.9, 0.0), (1.0, 10.0), (1.2, -15.0), (0.8, 20.0)]


def _pose_err(T_est, T_true):
    d = synth.se3_log(T_true @ T_est)
    return np.abs(d[:3]).max(), np.abs(d[3:]).max()


def test_accuracy_under_exposure_changes(oracle):
    """FAITHFUL, make_pair(seed) for seeds 0..11, 640x480, levels 4..0: on the changed frames the photometric mode's median
    translation error is at least 3x below the default mode's, and on unchanged frames at most 1.5x the default's."""
    cfg = oracle.config(first_level=4, last_level=0, max_iterations_per_level=50, precision=1e-4)
    m = oracle.mode("faithful")
    err = {}
    for seed in range(12):
        pair = synth.make_pair(seed)
        K = synth.FR1_INTRINSICS
        oref = oracle.Pyramid(pair["I_ref"].numpy(), pair["Z_ref"].numpy(), K, 5)
        for g, b in EXPOSURES:
            Ic = synth.exposure(pair["I_cur"].numpy(), g, b)
            ocur = oracle.Pyramid(Ic, pair["Z_cur"].numpy(), K, 5)
            d = oracle.match(oref, ocur, cfg, m)
            p = oracle.match(oref, ocur, cfg, m, photometric=True)
            err.setdefault((g, b), []).append((_pose_err(d["T"], pair["T_true"])[0], _pose_err(p["T"], pair["T_true"])[0]))
    for (g, b), e in err.items():
        dflt, phot = np.median([x[0] for x in e]), np.median([x[1] for x in e])
        if (g, b) == (1.0, 0.0):
            assert phot <= 1.5 * dflt, (g, b, dflt, phot)
        else:
            assert phot * 3 <= dflt, (g, b, dflt, phot)


def test_bindings_match_the_header():
    """The three entry points are exported ABI symbols, and their ctypes argument lists have the header's arity."""
    from dvo_slam_b200 import engine
    src = open(os.path.join(ROOT, "include", "dvo_b200.h")).read()
    L = engine.load_library()
    for name, nargs in (("dvo_b200_match_batch_photometric", 11), ("dvo_b200_residual_image_photometric", 9),
                        ("dvo_b200_linearize_photometric", 14)):
        m = re.search(r"int " + name + r"\(([^;]*)\);", src)
        assert m and m.group(1).count(",") + 1 == nargs, name
        assert name in engine.ABI_SYMBOLS
        assert len(getattr(L, name).argtypes) == nargs, name


def test_refusals_without_a_context():
    """A NULL context is refused with INVALID_ARGUMENT by every photometric entry point, before anything else."""
    from dvo_slam_b200 import engine
    L = engine.load_library()
    ab = np.array([1.0, 0.0])
    out = np.zeros(2)
    cfg = engine.Config()
    assert L.dvo_b200_match_batch_photometric(None, C.byref(cfg), 1, None, None, None, None, None,
                                              out.ctypes.data_as(C.POINTER(C.c_double)), None, 0) == ERR_INVALID_ARGUMENT
    abp = ab.ctypes.data_as(C.POINTER(C.c_double))
    assert L.dvo_b200_residual_image_photometric(None, C.byref(cfg), None, None, 0, None, abp, None, None) == ERR_INVALID_ARGUMENT
    assert L.dvo_b200_linearize_photometric(None, C.byref(cfg), None, None, 0, None, abp, 0, None, None, None, None, None,
                                            None) == ERR_INVALID_ARGUMENT


def test_exposure_is_clipped_and_rounded():
    I = np.array([[0.0, 100.0, 250.0]], dtype=np.float32)
    assert np.array_equal(synth.exposure(I, 1.1, 0.0), np.array([[0.0, 110.0, 255.0]], dtype=np.float32))
    assert synth.exposure(I, 1.0, 0.0).dtype == np.float32 and np.array_equal(synth.exposure(I, 1.0, 0.0), I)


def test_cross_terms_match_finite_differences(oracle, pair_small, small_scene):
    """A[6, 7] is the mixed second difference of the EXACT objective (fixed P, unit weights) in (alpha, beta).  The pose /
    brightness terms A[0:6, 6] have the sign of d2f / dxi dalpha for a left-multiplied pose increment (how the engine applies
    one); their size differs from it by the approximation the whole pose block shares (the gradient averaged with the
    reference's, at the untransformed point), so only the sign is pinned here."""
    pref, pcur = _pyrs(oracle, pair_small, small_scene)
    T = np.linalg.inv(pair_small["T_true"])
    m = oracle.mode("exact")
    ab = np.array([1.05, -3.0])
    lin = oracle.linearize(pref, pcur, 1, T, m, ab=ab)
    P = lin["precision"]
    f = lambda TT, x: _objective(oracle, pref, pcur, TT, x, m, P, 1)
    ha, hb = 1e-2, 1.0
    a67 = (f(T, ab + [ha, hb]) - f(T, ab + [ha, -hb]) - f(T, ab + [-ha, hb]) + f(T, ab + [-ha, -hb])) / (4 * ha * hb)
    assert abs(a67 - lin["A"][6, 7]) <= 1e-3 * abs(a67), (a67, lin["A"][6, 7])
    assert lin["A"][6, 7] == lin["A"][7, 6]
    for k in range(6):
        e = np.zeros(6); e[k] = 1e-4
        g = lambda s: (f(synth.se3_exp(s * e) @ T, ab + [ha, 0]) - f(synth.se3_exp(s * e) @ T, ab - [ha, 0])) / (2 * ha)
        fd = (g(1) - g(-1)) / 2e-4
        assert np.sign(fd) == np.sign(lin["A"][k, 6]) and lin["A"][k, 6] == lin["A"][6, k], (k, fd, lin["A"][k, 6])
