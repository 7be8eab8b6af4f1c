"""The corrected estimator without a GPU: its C ABI entry points, and the oracle definition the GPU kernel is checked against.

"corrected" = the oracle's MIRROR mode with the four structural quirks of the reference off (helpers.corrected_mode):
scale = sum_i w_i r_i r_i^T / (n - 3), log-likelihood over all n points as the sum of their logs, the odd last point kept."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from helpers import GOLDEN_SEEDS, corrected_mode, golden_images, load_golden, odd_point_margin  # noqa: F401

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as ge
    ge.build_cuda()
    from dvo_slam_b200 import engine
    return engine.load_library()


def test_estimator_entry_points(lib):
    from dvo_slam_b200 import engine
    assert hasattr(lib, "dvo_b200_set_estimator") and hasattr(lib, "dvo_b200_get_estimator")
    src = open(os.path.join(ROOT, "include", "dvo_b200.h")).read()
    assert re.search(r"DVO_B200_ESTIMATOR_REFERENCE\s*=\s*0\b", src) and re.search(r"DVO_B200_ESTIMATOR_CORRECTED\s*=\s*1\b", src)
    assert engine.ESTIMATORS == {"reference": 0, "corrected": 1}
    # a NULL context is rejected whatever the value (DVO_B200_ERR_INVALID_ARGUMENT)
    for e in (0, 1, 2, -1):
        assert lib.dvo_b200_set_estimator(None, e) == -1
    assert lib.dvo_b200_get_estimator(None) == -1


def _student_t(E, P):
    """computeWeightsSse with mean 0 and nu = 5: w = 7 / (5 + r^T P r), in float as the oracle's IEEE modes compute it"""
    x, y = E[:, 0], E[:, 1]
    d = (x * P[0, 0] + y * P[1, 0]) * x + (x * P[0, 1] + y * P[1, 1]) * y
    return ((2.0 + 5.0) / (np.float32(5.0) + d).astype(np.float64)).astype(np.float32)


@pytest.mark.parametrize("seed", GOLDEN_SEEDS)
def test_oracle_corrected_scale_and_log_likelihood(oracle, seed):
    """P = inverse(sum w r r^T / (n - 3)) over the corrected residual image, LL over all n points."""
    g = load_golden(seed)
    im = golden_images(g, oracle)
    oref = oracle.Pyramid(im["I_ref"], im["Z_ref"], g["K"], 3)
    ocur = oracle.Pyramid(im["I_cur"], im["Z_cur"], g["K"], 3)
    m = corrected_mode(oracle)
    T = np.eye(4)
    T[:3, 3] = [0.01, -0.005, 0.02]
    pp = np.array([[2000.0, -30.0], [-30.0, 9000.0]], dtype=np.float32)
    for lvl in range(3):
        n_img, planes = oracle.residual_image(oref, ocur, lvl, T, m)
        E = planes[0:2].reshape(2, -1).T
        E = E[~np.isnan(E[:, 0])]
        assert E.shape[0] == n_img > 50
        for uw in (False, True):
            lin = oracle.linearize(oref, ocur, lvl, T, m, uw, pp)
            assert lin["n"] == n_img
            w = _student_t(E, pp) if uw else np.ones(n_img, np.float32)
            e = E.astype(np.float64)
            S = np.array([np.sum(w * e[:, 0] * e[:, 0]), np.sum(w * e[:, 0] * e[:, 1]), np.sum(w * e[:, 1] * e[:, 1])]) / (n_img - 3)
            Cov = S.astype(np.float32)
            det = Cov[0] * Cov[2] - Cov[1] * Cov[1]
            P = np.array([[Cov[2], -Cov[1]], [-Cov[1], Cov[0]]], dtype=np.float32) * (np.float32(1.0) / det)
            assert np.allclose(lin["precision"], P, rtol=1e-5), (lvl, uw, lin["precision"], P)
            # the log-likelihood over ALL n terms, from the P the oracle returned
            Pk = lin["precision"].astype(np.float32)
            x, y = E[:, 0], E[:, 1]
            d = (x * Pk[0, 0] + y * Pk[1, 0]) * x + (x * Pk[0, 1] + y * Pk[1, 1]) * y
            detP = np.float32(Pk[0, 0] * Pk[1, 1] - Pk[0, 1] * Pk[1, 0])
            ll = 0.5 * n_img * float(np.log(detP)) - 3.5 * float(np.sum(np.log1p(0.2 * d.astype(np.float64))))
            assert abs(lin["ll"] - ll) <= 1e-5 * abs(ll) + 1e-2, (lvl, uw, lin["ll"], ll)
            if n_img % 50:
                # and not what the reference's truncated sum gives
                kept = (n_img // 50) * 50
                ll_trunc = 0.5 * n_img * float(np.log(detP)) - 3.5 * float(np.sum(np.log1p(0.2 * d[:kept].astype(np.float64))))
                assert abs(ll - ll_trunc) > 1e-3 * abs(ll - lin["ll"]) + 1e-3


def test_oracle_corrected_keeps_the_odd_point(oracle):
    """On the odd-selection case of tests/helpers.py the corrected count is the MIRROR count plus one: the odd last point."""
    margin, im, oref, ocur = odd_point_margin(oracle)
    S, mask = oracle.select(oref, 0, 0.0, 0.0, None)
    assert S % 2 == 1
    last = np.flatnonzero(mask.reshape(-1))[-1]
    mir = oracle.linearize(oref, ocur, 0, np.eye(4), oracle.mode("mirror"))
    cor = oracle.linearize(oref, ocur, 0, np.eye(4), corrected_mode(oracle))
    assert cor["n"] == mir["n"] + 1
    _, pm = oracle.residual_image(oref, ocur, 0, np.eye(4), oracle.mode("mirror"))
    _, pc = oracle.residual_image(oref, ocur, 0, np.eye(4), corrected_mode(oracle))
    assert np.isnan(pm[0].reshape(-1)[last]) and not np.isnan(pc[0].reshape(-1)[last])
    other = np.ones(pm[0].size, bool)
    other[last] = False
    assert np.array_equal(np.isnan(pm[0].reshape(-1)[other]), np.isnan(pc[0].reshape(-1)[other]))


def overflow_state(orc):
    """golden pair 11, level 0, a small offset, weights from a previous precision of 1e10 I: the weighted scale is tiny, so
    r^T P r is ~1e9 and a 50-point product of (1 + 0.2 d) passes DBL_MAX -- (pyramids, T, prev_precision)"""
    g = load_golden(11)
    im = golden_images(g, orc)
    oref = orc.Pyramid(im["I_ref"], im["Z_ref"], g["K"], 3)
    ocur = orc.Pyramid(im["I_cur"], im["Z_cur"], g["K"], 3)
    T = np.eye(4)
    T[:3, 3] = [0.01, -0.005, 0.02]
    return im, g["K"], oref, ocur, T, np.array([[1e10, 0.0], [0.0, 1e10]], dtype=np.float32)


def test_oracle_corrected_log_likelihood_past_the_products_overflow(oracle):
    """The reference takes the log of fp64 products of (1 + 0.2 d) over groups of 50 points; where one overflows its
    log-likelihood is -inf and the iteration is rejected.  The corrected estimator sums the per-point logs (as the kernel
    does): finite, and equal to that sum computed here from the residual image and the returned P."""
    _, _, oref, ocur, T, pp = overflow_state(oracle)
    assert oracle.linearize(oref, ocur, 0, T, oracle.mode("mirror"), True, pp)["ll"] == -np.inf
    grouped = corrected_mode(oracle)
    grouped.ll_group_product = 1
    assert oracle.linearize(oref, ocur, 0, T, grouped, True, pp)["ll"] == -np.inf
    m = corrected_mode(oracle)
    lin = oracle.linearize(oref, ocur, 0, T, m, True, pp)
    n_img, planes = oracle.residual_image(oref, ocur, 0, T, m)
    E = planes[0:2].reshape(2, -1).T
    E = E[~np.isnan(E[:, 0])]
    assert E.shape[0] == n_img == lin["n"]
    Pk = lin["precision"].astype(np.float32)
    x, y = E[:, 0], E[:, 1]
    d = (x * Pk[0, 0] + y * Pk[1, 0]) * x + (x * Pk[0, 1] + y * Pk[1, 1]) * y
    detP = np.float32(Pk[0, 0] * Pk[1, 1] - Pk[0, 1] * Pk[1, 0])
    ll = 0.5 * n_img * float(np.log(detP)) - 3.5 * float(np.sum(np.log1p(0.2 * d.astype(np.float64))))
    assert np.isfinite(lin["ll"]) and abs(lin["ll"] - ll) <= 1e-5 * abs(ll), (lin["ll"], ll)
