"""The motion prior without a GPU: the argument checks of csrc/prior_args.h built for the host, and the prior's definition on
the CPU oracle (tests/native/prior_oracle.cpp) against the oracle's own mu path, in both modes."""
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np
import pytest

import prior_oracle as pro
from dvo_slam_b200 import synth
from dvo_slam_b200.engine import prior_from_result

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def checks():
    tmp = tempfile.mkdtemp(prefix="dvo_prior_args_")
    try:
        out = os.path.join(tmp, "libprior_args.so")
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-Wall", "-fPIC", "-shared", "-I", os.path.join(ROOT, "dvo_slam_b200", "csrc"),
                               "-o", out, os.path.join(ROOT, "tests", "native", "prior_args.cpp")])
        L = C.CDLL(out)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    L.prior_check.argtypes = [C.c_int, C.c_double, C.c_int, C.POINTER(C.c_double), C.c_int, C.c_int, C.c_char_p, C.c_int]

    def run(prior, mu=0.0, has_cfg=True, ab_init=False, ab=False, n=None):
        buf = C.create_string_buffer(256)
        p = None
        if prior is not None:
            prior = np.ascontiguousarray(np.asarray(prior, dtype=np.float64).reshape(-1, 36))
            p = prior.ctypes.data_as(C.POINTER(C.c_double))
            n = prior.shape[0] if n is None else n
        L.prior_check(int(has_cfg), mu, 1 if n is None else n, p, int(ab_init), int(ab), buf, 256)
        return buf.value.decode()
    return run


def _spd(rng, scale=1.0):
    M = rng.standard_normal((6, 6))
    S = M @ M.T * scale
    return 0.5 * (S + S.T)


def test_accepted_priors(checks):
    rng = np.random.default_rng(0)
    assert checks(np.zeros((6, 6))) == ""
    for k in range(6):
        e = np.zeros(6); e[k] = 1.0
        assert checks(1e6 * np.outer(e, e)) == ""
    assert checks(np.stack([_spd(rng), _spd(rng, 1e8), 0.05 * np.eye(6)])) == ""
    assert checks(np.stack([_spd(rng)]), ab_init=True, ab=True) == ""
    assert checks(np.stack([_spd(rng)]), ab=True) == ""
    # a PSD rank-deficient prior whose computed eigenvalues sit at rounding level around 0
    v = rng.standard_normal((6, 2))
    assert checks(0.5 * (v @ v.T + (v @ v.T).T) * 1e4) == ""


def test_refused_priors(checks):
    rng = np.random.default_rng(1)
    S = _spd(rng)
    asym = S.copy()
    asym[1, 4] = np.nextafter(asym[1, 4], np.inf)   # one ulp
    assert "pair 0 is not symmetric" in checks(asym)
    assert "pair 0 is not positive semi-definite" in checks(np.diag([1, 1, 1, 1, 1, -1e-3]))
    for bad in (np.nan, np.inf, -np.inf):
        M = S.copy(); M[2, 2] = bad
        assert "pair 0 is not finite" in checks(M)
    assert "pair 1 is not symmetric" in checks(np.stack([S, asym]))
    assert "prior_information is null" in checks(None)
    assert "mu must be 0" in checks(S, mu=0.05)
    assert "photometric_init without photometric" in checks(S, ab_init=True)
    assert checks(S).startswith("") and checks(asym).startswith("match_batch_prior: ")


def test_null_cfg_is_left_to_the_batch_checks(checks):
    assert checks(np.diag([1, 1, 1, 1, 1, -1.0]), has_cfg=False) == ""


def test_prior_from_result_is_symmetric_and_scaled():
    class R:
        information = np.arange(36, dtype=np.float64).reshape(6, 6) * 0.008 ** 2
    L = prior_from_result(R(), 0.5)
    assert np.array_equal(L, L.T)
    assert np.allclose(L, 0.25 * (np.arange(36).reshape(6, 6) + np.arange(36).reshape(6, 6).T))


# ---- the oracle ----
SCENE = synth.SceneConfig(width=160, height=120, intrinsics=tuple(v / 4 for v in synth.FR1_INTRINSICS))


@pytest.fixture(scope="module")
def pyrs():
    out = []
    for seed in (3, 5):
        pair = synth.make_pair(seed, SCENE)
        out.append((pro.Pyramid(pair["I_ref"].numpy(), pair["Z_ref"].numpy(), SCENE.intrinsics, 3),
                    pro.Pyramid(pair["I_cur"].numpy(), pair["Z_cur"].numpy(), SCENE.intrinsics, 3), pair))
    return out


def _cfg(oracle, mu=0.0):
    return oracle.config(first_level=2, last_level=0, max_iterations_per_level=40, precision=5e-7, mu=mu, use_initial_estimate=1)


def _T0(pair):
    """the initial estimate: the true estimate (the inverse of the true Result.transformation), perturbed"""
    return synth.se3_exp(np.array([4e-3, -3e-3, 2e-3, -2e-3, 3e-3, 1e-3])) @ pair["T_true"]


def _same(a, b, prior_tol=None):
    assert np.array_equal(a["T"], b["T"]) and np.array_equal(a["information"], b["information"], equal_nan=True)
    assert a["levels"] == b["levels"] and len(a["iterations"]) == len(b["iterations"])
    for x, y in zip(a["iterations"], b["iterations"]):
        for k in ("level", "id", "n", "nll"):
            assert x[k] == y[k], k
        for k in ("precision", "x", "A"):
            assert np.array_equal(x[k], y[k], equal_nan=True), k
        if prior_tol is None:
            assert x["prior"] == y["prior"]
        else:
            assert abs(x["prior"] - y["prior"]) <= prior_tol * abs(y["prior"])
    if prior_tol is None:
        assert a["log_likelihood"] == b["log_likelihood"] or (np.isnan(a["log_likelihood"]) and np.isnan(b["log_likelihood"]))
    else:
        assert abs(a["log_likelihood"] - b["log_likelihood"]) <= prior_tol * abs(b["log_likelihood"])


@pytest.mark.parametrize("photometric", [False, True])
@pytest.mark.parametrize("mode", ["faithful", "mirror"])
@pytest.mark.parametrize("mu", [0.05, 1.0, 25.0])
def test_scalar_prior_is_the_mu_path(oracle, pyrs, mode, photometric, mu):
    m = oracle.mode(mode)
    for ref, cur, pair in pyrs:
        T0 = _T0(pair)
        d = pro.match(ref, cur, _cfg(oracle, mu), m, T0, photometric=photometric)
        p = pro.match(ref, cur, _cfg(oracle), m, T0, prior=mu * np.eye(6), photometric=photometric)
        assert any(it["prior"] != 0.0 for it in d["iterations"])
        _same(p, d, prior_tol=1e-14)
        if photometric:
            assert np.array_equal(p["ab"], d["ab"])


@pytest.mark.parametrize("photometric", [False, True])
@pytest.mark.parametrize("mode", ["faithful", "mirror"])
def test_zero_prior_is_mu_zero(oracle, pyrs, mode, photometric):
    m = oracle.mode(mode)
    for ref, cur, pair in pyrs:
        T0 = _T0(pair)
        d = pro.match(ref, cur, _cfg(oracle), m, T0, photometric=photometric)
        p = pro.match(ref, cur, _cfg(oracle), m, T0, prior=np.zeros((6, 6)), photometric=photometric)
        _same(p, d)


# A at these sizes is ~1e10 on its diagonal: 1e18 is stiff.
STIFF = 1e18


@pytest.mark.parametrize("photometric", [False, True])
@pytest.mark.parametrize("mode", ["faithful", "mirror"])
def test_stiff_prior_returns_the_initial_estimate(oracle, pyrs, mode, photometric):
    m = oracle.mode(mode)
    for ref, cur, pair in pyrs:
        T0 = _T0(pair)
        p = pro.match(ref, cur, _cfg(oracle), m, T0, prior=STIFF * np.eye(6), photometric=photometric)
        assert np.abs(synth.se3_log(T0 @ p["T"])).max() < 1e-8


@pytest.mark.parametrize("photometric", [False, True])
@pytest.mark.parametrize("mode", ["faithful", "mirror"])
@pytest.mark.parametrize("k", [0, 4])
def test_stiff_rank_one_prior_holds_its_direction(oracle, pyrs, mode, photometric, k):
    """The prior holds component k of log(initial), the Revertable that the increments update from the left; it equals
    log(T0 Result.T) to first order in the increments, so the component returned is small rather than zero."""
    m = oracle.mode(mode)
    for ref, cur, pair in pyrs:
        T0 = _T0(pair)
        e = np.zeros(6); e[k] = 1.0
        p = pro.match(ref, cur, _cfg(oracle), m, T0, prior=STIFF * np.outer(e, e), photometric=photometric)
        d = synth.se3_log(T0 @ p["T"])
        assert abs(d[k]) < 2e-4, d
        assert np.abs(np.delete(d, k)).max() > 4e-3, d
