"""Every Gauss-Newton step of the level kernel against an fp64 replay of its own iteration log (tests/step_replay.py).

The replay rebuilds from the logged increments the pose (and brightness) each iteration linearised at, linearises the
oracle there (MIRROR, or helpers.corrected_mode for the corrected estimator), and checks every entry of every
alignment: constraint count, precision, log-likelihood, prior term, information (with the prior, or the photometric
Schur complement), the increment as a backward error in the reference system, the accept decisions, each level's
termination and length, and the final pose and (alpha, beta).  Whatever path rounding sends an alignment down, it is
checked along that path.

Prefix runs check the replay's SE(3) chain and (alpha, beta), which the log does not hold, against the kernel directly: on a
single-level config, a run capped at max_iterations_per_level = k ends after computing x_k without applying it, so it
returns the state iteration k - 1 linearised at, and its log is the uncapped log's first k entries bit for bit.
"""
import json

import numpy as np
import pytest

import step_replay as sr
from dvo_slam_b200.engine import Config

pytestmark = pytest.mark.gpu

PREFIX_MAX_K = 12


@pytest.fixture(scope="module")
def maxima(request):
    """mode -> quantity -> largest normalised error over the tests of this module that ran; at the module's end one line
    with them beside the bounds (step_replay's docstring defines each quantity), written past output capture"""
    found = {}
    yield found
    b = sr.Bounds()
    bounds = {"n": b.n, "precision": f"{b.P} ({sr.PHOTOMETRIC.P} photometric)", "nll": f"{b.rel} + {b.nll_abs} abs",
              "prior": b.prior_rel, "A": f"{b.A} ({sr.PHOTOMETRIC.A} photometric)", "x": b.tau, "pose": b.pose, "ab": b.ab}
    line = ("end-step replay maxima: " + json.dumps({m: {k: float("%.3g" % v) for k, v in d.items()} for m, d in found.items()})
            + "\nend-step replay bounds: " + json.dumps(bounds))
    cap = request.config.pluginmanager.getplugin("capturemanager")
    if cap is None:
        print("\n" + line)
    else:
        with cap.global_and_fixture_disabled():
            print("\n" + line)


def _record(found, mode, maxima):
    d = found.setdefault(mode, {})
    for k, v in maxima.items():
        d[k] = max(d.get(k, 0.0), v)


def _gpu_log(engine, c):
    kw = {} if c["mask"] is None else {"mask": c["mask"], "mask_roles": "both"}
    gref = engine.pyramid(c["I_ref"], c["Z_ref"], c["K"], c["levels"], **kw)
    gcur = engine.pyramid(c["I_cur"], c["Z_cur"], c["K"], c["levels"], **kw)
    cfg = Config(**c["cfg"])
    T0 = None if c["T_init"] is None else [c["T_init"]]
    prior = None if c["prior"] is None else np.asarray(c["prior"])[None]
    engine.set_estimator(c["estimator"])
    try:
        if c["photometric"]:
            res, ab = engine.match_batch_photometric([gref], [gcur], cfg, T0, None if c["ab0"] is None else [c["ab0"]],
                                                     with_iterations=True, prior_information=prior)
            return sr.as_log(res[0], ab[0])
        return sr.as_log(engine.match_batch([gref], [gcur], cfg, T0, with_iterations=True, prior_information=prior)[0])
    finally:
        engine.set_estimator("reference")


@pytest.mark.parametrize("name", list(sr.CASES))
def test_every_step_replays(engine, oracle, maxima, name):
    c = sr.case(name)
    log = _gpu_log(engine, c)
    rep = sr.replay_case(c, log, sr.PHOTOMETRIC if c["photometric"] else sr.Bounds())
    _record(maxima, name.split("/")[0], rep.maxima)
    assert not rep.failures, rep.failures[:5]


def _same_entry(a, b):
    return all(np.array_equal(np.asarray(a[k]), np.asarray(b[k]), equal_nan=True)
               for k in ("level", "id", "n", "nll", "precision", "prior", "x", "A"))


@pytest.mark.parametrize("name", ["reference/golden11", "photometric-reference/exposure0"])
def test_prefix_runs(engine, oracle, maxima, name):
    """level 0 alone, capped at k = 1 .. K iterations: the log is a prefix of the uncapped log, bit for bit, and the result
    is the replayed state of entry k - 1 (its pose; in the photometric mode its (alpha, beta))"""
    c = sr.case(name)
    c["cfg"].update(first_level=0, last_level=0)
    full = _gpu_log(engine, c)
    rep = sr.replay_case(c, full, sr.PHOTOMETRIC if c["photometric"] else sr.Bounds())
    assert not rep.failures, rep.failures[:5]
    K = min(len(full.iterations), PREFIX_MAX_K)
    assert K >= 4
    worst = {"pose": 0.0, "ab": 0.0}
    for k in range(1, K + 1):
        ck = dict(c, cfg=dict(c["cfg"], max_iterations_per_level=k))
        log = _gpu_log(engine, ck)
        assert len(log.iterations) == k
        assert all(_same_entry(a, b) for a, b in zip(log.iterations, full.iterations)), k
        estimate, ab, path = rep.states[k - 1]
        worst["pose"] = max(worst["pose"], np.abs(log.T - sr.se3_inv(estimate)).max())
        assert np.abs(log.T - sr.se3_inv(estimate)).max() <= sr.Bounds().pose, k
        if c["photometric"]:
            worst["ab"] = max(worst["ab"], sr.ab_error(log.ab, ab, path))
            assert sr.ab_error(log.ab, ab, path) <= sr.Bounds().ab, (k, log.ab, ab, path)
    _record(maxima, "prefix-" + name.split("/")[0], worst)



def test_corrected_log_likelihood_past_the_products_overflow(engine, oracle):
    """Where the reference's 50-point products overflow (-ll = +inf, the step rejected), the corrected estimator's
    log-likelihood is the finite per-point sum (helpers.corrected_mode): the kernel's hook gives it to the suite's bound"""
    from helpers import corrected_mode
    from test_corrected_estimator import overflow_state
    im, K, oref, ocur, T, pp = overflow_state(oracle)
    o = oracle.linearize(oref, ocur, 0, T, corrected_mode(oracle), True, pp)
    assert np.isfinite(o["ll"]) and oracle.linearize(oref, ocur, 0, T, oracle.mode("mirror"), True, pp)["ll"] == -np.inf
    gref = engine.pyramid(im["I_ref"], im["Z_ref"], K, 3)
    gcur = engine.pyramid(im["I_cur"], im["Z_cur"], K, 3)
    engine.set_estimator("corrected")
    try:
        g = engine.linearize(gref, gcur, 0, T, True, pp)
    finally:
        engine.set_estimator("reference")
    assert g["n"] == o["n"]
    assert np.allclose(g["precision"], o["precision"], rtol=0, atol=2e-6 * np.abs(o["precision"]).max())
    assert abs(g["ll"] - o["ll"]) <= 2e-6 * abs(o["ll"]) + 0.5, (g["ll"], o["ll"])
