"""The statistics of an alignment: the per-iteration log (dvo_b200_iteration_stats, DenseTracker::IterationStats) and the
LevelStats helper fields of dvo_b200_level_stats, against the oracle's MIRROR log and against the reference's definition of
HasIterationWithIncrement / LastIterationWithIncrement (tests/helpers.py level_fields).  Also the device-result entry point,
per-pair initial estimates in a fused batch, and an iteration log smaller than the iterations it has to hold.

Every termination path is reached here, each asserted from the oracle: IncrementTooSmall, IterationsExceeded
(max_iterations_per_level 1 and 0), LogLikelihoodDecreased, TooFewConstraints on the first iteration of the last level,
TooFewConstraints on the first iteration turned into IncrementTooSmall by the post-loop check, and TooFewConstraints after
an accepted iteration on the last level.  The last two are where LastIterationWithIncrement() is the entry with n < 6
constraints.  The cases are 160x120 (the oracle finishes them in milliseconds) except where a fused launch needs 640x480.
"""
import ctypes as C

import numpy as np
import pytest

from helpers import STATISTICS_CASES as CASES
from helpers import STATISTICS_CFG as CFG
from helpers import (TERM_INCREMENT_TOO_SMALL, TERM_ITERATIONS_EXCEEDED, TERM_LOG_LIKELIHOOD_DECREASED,
                     TERM_TOO_FEW_CONSTRAINTS, level_fields, split_levels)
from helpers import statistics_case as _case

FIELDS = ("has_iteration_with_increment", "last_valid_constraints", "last_increment_valid_constraints",
          "last_increment_log_likelihood")


def _oracle_match(orc, c, mode="mirror"):
    oref = orc.Pyramid(c["I_ref"], c["Z_ref"], c["K"], c["levels"])
    ocur = orc.Pyramid(c["I_cur"], c["Z_cur"], c["K"], c["levels"])
    return orc.match(oref, ocur, orc.config(**c["cfg"]), orc.mode(mode), T_init=c["T_init"])


def _flow(levels):
    return [(l["termination"], l["num_iterations"]) for l in levels]


@pytest.fixture(scope="module")
def oracle_runs(oracle):
    return {name: _oracle_match(oracle, _case(name)) for name in CASES}


def _expect_flows(runs):
    """the flows each construction is there for, from the oracle's MIRROR mode"""
    last = {k: r["levels"][-1] for k, r in runs.items()}
    assert all(l["termination"] == TERM_ITERATIONS_EXCEEDED and l["num_iterations"] == 1 for l in runs["iterations_1"]["levels"])
    assert all(l["termination"] == TERM_ITERATIONS_EXCEEDED and l["num_iterations"] == 1 for l in runs["iterations_0"]["levels"])
    assert any(l["termination"] == TERM_INCREMENT_TOO_SMALL for l in runs["increment_too_small"]["levels"])
    assert any(l["termination"] == TERM_LOG_LIKELIHOOD_DECREASED and l["num_iterations"] >= 2
               for k in ("golden11", "golden12", "golden13") for l in runs[k]["levels"])
    assert last["tfc_first_iteration"]["termination"] == TERM_TOO_FEW_CONSTRAINTS and last["tfc_first_iteration"]["num_iterations"] == 1
    assert all(l["termination"] != TERM_TOO_FEW_CONSTRAINTS for l in runs["tfc_first_iteration"]["levels"][:-1])
    assert all(l["termination"] == TERM_INCREMENT_TOO_SMALL and l["num_iterations"] == 1 for l in runs["tfc_overridden"]["levels"])
    assert all(it["n"] < 6 for it in runs["tfc_overridden"]["iterations"])
    assert last["tfc_after_accept"]["termination"] == TERM_TOO_FEW_CONSTRAINTS and last["tfc_after_accept"]["num_iterations"] >= 2
    lv = split_levels(runs["tfc_after_accept"])[-1]
    assert lv[-1]["n"] < 6 and all(it["n"] >= 6 for it in lv[:-1])


def test_level_fields_definition_on_oracle_logs(oracle, oracle_runs):
    """CPU: the flows are reached, and the definition of the level fields picks what the reference's match() picks.  The
    oracle chooses Result.Information / LogLikelihood (dense_tracking.cpp:368-373) with its own index arithmetic; the
    helper's LastIterationWithIncrement() of the last level must be that entry whenever it holds an increment."""
    _expect_flows(oracle_runs)
    fa = _oracle_match(oracle, _case("tfc_after_accept"), "faithful")
    assert _flow(fa["levels"]) == _flow(oracle_runs["tfc_after_accept"]["levels"])
    for name, r in oracle_runs.items():
        per_level = split_levels(r)
        for lv, l in zip(per_level, r["levels"]):
            f = level_fields(lv, l["termination"])
            assert f["last_valid_constraints"] == lv[-1]["n"]
            if l["termination"] == TERM_LOG_LIKELIHOOD_DECREASED:
                assert f["has_iteration_with_increment"] == (len(lv) >= 2)
                if len(lv) >= 2:   # the entry before a rejected one was accepted
                    assert np.isfinite(lv[-2]["x"]).all() and f["last_increment_valid_constraints"] == lv[-2]["n"]
            elif l["termination"] != TERM_TOO_FEW_CONSTRAINTS:
                assert f["has_iteration_with_increment"] and f["last_increment_valid_constraints"] == lv[-1]["n"]
        last, lv = r["levels"][-1], per_level[-1]
        f = level_fields(lv, last["termination"])
        if f["has_iteration_with_increment"] and np.isfinite(lv[-1 - (last["termination"] == TERM_LOG_LIKELIHOOD_DECREASED)]["x"]).all():
            assert r["log_likelihood"] == f["last_increment_log_likelihood"] + \
                lv[-1 - (last["termination"] == TERM_LOG_LIKELIHOOD_DECREASED)]["prior"], name
    # the two cases where the picked entry is the one with n < 6: its log-likelihood is the value-initialised 0
    for lv, l in zip(split_levels(oracle_runs["tfc_overridden"]), oracle_runs["tfc_overridden"]["levels"]):
        assert level_fields(lv, l["termination"]) == {"has_iteration_with_increment": True, "last_valid_constraints": lv[0]["n"],
                                                      "last_increment_valid_constraints": lv[0]["n"],
                                                      "last_increment_log_likelihood": 0.0}
    lv = split_levels(oracle_runs["tfc_after_accept"])[-1]
    f = level_fields(lv, TERM_TOO_FEW_CONSTRAINTS)
    assert f["has_iteration_with_increment"] and f["last_increment_valid_constraints"] == lv[-1]["n"] < 6
    assert f["last_increment_log_likelihood"] == 0.0
    lv = split_levels(oracle_runs["tfc_first_iteration"])[-1]
    f = level_fields(lv, TERM_TOO_FEW_CONSTRAINTS)
    assert not f["has_iteration_with_increment"] and f["last_increment_valid_constraints"] == -1
    assert np.isnan(f["last_increment_log_likelihood"])


# ---------------------------------------------------------------------------------------------------------------------
# GPU

def _gpu_match(engine, c, with_iterations=True):
    from dvo_slam_b200.engine import Config
    gref = engine.pyramid(c["I_ref"], c["Z_ref"], c["K"], c["levels"])
    gcur = engine.pyramid(c["I_cur"], c["Z_cur"], c["K"], c["levels"])
    return engine.match(gref, gcur, Config(**c["cfg"]), T_init=c["T_init"], with_iterations=with_iterations)


def _same_float(a, b):
    return (np.isnan(a) and np.isnan(b)) or a == b


@pytest.mark.gpu
@pytest.mark.parametrize("name", CASES)
def test_level_fields(engine, oracle_runs, name):
    """dvo_b200_level_stats' helper fields equal the reference's definition applied to the GPU's own iteration log, with and
    without a log requested; where the flow equals MIRROR's, also the definition applied to the oracle's log."""
    c = _case(name)
    r = _gpu_match(engine, c)
    plain = _gpu_match(engine, c, with_iterations=False)
    assert len(plain.levels) == len(r.levels)
    for a, b in zip(plain.levels, r.levels):   # the fields do not depend on whether a log is kept
        assert all(_same_float(a[k], b[k]) if isinstance(a[k], float) else a[k] == b[k] for k in a), (a, b)
    mi = oracle_runs[name]
    if name.startswith("tfc") or name.startswith("iterations"):
        assert _flow(r.levels) == _flow(mi["levels"]), (name, _flow(r.levels), _flow(mi["levels"]))
    for lv, l in zip(split_levels(r), r.levels):
        want = level_fields(lv, l["termination"])
        got = {k: l[k] for k in FIELDS}
        assert got["has_iteration_with_increment"] == want["has_iteration_with_increment"], (name, l, want)
        assert got["last_valid_constraints"] == want["last_valid_constraints"], (name, l, want)
        assert got["last_increment_valid_constraints"] == want["last_increment_valid_constraints"], (name, l, want)
        assert _same_float(got["last_increment_log_likelihood"], want["last_increment_log_likelihood"]), (name, l, want)
    if _flow(r.levels) == _flow(mi["levels"]):
        for lg, lo, l in zip(split_levels(r), split_levels(mi), r.levels):
            g, o = level_fields(lg, l["termination"]), level_fields(lo, l["termination"])
            assert g["has_iteration_with_increment"] == o["has_iteration_with_increment"]
            assert abs(g["last_increment_valid_constraints"] - o["last_increment_valid_constraints"]) <= 2
            a, b = g["last_increment_log_likelihood"], o["last_increment_log_likelihood"]
            assert _same_float(a, b) or abs(a - b) <= 1e-3 * abs(b), (name, a, b)


@pytest.mark.gpu
@pytest.mark.parametrize("name", CASES)
def test_iteration_log_structure(engine, name):
    """Exact properties of the GPU's own log: one entry per iteration, ids 0..k-1 per level, increment and information NaN
    exactly on the rejected (LogLikelihoodDecreased) and TooFewConstraints entries, and Result.Information / LogLikelihood
    taken from the entry dense_tracking.cpp:368-373 picks."""
    c = _case(name)
    r = _gpu_match(engine, c)
    assert sum(l["num_iterations"] for l in r.levels) == r.num_iterations_total == len(r.iterations)
    per_level = split_levels(r)
    for lv, l in zip(per_level, r.levels):
        assert [it["id"] for it in lv] == list(range(l["num_iterations"]))
        assert all(it["level"] == l["id"] for it in lv)
        for k, it in enumerate(lv):
            rejected = it["n"] < 6 or (k == len(lv) - 1 and l["termination"] == TERM_LOG_LIKELIHOOD_DECREASED)
            assert np.isnan(it["x"]).all() == rejected and np.isnan(it["A"]).all() == rejected, (name, k, it["n"])
            assert np.isfinite(it["x"]).all() != rejected and np.isfinite(it["A"]).all() != rejected
            if it["n"] < 6:   # the value-initialised entry of dense_tracking.cpp:247-284
                assert it["nll"] == 0.0 and it["prior"] == 0.0 and not it["precision"].any()
    last, lv = r.levels[-1], per_level[-1]
    pick = lv[-2] if last["termination"] == TERM_LOG_LIKELIHOOD_DECREASED else lv[-1]
    if pick["n"] >= 6:
        assert np.array_equal(r.information, pick["A"] * 0.008 * 0.008)
        assert r.log_likelihood == pick["nll"] + pick["prior"]
    else:   # the reference reads an entry without an estimate here (SURVEY Q24): NaN, so Result::isNaN() fires
        assert np.isnan(r.information).all() and r.is_nan()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["golden11", "golden12", "golden13", "initial_estimate"])
def test_first_iteration_against_oracle(engine, oracle_runs, name):
    """The first iteration of the first level runs at a known transform (the identity, or T_init): the same constraints as the
    oracle's MIRROR mode, and the same log-likelihood, precision and information up to summation order."""
    r = _gpu_match(engine, _case(name))
    g, o = r.iterations[0], oracle_runs[name]["iterations"][0]
    assert (g["level"], g["id"]) == (o["level"], o["id"]) == (CFG["first_level"], 0)
    assert g["n"] == o["n"] > 6
    assert abs(g["nll"] - o["nll"]) <= 2e-6 * abs(o["nll"]) + 0.5
    assert np.allclose(g["precision"], o["precision"], rtol=2e-6, atol=0)
    assert np.allclose(g["A"], o["A"], rtol=0, atol=2e-6 * np.abs(o["A"]).max())
    assert g["prior"] == pytest.approx(o["prior"], rel=1e-9, abs=1e-12)


@pytest.mark.gpu
def test_iteration_log_against_oracle(engine, oracle_runs):
    """Where the control flow equals MIRROR's, every entry's constraint count agrees within 2 (a pixel exactly on a bound may
    flip as the pose chains differ by ~1e-8), and log-likelihood and prior to 1e-3 relative."""
    compared = 0
    for name in CASES:
        r = _gpu_match(engine, _case(name))
        mi = oracle_runs[name]
        if _flow(r.levels) != _flow(mi["levels"]):
            continue
        compared += 1
        assert len(r.iterations) == len(mi["iterations"])
        for g, o in zip(r.iterations, mi["iterations"]):
            assert (g["level"], g["id"]) == (o["level"], o["id"])
            assert abs(g["n"] - o["n"]) <= 2, (name, g["n"], o["n"])
            assert abs(g["nll"] - o["nll"]) <= 1e-3 * abs(o["nll"]), (name, g["nll"], o["nll"])
            assert abs(g["prior"] - o["prior"]) <= 1e-3 * abs(o["prior"]) + 1e-9, (name, g["prior"], o["prior"])
            assert np.array_equal(np.isnan(g["x"]), np.isnan(o["x"]))
            if o["n"] < 6:
                assert not g["precision"].any() and not o["precision"].any()
    assert compared >= len(CASES) // 2, compared


def _golden_batch(engine, names):
    cs = [_case(n) for n in names]
    refs = [engine.pyramid(c["I_ref"], c["Z_ref"], c["K"], c["levels"]) for c in cs]
    curs = [engine.pyramid(c["I_cur"], c["Z_cur"], c["K"], c["levels"]) for c in cs]
    return refs, curs


@pytest.mark.gpu
def test_match_batch_device_equals_match_batch(engine):
    """dvo_b200_match_batch_device leaves the records in device memory: gathered into a torch CUDA buffer and read after the
    context's stream is synchronised, they are match_batch's records byte for byte (the buffer's 0x5A fill is gone)."""
    import torch
    from dvo_slam_b200.engine import CResult, Config
    names = ["golden11", "golden12", "golden13", "tfc_overridden", "golden12"]
    refs, curs = _golden_batch(engine, names)
    cfg = Config(**CFG)
    want = engine.match_batch(refs, curs, cfg, raw=True)
    n = len(names)
    buf = torch.full((n * C.sizeof(CResult),), 0x5A, dtype=torch.uint8, device="cuda:0")
    torch.cuda.synchronize()
    engine.match_batch_device(refs, curs, cfg, buf.data_ptr())
    engine.synchronize()
    got = (CResult * n).from_buffer_copy(buf.cpu().numpy().tobytes())
    for i in range(n):
        assert bytes(got[i]) == bytes(want[i]), i
        assert np.array_equal(np.array(got[i].transformation), np.array(want[i].transformation))
        assert got[i].num_iterations_total == want[i].num_iterations_total > 0


def _log_bytes(its):
    return [b"".join([np.int64(it["level"]).tobytes(), np.int64(it["id"]).tobytes(), np.int64(it["n"]).tobytes(),
                      np.float64(it["nll"]).tobytes(), it["precision"].tobytes(), np.float64(it["prior"]).tobytes(),
                      it["x"].tobytes(), it["A"].tobytes()]) for it in its]


@pytest.mark.gpu
def test_per_pair_initial_estimate_in_a_fused_batch(engine):
    """72 640x480 pairs (a batch that fills the GPU runs every level in one fused launch) with a different T_init per pair
    and use_initial_estimate: results and iteration logs are bit-equal to single alignments with the same T_init."""
    import os
    from dvo_slam_b200 import synth
    from dvo_slam_b200.engine import Config
    pairs = [synth.make_pair(s) for s in range(4)]
    K = pairs[0]["intrinsics"]
    refs = engine.pyramid_batch(np.stack([p["I_ref"].numpy() for p in pairs]), np.stack([p["Z_ref"].numpy() for p in pairs]), K, 5)
    curs = engine.pyramid_batch(np.stack([p["I_cur"].numpy() for p in pairs]), np.stack([p["Z_cur"].numpy() for p in pairs]), K, 5)
    n = 72
    idx = [i % 4 for i in range(n)]
    T0 = np.stack([synth.se3_exp(pairs[k]["xi"] * (0.3 + 0.01 * i)) for i, k in enumerate(idx)])
    cfg = Config(first_level=4, last_level=0, max_iterations_per_level=50, precision=1e-4, use_initial_estimate=1)
    b = [refs[k] for k in idx], [curs[k] for k in idx]
    l0 = engine.kernel_launches()
    batch = engine.match_batch(*b, cfg, T_init=T0, with_iterations=True)
    fused_launches = engine.kernel_launches() - l0
    os.environ["DVO_B200_NO_FUSE"] = "1"
    try:
        l0 = engine.kernel_launches()
        unfused = engine.match_batch(*b, cfg, T_init=T0, with_iterations=True)
        assert engine.kernel_launches() - l0 == fused_launches + 1     # coarse and fine levels: one launch instead of two
    finally:
        del os.environ["DVO_B200_NO_FUSE"]
    for i in range(n):
        single = engine.match(refs[idx[i]], curs[idx[i]], cfg, T_init=T0[i], with_iterations=True)
        for other in (single, unfused[i]):
            assert np.array_equal(batch[i].transformation, other.transformation), i
            assert np.array_equal(batch[i].information, other.information, equal_nan=True), i
            assert batch[i].log_likelihood == other.log_likelihood and batch[i].levels == other.levels, i
            assert _log_bytes(batch[i].iterations) == _log_bytes(other.iterations), i
    # the estimates differ per pair: the same images with different T_init do not all give the same bits
    assert not all(np.array_equal(batch[0].transformation, batch[i].transformation) for i in range(4, n, 4))


@pytest.mark.gpu
def test_truncated_iteration_log(engine):
    """max_iteration_stats smaller than the iterations run: each pair's slot holds its first max_iteration_stats entries,
    nothing is written past a slot or past the buffer, and the results are those of an untruncated call."""
    from dvo_slam_b200.engine import CResult, Config, IterationStats
    names = ["golden11", "tfc_overridden", "golden12", "golden13"]
    refs, curs = _golden_batch(engine, names)
    cfg = Config(**CFG)
    full = engine.match_batch(refs, curs, cfg, with_iterations=True)
    full_raw = engine.match_batch(refs, curs, cfg, raw=True)
    n, m, extra = len(names), 4, 3
    assert full[1].num_iterations_total < m < min(full[i].num_iterations_total for i in (0, 2, 3))
    log = (IterationStats * (n * m + extra))()
    C.memset(log, 0xA5, C.sizeof(log))
    sentinel = bytes([0xA5]) * C.sizeof(IterationStats)
    res = (CResult * n)()
    rh = (C.c_void_p * n)(*[p.handle for p in refs])
    ch = (C.c_void_p * n)(*[p.handle for p in curs])
    engine._check(engine.lib.dvo_b200_match_batch(engine.ctx, C.byref(cfg), n, rh, ch, None, res, log, m))
    for i in range(n):
        assert bytes(res[i]) == bytes(full_raw[i]), i
        assert res[i].num_iterations_total == full[i].num_iterations_total
        k = min(m, full[i].num_iterations_total)
        for j in range(k):
            s, want = log[i * m + j], full[i].iterations[j]
            got = {"level": s.level, "id": s.id, "n": s.valid_constraints, "nll": s.tdist_log_likelihood,
                   "precision": np.array(s.tdist_precision).reshape(2, 2), "prior": s.prior_log_likelihood,
                   "x": np.array(s.increment), "A": np.array(s.information).reshape(6, 6)}
            assert _log_bytes([got]) == _log_bytes([want]), (i, j)
        for j in range(k, m):   # the unused end of a slot is cleared, not left stale
            assert bytes(log[i * m + j]) == bytes(C.sizeof(IterationStats)), (i, j)
    for j in range(n * m, n * m + extra):
        assert bytes(log[j]) == sentinel, j
