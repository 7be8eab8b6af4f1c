"""The end-step replay model (tests/step_replay.py) on the CPU oracle's own iteration logs, before it judges the GPU's.

Self-replay: the oracle's logs of every replay case (default and corrected estimator, non-default selection thresholds, the
photometric mode with a mask and an initial (alpha, beta), full, rank-one and scalar priors with and without the
photometric mode, and the 640x480 and 1280x960 benchmark shapes) replay at step_replay.TIGHT: counts, precision and
log-likelihood exact, information, increments and poses to the fp64 rounding of a different solve and SE(3) formula.
The cases reach every termination, and the level start's re-application of the previous level's last increment after a
reject and after TooFewConstraints.

Mutation controls: each rule of the end step, broken once in the model or in a log, makes a named check fail at the bounds
the GPU is held to (step_replay.Bounds()), so the checks tell the kernel's rule from its neighbours at those bounds.
"""
import copy

import numpy as np
import pytest

import step_replay as sr
from helpers import (TERM_INCREMENT_TOO_SMALL, TERM_ITERATIONS_EXCEEDED, TERM_LOG_LIKELIHOOD_DECREASED,
                     TERM_TOO_FEW_CONSTRAINTS)

_logs = {}


def _oracle(name):
    if name not in _logs:
        c = sr.case(name)
        _logs[name] = (c, sr.oracle_log(c))
    return _logs[name]


@pytest.mark.parametrize("name", list(sr.CASES))
def test_oracle_self_replay(oracle, name):
    c, log = _oracle(name)
    rep = sr.replay_case(c, log, sr.TIGHT)
    assert not rep.failures, rep.failures[:5]
    assert len(rep.states) == len(log.iterations)


def test_self_replay_covers_every_path(oracle):
    """every termination in the default and the photometric mode; a level that starts after a reject and one that starts
    after TooFewConstraints with more levels to go (so the re-applied increment is one that was reverted)"""
    terms = {}
    after = set()
    for name in sr.CASES:
        c, log = _oracle(name)
        mode = "photometric" if c["photometric"] else "default"
        terms.setdefault(mode, set()).update(t for t, _ in log.levels)
        after.update(t for t, _ in log.levels[:-1])
    assert terms["default"] == {TERM_ITERATIONS_EXCEEDED, TERM_INCREMENT_TOO_SMALL, TERM_LOG_LIKELIHOOD_DECREASED,
                                TERM_TOO_FEW_CONSTRAINTS}
    assert {TERM_INCREMENT_TOO_SMALL, TERM_LOG_LIKELIHOOD_DECREASED} <= terms["photometric"]
    assert TERM_LOG_LIKELIHOOD_DECREASED in after
    _, log = _oracle("reference/tfc_overridden")   # TooFewConstraints on level 2 and 1, reported as IncrementTooSmall
    assert all(it["n"] < 6 for it in log.iterations) and len(log.levels) == 3


def _largest_applied_increment(log):
    """(entry, component) of the largest increment component that a later iteration applies (not a level's last entry)"""
    best, k0 = (None, None, 0.0), 0
    for _, count in log.levels:
        for j in range(count - 1):
            x = log.iterations[k0 + j]["x"]
            if np.isfinite(x).all() and np.abs(x).max() > best[2]:
                best = (k0 + j, int(np.abs(x).argmax()), np.abs(x).max())
        k0 += count
    return best[:2]


def _first_accepted_in_a_later_level(log):
    k0 = log.levels[0][1]
    for j in range(k0, len(log.iterations)):
        if np.isfinite(log.iterations[j]["x"]).all():
            return j
    raise AssertionError("no accepted entry after the first level")


# (mutation, case, the check that must fail)
CONTROLS = [("scaled_increment", "reference/golden11", "pose"),
            ("no_level_start_reapply", "reference/golden11", "pose"),
            ("li_from_estimate", "prior/spd1e9", "prior"),
            ("information_without_prior", "prior/mu", "A"),
            ("ab_not_reverted", "photometric-reference/exposure0", "ab"),
            ("schur_without_prior", "prior-photometric/spd1e9", "A"),
            ("flip_accept", "reference/golden12", "decision")]


@pytest.mark.parametrize("mutation,name,check", CONTROLS, ids=[m for m, _, _ in CONTROLS])
def test_mutation_is_caught(oracle, mutation, name, check):
    c, log = _oracle(name)
    assert not sr.replay_case(c, log, sr.Bounds()).failures   # the rule itself passes at the GPU's bounds
    if mutation == "scaled_increment":   # one logged increment component times 1 + 1e-5
        log = copy.deepcopy(log)
        k, i = _largest_applied_increment(log)
        log.iterations[k]["x"][i] *= 1 + 1e-5
        rep = sr.replay_case(c, log, sr.Bounds())
    else:
        entry = _first_accepted_in_a_later_level(log) if mutation == "flip_accept" else -1
        rep = sr.replay_case(c, log, sr.Bounds(), sr.Mutation(mutation, entry))
    assert check in rep.failed, (rep.failed, rep.maxima)
