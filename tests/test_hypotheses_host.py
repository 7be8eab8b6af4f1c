"""Multi-hypothesis alignment without a GPU: the argument checks of csrc/hypotheses_args.h built for the host, and its
selection rule on synthetic level statistics against the Python restatement in tests/hypotheses_model.py."""
import ctypes as C
import math
import os
import shutil
import subprocess
import tempfile

import numpy as np
import pytest

import hypotheses_model as hm

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MAX_HYPOTHESES = 64
NAN = float("nan")


@pytest.fixture(scope="module")
def lib():
    tmp = tempfile.mkdtemp(prefix="dvo_hypotheses_args_")
    try:
        out = os.path.join(tmp, "libhypotheses_args.so")
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-Wall", "-fPIC", "-shared", "-I", os.path.join(ROOT, "dvo_slam_b200", "csrc"),
                               "-o", out, os.path.join(ROOT, "tests", "native", "hypotheses_args.cpp")])
        L = C.CDLL(out)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    dp = C.POINTER(C.c_double)
    L.hyp_check.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, dp, C.c_int, C.c_double, C.c_int, C.c_int,
                            C.c_char_p, C.c_int]
    L.hyp_score.argtypes = [C.c_int, C.c_longlong, C.c_longlong, C.c_double, C.c_double]
    L.hyp_score.restype = C.c_double
    L.hyp_pick.argtypes = [dp, C.c_int]
    return L


def _eye(n, k):
    return np.tile(np.eye(4), (n, k, 1, 1))


@pytest.fixture(scope="module")
def check(lib):
    def run(H=None, n=None, k=None, first=4, last=0, use_init=1, screen=3, ratio=0.0, has_cfg=True, results=True, best=True):
        if H is not None:
            H = np.ascontiguousarray(np.asarray(H, dtype=np.float64))
            n = H.shape[0] if n is None else n
            k = H.shape[1] if k is None else k
        buf = C.create_string_buffer(256)
        p = H.ctypes.data_as(C.POINTER(C.c_double)) if H is not None else None
        lib.hyp_check(int(has_cfg), first, last, use_init, 1 if n is None else n, 1 if k is None else k, p, screen, ratio,
                      int(results), int(best), buf, 256)
        return buf.value.decode()
    return run


def test_refusals_each_with_its_message(check):
    H = _eye(2, 3)
    assert check(None, n=2, k=3) == "match_batch_hypotheses: hypotheses is null"
    assert check(H, results=False) == "match_batch_hypotheses: results is null"
    assert check(H, best=False) == "match_batch_hypotheses: best is null"
    assert check(_eye(1, 1), k=0) == "match_batch_hypotheses: k = 0 outside [1, 64]"
    assert check(_eye(1, 65)) == "match_batch_hypotheses: k = 65 outside [1, 64]"
    assert check(_eye(1, 1), k=-3) == "match_batch_hypotheses: k = -3 outside [1, 64]"
    assert check(H, use_init=0) == "match_batch_hypotheses: cfg->use_initial_estimate must be 1: the hypotheses are the initial estimates"
    assert check(H, screen=5) == "match_batch_hypotheses: screen_level = 5 outside [last_level, first_level] = [0, 4]"
    assert check(H, first=3, last=1, screen=0) == "match_batch_hypotheses: screen_level = 0 outside [last_level, first_level] = [1, 3]"
    for r in (NAN, math.inf, -math.inf, -1e-12, 1.0 + 1e-12, 2.0):
        assert check(H, ratio=r) == "match_batch_hypotheses: min_constraint_ratio is not a finite value in [0, 1]", r
    for bad in (NAN, math.inf, -math.inf):
        B = H.copy()
        B[1, 2, 0, 3] = bad
        assert check(B) == "match_batch_hypotheses: hypothesis 2 of pair 1 is not finite"
    for row in ((1e-300, 0, 0, 1), (0, 0, 0, 0.5), (0, -0.0, 1e-9, 1), (0, 0, 0, 2)):
        B = H.copy()
        B[0, 1, 3] = row
        want = "match_batch_hypotheses: hypothesis 1 of pair 0 has a bottom row other than (0, 0, 0, 1)"
        assert check(B) == want, row


def test_order_of_the_refusals(check):
    # the null pointers first, then k, then the config, then the ratio, then the matrices
    bad = _eye(1, 2)
    bad[0, 0, 0, 0] = NAN
    assert "hypotheses is null" in check(None, n=1, k=0, results=False)
    assert "results is null" in check(bad, k=0, results=False, best=False)
    assert "k = 0" in check(bad, k=0, use_init=0)
    assert "use_initial_estimate" in check(bad, use_init=0, screen=9, ratio=NAN)
    assert "screen_level" in check(bad, screen=9, ratio=NAN)
    assert "min_constraint_ratio" in check(bad, ratio=NAN)
    assert "is not finite" in check(bad)


def test_null_cfg_and_empty_batch_are_left_to_the_batch_checks(check):
    assert check(_eye(1, 2), has_cfg=False, use_init=0, screen=99) == ""
    bad = _eye(1, 1)
    bad[0, 0, 3, 3] = 0.0
    assert check(bad, n=0) == ""
    assert check(bad, n=-1) == ""


def test_valid_edge_cases(check):
    rng = np.random.default_rng(0)
    from dvo_slam_b200 import synth
    H = np.stack([np.stack([synth.se3_exp(rng.normal(scale=0.3, size=6)) for _ in range(64)]) for _ in range(2)])
    assert check(H[:, :1]) == ""                       # k = 1
    assert check(H) == ""                              # k = 64
    for screen in (4, 0):                              # screen_level at first_level and at last_level
        assert check(H, screen=screen) == ""
    assert check(H, first=2, last=2, screen=2) == ""   # one level: screening only
    for r in (0.0, 1.0, 0.5):                          # ratios 0 and 1 are inside
        assert check(H, ratio=r) == ""
    B = H.copy()
    B[:, :, 3, :3] = -0.0                              # -0 in the bottom row is 0
    assert check(B) == ""


# ---- the selection rule -------------------------------------------------------------------------------------------------
def _level(has=True, n=1000, vp=2000, nll=1500.0):
    return {"has_iteration_with_increment": has, "last_increment_valid_constraints": n, "valid_pixels": vp,
            "last_increment_log_likelihood": nll}


def _score(lib, l, r):
    return lib.hyp_score(int(l["has_iteration_with_increment"]), l["last_increment_valid_constraints"], l["valid_pixels"],
                         l["last_increment_log_likelihood"], r)


def _same(a, b):
    return (math.isnan(a) and math.isnan(b)) or a == b


def _pick(lib, scores):
    a = np.ascontiguousarray(scores, dtype=np.float64)
    return lib.hyp_pick(a.ctypes.data_as(C.POINTER(C.c_double)), len(a))


CASES = [
    (_level(), 0.0),
    (_level(), 0.5),                                   # ratio exactly at the threshold: eligible
    (_level(n=999), 0.5),                              # just below it
    (_level(n=1, vp=3), 1.0 / 3.0),                    # at a threshold that is not exact in binary
    (_level(n=2, vp=3), 2.0 / 3.0),
    (_level(vp=1000), 1.0),                            # every selected point a constraint, ratio 1
    (_level(has=False, n=-1, nll=NAN), 0.0),           # no iteration with an increment
    (_level(has=False), 0.0),                          # the flag decides, not the fields
    (_level(nll=NAN), 0.0),                            # NaN log-likelihood
    (_level(nll=math.inf), 0.0),
    (_level(nll=-math.inf), 0.0),
    (_level(n=0, nll=0.0), 0.0),                       # zero constraints (TooFewConstraints): 0 / 0
    (_level(n=0, nll=5.0), 0.0),                       # x / 0 = inf
    (_level(n=3, nll=0.0), 0.0),                       # TooFewConstraints with a few constraints: score 0
    (_level(n=5, vp=0), 0.0),                          # no selected pixel: the ratio is inf
    (_level(n=0, vp=0, nll=0.0), 0.0),                 # 0 / 0 ratio
    (_level(nll=-1500.0), 0.0),                        # negative scores compare like any other
    (_level(nll=1e308, n=1), 0.0),
    (_level(nll=1e308, n=3, vp=3), 0.0),
]


@pytest.mark.parametrize("level,ratio", CASES)
def test_score_matches_the_definition(lib, level, ratio):
    assert _same(_score(lib, level, ratio), hm.score(level, ratio))


def test_score_values(lib):
    assert _score(lib, _level(), 0.5) == 1.5
    assert math.isnan(_score(lib, _level(n=999), 0.5))
    assert _score(lib, _level(n=1, vp=3), 1.0 / 3.0) == 1500.0
    assert _score(lib, _level(n=3, nll=0.0), 0.0) == 0.0
    for l in (_level(has=False), _level(nll=NAN), _level(n=0, nll=0.0), _level(nll=math.inf)):
        assert math.isnan(_score(lib, l, 0.0))


@pytest.mark.parametrize("scores,want", [
    ([3.0, 1.0, 2.0], 1),
    ([1.0, 1.0, 1.0], 0),                              # ties: the lowest index
    ([2.0, 1.0, 1.0], 1),
    ([NAN, 1.0, NAN, 1.0], 1),
    ([NAN, NAN, NAN], 0),                              # none eligible
    ([NAN], 0),
    ([5.0], 0),
    ([0.0, -0.0], 0),                                  # -0 == 0: a tie
    ([-0.0, 0.0], 0),
    ([1.0, NAN, 0.5], 2),
])
def test_pick(lib, scores, want):
    assert _pick(lib, scores) == want == hm.pick(scores)


def test_random_batches_against_the_restatement(lib):
    rng = np.random.default_rng(7)
    for trial in range(400):
        k = int(rng.integers(1, 65))
        levels = []
        for j in range(k):
            vp = int(rng.choice([0, 1, 7, 1000, 76800]))
            n = int(rng.integers(0, vp + 1)) if vp else int(rng.integers(0, 3))
            nll = float(rng.choice([NAN, math.inf, 0.0, rng.uniform(-2, 2) * n, float(rng.integers(1, 4)) * n]))
            levels.append(_level(has=bool(rng.random() < 0.85), n=n, vp=vp, nll=nll))
        r = float(rng.choice([0.0, 1.0, 0.25, rng.random()]))
        got = [_score(lib, l, r) for l in levels]
        want = [hm.score(l, r) for l in levels]
        assert all(_same(a, b) for a, b in zip(got, want)), trial
        assert _pick(lib, got) == hm.pick(want), trial
        if all(math.isnan(s) for s in got):
            assert _pick(lib, got) == 0
