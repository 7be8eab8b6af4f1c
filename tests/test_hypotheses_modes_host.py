"""Multi-hypothesis alignment in the photometric mode, with motion priors and with weight maps, without a GPU: the argument
checks of dvo_b200_match_batch_hypotheses_modes (csrc/hypotheses_args.h) built for the host with a fake in place of
cudaPointerGetAttributes, each refusal with its message and hypothesis index and the order of the refusals; and the score and
pick rules, unchanged by the modes, on level statistics of photometric and prior alignments."""
import ctypes as C
import math
import os
import shutil
import subprocess
import tempfile

import numpy as np
import pytest

import hypotheses_model as hm
from dvo_slam_b200.engine import MAPS_MEMORY, MapPlane, WeightMaps

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAN = float("nan")
FN = "match_batch_hypotheses: "
DEV, REGION = 0x10000000, 0x10000000          # the fake's device memory
N, K = 2, 3
LW, LH, W0, H0 = 160, 120, 320, 240   # the maps' extents: level L and level 0


@pytest.fixture(scope="module")
def lib():
    tmp = tempfile.mkdtemp(prefix="dvo_hypotheses_modes_args_")
    try:
        out = os.path.join(tmp, "libhypotheses_modes_args.so")
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-Wall", "-fPIC", "-shared", "-I", os.path.join(ROOT, "dvo_slam_b200", "csrc"),
                               "-o", out, os.path.join(ROOT, "tests", "native", "hypotheses_modes_args.cpp")])
        L = C.CDLL(out)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    dp = C.POINTER(C.c_double)
    L.hm_check.argtypes = [C.c_int, C.c_int, C.c_int, C.c_double, C.c_int, C.c_int, dp, C.c_int, C.c_double, dp, dp, C.c_int, C.c_int,
                           C.POINTER(WeightMaps), C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_longlong, C.c_longlong, C.c_char_p,
                           C.c_int]
    return L


def _eye(n=N, k=K):
    return np.tile(np.eye(4), (n, k, 1, 1))


def _spd(seed):
    M = np.random.default_rng(seed).normal(size=(6, 6)) * 30.0
    L = M @ M.T
    return 0.5 * (L + L.T)


def _lam(n=N, k=K):
    return np.stack([np.stack([_spd(p * k + j) if j else np.zeros((6, 6)) for j in range(k)]) for p in range(n)])


def _ab0(n=N, k=K):
    return np.tile([1.05, -3.0], (n, k, 1))


def _maps(memory="device", mask_weight=0.3, base=DEV):
    m = WeightMaps()
    m.memory = MAPS_MEMORY[memory] if isinstance(memory, str) else memory
    m.weight = MapPlane(base, 4 * LW, 4 * LW * LH)
    m.mask = MapPlane(base + 0x1000000, W0, W0 * H0)
    m.mask_weight = mask_weight
    return m


@pytest.fixture(scope="module")
def check(lib):
    def run(H=None, n=N, k=K, first=3, last=0, mu=0.0, screen=2, ratio=0.0, lam=None, ab0=None, photometric=False,
            screen_photometric=False, maps=None, has_cfg=True, extent=True):
        H = _eye(n, k) if H is None else H
        dp = C.POINTER(C.c_double)
        arr = lambda a: None if a is None else np.ascontiguousarray(a, dtype=np.float64)
        H, lam, ab0 = arr(H), arr(lam), arr(ab0)
        ptr = lambda a: None if a is None else a.ctypes.data_as(dp)
        buf = C.create_string_buffer(512)
        lib.hm_check(int(has_cfg), first, last, mu, n, k, ptr(H), screen, ratio, ptr(lam), ptr(ab0), int(photometric),
                     int(screen_photometric), C.byref(maps) if maps is not None else None, int(extent), LW, LH, W0, H0,
                     DEV, DEV + REGION, buf, 512)
        return buf.value.decode()
    return run


def test_valid_calls_pass(check):
    assert check() == ""
    assert check(lam=_lam()) == ""
    assert check(photometric=True, ab0=_ab0(), screen_photometric=True) == ""
    assert check(lam=_lam(), ab0=_ab0(), photometric=True, screen_photometric=True, maps=_maps()) == ""
    assert check(lam=np.zeros((N, K, 6, 6)), maps=_maps(), screen=0) == ""          # Lambda = 0, s = last_level
    assert check(photometric=True) == ""                                           # (alpha, beta)_0 = (1, 0) each


def test_the_hypotheses_checks_come_first_and_are_unchanged(check):
    bad = _eye()
    bad[1, 2, 0, 0] = NAN
    assert check(bad, lam=_lam(), ab0=_ab0(), maps=_maps(memory=7)) == FN + "hypothesis 2 of pair 1 is not finite"
    assert check(k=65, H=_eye(N, 65), ab0=_ab0(N, 65)) == FN + "k = 65 outside [1, 64]"
    assert check(screen=5, lam=_lam(), mu=1.0) == FN + "screen_level = 5 outside [last_level, first_level] = [0, 3]"
    assert check(ratio=2.0, ab0=_ab0()) == FN + "min_constraint_ratio is not a finite value in [0, 1]"


def test_photometric_outputs_and_inputs(check):
    assert check(ab0=_ab0()) == FN + "photometric_init without photometric"
    assert check(screen_photometric=True) == FN + "screen_photometric without photometric"
    for p, j in ((0, 0), (1, 2), (0, 1)):
        for bad in (NAN, math.inf, -math.inf):
            for c in (0, 1):
                ab0 = _ab0()
                ab0[p, j, c] = bad
                assert check(photometric=True, ab0=ab0) == FN + f"photometric_init of hypothesis {j} of pair {p} is not finite"


def test_prior_refusals_name_the_hypothesis(check):
    assert check(lam=_lam(), mu=0.5) == FN + "cfg->mu must be 0: the prior replaces mu I"
    cases = []
    L = _lam(); L[1, 1, 2, 4] += 1.0
    cases.append((L, "prior_information of hypothesis 1 of pair 1 is not symmetric"))
    L = _lam(); L[0, 2, 5, 5] = NAN
    cases.append((L, "prior_information of hypothesis 2 of pair 0 is not finite"))
    L = _lam(); L[1, 0] = -np.eye(6)
    cases.append((L, "prior_information of hypothesis 0 of pair 1 is not positive semi-definite"))
    L = _lam(); L[0, 1, 0, 0] = math.inf
    cases.append((L, "prior_information of hypothesis 1 of pair 0 is not finite"))
    for lam, want in cases:
        assert check(lam=lam) == FN + want
    # rank-deficient and tiny negative eigenvalues inside the tolerance are accepted, as by dvo_b200_match_batch_prior
    L = _lam(); L[0, 1] = np.diag([1e4, 0, 0, 0, 0, 0])
    assert check(lam=L) == ""


def test_maps_refusals_under_this_call_s_prefix(check):
    assert check(maps=_maps(memory=7)) == FN + "unknown memory 7"
    empty = WeightMaps()
    assert check(maps=empty) == FN + "no output requested"
    assert check(maps=_maps(mask_weight=0.0)) == FN + "mask_weight must be finite and > 0"
    assert check(maps=_maps(mask_weight=NAN)) == FN + "mask_weight must be finite and > 0"
    assert check(maps=_maps(base=0x70000000)) == FN + "weight is not device or managed memory of device 0"
    assert check(maps=_maps(memory="host")) == FN + "weight lies in device memory"
    short = _maps()
    short.weight = MapPlane(DEV, 4 * LW - 4, 4 * LW * LH)
    assert check(maps=short).startswith(FN + "weight.row_bytes 636 is below 160 x 4")
    # a batch the match would refuse: the maps are checked as for n = 0 (the pointers are not looked at)
    assert check(maps=_maps(base=0x70000000), extent=False) == ""
    assert check(maps=_maps(memory=7), extent=False) == FN + "unknown memory 7"


def test_order_of_the_mode_refusals(check):
    """the header's order: photometric_init / screen_photometric without photometric, mu, each Lambda, each (alpha, beta)_0,
    then the maps"""
    bad_lam = _lam(); bad_lam[0, 1, 0, 1] += 1.0
    bad_ab = _ab0(); bad_ab[0, 0, 0] = NAN
    bad_maps = _maps(memory=7)
    assert "photometric_init without photometric" in check(ab0=bad_ab, screen_photometric=True, lam=bad_lam, mu=1.0, maps=bad_maps)
    assert "screen_photometric without photometric" in check(screen_photometric=True, lam=bad_lam, mu=1.0, maps=bad_maps)
    assert "cfg->mu must be 0" in check(lam=bad_lam, mu=1.0, photometric=True, ab0=bad_ab, maps=bad_maps)
    assert "prior_information of hypothesis 1 of pair 0" in check(lam=bad_lam, photometric=True, ab0=bad_ab, maps=bad_maps)
    assert "photometric_init of hypothesis 0 of pair 0" in check(lam=_lam(), photometric=True, ab0=bad_ab, maps=bad_maps)
    assert "unknown memory 7" in check(lam=_lam(), photometric=True, ab0=_ab0(), maps=bad_maps)
    # the first bad hypothesis in (p, j) order is the one named
    two = _lam(); two[1, 0, 0, 1] += 1.0; two[0, 2, 0, 1] += 1.0
    assert check(lam=two) == FN + "prior_information of hypothesis 2 of pair 0 is not symmetric"


def test_null_cfg_and_empty_batch_are_left_to_the_batch_checks(check):
    bad_lam = _lam(); bad_lam[0, 1, 0, 1] += 1.0
    assert check(has_cfg=False, lam=bad_lam) == ""        # as dvo_b200_match_batch_prior: the cfg check refuses first
    assert check(n=0, lam=bad_lam, photometric=True, ab0=_ab0()[:0]) == ""


# ---- the score and the pick, unchanged by the modes --------------------------------------------------------------------
@pytest.fixture(scope="module")
def rules():
    tmp = tempfile.mkdtemp(prefix="dvo_hypotheses_args_")
    try:
        out = os.path.join(tmp, "libhypotheses_args.so")
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-Wall", "-fPIC", "-shared", "-I", os.path.join(ROOT, "dvo_slam_b200", "csrc"),
                               "-o", out, os.path.join(ROOT, "tests", "native", "hypotheses_args.cpp")])
        L = C.CDLL(out)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    L.hyp_score.argtypes = [C.c_int, C.c_longlong, C.c_longlong, C.c_double, C.c_double]
    L.hyp_score.restype = C.c_double
    L.hyp_pick.argtypes = [C.POINTER(C.c_double), C.c_int]
    return L


def _score(L, level, ratio):
    return L.hyp_score(int(level["has_iteration_with_increment"]), level["last_increment_valid_constraints"], level["valid_pixels"],
                       level["last_increment_log_likelihood"], ratio)


def _pick(L, scores):
    a = np.ascontiguousarray(scores, dtype=np.float64)
    return L.hyp_pick(a.ctypes.data_as(C.POINTER(C.c_double)), len(a))


def test_a_hypothesis_s_own_prior_does_not_make_it_win(rules):
    """The level statistics of a prior alignment: last_increment_log_likelihood is the data term alone (the level kernel's
    nll), the prior term li^T Lambda li only enters Result.log_likelihood.  Hypothesis 0 has the better data term and a large
    prior term, hypothesis 1 the better total: the score and the pick follow the data term."""
    data = [1200.0, 1500.0]
    prior = [900.0, 0.0]
    levels = [{"has_iteration_with_increment": True, "last_increment_valid_constraints": 1000, "valid_pixels": 1800,
               "last_increment_log_likelihood": d} for d in data]
    scores = [_score(rules, l, 0.3) for l in levels]
    assert scores == [hm.score(l, 0.3) for l in levels] == [1.2, 1.5]
    assert _pick(rules, scores) == hm.pick(scores) == 0
    totals = [(d + q) / 1000 for d, q in zip(data, prior)]
    assert np.argmin(totals) == 1                     # a score with the prior would pick the other one


def test_photometric_level_statistics_score_as_any_other(rules):
    """The photometric mode changes the residuals, not the statistics the rule reads: random level statistics with the spread
    an exposure change gives (more or fewer constraints, a larger nll) score and pick as the restatement says."""
    rng = np.random.default_rng(11)
    for trial in range(200):
        k = int(rng.integers(1, 9))
        levels = []
        for _ in range(k):
            vp = int(rng.integers(500, 4800))
            n = int(rng.integers(0, vp + 1))
            nll = float(rng.choice([NAN, rng.uniform(0.5, 4.0) * n, rng.uniform(-1.0, 0.0) * n]))
            levels.append({"has_iteration_with_increment": bool(rng.random() < 0.9), "last_increment_valid_constraints": n,
                           "valid_pixels": vp, "last_increment_log_likelihood": nll})
        r = float(rng.choice([0.0, 0.3, 0.6]))
        got = [_score(rules, l, r) for l in levels]
        want = [hm.score(l, r) for l in levels]
        assert all((math.isnan(a) and math.isnan(b)) or a == b for a, b in zip(got, want)), trial
        assert _pick(rules, got) == hm.pick(want), trial
