"""Multi-hypothesis alignment on the GPU (dvo_b200_match_batch_hypotheses): k = 1 is dvo_b200_match_batch; the continued
result is the single alignment from the chosen hypothesis and the screening results those of the screening levels alone, bit
for bit, under both estimators; scores and choice follow the rule of tests/hypotheses_model.py; batch position, batch size and
launch plan change nothing; masks and mixed intrinsics; a large rotation that the identity start gets wrong and a near
hypothesis gets right; refusals before any upload or launch; the C++ adapter."""
import ctypes as C
import json
import os
import subprocess

import numpy as np
import pytest

import hypotheses_model as hm
from dvo_slam_b200 import synth
from dvo_slam_b200.engine import CResult, Config

pytestmark = pytest.mark.gpu
SCENE = synth.SceneConfig(width=320, height=240, intrinsics=tuple(v / 2 for v in synth.FR1_INTRINSICS))
DELTA = np.array([4e-3, -3e-3, 2e-3, -2e-3, 3e-3, 1e-3])
FIRST, LAST = 2, 0


def _cfg(first=FIRST, last=LAST, **kw):
    kw = {"use_initial_estimate": 1, **kw}
    return Config(first_level=first, last_level=last, max_iterations_per_level=50, precision=1e-4, **kw)


def _mask(k):
    m = np.ones((240, 320), np.uint8)
    m[40 + 10 * k:110 + 10 * k, 60:150] = 0
    return m


def _hypotheses(p, k, i):
    """k poses for pair p (reference -> current, as T_init): the identity, a near start, a far start and decoys"""
    T = p["T_true"]
    out = [np.eye(4), synth.se3_exp(DELTA * (1 + 0.3 * i)) @ T, synth.se3_exp(6 * DELTA) @ T,
           synth.se3_exp(np.array([0.05, -0.04, 0.0, 0.2, -0.15, 0.1])) @ T]
    rng = np.random.default_rng(100 + i)
    while len(out) < k:
        out.append(synth.se3_exp(rng.normal(scale=[0.01] * 3 + [0.02] * 3)) @ T)
    return np.stack(out[:k])


@pytest.fixture(scope="module")
def batch(engine):
    """six 320 x 240 pairs, 3 levels"""
    out = []
    for i in range(6):
        p = synth.make_pair(80 + i, SCENE)
        out.append({"ref": engine.pyramid(p["I_ref"].numpy(), p["Z_ref"].numpy(), SCENE.intrinsics, 3),
                    "cur": engine.pyramid(p["I_cur"].numpy(), p["Z_cur"].numpy(), SCENE.intrinsics, 3), "pair": p})
    return out


def _eq(a, b):
    return np.array_equal(np.asarray(a), np.asarray(b), equal_nan=True)


def _same(r0, r1, iterations=True):
    """every field of two Results bit for bit (NaN == NaN), the iteration logs too"""
    if not (_eq(r0.transformation, r1.transformation) and _eq(r0.information, r1.information)):
        return False
    if r0.num_iterations_total != r1.num_iterations_total or len(r0.levels) != len(r1.levels):
        return False
    if not (r0.log_likelihood == r1.log_likelihood or (r0.log_likelihood != r0.log_likelihood and r1.log_likelihood != r1.log_likelihood)):
        return False
    for a, b in zip(r0.levels, r1.levels):
        if a.keys() != b.keys() or not all(a[k] == b[k] or (a[k] != a[k] and b[k] != b[k]) for k in a):
            return False
    if not iterations:
        return True
    if len(r0.iterations) != len(r1.iterations):
        return False
    for x, y in zip(r0.iterations, r1.iterations):
        for k in ("level", "id", "n", "nll", "precision", "prior", "x", "A"):
            if not _eq(x[k], y[k]):
                return False
    return True


def _check_call(engine, refs, curs, H, s, ratio, cfg):
    """one call against its definition: the continued results (with their logs), the screening results, scores and best"""
    n, k = H.shape[:2]
    res, best, scores, screen = engine.match_batch_hypotheses(refs, curs, H, s, ratio, cfg, with_iterations=True, screen_results=True)
    cfg_s = _cfg(cfg.first_level, s, mu=cfg.mu)
    want_screen = engine.match_batch([r for r in refs for _ in range(k)], [c for c in curs for _ in range(k)], cfg_s,
                                     H.reshape(n * k, 4, 4))
    for p in range(n):
        want_scores = [hm.score(want_screen[p * k + j].levels[-1], ratio) for j in range(k)]
        assert _eq(scores[p], want_scores), (p, scores[p], want_scores)
        assert best[p] == hm.pick(want_scores), p
        for j in range(k):
            assert _same(screen[p][j], want_screen[p * k + j], iterations=False), (p, j)
        single = engine.match_batch([refs[p]], [curs[p]], cfg, [H[p, best[p]]], with_iterations=True)[0]
        assert _same(res[p], single), p
        assert res[p].iterations and len(res[p].levels) == cfg.first_level - cfg.last_level + 1
    return res, best, scores


@pytest.mark.parametrize("estimator", ["reference", "corrected"])
def test_one_hypothesis_is_match_batch(engine, batch, estimator):
    refs, curs = [q["ref"] for q in batch], [q["cur"] for q in batch]
    H = np.stack([_hypotheses(q["pair"], 2, i)[1:2] for i, q in enumerate(batch)])
    engine.set_estimator(estimator)
    try:
        want = engine.match_batch(refs, curs, _cfg(), H[:, 0], with_iterations=True)
        for s in (FIRST, FIRST - 1, LAST):
            res, best, scores = engine.match_batch_hypotheses(refs, curs, H, s, 0.0, _cfg(), with_iterations=True)
            assert np.array_equal(best, np.zeros(len(refs))) and scores.shape == (len(refs), 1)
            for p in range(len(refs)):
                assert _same(res[p], want[p]), (s, p)
    finally:
        engine.set_estimator("reference")


@pytest.mark.parametrize("estimator", ["reference", "corrected"])
@pytest.mark.parametrize("s,ratio", [(FIRST, 0.0), (FIRST - 1, 0.5), (LAST, 0.6)])
def test_continuation_equals_the_single_alignment_from_the_chosen_hypothesis(engine, batch, estimator, s, ratio):
    refs, curs = [q["ref"] for q in batch], [q["cur"] for q in batch]
    H = np.stack([_hypotheses(q["pair"], 4, i) for i, q in enumerate(batch)])
    engine.set_estimator(estimator)
    try:
        _check_call(engine, refs, curs, H, s, ratio, _cfg())
        # cfg->mu carries over
        _check_call(engine, refs[:3], curs[:3], H[:3], s, ratio, _cfg(mu=0.05))
    finally:
        engine.set_estimator("reference")


def test_plan_and_batch_position_change_nothing(engine, batch, monkeypatch):
    k, s = 8, FIRST - 1
    H = np.stack([_hypotheses(q["pair"], k, i) for i, q in enumerate(batch)])
    single = [engine.match_batch_hypotheses([q["ref"]], [q["cur"]], H[i:i + 1], s, 0.3, _cfg(), with_iterations=True)
              for i, q in enumerate(batch)]
    big = 512
    idx = [i % len(batch) for i in range(big)]
    idx[511] = 0
    refs, curs = [batch[i]["ref"] for i in idx], [batch[i]["cur"] for i in idx]
    for knob, value in ((None, None), ("DVO_B200_NO_WALK", "1"), ("DVO_B200_FINE_G", "2"), ("DVO_B200_NO_FUSE", "1")):
        if knob:
            monkeypatch.setenv(knob, value)
        for order in (1, -1):
            o = list(range(big))[::order]
            res, best, scores = engine.match_batch_hypotheses([refs[i] for i in o], [curs[i] for i in o], H[[idx[i] for i in o]], s,
                                                              0.3, _cfg(), with_iterations=(knob is None))
            for pos, i in enumerate(o):
                r1, b1, s1 = single[idx[i]]
                assert best[pos] == b1[0] and _eq(scores[pos], s1[0]), (knob, order, i)
                assert _same(res[pos], r1[0], iterations=(knob is None)), (knob, order, i)
        if knob:
            monkeypatch.delenv(knob)


@pytest.mark.parametrize("estimator", ["reference", "corrected"])
def test_masks_and_mixed_intrinsics(engine, estimator):
    other = synth.SceneConfig(width=320, height=240, intrinsics=(287.0, 291.5, 161.0, 118.5))
    pyr, H = [], []
    for i, (scene, kw) in enumerate(((SCENE, {}), (SCENE, {"mask": _mask(1), "mask_roles": "reference"}),
                                     (SCENE, {"mask": _mask(2), "mask_roles": "both"}), (other, {}),
                                     (other, {"mask": _mask(4), "mask_roles": "both"}))):
        p = synth.make_pair(90 + i, scene)
        pyr.append((engine.pyramid(p["I_ref"].numpy(), p["Z_ref"].numpy(), scene.intrinsics, 3, **kw),
                    engine.pyramid(p["I_cur"].numpy(), p["Z_cur"].numpy(), scene.intrinsics, 3, **kw)))
        H.append(_hypotheses(p, 3, i))
    engine.set_estimator(estimator)
    try:
        for s, ratio in ((FIRST - 1, 0.4), (FIRST, 0.0)):
            _check_call(engine, [a for a, _ in pyr], [b for _, b in pyr], np.stack(H), s, ratio, _cfg())
    finally:
        engine.set_estimator("reference")


# A fast rotation: seed 0 of this scene turns by about 0.2 rad per axis.  The identity start converges to a wrong pose (the
# premise, checked below); the true pose perturbed by NEAR converges to the right one.
WIDE = synth.SceneConfig(width=320, height=240, intrinsics=tuple(v / 2 for v in synth.FR1_INTRINSICS), max_rotation=0.2,
                         max_translation=0.05)
NEAR = np.array([0.01, -0.008, 0.006, 0.02, -0.015, 0.01])
WRONG_MARGIN = 0.05                # rad: the identity start ends at least this far from the true rotation
TOL_T, TOL_R = 5e-3, 2e-3          # m, rad: the chosen hypothesis's final pose


def _pose_err(T, T_true):
    """translation and rotation norms of the error of Result.transformation T, which estimates T_true^-1"""
    d = synth.se3_log(T_true @ T)
    return np.linalg.norm(d[:3]), np.linalg.norm(d[3:])


@pytest.mark.parametrize("estimator", ["reference", "corrected"])
def test_the_near_hypothesis_wins_where_the_identity_fails(engine, estimator):
    p = synth.make_pair(0, WIDE)
    T = p["T_true"]
    ref = engine.pyramid(p["I_ref"].numpy(), p["Z_ref"].numpy(), WIDE.intrinsics, 3)
    cur = engine.pyramid(p["I_cur"].numpy(), p["Z_cur"].numpy(), WIDE.intrinsics, 3)
    decoys = [synth.se3_exp(np.array([0.0, 0.0, 0.0, 0.35, -0.3, 0.25])) @ T, np.linalg.inv(T)]
    H = np.stack([np.eye(4), synth.se3_exp(NEAR) @ T] + decoys)[None]
    engine.set_estimator(estimator)
    try:
        plain = engine.match(ref, cur, _cfg(), np.eye(4))
        assert _pose_err(plain.transformation, T)[1] > WRONG_MARGIN, _pose_err(plain.transformation, T)
        for s in (FIRST, FIRST - 1):
            res, best, scores = engine.match_batch_hypotheses([ref], [cur], H, s, 0.3, _cfg())
            assert best[0] == 1, scores
            dt, dr = _pose_err(res[0].transformation, T)
            assert dt < TOL_T and dr < TOL_R, (dt, dr)
    finally:
        engine.set_estimator("reference")


def test_refusals_move_no_counters(engine, batch):
    q = batch[0]
    engine.synchronize()
    L, ctx = engine.lib, engine.ctx
    h0, k0 = engine.h2d_bytes(), engine.kernel_launches()
    rh, ch = (C.c_void_p * 1)(q["ref"].handle), (C.c_void_p * 1)(q["cur"].handle)
    res, scr = (CResult * 1)(), (CResult * 64)()
    best = (C.c_int32 * 1)()
    sc = (C.c_double * 64)()
    dp = C.POINTER(C.c_double)
    H = np.tile(np.eye(4), (65, 1, 1))
    P = lambda a: np.ascontiguousarray(a, dtype=np.float64).ctypes.data_as(dp)
    nan, row = H.copy(), H.copy()
    nan[0, 1, 1] = np.nan
    row[0, 3, 3] = 1.5

    def call(cfg=None, n=1, k=2, h=H, s=1, ratio=0.0, r=res, b=best, refs=rh):
        return L.dvo_b200_match_batch_hypotheses(ctx, C.byref(cfg or _cfg()), n, refs, ch, k, None if h is None else P(h), s, ratio, r,
                                                 b, sc, scr, None, 0)
    cases = [dict(k=0), dict(k=65), dict(h=None), dict(r=None), dict(b=None), dict(h=nan), dict(h=row), dict(s=3), dict(s=-1),
             dict(ratio=float("nan")), dict(ratio=1.5), dict(cfg=_cfg(use_initial_estimate=0)),
             dict(cfg=Config(first_level=0, last_level=1, use_initial_estimate=1), s=0), dict(n=0),
             dict(cfg=_cfg(first=3), s=3), dict(refs=(C.c_void_p * 1)(None))]
    for kw in cases:
        assert call(**kw) == -1, kw    # DVO_B200_ERR_INVALID_ARGUMENT
        assert engine.lib.dvo_b200_last_error(ctx), kw
    assert engine.h2d_bytes() == h0 and engine.kernel_launches() == k0
    assert call() == 0 and engine.kernel_launches() > k0


def test_cpp_adapter(engine, tmp_path):
    """DenseTracker::matchWithHypotheses: the pose and index of Engine.match_batch_hypotheses, and false on a refusal; the
    overload with one prior per start and a weight map: the pose, index and weight map of the same call with
    prior_information and maps"""
    from helpers import nan_equal
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    lib = os.path.join(root, "dvo_slam_b200")
    exe = str(tmp_path / "hypotheses_adapter")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-I", os.path.join(root, "include"), "-o", exe,
                           os.path.join(root, "tests", "native", "hypotheses_adapter.cpp"), "-L" + lib, "-ldvo_core_b200", "-ldvo_b200",
                           "-Wl,-rpath," + lib])
    scene = synth.SceneConfig(max_rotation=0.1, max_translation=0.05)
    pair = synth.make_pair(5, scene)
    K = pair["intrinsics"]
    path = tmp_path / "pair.bin"
    with open(path, "wb") as f:
        for k in ("I_ref", "Z_ref", "I_cur", "Z_cur"):
            f.write(np.ascontiguousarray(pair[k].numpy(), dtype=np.float32).tobytes())
    H = _hypotheses(pair, 4, 0)
    hpath = tmp_path / "hypotheses.bin"
    np.ascontiguousarray(H, dtype=np.float64).tofile(hpath)
    rng = np.random.default_rng(11)
    lam = np.stack([0.5 * (S + S.T) for S in ((M @ M.T + 0.5 * np.eye(6)) * 10.0 ** rng.uniform(6, 9)
                                              for M in rng.standard_normal((4, 6, 6)))])
    lpath, wpath = tmp_path / "priors.bin", str(tmp_path / "weights.bin")
    lam.tofile(lpath)
    r = subprocess.run([exe, str(path), "640", "480"] + [repr(float(v)) for v in K] + [str(hpath), "4", str(lpath), wpath],
                       capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    out = json.loads(r.stdout.strip().splitlines()[-1])
    assert out["ok"] == 1 and out["refused_ok"] == 0 and out["refused_best"] == -1 and out["levels"] == 3
    refs = [engine.pyramid(pair["I_ref"].numpy(), pair["Z_ref"].numpy(), K, 4)]
    curs = [engine.pyramid(pair["I_cur"].numpy(), pair["Z_cur"].numpy(), K, 4)]
    cfg = Config(first_level=3, last_level=1, max_iterations_per_level=50, precision=1e-4, use_initial_estimate=1)
    res, best, _ = engine.match_batch_hypotheses(refs, curs, H[None], 2, 0.0, cfg)
    assert out["best"] == best[0]
    assert np.array_equal(np.array(out["T"]).reshape(4, 4), res[0].transformation)
    res, best, _, maps = engine.match_batch_hypotheses(refs, curs, H[None], 2, 0.0, cfg, prior_information=lam[None], maps=True)
    assert out["prior_ok"] == 1 and out["prior_best"] == best[0]
    assert np.array_equal(np.array(out["prior_T"]).reshape(4, 4), res[0].transformation)
    assert (out["rows"], out["cols"]) == (240, 320)
    weights = np.fromfile(wpath, dtype=np.float32).reshape(240, 320)
    assert nan_equal(weights, maps["weight"][0].cpu().numpy()) and np.isfinite(weights).sum() > 10000
