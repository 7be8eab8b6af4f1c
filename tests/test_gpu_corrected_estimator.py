"""The corrected estimator on the GPU (dvo_b200_set_estimator(ctx, DVO_B200_ESTIMATOR_CORRECTED)) against the oracle's
MIRROR mode with the reference's three structural quirks off (tests/test_corrected_estimator.py pins that definition):
residual records bit-exact including the re-admitted odd last point, counts exact, P / LL / A / b to 2e-6, the generic
pixel loop, whole alignments on the 512 benchmark pairs, determinism across plans, and isolation from reference-mode
contexts that share the pyramids."""
import json
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

from helpers import nan_equal, odd_point_margin, pose_delta
from test_corrected_estimator import corrected_mode
from test_gpu_generic_tiles import partial_pair, partial_pose, _rot_z, _shift_z
from tile_geometry import TILE_H, TILE_W, WIN_ROWS, assert_partial_band

pytestmark = pytest.mark.gpu

PP = np.array([[2000.0, -30.0], [-30.0, 9000.0]], dtype=np.float32)


@pytest.fixture(scope="module")
def corrected(engine):
    from dvo_slam_b200.engine import Engine
    eng = Engine(device=0, estimator="corrected")
    assert eng.estimator == "corrected" and engine.estimator == "reference"
    yield eng
    eng.close()


@pytest.fixture(scope="module")
def pair(engine, oracle):
    from dvo_slam_b200 import synth
    p = synth.make_pair(0)
    a = {k: p[k].numpy() for k in ("I_ref", "Z_ref", "I_cur", "Z_cur")}
    a["K"] = p["intrinsics"]
    a["gref"] = engine.pyramid(a["I_ref"], a["Z_ref"], a["K"], 5)
    a["gcur"] = engine.pyramid(a["I_cur"], a["Z_cur"], a["K"], 5)
    a["oref"] = oracle.Pyramid(a["I_ref"], a["Z_ref"], a["K"], 5)
    a["ocur"] = oracle.Pyramid(a["I_cur"], a["Z_cur"], a["K"], 5)
    return a


@pytest.fixture(scope="module")
def pair720(engine, oracle):
    """the partial-band scene of test_gpu_generic_tiles"""
    a = partial_pair(0)
    a["gref"] = engine.pyramid(a["I_ref"], a["Z_ref"], a["K"], 5)
    a["gcur"] = engine.pyramid(a["I_cur"], a["Z_cur"], a["K"], 5)
    a["oref"] = oracle.Pyramid(a["I_ref"], a["Z_ref"], a["K"], 5)
    a["ocur"] = oracle.Pyramid(a["I_cur"], a["Z_cur"], a["K"], 5)
    return a


def _check_level(eng, oracle, a, lvl, T):
    """records bit-exact, counts exact, P / LL / A / b to 2e-6 (use_weights 0 and 1); returns the oracle's linearisations"""
    m = corrected_mode(oracle)
    n_g, img_g = eng.residual_image(a["gref"], a["gcur"], lvl, T)
    n_o, img_o = oracle.residual_image(a["oref"], a["ocur"], lvl, T, m)
    assert n_g == n_o and n_g > 0 and nan_equal(img_g, img_o), (lvl, n_g, n_o)
    out = []
    for uw in (False, True):
        lg = eng.linearize(a["gref"], a["gcur"], lvl, T, uw, PP)
        lo = oracle.linearize(a["oref"], a["ocur"], lvl, T, m, uw, PP)
        assert lg["n"] == lo["n"] == n_o
        assert np.allclose(lg["precision"], lo["precision"], rtol=2e-6), (lvl, uw, lg["precision"], lo["precision"])
        assert abs(lg["ll"] - lo["ll"]) <= 2e-6 * abs(lo["ll"]) + 0.5, (lvl, uw, lg["ll"], lo["ll"])
        assert np.allclose(lg["A"], lo["A"], rtol=0, atol=2e-6 * np.abs(lo["A"]).max())
        assert np.allclose(lg["b"], lo["b"], rtol=0, atol=2e-6 * np.abs(lo["b"]).max())
        out.append((lg, lo))
    return out


def _pose():
    T = _rot_z(1.5) @ _shift_z(0.015)
    T[0, 3] = 0.01
    return T


@pytest.mark.parametrize("lvl", [0, 1, 2, 3, 4])
def test_records_and_linearisation(engine, corrected, oracle, pair, lvl):
    T = _pose()
    lin = _check_level(corrected, oracle, pair, lvl, T)
    S, _ = pair["gref"].select(lvl)
    n = lin[0][1]["n"]
    if n % 50:
        # the switch takes effect: the reference-mode context drops the last n mod 50 log-likelihood terms (and pairs the scale)
        for uw, (lg, _) in zip((False, True), lin):
            lr = engine.linearize(pair["gref"], pair["gcur"], lvl, T, uw, PP)
            assert lr["ll"] != lg["ll"] and not np.array_equal(lr["precision"], lg["precision"]), (lvl, uw)
    print(f"level {lvl}: S={S} n={n} n%50={n % 50}")


def test_a_level_with_a_log_likelihood_tail(corrected, oracle, pair):
    """at least one of the levels above has n mod 50 != 0, so the tail comparison there is not vacuous"""
    T = _pose()
    ns = [oracle.residual_image(pair["oref"], pair["ocur"], l, T, corrected_mode(oracle))[0] for l in range(5)]
    assert any(n % 50 for n in ns), ns


def test_odd_last_point_is_readmitted(engine, corrected, oracle):
    """The odd-selection case of tests/helpers.py: the corrected kernel gives the odd last point a residual record and an error
    image entry; the reference-mode context sharing the pyramids still drops it."""
    margin, im, oref, ocur = odd_point_margin(oracle)
    from helpers import GOLDEN_SEEDS, load_golden
    K = load_golden(GOLDEN_SEEDS[0])["K"]
    Z = im["Z_ref"].copy()
    Z[-margin:, :] = np.nan
    Z[:, -margin:] = np.nan
    gref = engine.pyramid(im["I_ref"], Z, K, 1)
    gcur = engine.pyramid(im["I_ref"], im["Z_ref"], K, 1)
    S, mask = gref.select(0)
    assert S % 2 == 1
    last = np.flatnonzero(mask.reshape(-1))[-1]
    T = np.eye(4)
    m = corrected_mode(oracle)
    n_c, img_c = corrected.residual_image(gref, gcur, 0, T)
    n_o, img_o = oracle.residual_image(oref, ocur, 0, T, m)
    n_r, img_r = engine.residual_image(gref, gcur, 0, T)
    assert n_c == n_o == n_r + 1 and nan_equal(img_c, img_o)
    assert not np.isnan(img_c[0].reshape(-1)[last]) and np.isnan(img_r[0].reshape(-1)[last])
    ne_c, err_c = corrected.intensity_error_image(gref, gcur, 0, T)
    ne_o, err_o = oracle.intensity_error_image(oref, ocur, 0, T, m)
    assert ne_c == ne_o == n_c and np.array_equal(err_c, err_o) and err_c.reshape(-1)[last] > 0
    for uw in (False, True):
        lg = corrected.linearize(gref, gcur, 0, T, uw, PP)
        lo = oracle.linearize(oref, ocur, 0, T, m, uw, PP)
        assert lg["n"] == lo["n"] == n_c
        assert np.allclose(lg["precision"], lo["precision"], rtol=2e-6)
        assert abs(lg["ll"] - lo["ll"]) <= 2e-6 * abs(lo["ll"]) + 0.5


# ---- the generic pixel loop (the cases of tests/test_gpu_generic_tiles.py) in corrected mode ----
def test_window_too_small(corrected, oracle, pair):
    fx, fy, ox, oy = pair["K"]
    T = _rot_z(20.0)
    h, w = pair["I_ref"].shape
    spans = []
    for y0 in range(0, h - TILE_H + 1, TILE_H):
        for x0 in range(0, w - TILE_W + 1, TILE_W):
            u = np.array([x0, x0 + TILE_W - 1, x0, x0 + TILE_W - 1], dtype=np.float64)
            v = np.array([y0, y0, y0 + TILE_H - 1, y0 + TILE_H - 1], dtype=np.float64)
            q = T[:3, :3] @ np.stack([(u - ox) / fx, (v - oy) / fy, np.ones(4)])
            vv = fy * q[1] / q[2] + oy
            if (vv >= 0).all() and (vv <= h - 1).all():
                spans.append(vv.max() - vv.min())
    assert spans and min(spans) > WIN_ROWS, min(spans)
    _check_level(corrected, oracle, pair, 0, T)


def test_corner_behind_camera(corrected, oracle, pair):
    Z = pair["Z_ref"]
    T = _shift_z(-float(np.nanmedian(Z)))
    zt = Z + T[2, 3]
    finite = np.isfinite(zt)
    assert (zt[finite] < -0.05).any() and (zt[finite] > 0.05).any()
    _check_level(corrected, oracle, pair, 0, T)


@pytest.mark.parametrize("lvl", [1, 2])
def test_partial_band(corrected, oracle, pair720, lvl):
    assert_partial_band(pair720["oref"].level_info(lvl)[0])
    _check_level(corrected, oracle, pair720, lvl, partial_pose())


# ---- whole alignments ----
B = 512
LEVELS, FIRST, LAST = 5, 4, 0
# Bounds from the corrected oracle's own spread between its two arithmetic variants (fused_pixel_math on / off: the kernel's
# operation order vs the reference's unfused order), measured on the CPU on the 512 pairs of seeds 0-511: pose |dt| median
# 1.6e-7 m, p99 5.3e-5 m, max 2.2e-4 m; |dr| max 6.7e-5 rad; identical terminations on every level for 484 / 512 pairs
# (94.5 %), identical terminations and iteration counts for 350 / 512 (68.4 %), iteration counts within +-1 for 453 / 512.
SPREAD_DT_MAX, SPREAD_DR_MAX = 2.2e-4, 6.7e-5
SPREAD_TERM, SPREAD_EXACT = 0.945, 0.684


def _flow(levels):
    return ([l["termination"] for l in levels], [l["num_iterations"] for l in levels])


def _pct(v, q):
    return float(np.percentile(np.asarray(v, dtype=np.float64), q))


@pytest.fixture(scope="module")
def batch(engine):
    import torch
    from dvo_slam_b200 import synth
    dev = torch.device("cuda", 0)
    scfg = synth.SceneConfig()
    K = synth.FR1_INTRINSICS
    H, W = scfg.height, scfg.width
    d = {k: np.empty((B, H, W), np.float32) for k in ("Ir", "Zr", "Ic", "Zc")}
    truth = []
    for i in range(B):                      # the bench's seeds: rank 0 uses seeds 0 .. B-1
        p = synth.make_pair(i, scfg, device=dev)
        d["Ir"][i] = p["I_ref"].cpu().numpy(); d["Zr"][i] = p["Z_ref"].cpu().numpy()
        d["Ic"][i] = p["I_cur"].cpu().numpy(); d["Zc"][i] = p["Z_cur"].cpu().numpy()
        truth.append(np.asarray(p["T_true"]))
    d["K"] = K
    d["truth"] = truth
    d["refs"] = engine.pyramid_batch(d["Ir"], d["Zr"], K, LEVELS)
    d["curs"] = engine.pyramid_batch(d["Ic"], d["Zc"], K, LEVELS)
    return d


def _cfg():
    from dvo_slam_b200.engine import Config
    return Config(first_level=FIRST, last_level=LAST, max_iterations_per_level=50, precision=1e-4)


def _vs_truth(T, T_true):
    """max |translation| of the residual motion: Result.Transformation maps the other way than the synthetic T_true"""
    from dvo_slam_b200 import synth
    return float(np.abs(synth.se3_log(np.asarray(T) @ np.asarray(T_true))[:3]).max())


def _same(a, b):
    return (np.array_equal(a.transformation, b.transformation) and np.array_equal(a.information, b.information)
            and a.log_likelihood == b.log_likelihood and a.levels == b.levels)


def test_batch_512_against_the_corrected_oracle(engine, corrected, oracle, batch):
    cfg = _cfg()
    refs, curs = batch["refs"], batch["curs"]
    # isolation: reference-mode alignments on the same pyramids before, between and after corrected ones are bit-identical
    ref0 = engine.match_batch(refs, curs, cfg)
    res = corrected.match_batch(refs, curs, cfg)
    ref1 = engine.match_batch(refs, curs, cfg)
    again = corrected.match_batch(refs, curs, cfg)
    rev = corrected.match_batch(refs[::-1], curs[::-1], cfg)[::-1]
    for i in range(B):
        assert _same(ref0[i], ref1[i]), i
        assert _same(res[i], again[i]) and _same(res[i], rev[i]), i
    for i in (0, 1, 200, 333, 334, 452, 453, 511):     # both sides of the slice boundaries of the fused launch
        assert _same(res[i], corrected.match(refs[i], curs[i], cfg)), i
    assert any(not _same(res[i], ref0[i]) for i in range(B))

    ocfg = oracle.config(first_level=FIRST, last_level=LAST, max_iterations_per_level=50, precision=1e-4)
    m = corrected_mode(oracle)

    def cpu(i):
        oref = oracle.Pyramid(batch["Ir"][i], batch["Zr"][i], batch["K"], LEVELS)
        ocur = oracle.Pyramid(batch["Ic"][i], batch["Zc"][i], batch["K"], LEVELS)
        return oracle.match(oref, ocur, ocfg, m)

    with ThreadPoolExecutor(os.cpu_count() or 8) as ex:
        orc = list(ex.map(cpu, range(B)))
    dts, drs, truth_gpu, truth_orc = [], [], [], []
    term = exact = within1 = 0
    for i in range(B):
        o, r = orc[i], res[i]
        dt, dr = pose_delta(o["T"], r.transformation)
        dts.append(dt); drs.append(dr)
        truth_gpu.append(_vs_truth(r.transformation, batch["truth"][i]))
        truth_orc.append(_vs_truth(o["T"], batch["truth"][i]))
        assert [l["valid_pixels"] for l in r.levels] == [l["valid_pixels"] for l in o["levels"]]
        assert not r.is_nan()
        (tg, ig), (to, io) = _flow(r.levels), _flow(o["levels"])
        term += tg == to
        exact += tg == to and ig == io
        within1 += all(abs(a - b) <= 1 for a, b in zip(ig, io))
    its_gpu = float(np.mean([r.num_iterations_total for r in res]))
    its_ref = float(np.mean([r.num_iterations_total for r in ref0]))
    summary = {"pairs": B,
               "pose_dt_m_vs_oracle": {"median": _pct(dts, 50), "p99": _pct(dts, 99), "max": max(dts)},
               "pose_dr_rad_vs_oracle": {"median": _pct(drs, 50), "max": max(drs)},
               "same_termination": term / B, "same_termination_and_iterations": exact / B, "iterations_within_1": within1 / B,
               "dt_vs_truth_gpu": {"median": _pct(truth_gpu, 50), "p90": _pct(truth_gpu, 90), "max": max(truth_gpu)},
               "dt_vs_truth_oracle": {"median": _pct(truth_orc, 50), "p90": _pct(truth_orc, 90), "max": max(truth_orc)},
               "iterations_per_alignment": {"corrected": its_gpu, "reference": its_ref}}
    print("\nbatch-512 corrected estimator vs corrected oracle:", json.dumps(summary))
    # the GPU is an IEEE restatement in the kernel's order, so it is at most as far from the oracle as the oracle's two orders
    # are from each other (x2 for the pose, -5 points for the control flow)
    assert max(dts) <= 2 * SPREAD_DT_MAX and max(drs) <= 2 * SPREAD_DR_MAX, summary
    assert term / B >= SPREAD_TERM - 0.05 and exact / B >= SPREAD_EXACT - 0.05, summary
    assert _pct(truth_gpu, 90) <= 1.1 * _pct(truth_orc, 90) + 1e-5, summary


def test_sharded_equals_one_context(corrected, batch):
    from dvo_slam_b200.engine import ShardedEngine
    n = 48
    cfg = _cfg()
    one = corrected.match_batch(batch["refs"][:n], batch["curs"][:n], cfg, raw=True)
    sh = ShardedEngine([0, 0])
    try:
        sh.set_estimator("corrected")
        # pyramid i on the shard that owns index i of n: references and currents are built as two batches of n
        refs = sh.pyramid_batch(batch["Ir"][:n], batch["Zr"][:n], batch["K"], LEVELS)
        curs = sh.pyramid_batch(batch["Ic"][:n], batch["Zc"][:n], batch["K"], LEVELS)
        got = sh.match_batch(refs, curs, cfg)
        for i in range(n):
            assert bytes(got[i]) == bytes(one[i]), i
        sh.release(refs + curs)
    finally:
        sh.close()


def test_unknown_estimator_is_rejected(corrected):
    assert corrected.lib.dvo_b200_set_estimator(corrected.ctx, 2) == -1
    assert corrected.lib.dvo_b200_set_estimator(corrected.ctx, -1) == -1
    assert corrected.estimator == "corrected"
    with pytest.raises(ValueError):
        corrected.set_estimator("paired")
