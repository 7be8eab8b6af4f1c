"""Parity at the BENCHMARKED configuration (BASELINE.json configs[2]): the first 512 seeded 640x480 pairs of bench.py,
one dvo_b200_match_batch call (the same plan_level outcome as the bench), against the oracle's FAITHFUL mode -- the mode
that tests/test_reference_pin.py pins bit for bit to the reference's own object code -- run on all host threads.

Asserted for 100 % of the pairs: pose within the stated SE(3) tolerance, identical selected-pixel counts.

Control flow (per-level TerminationCriterion and iteration counts, dense_tracking.cpp:276-284, 312-322, 357-363) is decided
by accept tests `Error < LastError` that near convergence compare numbers equal to ~1e-7: it is sensitive to ANY change of
rounding.  The oracle's own two arithmetic variants (FAITHFUL = the reference's SSE numerics, MIRROR = IEEE operations in
another order) agree on every termination for only ~70 % of pairs and on every iteration count (+-1) for ~50 %
(scripts/oracle_controlflow.py).  The meaningful statement is therefore relative: the CUDA path is no farther from the
reference's numerics than that independent IEEE restatement is.  The test measures both distances on the same 512 pairs and
asserts GPU-vs-FAITHFUL agreement >= MIRROR-vs-FAITHFUL agreement - 5 percentage points, plus absolute floors; the
distributions of |dt|, |dr|, Information and LogLikelihood error are printed (pytest -s shows them)."""
import json
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

from helpers import POSE_TOL_R, POSE_TOL_T, pose_delta

pytestmark = pytest.mark.gpu

B = 512
LEVELS, FIRST, LAST = 5, 4, 0


def _pct(v, q):
    return float(np.percentile(np.asarray(v, dtype=np.float64), q))


def test_batch_512_against_reference_numerics(engine, oracle):
    import torch
    from dvo_slam_b200 import synth
    from dvo_slam_b200.engine import Config

    dev = torch.device("cuda", 0)
    scfg = synth.SceneConfig()
    K = synth.FR1_INTRINSICS
    H, W = scfg.height, scfg.width
    Ir = np.empty((B, H, W), np.float32); Zr = np.empty((B, H, W), np.float32)
    Ic = np.empty((B, H, W), np.float32); Zc = np.empty((B, H, W), np.float32)
    for i in range(B):                      # the bench's seeds: rank 0 uses seeds 0 .. B-1
        p = synth.make_pair(i, scfg, device=dev)
        Ir[i] = p["I_ref"].cpu().numpy(); Zr[i] = p["Z_ref"].cpu().numpy()
        Ic[i] = p["I_cur"].cpu().numpy(); Zc[i] = p["Z_cur"].cpu().numpy()
    cfg = Config(first_level=FIRST, last_level=LAST, max_iterations_per_level=50, precision=1e-4)
    ocfg = oracle.config(first_level=FIRST, last_level=LAST, max_iterations_per_level=50, precision=1e-4)
    refs, curs = engine.pyramid_batch(Ir, Zr, K, LEVELS), engine.pyramid_batch(Ic, Zc, K, LEVELS)
    res = engine.match_batch(refs, curs, cfg)

    # Every floating-point sum above an image row is taken in an order fixed by the level's geometry (rows of a strip in
    # order, strips in order, fp64), never by how strips are spread over CTAs: the fused 512-pair launch -- one CTA per pair
    # on the coarse levels, slices with squads of 3, 6 and 12 CTAs on level 0 (on an H100, 132 SMs x 2 CTAs: pairs
    # 0-392, 393-471, 472-511) -- returns bit for bit what the same call returns again, what the batch in reverse order
    # returns (other slices), and what SINGLE alignments (one launch per level, squads of up to 69 CTAs) return.  The oracle comparison below therefore also speaks for the single-pair path
    # and vice versa (tests/test_gpu_parity.py compares that path with the oracle record by record).
    again = engine.match_batch(refs, curs, cfg)
    rev = engine.match_batch(refs[::-1], curs[::-1], cfg)[::-1]
    for other in (again, rev):
        for i in range(B):
            assert np.array_equal(res[i].transformation, other[i].transformation) and np.array_equal(res[i].information, other[i].information), i
            assert res[i].log_likelihood == other[i].log_likelihood and res[i].levels == other[i].levels, i
    for i in (0, 1, 200, 392, 393, 430, 471, 472, 500, 511):       # both sides of the slice boundaries 393 | 79 | 40
        single = engine.match(refs[i], curs[i], cfg)
        assert np.array_equal(res[i].transformation, single.transformation) and np.array_equal(res[i].information, single.information), i
        assert res[i].log_likelihood == single.log_likelihood and res[i].levels == single.levels, i

    def cpu(i):
        oref, ocur = oracle.Pyramid(Ir[i], Zr[i], K, LEVELS), oracle.Pyramid(Ic[i], Zc[i], K, LEVELS)
        return (oracle.match(oref, ocur, ocfg, oracle.mode("faithful")), oracle.match(oref, ocur, ocfg, oracle.mode("mirror")))

    with ThreadPoolExecutor(os.cpu_count() or 8) as ex:
        cpu_res = list(ex.map(cpu, range(B)))

    def flow(levels):
        return ([l["termination"] for l in levels], [l["num_iterations"] for l in levels])

    def rel_info(a, b):
        return float(np.linalg.norm(a - b) / np.linalg.norm(b))

    dts, drs = [], []
    err = {k: {"info": [], "ll": [], "info_same_flow": [], "ll_same_flow": [], "dt": []} for k in ("gpu", "mirror")}
    agree = {"gpu": {"term": 0, "it1": 0, "both": 0, "exact": 0}, "mirror": {"term": 0, "it1": 0, "both": 0, "exact": 0}}
    for i in range(B):
        fa, mi = cpu_res[i]
        r = res[i]
        dt, dr = pose_delta(fa["T"], r.transformation)
        assert dt < POSE_TOL_T and dr < POSE_TOL_R, (i, dt, dr)
        assert [l["valid_pixels"] for l in r.levels] == [l["valid_pixels"] for l in fa["levels"]]
        assert not r.is_nan()
        dts.append(dt); drs.append(dr)
        ft, fi = flow(fa["levels"])
        cand = (("gpu", flow(r.levels), r.information, r.log_likelihood, r.transformation),
                ("mirror", flow(mi["levels"]), mi["information"], mi["log_likelihood"], mi["T"]))
        for name, (t, it), info, ll, T in cand:
            same_t = t == ft
            within1 = all(abs(a - b) <= 1 for a, b in zip(it, fi))
            exact = same_t and it == fi
            agree[name]["term"] += same_t; agree[name]["it1"] += within1; agree[name]["both"] += same_t and within1
            agree[name]["exact"] += exact
            e_info, e_ll = rel_info(info, fa["information"]), abs(ll - fa["log_likelihood"]) / abs(fa["log_likelihood"])
            err[name]["info"].append(e_info); err[name]["ll"].append(e_ll); err[name]["dt"].append(pose_delta(fa["T"], T)[0])
            if exact:
                err[name]["info_same_flow"].append(e_info); err[name]["ll_same_flow"].append(e_ll)
    rate = {k: {m: v / B for m, v in d.items()} for k, d in agree.items()}

    def dist(v):
        return {"median": _pct(v, 50), "p95": _pct(v, 95), "max": float(max(v))} if len(v) else None

    summary = {
        "pairs": B,
        "bit_equal": "same call again, reversed batch (all 512), single alignments (10 pairs across the slices)",
        "pose_dt_m": {"median": _pct(dts, 50), "p95": _pct(dts, 95), "p99": _pct(dts, 99), "max": max(dts)},
        "pose_dr_rad": {"median": _pct(drs, 50), "p95": _pct(drs, 95), "p99": _pct(drs, 99), "max": max(drs)},
        "control_flow_vs_faithful": rate,
        "vs_faithful": {k: {m: dist(v) for m, v in d.items()} for k, d in err.items()},
    }
    print("\nbatch-512 parity vs FAITHFUL:", json.dumps(summary))
    # the CUDA path is as close to the reference's numerics as an independent IEEE restatement of the same algorithm:
    # control flow ...
    for m in ("term", "it1", "both"):
        assert rate["gpu"][m] >= rate["mirror"][m] - 0.05, (m, rate)
    assert rate["gpu"]["term"] >= 0.55 and rate["gpu"]["it1"] >= 0.35, rate
    # ... and Result.Information / Result.LogLikelihood / pose (they depend on which iteration was the last one)
    g, m = summary["vs_faithful"]["gpu"], summary["vs_faithful"]["mirror"]
    for key in ("info", "ll", "dt"):
        assert g[key]["median"] <= 1.25 * m[key]["median"] + 1e-6, (key, g[key], m[key])
        assert g[key]["p95"] <= 1.25 * m[key]["p95"] + 1e-6, (key, g[key], m[key])
    # pairs whose control flow is identical to FAITHFUL's.  Even there Information (= A of the last iteration, weighted with
    # the scale P_k) differs by several percent between ANY two roundings of the reference's algorithm: the scale estimator
    # pairs the weight of one point with the residual of its neighbour (computeScaleSse, dense_tracking_impl.cpp:556-599),
    # so a single point that flips validity (~20 of 263 000 at level 0 between FAITHFUL and MIRROR) shifts the pairing of
    # every later point and moves P_k by percents (measured at a fixed pose: P11 15563 vs 16134).  Asserted: the CUDA path
    # is not farther from FAITHFUL than MIRROR is, and stays inside the measured spread (info 7.5 %, LL 0.4 % median).
    if g["info_same_flow"] is not None and m["info_same_flow"] is not None:
        assert g["info_same_flow"]["median"] <= 1.25 * m["info_same_flow"]["median"] + 1e-6, (g, m)
        assert g["ll_same_flow"]["median"] <= 1.25 * m["ll_same_flow"]["median"] + 1e-6, (g, m)
    if g["info_same_flow"] is not None:
        assert g["info_same_flow"]["median"] < 0.15 and g["ll_same_flow"]["median"] < 0.01, g
    # typical agreement is far inside the tolerance
    assert summary["pose_dt_m"]["median"] < 5e-4 and summary["pose_dr_rad"]["median"] < 1e-4
    assert summary["pose_dt_m"]["p99"] < POSE_TOL_T and summary["pose_dr_rad"]["p99"] < POSE_TOL_R
