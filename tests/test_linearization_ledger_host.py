"""The fp64 ledger of tests/linearization_ledger.py on the CPU: validated against the oracle's MIRROR mode, shown not too
tight for the kernel's fp32 summation order, and shown to catch the defects the suite's max-normalised checks let through.

MIRROR restates the level kernel's operation order, so its outputs are a stand-in for the kernel's: fed its own records
and P_k, the ledger must hold every entry of P, the log-likelihood, A and b far inside its bound (the bound is derived
for the kernel's order; MIRROR sums in fp64, so it sits well inside).  Each mutation below is a defect a kernel could have;
the ledger must report it.  For the first two the suite's check of the form 2e-6 max|A| (max|b|) passes: the gap the
ledger closes.
"""
import numpy as np
import pytest

import linearization_ledger as L
import step_replay
from helpers import corrected_mode, odd_point_margin

PP = np.array([[2000.0, -30.0], [-30.0, 9000.0]], dtype=np.float32)    # the suite's prev_precision
ABS = [(1.0, 0.0), (1.1, -7.5), (0.85, 12.0)]                           # tests/test_gpu_photometric.py
EXPOSURE = (1.1, -7.5)


def _synth(width):
    from dvo_slam_b200 import synth
    p = synth.make_pair(3, step_replay._scene320() if width == 320 else None)
    a = {k: p[k].numpy() for k in ("I_ref", "Z_ref", "I_cur", "Z_cur")}
    a["K"], a["T_true"], a["xi"] = p["intrinsics"], p["T_true"], p["xi"]
    return a


def _poses(a):
    """the true motion (where b nearly cancels once weighted) and a pose perturbed from it"""
    from dvo_slam_b200 import synth
    return {"true": a["T_true"], "perturbed": synth.se3_exp(a["xi"] * 0.9) @ synth.se3_exp([4e-3, -3e-3, 2e-3, -2e-3, 3e-3, 1e-3])}


@pytest.fixture(scope="module")
def scenes(oracle):
    out = {}
    for width in (320, 640):
        a = _synth(width)
        a["oref"] = oracle.Pyramid(a["I_ref"], a["Z_ref"], a["K"], 5)
        a["ocur"] = oracle.Pyramid(a["I_cur"], a["Z_cur"], a["K"], 5)
        out[width] = a
    return out


@pytest.fixture(scope="module")
def photometric_scene():
    import photometric_oracle as pho
    from dvo_slam_b200 import synth
    a = _synth(320)
    a["I_cur"] = synth.exposure(a["I_cur"], *EXPOSURE)
    a["pref"] = pho.Pyramid(a["I_ref"], a["Z_ref"], a["K"], 3)
    a["pcur"] = pho.Pyramid(a["I_cur"], a["Z_cur"], a["K"], 3)
    return a


def _mode(oracle, estimator):
    return oracle.mode("mirror") if estimator == "reference" else corrected_mode(oracle)


def _mirror(oracle, a, level, T, estimator, uw, pp=PP):
    """(records, linearisation) of the oracle's MIRROR mode (or the corrected estimator's definition)"""
    m = _mode(oracle, estimator)
    _, rec = oracle.residual_image(a["oref"], a["ocur"], level, T, m)
    return rec, oracle.linearize(a["oref"], a["ocur"], level, T, m, uw, pp)


def _pho_intensity(p, level):
    import photometric_oracle as pho
    w, h = p.level_info(level)
    return np.ctypeslib.as_array(pho.lib().orc_pyramid_plane(p.h, level, 0), shape=(h, w)).copy()


def _pho_mirror(oracle, a, level, T, ab, estimator, uw):
    import photometric_oracle as pho
    m = _mode(oracle, estimator)
    _, rec = pho.residual_image(a["pref"], a["pcur"], level, T, ab, m)
    return rec, pho.linearize(a["pref"], a["pcur"], level, T, ab, m, uw, PP), _pho_intensity(a["pref"], level)


def _assert_holds(rep, limit=0.5):
    """every entry inside its bound, and far inside: MIRROR sums in fp64"""
    assert not rep.failures, rep.failures[:8]
    assert max(rep.maxima.values()) < limit, rep.maxima


def _old_check(out, ref):
    """the suite's check of A and b, relative to the largest entry"""
    return (np.allclose(out["A"], ref["A"], rtol=0, atol=2e-6 * np.abs(ref["A"]).max())
            and np.allclose(out["b"], ref["b"], rtol=0, atol=2e-6 * np.abs(ref["b"]).max()))


# ---- the ledger against MIRROR -------------------------------------------------------------------------------------------
LEVELS = [(320, 0), (320, 1), (320, 2), (640, 0), (640, 4)]


@pytest.mark.parametrize("pose", ["true", "perturbed"])
@pytest.mark.parametrize("uw", [0, 1])
@pytest.mark.parametrize("width,level", LEVELS, ids=[f"{w}-l{l}" for w, l in LEVELS])
@pytest.mark.parametrize("estimator", ["reference", "corrected"])
def test_ledger_holds_mirror(oracle, scenes, estimator, width, level, uw, pose):
    a = scenes[width]
    T = _poses(a)[pose]
    rec, out = _mirror(oracle, a, level, T, estimator, uw)
    led = L.ledger(rec, a["K"], level, out["precision"], estimator, uw, PP)
    assert led.n == out["n"] > 6
    _assert_holds(L.compare(led, out))


def test_b_nearly_cancels_at_the_true_motion(oracle, scenes):
    """where b is far below its absolute sum, a max-normalised bound says nothing about it; the ledger still holds it"""
    a = scenes[640]
    rec, out = _mirror(oracle, a, 0, a["T_true"], "reference", 1)
    led = L.ledger(rec, a["K"], 0, out["precision"], "reference", 1, PP)
    assert (np.abs(led.b) / led.M["b"]).max() < 0.02
    _assert_holds(L.compare(led, out))


@pytest.mark.parametrize("level", [0, 1, 2])
@pytest.mark.parametrize("ab", ABS, ids=[f"{x}_{y}" for x, y in ABS])
@pytest.mark.parametrize("estimator", ["reference", "corrected"])
def test_ledger_holds_photometric_mirror(oracle, photometric_scene, estimator, ab, level):
    a = photometric_scene
    for uw in (0, 1):
        for T in _poses(a).values():
            rec, out, Ir = _pho_mirror(oracle, a, level, T, ab, estimator, uw)
            led = L.ledger(rec, a["K"], level, out["precision"], estimator, uw, PP, I_ref=Ir)
            assert led.A.shape == (8, 8) and led.n == out["n"] > 6
            _assert_holds(L.compare(led, out))


# ---- the kernel's summation order in fp32 ------------------------------------------------------------------------------
@pytest.mark.parametrize("width", [320, 640])
def test_fp32_row_order_stays_inside_the_bound(oracle, scenes, width):
    """MIRROR's per-point terms, split as the kernel splits them and summed in fp32 lane chains of ceil(w/32) pixels (two
    rank-1 updates each), the halving exchange and fp64 rows, against the ledger: inside the bound, and not exact"""
    a = scenes[width]
    rec, out = _mirror(oracle, a, 0, a["T_true"], "reference", 1)
    led = L.ledger(rec, a["K"], 0, out["precision"], "reference", 1, PP)
    pts = L.points(rec, a["K"], 0)
    w, _ = L.weights(pts, True, PP)
    Pk = np.asarray(out["precision"], np.float64)
    T0, T1, t0, t1 = L.ldl_terms(pts, w, Pk)
    A = L.emulate_row_order(pts, T0, T1)
    b = L.emulate_row_order(pts, t0, t1)
    rA = np.abs(A - led.A) / led.A_bound
    rb = np.abs(b - led.b) / led.b_bound
    assert rA.max() < 1.0 and rb.max() < 1.0, (rA.max(), rb.max())
    assert rA.max() > 1e-3         # the fp32 order is visible to the ledger
    print(f"{width}x: fp32 row order / bound: A {rA.max():.3g}, b {rb.max():.3g}")


# ---- mutations of MIRROR's outputs ---------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def photometric_l0(oracle, photometric_scene):
    a = photometric_scene
    rec, out, Ir = _pho_mirror(oracle, a, 0, _poses(a)["perturbed"], (1.1, -7.5), "reference", 1)
    return a, rec, out, Ir


def _mutated(out, **kw):
    m = {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in out.items()}
    m.update(kw)
    return m


def test_mutation_beta_diagonal(photometric_l0):
    a, rec, out, Ir = photometric_l0
    led = L.ledger(rec, a["K"], 0, out["precision"], "reference", 1, PP, I_ref=Ir)
    _assert_holds(L.compare(led, out))
    A = out["A"].copy()
    A[7, 7] *= 1 + 1e-3
    bad = _mutated(out, A=A)
    assert _old_check(bad, out)
    assert "A" in L.compare(led, bad).failed


def test_mutation_beta_gradient(photometric_l0):
    a, rec, out, Ir = photometric_l0
    led = L.ledger(rec, a["K"], 0, out["precision"], "reference", 1, PP, I_ref=Ir)
    b = out["b"].copy()
    b[7] += 1e-3 * abs(b[7])
    bad = _mutated(out, b=b)
    assert _old_check(bad, out)
    assert "b" in L.compare(led, bad).failed


# values 32..44 of the photometric row exchange: A[5][6], A[5][7], A[6][6], A[6][7], A[7][7] and all of b
SECOND_WINDOW_A = [(5, 6), (5, 7), (6, 6), (6, 7), (7, 7)]


def test_mutation_row_missing_from_the_second_window(photometric_l0):
    a, rec, out, Ir = photometric_l0
    led = L.ledger(rec, a["K"], 0, out["precision"], "reference", 1, PP, I_ref=Ir)
    y = rec.shape[1] // 2
    cut = rec.copy()
    cut[:, y, :] = np.nan
    part = L.ledger(cut, a["K"], 0, out["precision"], "reference", 1, PP, I_ref=Ir)
    dA, db = led.A - part.A, led.b - part.b
    A, b = out["A"].copy(), out["b"] - db
    for r, c in SECOND_WINDOW_A:
        A[r, c] -= dA[r, c]
        A[c, r] = A[r, c]
    rep = L.compare(led, _mutated(out, A=A, b=b))
    assert {"A", "b"} <= rep.failed, rep.failures


def test_mutation_median_point_missing(oracle, scenes):
    a = scenes[320]
    rec, out = _mirror(oracle, a, 2, a["T_true"], "reference", 1)
    led = L.ledger(rec, a["K"], 2, out["precision"], "reference", 1, PP)
    _assert_holds(L.compare(led, out))
    pix = np.flatnonzero(np.isfinite(rec[0]).reshape(-1))
    cut = rec.copy()
    cut.reshape(7, -1)[:, pix[len(pix) // 2]] = np.nan
    part = L.ledger(cut, a["K"], 2, out["precision"], "reference", 1, PP)
    rep = L.compare(led, _mutated(out, A=out["A"] - (led.A - part.A), b=out["b"] - (led.b - part.b)))
    assert {"A", "b"} <= rep.failed, rep.failures


def test_mutation_tail_from_the_first_ranks(oracle, scenes):
    a = scenes[320]
    rec, out = _mirror(oracle, a, 0, a["T_true"], "reference", 1)
    led = L.ledger(rec, a["K"], 0, out["precision"], "reference", 1, PP)
    t = led.n % 50
    assert t > 0
    lg, _ = L.log_terms(L.points(rec, a["K"], 0), np.asarray(out["precision"], np.float64))
    ll = out["ll"] - 3.5 * (lg[-t:].sum() - lg[:t].sum())
    assert "ll" in L.compare(led, _mutated(out, ll=ll)).failed


@pytest.mark.parametrize("width,level", [(320, 2), (640, 0)])
def test_mutation_unpaired_scale_in_reference_mode(oracle, scenes, width, level):
    a = scenes[width]
    rec, out = _mirror(oracle, a, level, a["T_true"], "reference", 1)
    led = L.ledger(rec, a["K"], level, out["precision"], "reference", 1, PP)
    pts = L.points(rec, a["K"], level)
    w, eps = L.weights(pts, True, PP)
    S, _, _ = L.scale_sum(pts, w, eps, "corrected")
    P = np.linalg.inv(np.array([[S[0], S[1]], [S[1], S[2]]]) / (led.n - 3)).astype(np.float32)
    assert "P" in L.compare(led, _mutated(out, precision=P)).failed


def test_mutation_odd_point_counted_in_reference_mode(oracle):
    margin, im, oref, ocur = odd_point_margin(oracle)
    from helpers import GOLDEN_SEEDS, load_golden
    K = load_golden(GOLDEN_SEEDS[0])["K"]
    m = oracle.mode("mirror")
    _, rec = oracle.residual_image(oref, ocur, 0, np.eye(4), m)
    out = oracle.linearize(oref, ocur, 0, np.eye(4), m, True, PP)
    led = L.ledger(rec, K, 0, out["precision"], "reference", 1, PP)
    _assert_holds(L.compare(led, out))
    m.drop_odd_point = 0
    bad = oracle.linearize(oref, ocur, 0, np.eye(4), m, True, PP)
    assert bad["n"] == out["n"] + 1
    rep = L.compare(led, bad)
    assert {"n", "A"} <= rep.failed, rep.failures


def test_lane_chains_follow_the_rounds_of_32():
    """A lane adds one pixel per round of 32 columns: 5 per full 160-column band, ceil(bw / 32) in a partial band of bw.  k
    is the same at 640 and 1280 columns as when bands were 128 wide (DESIGN 5), and shorter where a partial band is narrow."""
    assert [L.rounds(w) for w in (640, 1280, 400, 161, 288, 319, 32)] == [20, 40, 13, 6, 9, 10, 1]
    assert [L.k_counts(w, "reference")["A"] for w in (640, 1280)] == [79, 119]
    assert [L.k_counts(w, "reference")["b"] for w in (640, 1280)] == [68, 108]
    assert L.k_counts(161, "reference") == {"A": 51, "b": 40, "ll": 13, "scale": 20}
    assert L.k_counts(161, "corrected")["scale"] == 12
