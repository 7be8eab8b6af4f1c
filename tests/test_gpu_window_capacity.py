"""The level kernel's tile windows at their capacity (csrc/stages.cuh: produce_tiles), against the oracle.

A fronto-parallel textured plane at constant depth (tests/window_model.py), under poses that put tiles on either side of
every window rule: a roll sweep to 19 rows (exact) and 20-21 (clipped), forward moves to 184 columns (exact), 186 (clipped)
and past both limits, exact windows on the replica rows and the first and last column, and shifts that keep a tile's hull
just inside or just outside each image edge.  tests/window_model.py restates the decision in fp32 and shows which class
each tile takes; it prints the count per class.  Per case: residual records bit-exact against MIRROR, counts exact,
P / LL / A / b to 2e-6, for both estimators, with and without a mask in the current role, and in the photometric hooks.
P, A and b are held to 2e-6 of their largest entry or to the oracle's own spread between its fused and unfused pixel
arithmetic where that is larger (the rule of test_gpu_geometry): on this plane a one-pixel shift leaves small, coherent
residuals, and the two arithmetic orders give P, A and b up to 4.7e-6 apart.
"""
import numpy as np
import pytest

import window_model as wm
from test_corrected_estimator import corrected_mode
from test_gpu_geometry import _check_linearisation, _unfused
from test_gpu_mask_roles import _pyrs
from test_gpu_photometric import AB_FORCED

PP = np.array([[2000.0, -30.0], [-30.0, 9000.0]], dtype=np.float32)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def corrected(engine):
    from dvo_slam_b200.engine import Engine
    eng = Engine(device=0, estimator="corrected")
    yield eng
    eng.close()


@pytest.fixture(scope="module")
def plane(engine, oracle):
    I, Z = wm.plane()
    # a current frame unlike the reference, so that both residuals vary: with a constant depth in both frames and no motion
    # along the axis every depth residual would be zero, and P the inverse of a singular covariance
    Ic = np.roll(I, 1, axis=1)
    Zc = (Z + 0.05 * (wm.plane(1)[0] - 128.0) / 64.0).astype(np.float32)
    m = np.ones((wm.H, wm.W), np.uint8)
    m[30:60, 90:140] = 0
    m[90:110, 330:370] = 0
    out = {"Z": Z}
    out["ref"] = _pyrs(engine, oracle, I, Z, wm.K, None, "both", 1)
    out["cur"] = _pyrs(engine, oracle, Ic, Zc, wm.K, None, "both", 1)
    out["cur_masked"] = _pyrs(engine, oracle, Ic, Zc, wm.K, m, "both", 1)
    return out


def _check(eng, mode, gref, gcur, oref, ocur, T, lin):
    """records and the intensity error image bit-exact, counts exact, linearisations (weights off and on) to the bounds;
    lin(pyramids, mode, use_weights) -> the oracle's linearisation"""
    n_g, img_g = eng.residual_image(gref, gcur, 0, T, ab=lin.ab)
    n_o, img_o = lin.records(oref, ocur, T, mode)
    assert n_g == n_o and n_g > 0 and np.array_equal(img_g, img_o, equal_nan=True), (n_g, n_o)
    for uw in (False, True):
        lg = eng.linearize(gref, gcur, 0, T, uw, PP, ab=lin.ab)
        _check_linearisation(lg, lin(oref, ocur, T, mode, uw), lin(oref, ocur, T, _unfused(mode), uw))


class _Hooks:
    """the oracle's records and linearisation at level 0, in the photometric mode at ab, or the default mode for ab None"""

    def __init__(self, oracle, ab=None):
        self.o, self.ab = oracle, ab

    def records(self, oref, ocur, T, mode):
        return self.o.residual_image(oref, ocur, 0, T, mode, ab=self.ab)

    def __call__(self, oref, ocur, T, mode, uw):
        return self.o.linearize(oref, ocur, 0, T, mode, uw, PP, ab=self.ab)


def _both_estimators(engine, corrected, oracle, gref, gcur, oref, ocur, T, lin):
    _check(engine, oracle.mode("mirror"), gref, gcur, oref, ocur, T, lin)
    _check(corrected, corrected_mode(oracle), gref, gcur, oref, ocur, T, lin)


@pytest.mark.parametrize("case", list(wm.CASES))
def test_records_at_the_window_limits(engine, corrected, oracle, plane, case):
    T = wm.CASES[case]
    wins = wm.level_windows(wm.K, T, plane["Z"])
    print(f"\n{case}: {wm.census(wins)}")
    (gref, oref), (gcur, ocur) = plane["ref"], plane["cur"]
    _both_estimators(engine, corrected, oracle, gref, gcur, oref, ocur, T, _Hooks(oracle))
    gcm, ocm = plane["cur_masked"]
    _both_estimators(engine, corrected, oracle, gref, gcm, oref, ocm, T, _Hooks(oracle))


@pytest.mark.parametrize("case", ["edges", "roll2.6", "roll2.9", "forward1.112", "forward1.12", "forward2.5", "right_in",
                                  "bottom_in"])
def test_photometric_records_at_the_window_limits(engine, corrected, oracle, plane, case):
    T = wm.CASES[case]
    gref, oref = plane["ref"]
    for key in ("cur", "cur_masked"):
        gcur, ocur = plane[key]
        _both_estimators(engine, corrected, oracle, gref, gcur, oref, ocur, T, _Hooks(oracle, AB_FORCED))
