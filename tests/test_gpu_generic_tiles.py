"""The level kernel's generic pixel loop, against the oracle's MIRROR mode.

Almost every tile of an alignment takes the exact loop (window holds all taps, full band).  The generic loop serves the
rest: windows the taps do not fit, tiles with a corner behind the camera (no window at all: every tap is gathered), and
partial bands at the right edge.  Each case is forced here by the pose or the level, shown from the geometry, and checked
as test_gpu_parity checks the exact loop: residual records bit-exact, counts exact, P / LL / A / b to 2e-6.

The partial bands come from a 720 x 540 scene (PARTIAL): levels 0, 1 and 2 are 720, 360 and 180 columns wide, so each has
full 160-column bands and a partial last band of 80, 40 and 20 columns.  The other modules that force the generic loop
take their partial-band case from here.
"""
import numpy as np
import pytest

from helpers import nan_equal
from tile_geometry import TILE_H, TILE_W, WIN_ROWS, assert_partial_band

pytestmark = pytest.mark.gpu

PARTIAL_W, PARTIAL_H = 720, 540


def partial_scene():
    """the scene config of the partial-band cases: fr1 intrinsics scaled to 720 x 540"""
    from dvo_slam_b200 import synth
    s = PARTIAL_W / 640
    return synth.SceneConfig(width=PARTIAL_W, height=PARTIAL_H, intrinsics=tuple(v * s for v in synth.FR1_INTRINSICS))


def partial_pair(seed=0):
    """images and intrinsics of one pair of the partial-band scene"""
    from dvo_slam_b200 import synth
    p = synth.make_pair(seed, partial_scene())
    a = {k: p[k].numpy() for k in ("I_ref", "Z_ref", "I_cur", "Z_cur")}
    a["K"] = p["intrinsics"]
    return a


def partial_pose():
    """a small motion under which most tiles of levels 1 and 2 keep a window"""
    return _rot_z(3.0) @ _shift_z(0.02)


def _rot_z(deg):
    a = np.deg2rad(deg)
    T = np.eye(4)
    T[:2, :2] = [[np.cos(a), -np.sin(a)], [np.sin(a), np.cos(a)]]
    return T


def _shift_z(dz):
    T = np.eye(4)
    T[2, 3] = dz
    return T


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
    a = partial_pair(0)
    a["gref"] = engine.pyramid(a["I_ref"], a["Z_ref"], a["K"], 5)
    a["gcur"] = engine.pyramid(a["I_cur"], a["Z_cur"], a["K"], 5)
    a["oref"] = oracle.Pyramid(a["I_ref"], a["Z_ref"], a["K"], 5)
    a["ocur"] = oracle.Pyramid(a["I_cur"], a["Z_cur"], a["K"], 5)
    return a


def _check_level(engine, oracle, a, lvl, T):
    mir = oracle.mode("mirror")
    n_g, img_g = engine.residual_image(a["gref"], a["gcur"], lvl, T)
    n_o, img_o = oracle.residual_image(a["oref"], a["ocur"], lvl, T, mir)
    assert n_g == n_o and n_g > 0 and nan_equal(img_g, img_o)
    pp = np.array([[2000.0, -30.0], [-30.0, 9000.0]], dtype=np.float32)
    for uw in (False, True):
        lg = engine.linearize(a["gref"], a["gcur"], lvl, T, uw, pp)
        lo = oracle.linearize(a["oref"], a["ocur"], lvl, T, mir, uw, pp)
        assert lg["n"] == lo["n"]
        assert np.allclose(lg["precision"], lo["precision"], rtol=2e-6)
        assert abs(lg["ll"] - lo["ll"]) <= 2e-6 * abs(lo["ll"]) + 0.5
        assert np.allclose(lg["A"], lo["A"], rtol=0, atol=2e-6 * np.abs(lo["A"]).max())
        assert np.allclose(lg["b"], lo["b"], rtol=0, atol=2e-6 * np.abs(lo["b"]).max())


def test_window_too_small(engine, oracle, pair):
    """A rotation about the optical axis tilts every tile row: a 160-pixel row then spans more image rows than the window
    holds.  A pure rotation maps pixels independently of depth, so the span is exact geometry."""
    fx, fy, ox, oy = pair["K"]
    T = _rot_z(20.0)
    h, w = pair["I_ref"].shape
    spans = []
    for y0 in range(0, h - TILE_H + 1, TILE_H):
        for x0 in range(0, w - TILE_W + 1, TILE_W):
            u = np.array([x0, x0 + TILE_W - 1, x0, x0 + TILE_W - 1], dtype=np.float64)
            v = np.array([y0, y0, y0 + TILE_H - 1, y0 + TILE_H - 1], dtype=np.float64)
            ray = np.stack([(u - ox) / fx, (v - oy) / fy, np.ones(4)])
            q = T[:3, :3] @ ray
            vv = fy * q[1] / q[2] + oy
            inside = (vv >= 0).all() and (vv <= h - 1).all()
            if inside:
                spans.append(vv.max() - vv.min())
    assert spans and min(spans) > WIN_ROWS, min(spans)      # every tile inside the image overflows the window
    _check_level(engine, oracle, pair, 0, T)


def test_corner_behind_camera(engine, oracle, pair):
    """Moving the camera forward past the nearest surfaces puts reference points behind it.  Z' is affine in the point, so
    a tile holding such a point has a corner ray (at its min or max depth) with Z' < 0 and takes no window."""
    Z = pair["Z_ref"]
    dz = float(np.nanmedian(Z))
    T = _shift_z(-dz)
    zt = Z + T[2, 3]
    finite = np.isfinite(zt)
    assert (zt[finite] < -0.05).any() and (zt[finite] > 0.05).any()
    _check_level(engine, oracle, pair, 0, T)


@pytest.mark.parametrize("lvl", [1, 2])
def test_partial_band(engine, oracle, pair720, lvl):
    """720 / 2 and 720 / 4 columns are full 160-column bands followed by a partial one in every strip."""
    assert_partial_band(pair720["oref"].level_info(lvl)[0])
    _check_level(engine, oracle, pair720, lvl, partial_pose())
