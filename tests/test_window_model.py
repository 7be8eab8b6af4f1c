"""The restatement of the level kernel's window decision (tests/window_model.py) against fp64 projections: for every case
of test_gpu_window_capacity.py, every tile it calls exact holds every bilinear tap and gradient tap of every pixel of the
tile that projects inside the image, and the cases reach every class they are there for."""
import numpy as np
import pytest

import window_model as wm
from tile_geometry import TILE_H, TILE_W, WIN_COLS, WIN_ROWS


def _taps_inside(win, s, b, T):
    """every pixel of tile (s, b), projected in fp64: its taps (columns u0-1 .. u0+2 clamped to the image, rows v0-1 .. v0+2
    clamped to the replica rows -1 and h) lie in the window"""
    fx, fy, ox, oy = wm.K
    ys, xs = np.mgrid[s * TILE_H:min((s + 1) * TILE_H, wm.H), b * TILE_W:min((b + 1) * TILE_W, wm.W)]
    z = wm.DEPTH
    p = np.stack([(xs.ravel() - ox) / fx * z, (ys.ravel() - oy) / fy * z, np.full(xs.size, z)])
    q = T[:3, :3] @ p + T[:3, 3:4]
    u, v = fx * q[0] / q[2] + ox, fy * q[1] / q[2] + oy
    inside = (u >= 0) & (u < wm.W - 1) & (v >= 0) & (v < wm.H - 1)
    u0, v0 = np.floor(u[inside]).astype(int), np.floor(v[inside]).astype(int)
    c_lo, c_hi = np.maximum(u0 - 1, 0), np.minimum(u0 + 2, wm.W - 1)
    r_lo, r_hi = np.maximum(v0 - 1, -1), np.minimum(v0 + 2, wm.H)
    ok = ((c_lo >= win["bx0"]) & (c_hi <= win["bx0"] + win["ncols"] - 1) &
          (r_lo >= win["row_lo"]) & (r_hi <= win["row_lo"] + win["nrows"] - 1))
    return bool(ok.all()), int(inside.sum())


@pytest.mark.parametrize("case", list(wm.CASES))
def test_exact_windows_hold_every_tap(case):
    T = wm.CASES[case]
    _, Z = wm.plane()
    wins = wm.level_windows(wm.K, T, Z)
    checked = 0
    for (s, b), win in wins.items():
        assert win["ncols"] <= WIN_COLS and win["nrows"] <= WIN_ROWS and win["ncols"] % 2 == 0
        if win["kind"] == "exact" and wm.safe(win):
            ok, n = _taps_inside(win, s, b, T)
            assert ok, (case, s, b, win)
            checked += n
        if win["kind"] == "skip" and win["corners"]:
            assert _taps_inside({"bx0": 0, "ncols": 0, "row_lo": 0, "nrows": 0}, s, b, T)[1] == 0, (case, s, b)
    assert checked > 0 or case.endswith("2.5")


def test_every_class_is_reached():
    """nrows 19 exact and 20-21 clipped, ncols 184 exact and 186 clipped, column clips alone and with rows, exact windows on
    the replica rows and the first and last column, and tiles just inside and just outside each image edge"""
    _, Z = wm.plane()
    wins = {name: wm.level_windows(wm.K, T, Z) for name, T in wm.CASES.items()}
    safe = [w for ws in wins.values() for w in ws.values() if wm.safe(w) and w["kind"] != "skip"]
    exact = [w for w in safe if w["kind"] == "exact"]
    assert any(w["nrows"] == WIN_ROWS for w in exact)
    assert {20, 21} <= {w["nrows_hull"] for w in safe if w["kind"] == "rows"}
    assert any(w["ncols"] == WIN_COLS for w in exact)
    assert any(w["ncols_hull"] == WIN_COLS + 2 for w in safe if w["kind"] == "cols")
    assert wm.census(wins["forward1.2"]).get("cols") and not wm.census(wins["forward1.2"]).get("rows")
    assert wm.census(wins["forward2.5"]).get("both")
    e = [w for w in exact if w in wins["edges"].values()]
    assert any(w["row_lo"] == -1 for w in e) and any(w["row_lo"] + w["nrows"] - 1 == wm.H for w in e)
    assert any(w["bx0"] == 0 for w in e) and any(w["bx0"] + w["ncols"] - 1 >= wm.W - 1 for w in e)
    for edge in ("left", "right", "top", "bottom"):
        kept, skipped = wm.edge_tiles(wins[f"{edge}_in"], edge)
        assert kept > 0 and skipped == 0, edge
        kept, skipped = wm.edge_tiles(wins[f"{edge}_out"], edge)
        assert skipped > 0 and kept == 0, edge
