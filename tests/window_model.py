"""The level kernel's window decision for one tile (csrc/stages.cuh: produce_tiles), restated in fp32 in its operation order.

The producer sizes the window of the current image a tile's taps may read from eight projections: the four corner rays of
the tile (template tx at its first and last column, ty at its first and last row) at the tile's minimum and maximum
reference depth, through K float(T).  The result is one of
  skip      no reference depth in the tile, or the whole hull outside the image (umax < -1, vmax < -1, umin > w, vmin > h)
  none      a corner behind the camera (Z' <= 1e-6 or NaN), or a window smaller than 4 x 4 (the sliver rule): no window,
            every tap is gathered.  A hull that is not skipped spans at least 4 columns and 4 rows unless umin == w or
            vmin == h exactly, so the sliver rule is met only at those float equalities
  exact     the window holds the hull's taps: at most WIN_COLS columns and WIN_ROWS rows
  cols / rows / both   the window was centred and clipped to WIN_COLS columns, WIN_ROWS rows, or both
together with the window's first column bx0, its width ncols (even), its first row row_lo (-1 is the replica row above
the image) and its height nrows.  test_gpu_window_capacity.py uses it to show that each class is reached; the restatement
is checked against fp64 projections of every pixel in test_window_model.py.  The cases both use are at the end.
"""
import numpy as np

import linearization_ledger as led
from tile_geometry import TILE_H, TILE_W, WIN_COLS, WIN_ROWS, bands, strips

F = np.float32


def _fma(a, b, c):
    return F(np.float64(a) * np.float64(b) + np.float64(c))


def kt(K, T):
    """K float(T) as the tracker forms it: rows fx t0 + ox t2, fy t1 + oy t2, t2 in fp32 (tracker.cu, kt_of)"""
    fx, fy, ox, oy = (F(v) for v in K)
    out = np.zeros(12, np.float32)
    for j in range(4):
        t0, t1, t2 = F(T[0][j]), F(T[1][j]), F(T[2][j])
        out[j] = F(fx * t0) + F(ox * t2)
        out[4 + j] = F(fy * t1) + F(oy * t2)
        out[8 + j] = t2
    return out


def tile_ranges(Z, usable=None):
    """(zmin, zmax) per tile of non-NaN depth (and usable pixels, under a mask), strips x bands; zmin > zmax: none"""
    h, w = Z.shape
    nb, ns = len(bands(w)), len(strips(h))
    zr = np.empty((ns, nb, 2), np.float32)
    for s in range(ns):
        for b in range(nb):
            t = Z[s * TILE_H:(s + 1) * TILE_H, b * TILE_W:(b + 1) * TILE_W]
            if usable is not None:
                t = np.where(usable[s * TILE_H:(s + 1) * TILE_H, b * TILE_W:(b + 1) * TILE_W], t, np.nan)
            v = t[~np.isnan(t)]
            zr[s, b] = (v.min(), v.max()) if v.size else (np.inf, -np.inf)
    return zr


def window(k, tx, ty, w, h, s, b, zr):
    """one tile's decision: dict(kind, bx0, ncols, row_lo, nrows, corners = the eight (u, v) before the clamp)"""
    y0, x0 = s * TILE_H, b * TILE_W
    rows, bw = min(TILE_H, h - y0), min(TILE_W, w - x0)
    zmin, zmax = zr
    out = {"kind": "skip", "bx0": 0, "ncols": 0, "row_lo": 0, "nrows": 0, "corners": []}
    if not zmin <= zmax:
        return out
    us, vs, front = [], [], True
    for lane in range(8):
        txc = tx[x0 + bw - 1] if lane & 1 else tx[x0]
        tyc = ty[y0 + rows - 1] if lane & 2 else ty[y0]
        z = F(zmax if lane & 4 else zmin)
        px, py = F(txc * z), F(tyc * z)
        X = _fma(k[0], px, _fma(k[1], py, _fma(k[2], z, k[3])))
        Y = _fma(k[4], px, _fma(k[5], py, _fma(k[6], z, k[7])))
        Zt = _fma(k[8], px, _fma(k[9], py, _fma(k[10], z, k[11])))
        with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
            iz = F(F(1.0) / Zt)
            u, v = F(X * iz), F(Y * iz)
        front = front and bool(Zt > F(1e-6)) and u == u and v == v
        us.append(u); vs.append(v)
    out["corners"] = list(zip(us, vs))
    umin, umax, vmin, vmax = min(us), max(us), min(vs), max(vs)
    umin, vmin = max(umin, F(-8.0)), max(vmin, F(-8.0))
    umax, vmax = min(umax, F(w + 8.0)), min(vmax, F(h + 8.0))
    if not front:
        out["kind"] = "none"
        return out
    if umax < -1 or vmax < -1 or umin > w or vmin > h:
        return out
    col_lo, col_hi = max(int(np.floor(umin)) - 2, 0), min(int(np.floor(umax)) + 3, w - 1)
    row_lo = max(int(np.floor(vmin)) - 2, -1)
    row_hi = min(int(np.floor(vmax)) + 3, h)
    bx0 = col_lo & ~1
    ncols = (col_hi + 2 - bx0) & ~1
    nrows = row_hi - row_lo + 1
    out.update(ncols_hull=ncols, nrows_hull=nrows)
    clip_c = clip_r = False
    if ncols > WIN_COLS:
        bx0 += ((ncols - WIN_COLS) // 2) & ~1
        ncols, clip_c = WIN_COLS, True
    if nrows > WIN_ROWS:
        row_lo += (nrows - WIN_ROWS) // 2
        nrows, clip_r = WIN_ROWS, True
    out.update(bx0=bx0, ncols=ncols, row_lo=row_lo, nrows=nrows)
    if ncols < 4 or nrows < 4:
        out.update(kind="none", bx0=0, ncols=0, row_lo=0, nrows=0)
    else:
        out["kind"] = "both" if clip_c and clip_r else "cols" if clip_c else "rows" if clip_r else "exact"
    return out


def level_windows(K, T, Z, usable=None):
    """every tile's decision at level 0 of an image with depth Z and intrinsics K under T: {(s, b): window}"""
    h, w = Z.shape
    tx, ty = led.template(w, h, K)
    tx, ty = tx.astype(np.float32), ty.astype(np.float32)
    k = kt(K, T)
    zr = tile_ranges(Z, usable)
    return {(s, b): window(k, tx, ty, w, h, s, b, zr[s, b]) for s in range(zr.shape[0]) for b in range(zr.shape[1])}


def safe(win, margin=1e-3):
    """every corner coordinate at least margin from the nearest integer: the floors and the edge tests cannot differ from
    the device's by a last-bit difference of the projection"""
    return all(abs(c - np.round(c)) >= margin for uv in win["corners"] for c in uv)


def census(wins):
    """{kind: number of safe tiles}"""
    out = {}
    for wv in wins.values():
        if safe(wv):
            out[wv["kind"]] = out.get(wv["kind"], 0) + 1
    return out


# ---- the cases: a fronto-parallel textured plane at constant depth ----------------------------------------------------------
# 400 x 126: bands of 160, 160 and 80 columns, 18 strips.  At constant depth each tile's footprint is the image of its
# corners, so the hull is the footprint.  The principal point is off the pixel grid and every pose carries a small
# sub-pixel shift, so the corner coordinates stay clear of integers.
W, H, DEPTH = 400, 126, 2.0
K = (300.3, 300.7, 199.37, 62.61)


def plane(seed=0):
    """(I, Z) of the textured plane: smooth random intensity, constant depth"""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[:H, :W].astype(np.float64)
    I = 128 + 0 * xx
    for _ in range(12):
        fx_, fy_, ph = rng.uniform(0.02, 0.25), rng.uniform(0.02, 0.25), rng.uniform(0, 2 * np.pi)
        I += rng.uniform(5, 15) * np.sin(fx_ * xx + fy_ * yy + ph)
    return np.clip(I, 0, 255).astype(np.float32), np.full((H, W), DEPTH, np.float32)


def _pose(roll_deg=0.0, dx_px=0.0, dy_px=0.0, scale=1.0):
    """roll about the optical axis, then a shift of the plane by (dx, dy) pixels and a move along the axis that scales it"""
    a = np.deg2rad(roll_deg)
    T = np.eye(4)
    T[:2, :2] = [[np.cos(a), -np.sin(a)], [np.sin(a), np.cos(a)]]
    T[0, 3] = (dx_px + 0.173) * DEPTH / K[0]
    T[1, 3] = (dy_px + 0.137) * DEPTH / K[1]
    T[2, 3] = DEPTH / scale - DEPTH
    return T


CASES = {
    "edges": _pose(),                                        # exact windows on replica rows -1, h and columns 0, w - 1
    **{f"roll{r}": _pose(roll_deg=r) for r in (2.3, 2.6, 2.9, 3.2)},
    **{f"forward{s}": _pose(scale=s) for s in (1.104, 1.112, 1.12, 1.128, 1.2)},
    "forward2.5": _pose(scale=2.5),                          # clips rows and columns
    "left_in": _pose(dx_px=-160.0),                          # band 0's hull ends at u = -0.83: kept
    "left_out": _pose(dx_px=-161.0),                         # and at u = -1.83: skipped
    "right_in": _pose(dx_px=79.5),                           # band 2's hull starts at u = 399.67 <= w: kept
    "right_out": _pose(dx_px=80.5),                          # and at u = 400.67 > w: skipped
    "top_in": _pose(dy_px=-7.0),                             # strip 0's hull ends at v = -0.86: kept
    "top_out": _pose(dy_px=-8.0),
    "bottom_in": _pose(dy_px=6.5),                           # the last strip (rows 119..125) starts at v = 125.64 <= h
    "bottom_out": _pose(dy_px=7.5),
}


def edge_tiles(wins, edge):
    """the safe tiles along an image edge: (kept, skipped) counts among tiles whose hull lies within 2 px of the edge"""
    kept = skipped = 0
    for wv in wins.values():
        if not wv["corners"] or not safe(wv):
            continue
        us, vs = [c[0] for c in wv["corners"]], [c[1] for c in wv["corners"]]
        near = {"left": -3 < max(us) < 1, "right": W - 1 < min(us) < W + 2, "top": -3 < max(vs) < 1,
                "bottom": H - 1 < min(vs) < H + 2}[edge]
        if near:
            skipped += wv["kind"] == "skip"
            kept += wv["kind"] != "skip"
    return kept, skipped
