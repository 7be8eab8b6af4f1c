"""The level kernel's tile geometry, in one place for the whole suite.

The kernel cuts every pyramid level into strips of TILE_H rows and bands of TILE_W columns (kTileW, kTileH of
csrc/create_args.h); the last band of a strip is partial when the level's width is not a multiple of TILE_W, and partial
bands take the generic pixel loop.  Each tile stages a window of the current image of at most WIN_COLS x WIN_ROWS
(kWinCols, kWinRows of csrc/stages.cuh).  test_band_width.py::test_tile_geometry compares these numbers with the compiled
header, so that a kernel change that moves them fails a CPU test instead of leaving the GPU tests' geometry claims
describing a kernel that no longer exists.
"""
TILE_W, TILE_H = 160, 7
WIN_COLS = TILE_W + 24
WIN_ROWS = 19


def bands(w):
    """widths of the bands of a level of width w, left to right"""
    return [min(TILE_W, w - x0) for x0 in range(0, w, TILE_W)]


def strips(h):
    """heights of the strips of a level of height h, top to bottom"""
    return [min(TILE_H, h - y0) for y0 in range(0, h, TILE_H)]


def level_shapes(w, h, levels):
    """(w, h) of every pyramid level, level 0 first (each level halves, rounding down)"""
    out = []
    for _ in range(levels):
        out.append((w, h))
        w, h = w // 2, h // 2
    return out


def has_partial_band(w):
    return w % TILE_W != 0


def assert_partial_band(w):
    """a level of width w has at least one full band (exact loops) and a partial last band (generic loop)"""
    b = bands(w)
    assert len(b) >= 2 and b[-1] < TILE_W, f"{w} columns are bands {b}: not full bands followed by a partial one"
    return b


def in_partial_band(x, w):
    """pixel column x of a level of width w lies in its partial last band"""
    return has_partial_band(w) and x >= (w // TILE_W) * TILE_W
