"""Reference masks on top of the CPU oracle (test infrastructure; the oracle itself has no masks, as the reference has none).

The engine's rule (include/dvo_b200.h, dvo_b200_pyramid_create_masked_batch): a pixel of level l is usable iff every level-0
pixel of its footprint [x 2^l, (x+1) 2^l) x [y 2^l, (y+1) 2^l) is, and the selection is isPointOk(ti, td) AND usable.

The oracle's isPointOk needs a non-NaN depth (point_selection.h:63-66), and once a level is built its depth plane is read by
the point selection alone: the depth derivatives were taken at creation, and a pyramid in the reference role is never
sampled as bilinear taps.  So the masked oracle pyramid is the unmasked one with NaN written into the depth plane of every
unusable pixel after the build.  The gradients of the neighbours and the depth of every selected point stay as they are;
in every mode and every entry point (select, residual_image, linearize, intensity_error_image, match) the selection is then
isPointOk AND usable, and S, the odd last point and everything else follow from it.  Such a pyramid must only be used as the
REFERENCE of an alignment (a mask acts in that role only).
"""
import ctypes as C

import numpy as np


def usable_by_footprint(mask, levels):
    """per level, the (h_l, w_l) bool array of usable pixels: the direct footprint test, by block reduction of level 0"""
    h, w = mask.shape
    out = []
    lh, lw = h, w
    for l in range(levels):
        f = 1 << l
        out.append((np.asarray(mask)[:lh * f, :lw * f] != 0).reshape(lh, f, lw, f).all(axis=(1, 3)))
        lh, lw = lh // 2, lw // 2
    return out


def masked_pyramid(orc, intensity, depth, intrinsics, levels, mask=None):
    """oracle Pyramid for the REFERENCE role with a reference mask (h, w; nonzero = usable); mask=None: orc.Pyramid"""
    p = orc.Pyramid(intensity, depth, intrinsics, levels)
    if mask is None:
        return p
    assert np.asarray(mask).shape == np.asarray(intensity).shape
    for l, usable in enumerate(usable_by_footprint(mask, levels)):
        w, h, _ = p.level_info(l)
        assert usable.shape == (h, w)
        z = np.ctypeslib.as_array(C.cast(orc.lib().orc_pyramid_plane(p.h, l, 1), C.POINTER(C.c_float)), shape=(h, w))
        z[~usable] = np.nan
    return p
