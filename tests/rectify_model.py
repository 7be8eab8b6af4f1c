"""numpy restatement of the rectifying remap (include/dvo_b200.h, dvo_b200_pyramid_create_rectified_batch) and of
dvo_b200_undistort_map, operation for operation: the rectified pyramids must equal, bit for bit, the float32 pyramids
built from what remap() returns, and undistort_map() must equal the library's map exactly."""
import numpy as np

F32 = np.float32


def undistort_map(width, height, K, dist, K_new=None):
    """(map_x, map_y) float32 [height, width]: the header's operation order in float64, rounded once to float32"""
    fx, fy, cx, cy = (float(v) for v in K)
    nfx, nfy, ncx, ncy = (float(v) for v in (K if K_new is None else K_new))
    k1, k2, p1, p2, k3 = (float(v) for v in dist)
    u = np.arange(width, dtype=np.float64)[None, :]
    v = np.arange(height, dtype=np.float64)[:, None]
    x = (u - ncx) / nfx
    y = (v - ncy) / nfy
    r2 = x * x + y * y
    kr = ((k3 * r2 + k2) * r2 + k1) * r2
    dx = x * kr + ((2 * p1) * x * y + p2 * (r2 + 2 * x * x))
    dy = y * kr + (p1 * (r2 + 2 * y * y) + (2 * p2) * x * y)
    mx = (cx + (fx / nfx) * (u - ncx)) + fx * dx
    my = (cy + (fy / nfy) * (v - ncy)) + fy * dy
    return mx.astype(F32), my.astype(F32)


def grey_of_bgr(bgr):
    """OpenCV's 8-bit BGR2GRAY, as dvo_b200_pyramid_create_bgr_batch reduces BGR"""
    b, g, r = (bgr[..., k].astype(np.int64) for k in range(3))
    return ((1868 * b + 9617 * g + 4899 * r + 8192) >> 14).astype(np.uint8)


def remap(image, depth, map_x, map_y, mask=None, depth_scale=None):
    """One frame through the map: (I, Z, usable) float32 / float32 / uint8 of the map's shape.  image: float32 or uint8
    grey [h, w] (reduce BGR with grey_of_bgr first); depth: float32 metres or uint16 raw (then depth_scale); mask: None or
    [h, w], nonzero = usable (usable is then None too)."""
    h, w = depth.shape
    sx, sy = np.asarray(map_x, F32), np.asarray(map_y, F32)
    with np.errstate(invalid="ignore"):
        valid = (sx >= 0) & (sx <= F32(w - 1)) & (sy >= 0) & (sy <= F32(h - 1))
    x0 = np.where(valid, np.minimum(np.floor(np.where(valid, sx, 0)), w - 2), 0).astype(np.int64)
    y0 = np.where(valid, np.minimum(np.floor(np.where(valid, sy, 0)), h - 2), 0).astype(np.int64)
    ax = (np.where(valid, sx, 0) - x0.astype(F32)).astype(F32)
    ay = (np.where(valid, sy, 0) - y0.astype(F32)).astype(F32)
    bx, by = F32(1) - ax, F32(1) - ay
    I = np.asarray(image).astype(F32)
    i00, i10, i01, i11 = I[y0, x0], I[y0, x0 + 1], I[y0 + 1, x0], I[y0 + 1, x0 + 1]
    with np.errstate(invalid="ignore"):
        top = bx * i00 + ax * i10
        bot = bx * i01 + ax * i11
        v = by * top + ay * bot
    xn, yn = x0 + (ax >= F32(0.5)), y0 + (ay >= F32(0.5))
    if depth.dtype == np.uint16:
        raw = depth[yn, xn]
        z = np.where(raw == 0, F32(np.nan), raw.astype(F32) * F32(depth_scale)).astype(F32)
    else:
        z = np.asarray(depth, F32)[yn, xn]
    nan = F32(np.nan)
    v = np.where(valid, v, nan).astype(F32)
    z = np.where(valid, z, nan).astype(F32)
    if mask is None:
        return v, z, None
    m = np.asarray(mask) != 0
    usable = valid & m[y0, x0] & m[y0, x0 + 1] & m[y0 + 1, x0] & m[y0 + 1, x0 + 1]
    return v, z, usable.astype(np.uint8)


def remap_batch(image, depth, map_x, map_y, masks=None, depth_scale=None):
    """remap over n frames: image [n,h,w] (float32 or uint8 grey) or [n,h,w,3] BGR, depth [n,h,w]; masks None, [h,w] or
    [n,h,w].  Returns (I, Z, M) stacked, M None without masks."""
    image = np.asarray(image)
    if image.ndim == 4:
        image = grey_of_bgr(image)
    n = image.shape[0]
    if masks is not None:
        masks = np.broadcast_to(np.asarray(masks), depth.shape)
    out = [remap(image[i], depth[i], map_x, map_y, None if masks is None else masks[i], depth_scale) for i in range(n)]
    I = np.stack([o[0] for o in out])
    Z = np.stack([o[1] for o in out])
    M = None if masks is None else np.stack([o[2] for o in out])
    return I, Z, M


def oracle_pyramid(orc, intensity, depth, intrinsics, levels):
    """The oracle pyramid of rectified planes under the engine's rule for NaN channels: a pixel with a NaN intensity or
    intensity gradient is neither a reference point nor a bilinear tap (include/dvo_b200.h, dvo_b200_pyramid_download: Z is
    NaN wherever any channel is).  The reference's isPointOk tests the depth channels only, because an intensity read from
    an image file is never NaN; rectified planes have NaN intensities, and at coarse levels the 2x2 mean carries them onto
    pixels whose subsampled depth is valid.  Such a pixel would be selected by the bare oracle and its NaN residual would
    poison the level's scale estimate.  So, as tests/masked_oracle.py does for masks, NaN is written into the depth plane of
    every level wherever I, Ix or Iy is NaN, after the build.  At level 0 this changes nothing: an invalid pixel has NaN
    depth too, and so do the depth derivatives of its neighbours."""
    import ctypes as C
    p = orc.Pyramid(intensity, depth, intrinsics, levels)
    for l in range(levels):
        w, h, _ = p.level_info(l)
        ch = [np.ctypeslib.as_array(C.cast(orc.lib().orc_pyramid_plane(p.h, l, c), C.POINTER(C.c_float)), shape=(h, w)) for c in (0, 1, 2, 3)]
        ch[1][np.isnan(ch[0]) | np.isnan(ch[2]) | np.isnan(ch[3])] = np.nan
    return p
