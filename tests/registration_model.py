"""numpy restatement of dvo_b200_depth_rays and of the depth registration (include/dvo_b200.h,
dvo_b200_pyramid_create_registered_batch), operation for operation: depth_rays() must equal the library's tables exactly,
and the registered pyramids must equal, bit for bit, the float32 pyramids built from what register_batch() returns.
Every float32 operation runs on float32 arrays and np.float32 scalars, so nothing promotes to float64."""
import numpy as np

import rectify_model as rm

F32 = np.float32
MAX_FOOTPRINT = 8          # DVO_B200_REGISTRATION_MAX_FOOTPRINT
MAX_ITER = 100             # DVO_B200_DEPTH_RAYS_MAX_ITER
TOL = 1e-12


def _undistort(xd, yd, dist):
    """Newton's method per point, in the header's order; a point stops updating once its residual is below TOL"""
    k1, k2, p1, p2, k3 = (float(v) for v in dist)
    x, y = xd.copy(), yd.copy()
    active = np.ones(x.shape, bool)
    for it in range(MAX_ITER + 1):
        r2 = x * x + y * y
        R = 1 + ((k3 * r2 + k2) * r2 + k1) * r2
        dR = k1 + (2 * k2 + 3 * k3 * r2) * r2
        ex = x * R + 2 * p1 * x * y + p2 * (r2 + 2 * x * x) - xd
        ey = y * R + p1 * (r2 + 2 * y * y) + 2 * p2 * x * y - yd
        with np.errstate(invalid="ignore"):
            active &= ~((np.abs(ex) < TOL) & (np.abs(ey) < TOL))
        if not active.any():
            return x, y
        if it == MAX_ITER:
            raise ValueError("depth_rays: no convergence")
        a = R + 2 * x * x * dR + 2 * p1 * y + 6 * p2 * x
        b = 2 * x * y * dR + 2 * p1 * x + 2 * p2 * y
        d = R + 2 * y * y * dR + 6 * p1 * y + 2 * p2 * x
        det = a * d - b * b
        nx, ny = x - (d * ex - b * ey) / det, y - (a * ey - b * ex) / det
        x, y = np.where(active, nx, x), np.where(active, ny, y)
    raise AssertionError("unreachable")


def depth_rays(size, K, dist=None):
    """(cx_ray, cy_ray, kx_ray, ky_ray): float32 [dh, dw] centre rays and [dh+1, dw+1] corner rays"""
    dw, dh = size
    fx, fy, cx, cy = (float(v) for v in K)

    def rays(u, v):
        xd, yd = (u - cx) / fx, (v - cy) / fy
        xd, yd = np.broadcast_arrays(xd, yd)
        x, y = (xd.copy(), yd.copy()) if dist is None else _undistort(xd.copy(), yd.copy(), dist)
        return x.astype(F32), y.astype(F32)

    c = rays(np.arange(dw, dtype=np.float64)[None, :], np.arange(dh, dtype=np.float64)[:, None])
    k = rays(np.arange(dw + 1, dtype=np.float64)[None, :] - 0.5, np.arange(dh + 1, dtype=np.float64)[:, None] - 0.5)
    return c[0], c[1], k[0], k[1]


def depth_metres(depth, depth_scale=None):
    """float32 metres: as given, or u16 * depth_scale with 0 -> NaN"""
    depth = np.asarray(depth)
    if depth.dtype == np.uint16:
        return np.where(depth == 0, F32(np.nan), depth.astype(F32) * F32(depth_scale)).astype(F32)
    return depth.astype(F32)


def _row(R, t, r, X, Y, Z):
    return ((R[r, 0] * X + R[r, 1] * Y) + R[r, 2] * Z) + t[r]


def register(depth, rays, T, size, K, depth_scale=None):
    """One depth frame [dh, dw] -> the registered float32 depth plane [h, w] of the colour camera (NaN: uncovered)"""
    w, h = size
    R = np.asarray(T, np.float64)[:3, :3].astype(F32)
    t = np.asarray(T, np.float64)[:3, 3].astype(F32)
    fx, fy, cx, cy = (F32(v) for v in K)
    crx, cry, kx, ky = rays
    d = depth_metres(depth, depth_scale)
    dh, dw = d.shape
    ok = np.isfinite(d) & (d > F32(0))
    d = np.where(ok, d, F32(1)).astype(F32)
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        zc = _row(R, t, 2, crx * d, cry * d, d)
        ok &= zc > F32(0)
        xs, ys = [], []
        for a, b in ((0, 0), (0, 1), (1, 0), (1, 1)):
            X, Y = kx[a:a + dh, b:b + dw] * d, ky[a:a + dh, b:b + dw] * d
            zk = _row(R, t, 2, X, Y, d)
            ok &= zk > F32(0)
            x = fx * (_row(R, t, 0, X, Y, d) / zk) + cx
            y = fy * (_row(R, t, 1, X, Y, d) / zk) + cy
            ok &= (np.abs(x) < F32(2 ** 20)) & (np.abs(y) < F32(2 ** 20))
            xs.append(x)
            ys.append(y)
    xs = np.where(ok, np.stack(xs), F32(0))
    ys = np.where(ok, np.stack(ys), F32(0))
    x0, x1 = np.ceil(xs.min(0)).astype(np.int64), np.ceil(xs.max(0)).astype(np.int64)
    y0, y1 = np.ceil(ys.min(0)).astype(np.int64), np.ceil(ys.max(0)).astype(np.int64)
    ok &= (x1 - x0 <= MAX_FOOTPRINT) & (y1 - y0 <= MAX_FOOTPRINT)
    zbuf = np.full(h * w, 0xFFFFFFFF, np.uint32)
    bits = zc.astype(F32).view(np.uint32)
    for oy in range(MAX_FOOTPRINT):
        for ox in range(MAX_FOOTPRINT):
            xx, yy = x0 + ox, y0 + oy
            sel = ok & (xx < x1) & (yy < y1) & (xx >= 0) & (xx < w) & (yy >= 0) & (yy < h)
            np.minimum.at(zbuf, yy[sel] * w + xx[sel], bits[sel])
    Z = zbuf.view(F32).copy()
    Z[zbuf == 0xFFFFFFFF] = F32(np.nan)
    return Z.reshape(h, w)


def register_batch(image, depth, rays, T, size, K, masks=None, depth_scale=None, rect_map=None):
    """The planes the registered create builds from: (I, Z, M) float32 / float32 / uint8 stacked over n frames, M None
    without masks.  image: float32 or uint8 grey [n, h, w] or BGR [n, h, w, 3] of the colour frames; depth [n, dh, dw];
    masks None, [h, w] or [n, h, w] in the colour frames' geometry; rect_map: None or (map_x, map_y) of a rectifier."""
    image = np.asarray(image)
    if image.ndim == 4:
        image = rm.grey_of_bgr(image)
    n = image.shape[0]
    Z = np.stack([register(depth[i], rays, T, size, K, depth_scale) for i in range(n)])
    if masks is not None:
        masks = np.broadcast_to(np.asarray(masks), image.shape)
    if rect_map is None:
        I = image.astype(F32)
        M = None if masks is None else (masks != 0).astype(np.uint8)
        return I, Z, M
    dummy = np.zeros(image.shape[1:], F32)
    out = [rm.remap(image[i], dummy, rect_map[0], rect_map[1], None if masks is None else masks[i]) for i in range(n)]
    I = np.stack([o[0] for o in out])
    M = None if masks is None else np.stack([o[2] for o in out])
    return I, Z, M
