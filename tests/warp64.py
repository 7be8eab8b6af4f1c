"""The weight maps of dvo_b200_match_batch_maps computed in plain fp64, and the forward-error bounds that hold a float32
kernel to them.

For each selected reference pixel (x, y) of level L -- Pyramid.select, without the odd last point under the reference
estimator (k_drop_odd_last), with it under the corrected one -- from the downloaded planes (Pyramid.download: I, Z):

  point      p = (tx z, ty z, z), tx = (x - ox) / fx, ty = (y - oy) / fy, z = Z_ref(x, y)        rgbd_image.cpp:197-198
  warp       (X, Y, Z') = K_cur [R | t] p with T^ = [R | t] (maps "estimate", reference -> current); (u, v) = (X, Y) / Z'
  bounds     0 <= u <= w - 2 and 0 <= v <= h - 2
  taps       (u0, v0) = floor(u, v); the (I, Z) of the current level at (u0 + {0, 1}, v0 + {0, 1})
  blend      bilinear I and Z with the weights of dense_tracking.cpp:215-220
  validity   Z finite (dense_tracking.cpp:261) and e_z > -20 sigma(z) (line 275), sigma of dense_tracking_impl.cpp:122-128
  residuals  e_i = (I - (alpha I_ref + beta)) / 255, e_z = Z - Z'
  weight     w = 7 / (5 + r^T P r), r = (e_i, e_z), P the kept precision P^
  mask       level 0: 0 where the level-L parent (X >> L, Y >> L) exists and is a constraint with w < mask_weight, else 1

Everything above is fp64 except the inputs themselves (float32 planes, intrinsics, P^; T^ and (alpha, beta) are fp64).

Bounds.  u = 2^-24 and gamma_k = k u / (1 - k u), as in tests/linearization_ledger.py.  A float32 evaluation of the operation
(the kernel's project_pixel / DVO_BLEND2 / residual sequence in stages.cuh, or the oracle's unfused one) rounds:
  K T       each entry fl(fl(f T0j) + fl(o T2j)) from fl(Tij): 3 roundings           -> |dKT_ij| <= gamma_3 KTa_ij
  p         fl(fl(fl(x - o) / f) z): 3 roundings                                      -> |dp_j| <= gamma_3 |p_j|
  X, Y, Z'  a dot product of 4 terms: 3 roundings fused, 4 unfused; Z' from fl(T2j)   -> gamma_10 S_X, gamma_8 S_Z
            with S_X = sum_j KTa_0j |p_j| (KTa = |f T0j| + |o T2j|, the last column times 1), S_Z = sum_j |T2j| |p_j|
  u = X/Z'  rcp_rn (2 ulp) and the multiply                                           -> gamma_3 |u|
so  delta_u = (gamma_10 S_X + gamma_8 |u| S_Z) / (|Z'| - gamma_8 S_Z) + gamma_3 |u|, and the same for v.
The blend is Lipschitz in (u, v) with the largest difference D of horizontally or vertically adjacent taps of the 4 x 4
neighbourhood of the cell (a position error that crosses a cell edge moves onto a neighbouring cell); its own rounding,
with g = 1 - f rounded, is at most gamma_8 max |tap|.  Per pixel:
  |dI| <= (delta_u + delta_v) D_I + gamma_8 max |I tap|       |dZ| <= (delta_u + delta_v) D_Z + gamma_8 max |Z tap|
  |e_i - e_i64| <= (|dI| + gamma_3 (|alpha I_ref| + |beta|) + gamma_3 (|I| + |alpha I_ref + beta|)) / 255
  |e_z - e_z64| <= |dZ| + gamma_8 S_Z + u |e_z|
Tie band: a pixel whose fp64 u or v lies within delta of a bound or of an integer (the tap cell, hence a NaN tap, can
change), or whose e_z lies within its bound plus gamma_4 |20 sigma| of the occlusion threshold.  Only there may the NaN
pattern differ.  Weights: |dw| <= 7 dd / ((5 + d)(5 + d - dd)) + 2^-21 w, dd the first- and second-order change of
d = r^T P r under the residual bounds plus gamma_4 sum |P_ij r_i r_j|; the mask may differ from the fp64 weights' mask only
where some parent lies in the tie band or within |dw| of mask_weight.
"""
from dataclasses import dataclass, field

import numpy as np

U32 = 2.0 ** -24
SIGMA = (np.float64(np.float32(0.0019)), np.float64(np.float32(0.4)), np.float64(np.float32(0.0012)))   # depth_sigma's constants


def gamma(k):
    return k * U32 / (1.0 - k * U32)


def selection(mask, estimator):
    """the constraint candidates of a level: the selection mask, less its odd last point under the reference estimator"""
    sel = np.asarray(mask).astype(bool)
    flat = np.flatnonzero(sel.reshape(-1))
    if estimator == "reference" and len(flat) % 2 == 1:
        sel.reshape(-1)[flat[-1]] = False
    return sel


def _adjacent_max(P, ys, xs, h, w):
    """largest |difference| of horizontally or vertically adjacent entries of P in the 4 x 4 block at rows ys - 1 .. ys + 2,
    columns xs - 1 .. xs + 2 (clipped to the image), NaN-free differences only"""
    best = np.zeros(len(ys))
    for dy in range(-1, 3):
        for dx in range(-1, 3):
            y0, x0 = np.clip(ys + dy, 0, h - 1), np.clip(xs + dx, 0, w - 1)
            for ey, ex in ((0, 1), (1, 0)):
                y1, x1 = np.clip(y0 + ey, 0, h - 1), np.clip(x0 + ex, 0, w - 1)
                d = np.abs(P[y1, x1].astype(np.float64) - P[y0, x0])
                best = np.fmax(best, np.where(np.isfinite(d), d, 0.0))
    return best


def warp64(ref_planes, cur_planes, sel, K_ref, K_cur, T, P, ab=None):
    """the fp64 maps of one pair at one level.  ref_planes / cur_planes: [>= 2, h, w] (I, Z, ...); sel: bool [h, w], the
    constraint candidates (selection()); K_*: (fx, fy, ox, oy) of the level; T: 4 x 4 fp64 reference -> current; P: 2 x 2.
    Returns a dict of [h, w] arrays: e_i, e_z, w (NaN where not a constraint), valid, tie, bound_i, bound_z."""
    Ir, Zr = ref_planes[0], ref_planes[1]
    Ic, Zc = cur_planes[0], cur_planes[1]
    h, w = Ir.shape
    fxr, fyr, oxr, oyr = (np.float64(np.float32(k)) for k in K_ref)
    fx, fy, ox, oy = (np.float64(np.float32(k)) for k in K_cur)
    T = np.asarray(T, dtype=np.float64).reshape(4, 4)
    alpha, beta = (1.0, 0.0) if ab is None else (float(ab[0]), float(ab[1]))
    ys, xs = np.nonzero(sel)
    z = Zr[ys, xs].astype(np.float64)
    p = np.stack([(xs - oxr) / fxr * z, (ys - oyr) / fyr * z, z, np.ones_like(z)])
    KT = np.stack([fx * T[0] + ox * T[2], fy * T[1] + oy * T[2], T[2]])
    KTa = np.stack([np.abs(fx * T[0]) + np.abs(ox * T[2]), np.abs(fy * T[1]) + np.abs(oy * T[2]), np.abs(T[2])])
    X, Y, Zt = KT @ p
    SX, SY, SZ = KTa @ np.abs(p)
    with np.errstate(divide="ignore", invalid="ignore"):
        u, v = X / Zt, Y / Zt
        den = np.abs(Zt) - gamma(8) * SZ
        du = (gamma(10) * SX + gamma(8) * np.abs(u) * SZ) / den + gamma(3) * np.abs(u)
        dv = (gamma(10) * SY + gamma(8) * np.abs(v) * SZ) / den + gamma(3) * np.abs(v)
    du = np.where(den > 0, du, np.inf)
    dv = np.where(den > 0, dv, np.inf)
    inb = (u >= 0) & (u <= w - 2) & (v >= 0) & (v <= h - 2)
    uc, vc = np.where(inb, u, 0.0), np.where(inb, v, 0.0)
    u0, v0 = np.floor(uc).astype(np.int64), np.floor(vc).astype(np.int64)
    fu, fv = uc - u0, vc - v0
    gu, gv = 1.0 - fu, 1.0 - fv

    def blend(Pl):
        c00, c10 = Pl[v0, u0].astype(np.float64), Pl[v0, u0 + 1].astype(np.float64)
        c01, c11 = Pl[v0 + 1, u0].astype(np.float64), Pl[v0 + 1, u0 + 1].astype(np.float64)
        with np.errstate(invalid="ignore"):
            val = fv * (fu * c11 + gu * c01) + gv * (fu * c10 + gu * c00)
        taps = np.abs(np.stack([c00, c10, c01, c11]))
        big = np.where(np.isnan(taps), 0.0, taps).max(axis=0) if len(c00) else np.zeros(0)
        return val, big
    I_b, I_big = blend(Ic)
    Z_b, Z_big = blend(Zc)
    Ir_ab = alpha * Ir[ys, xs].astype(np.float64) + beta
    ei = (I_b - Ir_ab) / 255.0
    ez = Z_b - Zt
    sig = SIGMA[0] * (z - SIGMA[1]) ** 2 + SIGMA[2]
    thr = -20.0 * sig
    with np.errstate(invalid="ignore"):
        valid = inb & np.isfinite(Z_b) & (ez > thr)
    DI, DZ = _adjacent_max(Ic, v0, u0, h, w), _adjacent_max(Zc, v0, u0, h, w)
    dpos = du + dv
    with np.errstate(invalid="ignore"):
        bI = dpos * DI + gamma(8) * I_big
        bZ = dpos * DZ + gamma(8) * Z_big
        b_i = (bI + gamma(3) * (np.abs(alpha * Ir[ys, xs]) + abs(beta)) + gamma(3) * (np.abs(I_b) + np.abs(Ir_ab))) / 255.0
        b_z = bZ + gamma(8) * SZ + U32 * np.abs(ez)
    b_i, b_z = np.where(np.isfinite(b_i), b_i, np.inf), np.where(np.isfinite(b_z), b_z, np.inf)

    def near(a, d, lo, hi):
        with np.errstate(invalid="ignore"):
            return (np.abs(a - lo) <= d) | (np.abs(a - hi) <= d) | (np.abs(a - np.round(a)) <= d) | ~np.isfinite(a)
    with np.errstate(invalid="ignore"):
        tie = near(u, du, 0.0, w - 2.0) | near(v, dv, 0.0, h - 2.0)
        tie |= inb & np.isfinite(Z_b) & (np.abs(ez - thr) <= b_z + gamma(4) * np.abs(thr))
    Pd = np.asarray(P, dtype=np.float64).reshape(2, 2)
    a, b = np.where(valid, ei, 0.0), np.where(valid, ez, 0.0)
    d = Pd[0, 0] * a * a + (Pd[0, 1] + Pd[1, 0]) * a * b + Pd[1, 1] * b * b
    wgt = 7.0 / (5.0 + d)
    ai, bi = np.where(valid, b_i, 0.0), np.where(valid, b_z, 0.0)
    Pa = np.abs(Pd)
    dd = (2 * Pa[0, 0] * np.abs(a) * ai + (Pa[0, 1] + Pa[1, 0]) * (np.abs(a) * bi + np.abs(b) * ai) + 2 * Pa[1, 1] * np.abs(b) * bi
          + Pa[0, 0] * ai * ai + (Pa[0, 1] + Pa[1, 0]) * ai * bi + Pa[1, 1] * bi * bi
          + gamma(4) * (Pa[0, 0] * a * a + (Pa[0, 1] + Pa[1, 0]) * np.abs(a * b) + Pa[1, 1] * b * b))
    with np.errstate(divide="ignore", invalid="ignore"):
        bw = np.where(5.0 + d - dd > 0, 7.0 * dd / ((5.0 + d) * (5.0 + d - dd)), np.inf) + 2.0 ** -21 * wgt

    def img(vals, fill):
        out = np.full((h, w), fill, dtype=vals.dtype if vals.dtype == bool else np.float64)
        out[ys, xs] = vals
        return out
    nan = np.nan
    return {"sel": sel, "valid": img(valid, False), "tie": img(tie, False),
            "e_i": img(np.where(valid, ei, nan), nan), "e_z": img(np.where(valid, ez, nan), nan),
            "w": img(np.where(valid, wgt, nan), nan), "bound_i": img(b_i, 0.0), "bound_z": img(b_z, 0.0),
            "bound_w": img(np.where(valid, bw, 0.0), 0.0), "u": img(u, nan), "v": img(v, nan)}


def footprint(parent, level, shape0):
    """bool [h0, w0]: the level-L parent (x >> L, y >> L) of each level-0 pixel exists and `parent` holds there"""
    h0, w0 = shape0
    h, w = parent.shape
    ys, xs = np.mgrid[0:h0, 0:w0]
    py, px = ys >> level, xs >> level
    inside = (py < h) & (px < w)
    out = np.zeros((h0, w0), bool)
    out[inside] = parent[py[inside], px[inside]]
    return out


@dataclass
class Report:
    maxima: dict = field(default_factory=lambda: {"e_i": 0.0, "e_z": 0.0})   # largest |kernel - fp64| / bound
    tie: int = 0              # constraint candidates in the tie band
    candidates: int = 0
    failures: list = field(default_factory=list)


def compare(ref, e_i, e_z, weight=None, mask=None, level=0, mask_weight=None, report=None):
    """kernel maps (e_i, e_z [h, w] float32; weight; mask [h0, w0] uint8) against warp64's `ref`"""
    rep = report or Report()
    tie, valid = ref["tie"], ref["valid"]
    fin = np.isfinite(e_i)
    rep.tie += int(tie.sum())
    rep.candidates += int(ref["sel"].sum())
    if not np.array_equal(fin, np.isfinite(e_z)):
        rep.failures.append(("nan", "e_i and e_z have different NaN patterns"))
    off = (fin != valid) & ~tie
    if off.any():
        y, x = np.argwhere(off)[0]
        rep.failures.append(("validity", f"{int(off.sum())} pixels outside the tie band, first ({y}, {x}): kernel "
                                         f"{'valid' if fin[y, x] else 'NaN'}, fp64 {'valid' if valid[y, x] else 'NaN'}"))
    both = fin & valid
    for name, g, b in (("e_i", e_i, ref["bound_i"]), ("e_z", e_z, ref["bound_z"])):
        err = np.abs(g[both].astype(np.float64) - ref[name][both])
        bnd = b[both]
        if err.size:
            q = np.where(bnd > 0, err / np.where(bnd > 0, bnd, 1.0), np.where(err > 0, np.inf, 0.0))
            rep.maxima[name] = max(rep.maxima[name], float(q.max()))
            if (q > 1.0).any():
                k = int(np.argmax(q))
                rep.failures.append((name, f"{int((q > 1).sum())} pixels past the bound, worst {err[k]:.3e} > {bnd[k]:.3e}"))
    if weight is not None and not np.array_equal(np.isfinite(weight), fin):
        rep.failures.append(("weight", "weight and residuals have different NaN patterns"))
    if mask is not None:
        with np.errstate(invalid="ignore"):
            out64 = valid & (ref["w"] < mask_weight)
            wtie = tie | (valid & (np.abs(ref["w"] - mask_weight) <= ref["bound_w"]))
        shape0 = mask.shape
        want = np.where(footprint(out64, level, shape0), 0, 1).astype(np.uint8)
        free = footprint(wtie, level, shape0)
        bad = (mask != want) & ~free
        if bad.any():
            y, x = np.argwhere(bad)[0]
            rep.failures.append(("mask", f"{int(bad.sum())} bytes, first ({y}, {x}) = {mask[y, x]}, want {want[y, x]}"))
    return rep
