"""The fp64 warp of the weight maps (tests/warp64.py) established on the CPU: it agrees with the oracle's EXACT residual image
at the tile-edge sizes of test_gpu_geometry.py within its own bounds, and a float32 restatement shaped like k_weight_maps
(csrc/weight_maps.cu) passes against it while each planted defect of that restatement is reported -- the bounds are tight
enough to matter.

A transposed P is not among the defects: the weight reads P only through r^T P r = P00 ei^2 + (P01 + P10) ei ez + P11 ez^2,
which no transposition changes, so no test of the maps can see one.  Swapping P's diagonal stands in for a misread P.
"""
import numpy as np
import pytest

import warp64 as W
from test_gpu_geometry import SIZES, _edge_shift, _intrinsics, _scene, _small_motion
from tile_geometry import level_shapes
from weight_maps_model import _fma32

P_KEPT = np.array([[2100.0, -35.0], [-35.0, 8700.0]], dtype=np.float32)     # of the order of a kept precision at these sizes
AB = (1.1, -7.5)
MASK_WEIGHT = 0.3
DEFECTS = ("swap_fu_gu", "tap_row_off", "pitch_for_w", "footprint_unwritten", "P_diagonal_swapped")
SENTINEL_F, SENTINEL_B = np.float32(-12345.0), np.uint8(9)


def _planes(op, level):
    """the oracle pyramid's planes as Pyramid.download returns them: depth NaN where any channel is"""
    pl = op.planes(level)
    pl[1][np.isnan(pl).any(axis=0)] = np.nan
    return pl


def kernel32(ref, cur, sel, Kr, Kc, T, P, ab, level, shape0, defect=None):
    """k_weight_maps restated in float32 with its layout: a current plane of even row pitch, the template tx[0, w) then
    ty[0, h), padded outputs (rows w + 3 floats, mask rows w0 + 5 bytes) prefilled with a sentinel.  Returns the padded
    (weight, e_i, e_z, mask)."""
    f32 = np.float32
    h, w = ref.shape[1:]
    h0, w0 = shape0
    pitch = w + (w & 1)
    Ic = np.full((h, pitch), np.nan, f32); Ic[:, :w] = cur[0]
    Zc = np.full((h, pitch), np.nan, f32); Zc[:, :w] = cur[1]
    fxr, fyr, oxr, oyr = (f32(k) for k in Kr)
    tmpl = np.concatenate([(np.arange(w, dtype=f32) - oxr) / fxr, (np.arange(h, dtype=f32) - oyr) / fyr, np.zeros(2, f32)]).astype(f32)
    fx, fy, ox, oy = (f32(k) for k in Kc)
    t = np.asarray(T, dtype=np.float64).reshape(4, 4).astype(f32)
    kt = np.zeros((3, 4), f32)
    for j in range(4):
        kt[0, j] = f32(fx * t[0, j]) + f32(ox * t[2, j])
        kt[1, j] = f32(fy * t[1, j]) + f32(oy * t[2, j])
        kt[2, j] = t[2, j]
    Pk = np.asarray(P, f32).reshape(4).copy()
    if defect == "P_diagonal_swapped":
        Pk[0], Pk[3] = Pk[3], Pk[0]
    alpha, beta = f32(ab[0]), f32(ab[1])
    ys, xs = np.nonzero(sel)
    z = ref[1][ys, xs].astype(f32)
    ty = tmpl[(pitch if defect == "pitch_for_w" else w) + ys]
    px, py = (tmpl[xs] * z).astype(f32), (ty * z).astype(f32)

    def chain(r):
        return _fma32(np.full_like(px, kt[r, 0]), px, _fma32(np.full_like(py, kt[r, 1]), py, _fma32(np.full_like(z, kt[r, 2]), z,
                                                                                                   np.full_like(z, kt[r, 3]))))
    X, Y, Zt = chain(0), chain(1), chain(2)
    with np.errstate(divide="ignore", invalid="ignore"):
        rz = (f32(1.0) / Zt).astype(f32)
        u, v = (X * rz).astype(f32), (Y * rz).astype(f32)
        inb = (u >= 0) & (u <= f32(w - 2)) & (v >= 0) & (v <= f32(h - 2))
    u, v = np.where(inb, u, f32(0)), np.where(inb, v, f32(0))
    u0, v0 = np.floor(u).astype(np.int64), np.floor(v).astype(np.int64)
    fu, fv = (u - u0).astype(f32), (v - v0).astype(f32)
    gu, gv = (f32(1) - fu).astype(f32), (f32(1) - fv).astype(f32)
    if defect == "swap_fu_gu":
        fu, gu = gu, fu
    r1 = np.minimum(v0 + (2 if defect == "tap_row_off" else 1), h - 1)

    def blend(Pl):
        c00, c10, c01, c11 = Pl[v0, u0], Pl[v0, u0 + 1], Pl[r1, u0], Pl[r1, u0 + 1]
        with np.errstate(invalid="ignore"):
            a = _fma32(fu, c11, (gu * c01).astype(f32))
            b = _fma32(fu, c10, (gu * c00).astype(f32))
            return _fma32(fv, a, (gv * b).astype(f32))
    I_b, Z_b = blend(Ic), blend(Zc)
    ci = f32(1.0 / 255.0)
    Ir = _fma32(np.full_like(z, alpha), ref[0][ys, xs], np.full_like(z, beta))
    with np.errstate(invalid="ignore"):
        ez = (Z_b - Zt).astype(f32)
        ei = _fma32(np.full_like(z, ci), I_b, (-ci * Ir).astype(f32))
        s = (z - f32(0.4)).astype(f32)
        sig = _fma32((f32(0.0019) * s).astype(f32), s, np.full_like(s, f32(0.0012)))
        ok = inb & (Z_b == Z_b) & (ez > (f32(-20.0) * sig).astype(f32))
        q0 = _fma32(ez, np.full_like(ez, Pk[2]), (ei * Pk[0]).astype(f32))
        q1 = _fma32(ez, np.full_like(ez, Pk[3]), (ei * Pk[1]).astype(f32))
        d = _fma32(q0, ei, (q1 * ez).astype(f32))
        wg = (f32(7.0) * (f32(1.0) / (f32(5.0) + d)).astype(f32)).astype(f32)
    nan = f32(np.nan)
    planes = []
    for val in (wg, ei, ez):
        out = np.full((h + 1, w + 3), SENTINEL_F, f32)
        out[:h, :w] = nan
        out[ys, xs] = np.where(ok, val, nan)
        planes.append(out)
    outlier = np.zeros((h, w), bool)
    outlier[ys, xs] = ok & (wg < f32(MASK_WEIGHT))
    mask = np.full((h0, w0 + 5), SENTINEL_B, np.uint8)
    s_ = 1 << level
    gx = w if defect == "footprint_unwritten" else max(w, -(-w0 // s_))
    gy = h if defect == "footprint_unwritten" else max(h, -(-h0 // s_))
    for y in range(gy):
        for x in range(gx):
            y0, x0 = y << level, x << level
            if x0 < w0 and y0 < h0:
                b = 0 if (x < w and y < h and outlier[y, x]) else 1
                mask[y0:min(y0 + s_, h0), x0:min(x0 + s_, w0)] = b
    return planes[0], planes[1], planes[2], mask


def _case(oracle, w, h, levels, level, estimator):
    a = _scene(w, h)
    K = _intrinsics(w, h)
    op = oracle.Pyramid(a["I_ref"], a["Z_ref"], K, levels)
    oc = oracle.Pyramid(a["I_cur"], a["Z_cur"], K, levels)
    S, m = oracle.select(op, level)
    Kl = op.level_info(level)[2]
    return op, oc, W.selection(m, estimator), Kl


def _check_kernel32(oracle, w, h, levels, level, estimator, defect=None):
    op, oc, sel, Kl = _case(oracle, w, h, levels, level, estimator)
    T = _small_motion()
    ref, cur = _planes(op, level), _planes(oc, level)
    shape0 = level_shapes(w, h, levels)[0][::-1]
    want = W.warp64(ref, cur, sel, Kl, Kl, T, P_KEPT, AB)
    wg, ei, ez, mask = kernel32(ref, cur, sel, Kl, Kl, T, P_KEPT, AB, level, shape0, defect)
    lh, lw = ref.shape[1:]
    rep = W.compare(want, ei[:lh, :lw], ez[:lh, :lw], wg[:lh, :lw], mask[:, :shape0[1]], level, MASK_WEIGHT)
    # the restatement's weights are those of its own residuals and (possibly misread) P; against the fp64 weights of P^:
    fin = np.isfinite(wg[:lh, :lw]) & want["valid"]
    dw = np.abs(wg[:lh, :lw][fin] - want["w"][fin])
    if (dw > want["bound_w"][fin]).any():
        rep.failures.append(("weight", f"{int((dw > want['bound_w'][fin]).sum())} weights past their bound"))
    if (wg[lh:] != SENTINEL_F).any() or (wg[:, lw:] != SENTINEL_F).any() or (mask[:, shape0[1]:] != SENTINEL_B).any():
        rep.failures.append(("outside", "a byte outside the extents was written"))
    return rep, sel.sum()


ODD = [s for s in SIZES if s[0] % 2]


@pytest.mark.parametrize("estimator", ["reference", "corrected"])
@pytest.mark.parametrize("w,h,levels", SIZES, ids=[f"{w}x{h}" for w, h, _ in SIZES])
def test_warp64_agrees_with_the_exact_oracle(oracle, w, h, levels, estimator):
    """the oracle's EXACT residual image (fp32, unfused, exact division) within warp64's bounds, at every level, with the
    photometric (alpha, beta), at the two poses of test_gpu_geometry; the NaN pattern differs only in the tie band (not the
    identity pose: every pixel would warp onto an integer)"""
    a = _scene(w, h)
    K = _intrinsics(w, h)
    op = oracle.Pyramid(a["I_ref"], a["Z_ref"], K, levels)
    oc = oracle.Pyramid(a["I_cur"], a["Z_cur"], K, levels)
    mode = oracle.mode("exact")
    if estimator == "reference":
        mode.drop_odd_point = 1
    rep = W.Report()
    for level in range(levels):
        S, m = oracle.select(op, level)
        Kl = op.level_info(level)[2]
        ref, cur = _planes(op, level), _planes(oc, level)
        for T in (_small_motion(), _edge_shift(w, h, K, a["Z_ref"])):
            n, img = oracle.residual_image(op, oc, level, T, mode, ab=AB)
            want = W.warp64(ref, cur, W.selection(m, estimator), Kl, Kl, T, P_KEPT, AB)
            W.compare(want, img[0], img[1], report=rep)
    assert not rep.failures, rep.failures[:4]
    assert rep.candidates > 0 and rep.tie <= 0.01 * rep.candidates, (rep.tie, rep.candidates)
    print(f"{w}x{h} {estimator}: |oracle - fp64| / bound {rep.maxima}, tie band {rep.tie} of {rep.candidates}")


def test_exact_mode_is_a_different_evaluation(oracle):
    """the comparison above is not vacuous: EXACT's residuals are not warp64's fp64 values rounded to float32"""
    w, h, levels = SIZES[0]
    op, oc, sel, Kl = _case(oracle, w, h, levels, 0, "corrected")
    n, img = oracle.residual_image(op, oc, 0, _small_motion(), oracle.mode("exact"), ab=AB)
    want = W.warp64(_planes(op, 0), _planes(oc, 0), sel, Kl, Kl, _small_motion(), P_KEPT, AB)
    both = np.isfinite(img[0]) & want["valid"]
    assert both.sum() > 100 and (img[0][both] != want["e_i"][both].astype(np.float32)).any()


@pytest.mark.parametrize("estimator", ["reference", "corrected"])
@pytest.mark.parametrize("w,h,levels", ODD, ids=[f"{w}x{h}" for w, h, _ in ODD])
def test_kernel_restatement_passes(oracle, w, h, levels, estimator):
    for level in (0, levels - 1):
        rep, n = _check_kernel32(oracle, w, h, levels, level, estimator)
        assert n > 0 and not rep.failures, (level, rep.failures[:4])


@pytest.mark.parametrize("defect", DEFECTS)
def test_each_planted_defect_is_reported(oracle, defect):
    """at 161 x 50 (odd width: pitch != w; odd level sizes below it: level-0 pixels with no parent at the last level)"""
    w, h, levels = 161, 50, 3
    shapes = level_shapes(w, h, levels)
    assert w % 2 == 1 and (shapes[-1][0] << (levels - 1)) < w and (shapes[-1][1] << (levels - 1)) < h
    level = 0 if defect != "footprint_unwritten" else levels - 1
    rep, _ = _check_kernel32(oracle, w, h, levels, level, "corrected", defect)
    assert rep.failures, defect
    print(defect, "->", rep.failures[0])
