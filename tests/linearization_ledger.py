"""An fp64 ledger of one linearisation of the level kernel, entry by entry, from the kernel's own residual records.

Inputs, for one (reference, current, level, T[, alpha, beta], estimator, use_weights, prev_precision): the seven record
planes of residual_image (e_i, e_z, gx, gy, hx, hy, z; NaN where a pixel is not a valid point), the level's intrinsics
K 2^-l, the reference intensity of the level (the photometric columns), and the P_k the kernel returned.  From these, in
fp64 and in the plain mathematics of the reference's formulas:

  n        the number of finite records (raster order is rank order)
  w        7 / (5 + r^T P_{k-1} r), or 1 on a level's first iteration                  dense_tracking_impl.cpp:657-707
  scale    REFERENCE: each leader's residual with both weights of its pair over the compacted raster list, plus the odd
           last point with its own (computeScaleSse's pair quirk); CORRECTED: sum w r r^T.  Covariance = scale / (n - 3),
           P = its inverse
  ll       0.5 n log det P_k - 3.5 sum log(1 + 0.2 r^T P_k r); REFERENCE drops the last n mod 50 ranks, CORRECTED none
  A, b     A = sum w J^T P_k J, b = -sum w J^T P_k r, J at the untransformed reference point x = tx z, y = ty z
           (dense_tracking.cpp:448-476); the photometric mode adds -c_i I_ref and -c_i to the intensity row (8 x 8)

Every entry also gets M, its absolute sum: the same sum with every factor replaced by its absolute value, expanded down
to the record values (|gx| |Jw0| + |gy| |Jw1| with |Jw0| = [1/z, 0, |x|/z^2, |x y|/z^2, 1 + x^2/z^2, |y|/z], |w|, |P|).
The acceptance rule is |kernel - ledger| <= gamma_k M + E, gamma_k = k u / (1 - k u) (Higham), u = 2^-24, where E adds
the approximate operations' documented errors and the rounding of the output itself.  Nothing in it is fitted.

Counts (dvo_slam_b200/csrc/stages.cuh; "units" are multiples of u in a factor's relative error):

  A   stage_b_pixel (stages.cuh:1037-1060) forms each point's J^T P J as two rank-1 updates, d0 j0' j0'^T + d1 J1 J1^T with
      l = P01/P00, d0 = P00, d1 = P11 - P01 l (load_stage_b_consts, :1265-1267), j0' = J0 + l J1.  Since d1 + P01^2/P00 =
      P11, the absolute sum of that form is <= |J|^T |P| |J|: M bounds it.  One entry of V0 / V1 (:1052-1057) carries
      at most 13 units: rcp_fast(z) 2 (rcp.approx.f32: 1 ulp), zs = zi^2 5, a2 = -px zs 7 (px = tx z: 1), a3 = a2 py 9,
      b2 py - 1 and 1 - a2 px 9, Gp = G + l H 2 (l: the IEEE division, 1), and three products chained by two FMAs:
      gy' (b2 py - 1) = 2 + 9 + 2 = 13.  A term u_r v_c with u_r = v_r (w d) (:1017): 13 + 13 + 1 (u_r) + 1 (w d) + 6
      (d1: l, product, difference = 3 units of P11 + P01^2/P00 <= 2 P11) = 34, plus the weight's own error (below).
  b   u_r s with s = -(e_i + l e_z) (:1059, 2 units): 13 + 1 + 1 + 6 + 2 = 23.
  chain  a lane adds one pixel per round of 32 (stage_b_rounds, :1144-1148): 5 rounds per full 160-column band and
      ceil(bw/32) in a partial band of bw columns, so ceil(w/32) pixels per image row (160 is whole rounds), each into both
      rank-1 updates (:1059-1060): 2 ceil(w/32) FMAs per accumulator; then the 5 levels of the halving exchange
      (flush_row_window, :1088-1102), and the row's fp32 total.  A: k = 34 + 2 ceil(w/32) + 5; b: k = 23 + 2 ceil(w/32) + 5.
  ll  per point (:1040-1041): d = r^T P r unfused (4 units of |r|^T |P| |r|), 0.2f (< 1 unit), the FMA 1 + 0.2 d (1
      unit of x), then __log2f (CUDA C Programming Guide, intrinsic functions: absolute error <= 2^-22 for x in
      [0.5, 2], else 2 ulp); E_ll = sum over kept points of 0.2 gamma_5 |r|^T|P||r| / x + u + that log error.  The lane
      chain adds one term per pixel (ceil(w/32)), the exchange 5, the scaling by the fp32 ln 2 (:1068) 2:
      k = ceil(w/32) + 7 of sum log x.  The end step (tracker.cu:302-305): det in fp32 (gamma_2 of |P0 P3| + |P1 P2|), its
      log rounded to fp32 (u |log det|), times 0.5 n; the result rounded to fp32 (u |ll|).
  weights  student_weight (stages.cuh:684-689): d in three roundings (gamma_3 |r|^T |P_{k-1}| |r|), 5 + d (1), rcp_fast (2),
      7 * (1): the weight's relative error eps_w = gamma_3 |r|^T|P||r| / (5 + d) + 4 u, added per point to A, b and the
      scale as sum eps_w M_point.
  scale  stage A (scale_round32, :709-744): a term (w_k + w_next) r r^T: the product r r^T 1, the weight sum 1; a lane
      adds up to two FMAs per pixel (the pending leader of the previous round and its own), ceil(w/32) pixels per row:
      2 ceil(w/32), the exchange 5, and the export of each hypothesis as (float)(0.5 (all +- alt)) 1 (:820-826):
      k = 2 ceil(w/32) + 8.  The
      kernel sums both pairing hypotheses (leaders at even and at odd rank) in the same registers, so M is the sum over
      both: sum over every point i < n-1 of (w_i + w_{i+1}) |r_i r_i^T|, plus the last point alone.  CORRECTED
      (scale_add, :762-768): w r in 1, one FMA per pixel (ceil(w/32)), the exchange 5: k = ceil(w/32) + 6.
      pair_mid_warp (tracker.cu:163-173): C = (float)(S / (n - 3)) (u |C|), det = C0 C3 - C1^2 in fp32 (gamma_2 of
      |C0 C3| + C1^2), 1/det and C / det (2 units).  P gets the first-order bound |P| |dC| |P| / (1 - rho), rho the
      infinity norm of |P| |dC|, on top of eta |P| with eta = gamma_2 (|C0 C3| + C1^2) / |det C| + 2 u.
  fp64  the row totals go into fp64 strip and level sums (tracker.cu:266-298): gamma_{h+64} in u = 2^-53 of M.

The model reads nothing from the oracle: it sees records, the reference intensity, intrinsics and the kernel's outputs.
"""
from dataclasses import dataclass, field

import numpy as np

from tile_geometry import bands

U = 2.0 ** -24          # fp32 unit roundoff
U64 = 2.0 ** -53        # fp64 unit roundoff
C_I = float(np.float32(1.0) / np.float32(255.0))     # c.c_i = 1.0f / 255.0f (stages.cuh:258)
LOG2F_ABS = 2.0 ** -22  # __log2f: absolute error for x in [0.5, 2], in log2 units
LOG2F_REL = 2.0 ** -22  # __log2f: 2 ulp elsewhere, relative

K_TERM_A = 34           # units of one A term (module docstring)
K_TERM_B = 23
K_TERM_SCALE_REFERENCE = 3
K_TERM_SCALE_CORRECTED = 1
K_EXCHANGE = 5          # the halving exchange over 32 lanes


def gamma(k, u=U):
    return k * u / (1.0 - k * u)


def nbands(w):
    return len(bands(w))


def rounds(w):
    """pixels one lane adds per image row: one per round of 32 columns, and every band but the last is whole rounds"""
    return sum((bw + 31) // 32 for bw in bands(w))


def k_counts(w, estimator):
    """k of every quantity at an image width w (the lane chains grow with the rounds of 32 pixels per row)"""
    nr = rounds(w)
    scale = (2 * nr + K_EXCHANGE + K_TERM_SCALE_REFERENCE) if estimator == "reference" else \
        (nr + K_EXCHANGE + K_TERM_SCALE_CORRECTED)
    return {"A": K_TERM_A + 2 * nr + K_EXCHANGE, "b": K_TERM_B + 2 * nr + K_EXCHANGE, "ll": nr + K_EXCHANGE + 2,
            "scale": scale}


def level_intrinsics(K, level):
    """K 2^-l in fp32, as the pyramid halves the intrinsics (exact: a power of two)"""
    return tuple(float(np.float32(v) * np.float32(0.5 ** level)) for v in K)


def template(w, h, Kl):
    """tx[w], ty[h] of the level (pyramid.cu k_template: ((float) i - o) / f with IEEE fp32 division)"""
    fx, fy, ox, oy = (np.float32(v) for v in Kl)
    tx = (np.arange(w, dtype=np.float32) - ox) / fx
    ty = (np.arange(h, dtype=np.float32) - oy) / fy
    return tx.astype(np.float64), ty.astype(np.float64)


@dataclass
class Points:
    """the valid records in rank (raster) order, in fp64, with their Jacobians and absolute Jacobians"""
    pix: np.ndarray
    rows: np.ndarray
    r: np.ndarray           # (n, 2)
    J: np.ndarray           # (n, 2, k)
    Jabs: np.ndarray        # (n, 2, k)
    w: int
    h: int


def points(records, K, level, I_ref=None):
    """records: (7, h, w) float32 planes; I_ref: the level's reference intensity (h, w), which adds the two brightness
    columns (photometric mode)"""
    _, h, w = records.shape
    flat = records.reshape(7, -1)
    valid = np.isfinite(flat).all(axis=0)
    pix = np.flatnonzero(valid)
    rec = flat[:, pix].astype(np.float64)
    tx, ty = template(w, h, level_intrinsics(K, level))
    rows, cols = pix // w, pix % w
    z = rec[6]
    x, y = tx[cols] * z, ty[rows] * z
    zi, zs = 1.0 / z, 1.0 / (z * z)
    zero, one = np.zeros_like(z), np.ones_like(z)
    Jw0 = np.stack([zi, zero, -x * zs, -x * y * zs, 1.0 + x * x * zs, -y * zi], axis=1)
    Jw1 = np.stack([zero, zi, -y * zs, -1.0 - y * y * zs, x * y * zs, x * zi], axis=1)
    Aw0 = np.stack([np.abs(zi), zero, np.abs(x) * zs, np.abs(x * y) * zs, 1.0 + x * x * zs, np.abs(y * zi)], axis=1)
    Aw1 = np.stack([zero, np.abs(zi), np.abs(y) * zs, 1.0 + y * y * zs, np.abs(x * y) * zs, np.abs(x * zi)], axis=1)
    Jz = np.stack([zero, zero, one, y, -x, zero], axis=1)
    gx, gy, hx, hy = (rec[k][:, None] for k in (2, 3, 4, 5))
    J0 = gx * Jw0 + gy * Jw1
    J1 = hx * Jw0 + hy * Jw1 - Jz
    B0 = np.abs(gx) * Aw0 + np.abs(gy) * Aw1
    B1 = np.abs(hx) * Aw0 + np.abs(hy) * Aw1 + np.abs(Jz)
    if I_ref is not None:
        Ir = np.asarray(I_ref, dtype=np.float64).reshape(-1)[pix]
        J0 = np.concatenate([J0, np.stack([-C_I * Ir, -C_I * one], axis=1)], axis=1)
        B0 = np.concatenate([B0, np.stack([C_I * np.abs(Ir), C_I * one], axis=1)], axis=1)
        J1 = np.concatenate([J1, np.zeros((len(z), 2))], axis=1)
        B1 = np.concatenate([B1, np.zeros((len(z), 2))], axis=1)
    return Points(pix=pix, rows=rows, r=rec[:2].T.copy(), J=np.stack([J0, J1], axis=1), Jabs=np.stack([B0, B1], axis=1), w=w, h=h)


def quad(r, P):
    """r^T P r per point, P as given (row-major 2 x 2)"""
    return r[:, 0] * (P[0, 0] * r[:, 0] + P[1, 0] * r[:, 1]) + r[:, 1] * (P[0, 1] * r[:, 0] + P[1, 1] * r[:, 1])


def weights(pts, use_weights, prev_precision):
    """(w, eps_w): the Student-t weights in fp64 and the relative error bound of the kernel's"""
    n = len(pts.pix)
    if not use_weights:
        return np.ones(n), np.zeros(n)
    Pp = np.asarray(prev_precision, dtype=np.float32).reshape(2, 2).astype(np.float64)
    d = quad(pts.r, Pp)
    dabs = quad(np.abs(pts.r), np.abs(Pp))
    return 7.0 / (5.0 + d), gamma(3) * dabs / np.abs(5.0 + d) + 4.0 * U


def outer3(r):
    """the (00, 01, 11) components of r r^T per point"""
    return np.stack([r[:, 0] * r[:, 0], r[:, 0] * r[:, 1], r[:, 1] * r[:, 1]], axis=1)


def scale_sum(pts, w, eps, estimator):
    """(S, M, E): the scale sum (00, 01, 11), its absolute sum and the weights' error term"""
    n = len(w)
    o = outer3(pts.r)
    oa = np.abs(o)
    if estimator == "corrected":
        return (w[:, None] * o).sum(0), (np.abs(w)[:, None] * oa).sum(0), ((eps * np.abs(w))[:, None] * oa).sum(0)
    n2 = n - n % 2
    src = np.arange(n)
    src[1:n2:2] -= 1                   # a follower uses its leader's residual
    S = (w[:, None] * o[src]).sum(0)
    # both hypotheses: every point but the last with its weight and the next one's, the last alone
    ws = np.abs(w).copy()
    ws[:-1] += np.abs(w[1:])
    es = (eps * np.abs(w)).copy()
    es[:-1] += eps[1:] * np.abs(w[1:])
    return S, (ws[:, None] * oa).sum(0), (es[:, None] * oa).sum(0)


def _sym(c):
    return np.array([[c[0], c[1]], [c[1], c[2]]])


def normal_equations(pts, w, eps, P):
    """(A, b, M_A, M_b, E_A, E_b) with the precision P (2 x 2) in every point's W = w P"""
    J, Ja, r = pts.J, pts.Jabs, pts.r
    Pa = np.abs(P)
    PJ = np.einsum("ij,njc->nic", P, J)
    PaJa = np.einsum("ij,njc->nic", Pa, Ja)
    A = np.einsum("n,nic,nid->cd", w, J, PJ)
    b = -np.einsum("n,nic,ni->c", w, PJ, r)
    wa = np.abs(w)
    MA = np.einsum("n,nic,nid->cd", wa, Ja, PaJa)
    Mb = np.einsum("n,nic,ni->c", wa, PaJa, np.abs(r))
    we = eps * wa
    EA = np.einsum("n,nic,nid->cd", we, Ja, PaJa)
    Eb = np.einsum("n,nic,ni->c", we, PaJa, np.abs(r))
    return A, b, MA, Mb, EA, Eb


def kept(n, estimator):
    """the points whose log-likelihood term counts: REFERENCE drops the last n mod 50 ranks"""
    return n if estimator == "corrected" else n - n % 50


def log_terms(pts, P):
    """(log(1 + 0.2 r^T P r), its error bound per point) with the kernel's P"""
    d = quad(pts.r, P)
    dabs = quad(np.abs(pts.r), np.abs(P))
    x = 1.0 + 0.2 * d
    lg = np.log(x)
    err = 0.2 * gamma(5) * dabs / x + U + np.where(x <= 2.0, np.log(2.0) * LOG2F_ABS, LOG2F_REL * np.abs(lg))
    return lg, err


@dataclass
class Ledger:
    n: int
    estimator: str
    k: dict
    P: np.ndarray = None
    P_bound: np.ndarray = None
    ll: float = None
    ll_bound: float = None
    A: np.ndarray = None
    A_bound: np.ndarray = None
    b: np.ndarray = None
    b_bound: np.ndarray = None
    M: dict = field(default_factory=dict)


def ledger(records, K, level, P_kernel, estimator="reference", use_weights=False, prev_precision=None, I_ref=None):
    """The ledger of one linearisation (module docstring).  records: (7, h, w) float32; K: level-0 intrinsics; P_kernel:
    the kernel's P_k (2 x 2); I_ref: the level's reference intensity in the photometric mode, else None."""
    pts = points(records, K, level, I_ref)
    n = len(pts.pix)
    led = Ledger(n=n, estimator=estimator, k=k_counts(pts.w, estimator))
    if n < 6:
        return led
    f64 = gamma(pts.h + 64, U64)
    w, eps = weights(pts, use_weights, prev_precision)
    # scale, covariance, P
    S, MS, ES = scale_sum(pts, w, eps, estimator)
    C = _sym(S) / (n - 3)
    led.P = np.linalg.inv(C)
    dC = _sym(((gamma(led.k["scale"]) + f64) * MS + ES) / (n - 3)) + U * np.abs(C)
    Pa = np.abs(led.P)
    rho = np.abs(Pa @ dC).sum(axis=1).max()
    det = C[0, 0] * C[1, 1] - C[0, 1] ** 2
    eta = gamma(2) * (abs(C[0, 0] * C[1, 1]) + C[0, 1] ** 2) / abs(det) + 2.0 * U
    led.P_bound = Pa @ dC @ Pa / (1.0 - rho) + eta * Pa
    led.M["scale"] = MS
    # log-likelihood at the kernel's P
    Pk = np.asarray(P_kernel, dtype=np.float32).reshape(2, 2).astype(np.float64)
    lg, lerr = log_terms(pts, Pk)
    nk = kept(n, estimator)
    sl = lg[:nk].sum()
    pdet = Pk[0, 0] * Pk[1, 1] - Pk[0, 1] * Pk[1, 0]
    logdet = np.log(pdet)
    led.ll = 0.5 * n * logdet - 3.5 * sl
    e_det = 0.5 * n * (gamma(2) * (abs(Pk[0, 0] * Pk[1, 1]) + abs(Pk[0, 1] * Pk[1, 0])) / abs(pdet) + U * abs(logdet))
    led.ll_bound = 3.5 * (lerr[:nk].sum() + (gamma(led.k["ll"]) + f64) * sl) + e_det + U * abs(led.ll) + \
        f64 * (0.5 * n * abs(logdet) + 3.5 * sl)
    led.M["ll"] = sl
    # normal equations at the kernel's P
    A, b, MA, Mb, EA, Eb = normal_equations(pts, w, eps, Pk)
    led.A, led.b = A, b
    led.A_bound = (gamma(led.k["A"]) + f64) * MA + EA
    led.b_bound = (gamma(led.k["b"]) + f64) * Mb + Eb
    led.M["A"], led.M["b"] = MA, Mb
    return led


def _ratio(d, bound):
    d, bound = np.abs(np.asarray(d, dtype=np.float64)), np.asarray(bound, dtype=np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where(d == 0, 0.0, np.where(bound > 0, d / bound, np.inf))


@dataclass
class Report:
    ratios: dict = field(default_factory=dict)      # quantity -> array of |kernel - ledger| / bound
    failures: list = field(default_factory=list)    # (quantity, detail): the per-entry report

    @property
    def maxima(self):
        return {q: float(np.max(r)) if np.size(r) else 0.0 for q, r in self.ratios.items()}

    @property
    def failed(self):
        return {f[0] for f in self.failures}


def compare(led, out):
    """the kernel's (or any) linearisation `out` = {"n", "precision", "ll", "A", "b"} against the ledger, entry by entry"""
    rep = Report()
    if int(out["n"]) != led.n:
        rep.failures.append(("n", f"kernel {int(out['n'])} ledger {led.n}"))
    rep.ratios["n"] = np.array([0.0 if int(out["n"]) == led.n else np.inf])
    if led.n < 6:
        return rep
    Pk = np.asarray(out["precision"], dtype=np.float64).reshape(2, 2)
    items = [("P", Pk, led.P, led.P_bound), ("ll", float(out["ll"]), led.ll, led.ll_bound),
             ("A", np.asarray(out["A"]), led.A, led.A_bound), ("b", np.asarray(out["b"]), led.b, led.b_bound)]
    for q, got, want, bound in items:
        r = _ratio(np.asarray(got) - want, bound)
        rep.ratios[q] = np.atleast_1d(r)
        for idx in zip(*np.nonzero(np.atleast_1d(r) > 1.0)):
            g, wv, bd = (np.atleast_1d(v)[idx] for v in (got, want, bound))
            rep.failures.append((q, f"{list(map(int, idx)) if np.ndim(r) else ''} kernel {g:.9g} ledger {wv:.9g} "
                                    f"|d| {abs(g - wv):.3g} bound {bd:.3g} ratio {np.atleast_1d(r)[idx]:.3g}"))
    return rep


# ---- the kernel's summation order in fp32 (tests/test_linearization_ledger_host.py) ----------------------------------------
def ldl_terms(pts, w, P):
    """the two rank-1 parts of each point's w J^T P J and w J^T P r as stage_b_pixel splits them (l = P01 / P00,
    d0 = P00, d1 = P11 - P01 l): (T0, T1) of shape (n, k, k) and (t0, t1) of shape (n, k), in fp64"""
    l = P[0, 1] / P[0, 0]
    d0, d1 = P[0, 0], P[1, 1] - P[0, 1] * l
    j0 = pts.J[:, 0] + l * pts.J[:, 1]
    j1 = pts.J[:, 1]
    s0 = -(pts.r[:, 0] + l * pts.r[:, 1])
    s1 = -pts.r[:, 1]
    T0 = (w * d0)[:, None, None] * j0[:, :, None] * j0[:, None, :]
    T1 = (w * d1)[:, None, None] * j1[:, :, None] * j1[:, None, :]
    return T0, T1, (w * d0 * s0)[:, None] * j0, (w * d1 * s1)[:, None] * j1


def emulate_row_order(pts, *terms):
    """sum per-point terms (each (n, ...)) in the kernel's order: every term rounded to fp32, each lane's pixels of a row
    (columns = lane mod 32, in increasing column order, the terms of one pixel in the order given) in an fp32 chain, the
    32 lanes by the halving exchange in fp32, then the rows in fp64"""
    W = 32 * rounds(pts.w)
    shape = terms[0].shape[1:]
    out = np.zeros(shape)
    for e in np.ndindex(*shape):
        grids = []
        for t in terms:
            g = np.zeros((pts.h, W), np.float32)
            g.reshape(-1)[pts.rows * W + pts.pix % pts.w] = t[(slice(None),) + e].astype(np.float32)
            grids.append(g.reshape(pts.h, W // 32, 32))
        acc = np.zeros((pts.h, 32), np.float32)
        for c in range(W // 32):
            for g in grids:
                acc = acc + g[:, c]
        half = 16
        while half:
            acc = acc[:, :half] + acc[:, half:2 * half]
            half //= 2
        out[e] = acc[:, 0].astype(np.float64).sum()
    return out
