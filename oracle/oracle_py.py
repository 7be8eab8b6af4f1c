"""ctypes binding of oracle/liboracle.so -- TEST INFRASTRUCTURE ONLY (see oracle/dvo_oracle.h).

May be imported by tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference
legs; never by the product package dvo_slam_b200/.  The reference ships no goldens; the FAITHFUL mode is pinned,
bit for bit, against what the reference's own SSE translation units (oracle/_ref) compute on the golden cases
(tests/golden/reference_pin.npz, tests/test_reference_pin.py).
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "liboracle.so")
ORC_MAX_LEVELS = 8

TERMINATION_NAMES = ["IterationsExceeded", "IncrementTooSmall", "LogLikelihoodDecreased", "TooFewConstraints"]


class Mode(C.Structure):
    _fields_ = [(n, C.c_int) for n in ("rcp_approx", "rtz_residuals", "drop_odd_point", "scale_pair_bug",
                                       "ll_drop_tail", "f32_serial_accum", "fused_pixel_math", "ll_group_product")]


class Config(C.Structure):
    _fields_ = [("first_level", C.c_int), ("last_level", C.c_int), ("max_iterations_per_level", C.c_int),
                ("precision", C.c_double), ("mu", C.c_double), ("use_initial_estimate", C.c_int),
                ("intensity_derivative_threshold", C.c_float), ("depth_derivative_threshold", C.c_float)]


class IterationStats(C.Structure):
    _fields_ = [("level", C.c_int32), ("id", C.c_int32), ("valid_constraints", C.c_int64),
                ("tdist_log_likelihood", C.c_double), ("tdist_precision", C.c_double * 4),
                ("prior_log_likelihood", C.c_double), ("increment", C.c_double * 6),
                ("information", C.c_double * 36)]


class LevelStats(C.Structure):
    _fields_ = [("id", C.c_int32), ("termination", C.c_int32), ("max_valid_pixels", C.c_int64),
                ("valid_pixels", C.c_int64), ("num_iterations", C.c_int32), ("pad_", C.c_int32)]


class Result(C.Structure):
    _fields_ = [("transformation", C.c_double * 16), ("information", C.c_double * 36),
                ("log_likelihood", C.c_double), ("num_levels", C.c_int32), ("pad_", C.c_int32),
                ("levels", LevelStats * ORC_MAX_LEVELS)]


def build(force: bool = False) -> str:
    src = os.path.join(_HERE, "dvo_oracle.cpp")
    if force or not os.path.exists(_LIB_PATH) or (
            os.path.exists(src) and os.path.getmtime(src) > os.path.getmtime(_LIB_PATH)):
        subprocess.check_call(["make", "-C", _HERE, "liboracle.so"], stdout=subprocess.DEVNULL)
    return _LIB_PATH


_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(_LIB_PATH):
            build()
        L = C.CDLL(_LIB_PATH)
        fp = C.POINTER(C.c_float)
        dp = C.POINTER(C.c_double)
        L.orc_mode_faithful.restype = Mode
        L.orc_mode_exact.restype = Mode
        L.orc_mode_mirror.restype = Mode
        L.orc_config_default.restype = Config
        L.orc_pyramid_create.restype = C.c_void_p
        L.orc_pyramid_create.argtypes = [fp, fp, C.c_int, C.c_int, C.c_float, C.c_float, C.c_float, C.c_float, C.c_int]
        L.orc_pyramid_destroy.argtypes = [C.c_void_p]
        L.orc_pyramid_num_levels.argtypes = [C.c_void_p]
        L.orc_pyramid_plane.restype = fp
        L.orc_pyramid_plane.argtypes = [C.c_void_p, C.c_int, C.c_int]
        L.orc_pyramid_level_info.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int), fp]
        L.orc_select.restype = C.c_int64
        L.orc_select.argtypes = [C.c_void_p, C.c_int, C.c_float, C.c_float, C.POINTER(Mode), C.POINTER(C.c_uint8)]
        L.orc_residual_image.restype = C.c_int64
        L.orc_residual_image.argtypes = [C.c_void_p, C.c_void_p, C.c_int, dp, dp, C.c_float, C.c_float, C.POINTER(Mode), fp]
        L.orc_intensity_error_image.restype = C.c_int64
        L.orc_intensity_error_image.argtypes = [C.c_void_p, C.c_void_p, C.c_int, dp, C.c_float, C.c_float, C.POINTER(Mode), fp]
        L.orc_linearize.restype = C.c_int64
        L.orc_linearize.argtypes = [C.c_void_p, C.c_void_p, C.c_int, dp, dp, C.c_float, C.c_float, C.c_int, fp,
                                    C.POINTER(Mode), fp, fp, dp, dp]
        L.orc_match_with.restype = C.c_int
        L.orc_match_with.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(Config), dp, dp, dp, C.POINTER(Mode), C.POINTER(Result),
                                     dp, C.POINTER(IterationStats), C.c_int, C.POINTER(C.c_int)]
        L.orc_se3_exp.argtypes = [dp, dp]
        L.orc_se3_log.argtypes = [dp, dp]
        L.orc_ldlt_solve.argtypes = [dp, dp, dp, C.c_int]
        L.orc_schur_onto_pose.argtypes = [dp, dp]
        L.orc_convert_raw_depth.argtypes = [C.POINTER(C.c_uint16), fp, C.c_int64, C.c_float]
        L.orc_bgr_to_grey.argtypes = [C.POINTER(C.c_uint8), fp, C.c_int64]
        _lib = L
    return _lib


def _fptr(a):
    return a.ctypes.data_as(C.POINTER(C.c_float))


def _dptr(a):
    """a's data, or NULL for None"""
    return None if a is None else a.ctypes.data_as(C.POINTER(C.c_double))


def _doubles(a, n):
    """a as n contiguous float64 (kept alive by the caller), or None for None"""
    return None if a is None else np.ascontiguousarray(np.asarray(a, dtype=np.float64).reshape(n))


def mode(name: str) -> Mode:
    L = lib()
    return {"faithful": L.orc_mode_faithful, "exact": L.orc_mode_exact, "mirror": L.orc_mode_mirror}[name]()


def config(**kw) -> Config:
    c = lib().orc_config_default()
    for k, v in kw.items():
        if not hasattr(c, k):
            raise AttributeError(k)
        setattr(c, k, v)
    return c


class Pyramid:
    def __init__(self, intensity, depth, intrinsics, levels):
        I = np.ascontiguousarray(np.asarray(intensity, dtype=np.float32))
        Z = np.ascontiguousarray(np.asarray(depth, dtype=np.float32))
        assert I.shape == Z.shape and I.ndim == 2
        h, w = I.shape
        fx, fy, ox, oy = intrinsics
        self.h = lib().orc_pyramid_create(_fptr(I), _fptr(Z), w, h, fx, fy, ox, oy, levels)
        if not self.h:
            raise ValueError("orc_pyramid_create failed")
        self.levels = levels

    def __del__(self):
        h, self.h = getattr(self, "h", None), None
        if h and _lib is not None:   # at interpreter teardown the module globals may already be gone
            try:
                _lib.orc_pyramid_destroy(h)
            except Exception:
                pass

    def level_info(self, level):
        w, h = C.c_int(), C.c_int()
        K = (C.c_float * 4)()
        lib().orc_pyramid_level_info(self.h, level, C.byref(w), C.byref(h), K)
        return w.value, h.value, tuple(K)

    def plane(self, level, channel):
        w, h, _ = self.level_info(level)
        p = lib().orc_pyramid_plane(self.h, level, channel)
        return np.ctypeslib.as_array(p, shape=(h, w)).copy()

    def planes(self, level):
        return np.stack([self.plane(level, c) for c in range(6)])


def select(ref: Pyramid, level, ti=0.0, td=0.0, m: Mode | None = None):
    w, h, _ = ref.level_info(level)
    mask = np.zeros((h, w), dtype=np.uint8)
    S = lib().orc_select(ref.h, level, ti, td, C.byref(m) if m is not None else None,
                         mask.ctypes.data_as(C.POINTER(C.c_uint8)))
    return int(S), mask


def residual_image(ref: Pyramid, cur: Pyramid, level, T, m: Mode, ti=0.0, td=0.0, ab=None):
    """ab: None, or the photometric mode's (alpha, beta)"""
    w, h, _ = ref.level_info(level)
    out = np.empty((7, h, w), dtype=np.float32)
    T, ab = _doubles(T, 16), _doubles(ab, 2)
    n = lib().orc_residual_image(ref.h, cur.h, level, _dptr(T), _dptr(ab), ti, td, C.byref(m), _fptr(out))
    return int(n), out


def intensity_error_image(ref: Pyramid, cur: Pyramid, level, T, m: Mode, ti=0.0, td=0.0):
    """DenseTracker::computeIntensityErrorImage (dense_tracking.cpp:378-444) -> (n_written, image[h, w])."""
    w, h, _ = ref.level_info(level)
    out = np.empty((h, w), dtype=np.float32)
    T = np.ascontiguousarray(np.asarray(T, dtype=np.float64).reshape(16))
    n = lib().orc_intensity_error_image(ref.h, cur.h, level, _dptr(T), ti, td, C.byref(m), _fptr(out))
    return int(n), out


def linearize(ref: Pyramid, cur: Pyramid, level, T, m: Mode, use_weights=False, prev_precision=None, ti=0.0, td=0.0, ab=None):
    """ab: None, or the photometric mode's (alpha, beta), whose A is 8 x 8 and b 8 long"""
    T, ab = _doubles(T, 16), _doubles(ab, 2)
    pp = np.ascontiguousarray(np.asarray(prev_precision if prev_precision is not None else np.zeros(4), dtype=np.float32).reshape(4))
    P = np.zeros(4, dtype=np.float32)
    ll = C.c_float()
    nu = 6 if ab is None else 8
    A = np.zeros(nu * nu, dtype=np.float64)
    b = np.zeros(nu, dtype=np.float64)
    n = lib().orc_linearize(ref.h, cur.h, level, _dptr(T), _dptr(ab), ti, td, int(use_weights), _fptr(pp), C.byref(m),
                            _fptr(P), C.byref(ll), _dptr(A), _dptr(b))
    return {"n": int(n), "precision": P.reshape(2, 2), "ll": ll.value, "A": A.reshape(nu, nu), "b": b}


def match(ref: Pyramid, cur: Pyramid, cfg: Config, m: Mode, T_init=None, max_iters=1024, prior=None, photometric=False,
          ab_init=None):
    """prior: None for cfg.mu I, else a 6 x 6 prior information in its place.  photometric: estimate (alpha, beta) with the
    pose, from ab_init (None: (1, 0)); the result then holds the final ones as "ab"."""
    T0 = _doubles(T_init if T_init is not None else np.eye(4), 16)
    prior, ab_init = _doubles(prior, 36), _doubles(ab_init, 2)
    ab = np.zeros(2) if photometric else None
    res = Result()
    its = (IterationStats * max_iters)()
    n = C.c_int()
    rc = lib().orc_match_with(ref.h, cur.h, C.byref(cfg), _dptr(T0), _dptr(prior), _dptr(ab_init), C.byref(m),
                              C.byref(res), _dptr(ab), its, max_iters, C.byref(n))
    assert rc == 0
    levels = []
    for i in range(res.num_levels):
        l = res.levels[i]
        levels.append({"id": l.id, "termination": l.termination, "max_valid_pixels": l.max_valid_pixels,
                       "valid_pixels": l.valid_pixels, "num_iterations": l.num_iterations})
    iters = []
    for i in range(min(n.value, max_iters)):
        s = its[i]
        iters.append({"level": s.level, "id": s.id, "n": s.valid_constraints, "nll": s.tdist_log_likelihood,
                      "precision": np.array(s.tdist_precision).reshape(2, 2), "prior": s.prior_log_likelihood,
                      "x": np.array(s.increment), "A": np.array(s.information).reshape(6, 6)})
    out = {"T": np.array(res.transformation).reshape(4, 4), "information": np.array(res.information).reshape(6, 6),
           "log_likelihood": res.log_likelihood, "levels": levels, "iterations": iters}
    if photometric:
        out["ab"] = ab
    return out


def se3_exp(xi):
    xi = np.ascontiguousarray(np.asarray(xi, dtype=np.float64))
    T = np.zeros(16)
    lib().orc_se3_exp(_dptr(xi), _dptr(T))
    return T.reshape(4, 4)


def se3_log(T):
    T = np.ascontiguousarray(np.asarray(T, dtype=np.float64).reshape(16))
    xi = np.zeros(6)
    lib().orc_se3_log(_dptr(T), _dptr(xi))
    return xi


def ldlt_solve(A, b):
    """x = A^-1 b for an n x n A, n <= 8, by the oracle's pivoted LDL^T"""
    n = len(b)
    assert 1 <= n <= 8, n
    A, b = _doubles(A, n * n), _doubles(b, n)
    x = np.zeros(n)
    lib().orc_ldlt_solve(_dptr(A), _dptr(b), _dptr(x), n)
    return x


ldlt_solve6 = ldlt_solve   # the 6 x 6 case by its former name


def schur_pose(A):
    """the Schur complement of an 8 x 8 onto its first 6 unknowns (the photometric mode's information)"""
    A = _doubles(A, 64)
    S = np.zeros(36)
    lib().orc_schur_onto_pose(_dptr(A), _dptr(S))
    return S.reshape(6, 6)


def bgr_to_grey(bgr_u8):
    """(h, w, 3) uint8 BGR -> (h, w) float32 grey, as cv::cvtColor(CV_BGR2GRAY) + convertTo(CV_32F)."""
    bgr = np.ascontiguousarray(bgr_u8, dtype=np.uint8)
    assert bgr.shape[-1] == 3
    out = np.empty(bgr.shape[:-1], dtype=np.float32)
    lib().orc_bgr_to_grey(bgr.ctypes.data_as(C.POINTER(C.c_uint8)), _fptr(out), out.size)
    return out


def convert_raw_depth(raw_u16, scale):
    raw = np.ascontiguousarray(np.asarray(raw_u16, dtype=np.uint16))
    out = np.empty(raw.shape, dtype=np.float32)
    lib().orc_convert_raw_depth(raw.ctypes.data_as(C.POINTER(C.c_uint16)), _fptr(out), raw.size, scale)
    return out


# ---- oracle/_ref: the reference's own SSE translation units (see oracle/Makefile, oracle/ref_driver.cpp) ----------
_REF_DIR = os.path.join(_HERE, "_ref")
_ref = {}


def ref_available(variant: str = "") -> bool:
    return os.path.exists(os.path.join(_REF_DIR, f"libdvo_ref{variant}.so"))


def ref_lib(variant: str = ""):
    """libdvo_ref.so = dvo_core/src/{dense_tracking_impl,core/math_sse,core/intrinsic_matrix}.cpp of a dvo_slam checkout compiled
    unmodified + ref_driver.cpp (-O2; variant "_O3" = the reference's own optimisation level).  Built by __graft_entry__.build()
    when DVO_REFERENCE names that checkout (oracle/Makefile target `ref`)."""
    if variant not in _ref:
        L = C.CDLL(os.path.join(_REF_DIR, f"libdvo_ref{variant}.so"))
        fp, dp = C.POINTER(C.c_float), C.POINTER(C.c_double)
        L.ref_linearize.restype = C.c_int64
        L.ref_linearize.argtypes = [fp, fp, C.c_int, C.c_int, fp, dp, C.c_float, C.c_float, C.c_int, fp, C.POINTER(C.c_int64), fp,
                                    C.POINTER(C.c_int32), fp, fp, fp, fp, fp, fp]
        L.ref_pyramid_create.restype = C.c_void_p
        L.ref_pyramid_create.argtypes = [C.c_int, C.POINTER(fp), C.POINTER(C.c_int), C.POINTER(C.c_int), fp]
        L.ref_pyramid_destroy.argtypes = [C.c_void_p]
        L.ref_intensity_error_image.restype = C.c_int64
        L.ref_intensity_error_image.argtypes = [C.c_void_p, C.c_void_p, C.c_int, dp, C.c_float, C.c_float, fp]
        L.ref_match.restype = C.c_int
        L.ref_match.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_double, C.c_double, C.c_int, dp, C.c_float,
                                C.c_float, dp, dp, dp, C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.POINTER(C.c_int64)]
        _ref[variant] = L
    return _ref[variant]


class RefPyramid:
    """The reference's image model for one frame (acceleration images + cached point lists), filled from the planes of an
    oracle Pyramid (the pyramid / derivative code of the reference needs OpenCV proper and is not compiled)."""

    def __init__(self, pyr: "Pyramid", variant: str = ""):
        self.variant = variant
        n = pyr.levels
        self._planes = [np.ascontiguousarray(pyr.planes(l)) for l in range(n)]
        info = [pyr.level_info(l) for l in range(n)]
        w = (C.c_int * n)(*[i[0] for i in info]); h = (C.c_int * n)(*[i[1] for i in info])
        K = np.ascontiguousarray(np.array([i[2] for i in info], dtype=np.float32).reshape(-1))
        ptrs = (C.POINTER(C.c_float) * n)(*[_fptr(p) for p in self._planes])
        self.h = ref_lib(variant).ref_pyramid_create(n, ptrs, w, h, _fptr(K))
        self.levels = n
        self.size = [(i[0], i[1]) for i in info]

    def __del__(self):
        h, self.h = getattr(self, "h", None), None
        if h and self.variant in _ref:
            try:
                _ref[self.variant].ref_pyramid_destroy(h)
            except Exception:
                pass


def ref_match(ref: RefPyramid, cur: RefPyramid, cfg: Config, T_init=None):
    """DenseTracker::match() with every per-point pass run by the reference's own object code (oracle/ref_driver.cpp)."""
    T0 = np.ascontiguousarray(np.asarray(T_init if T_init is not None else np.eye(4), dtype=np.float64).reshape(16))
    nl = cfg.first_level - cfg.last_level + 1
    T = np.zeros(16); info = np.zeros(36); ll = C.c_double()
    term = (C.c_int32 * nl)(); its = (C.c_int32 * nl)(); vp = (C.c_int64 * nl)()
    rc = ref_lib(ref.variant).ref_match(ref.h, cur.h, cfg.first_level, cfg.last_level, cfg.max_iterations_per_level, cfg.precision, cfg.mu,
                                        cfg.use_initial_estimate, _dptr(T0), cfg.intensity_derivative_threshold,
                                        cfg.depth_derivative_threshold, _dptr(T), _dptr(info), C.byref(ll), term, its, vp)
    assert rc == 0
    levels = [{"id": cfg.first_level - i, "termination": term[i], "num_iterations": its[i], "valid_pixels": vp[i]} for i in range(nl)]
    return {"T": T.reshape(4, 4), "information": info.reshape(6, 6), "log_likelihood": ll.value, "levels": levels}


def ref_intensity_error_image(ref: RefPyramid, cur: RefPyramid, level, T, ti=0.0, td=0.0):
    """computeIntensityErrorImage with residuals and valid flags from the reference's computeResidualsAndValidFlagsSse."""
    L = ref_lib(ref.variant)
    w, h = ref.size[level]
    out = np.empty((h, w), dtype=np.float32)
    T = np.ascontiguousarray(np.asarray(T, dtype=np.float64).reshape(16))
    n = L.ref_intensity_error_image(ref.h, cur.h, level, _dptr(T), ti, td, _fptr(out))
    return int(n), out


def ref_linearize(ref_planes6, cur_planes6, K, T, use_weights=False, prev_precision=None, ti=0.0, td=0.0, variant=""):
    """One Gauss-Newton linearisation computed by the reference's own object code.  planes6: (6, h, w) float32."""
    rp = np.ascontiguousarray(ref_planes6, dtype=np.float32)
    cp = np.ascontiguousarray(cur_planes6, dtype=np.float32)
    _, h, w = rp.shape
    N = h * w
    K4 = np.ascontiguousarray(np.asarray(K, dtype=np.float32))
    T = np.ascontiguousarray(np.asarray(T, dtype=np.float64).reshape(16))
    pp = np.ascontiguousarray(np.asarray(prev_precision if prev_precision is not None else np.zeros(4), dtype=np.float32).reshape(4))
    nsel = C.c_int64()
    res = np.zeros((N, 2), dtype=np.float32)
    idx = np.zeros(N, dtype=np.int32)
    rec = np.zeros((N, 12), dtype=np.float32)
    wts = np.zeros(N, dtype=np.float32)
    P = np.zeros(4, dtype=np.float32)
    ll = C.c_float()
    A = np.zeros(36, dtype=np.float32)
    b = np.zeros(6, dtype=np.float32)
    n = ref_lib(variant).ref_linearize(_fptr(rp), _fptr(cp), w, h, _fptr(K4), _dptr(T), ti, td, int(use_weights), _fptr(pp), C.byref(nsel),
                                _fptr(res), idx.ctypes.data_as(C.POINTER(C.c_int32)), _fptr(rec), _fptr(wts), _fptr(P), C.byref(ll),
                                _fptr(A), _fptr(b))
    n = int(n)
    return {"n": n, "n_selected": int(nsel.value), "residuals": res[:n], "index": idx[:n], "records": rec[:n], "weights": wts[:n],
            "precision": P.reshape(2, 2), "ll": ll.value, "A": A.reshape(6, 6), "b": b}
