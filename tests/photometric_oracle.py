"""The photometric mode on the CPU oracle (tests/native/photometric_oracle.cpp), built with the oracle's flags once per
process into a temporary directory that is removed as soon as the library is loaded.  Pyramids are this library's own (the
oracle's translation unit is part of it); a mask follows the NaN-depth model of tests/masked_oracle.py."""
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np

from oracle import oracle_py as orc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_lib = None


def lib():
    global _lib
    if _lib is None:
        tmp = tempfile.mkdtemp(prefix="dvo_photometric_")
        try:
            out = os.path.join(tmp, "libphotometric_oracle.so")
            subprocess.check_call(["g++", "-std=c++17", "-O3", "-mavx2", "-mfma", "-msse3", "-ffp-contract=off", "-frounding-math",
                                   "-fPIC", "-Wall", "-Wno-subobject-linkage", "-shared", "-o", out,
                                   os.path.join(ROOT, "tests", "native", "photometric_oracle.cpp")])
            L = C.CDLL(out)
        finally:
            shutil.rmtree(tmp, ignore_errors=True)   # the loaded library stays mapped
        fp, dp, vp = C.POINTER(C.c_float), C.POINTER(C.c_double), C.c_void_p
        L.orc_pyramid_create.restype = vp
        L.orc_pyramid_create.argtypes = [fp, fp, C.c_int, C.c_int, C.c_float, C.c_float, C.c_float, C.c_float, C.c_int]
        L.orc_pyramid_destroy.argtypes = [vp]
        L.orc_pyramid_plane.restype = fp
        L.orc_pyramid_plane.argtypes = [vp, C.c_int, C.c_int]
        L.orc_pyramid_level_info.argtypes = [vp, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int), fp]
        L.orc_residual_image_photometric.restype = C.c_int64
        L.orc_residual_image_photometric.argtypes = [vp, vp, C.c_int, dp, dp, C.c_float, C.c_float, C.POINTER(orc.Mode), fp]
        L.orc_linearize_photometric.restype = C.c_int64
        L.orc_linearize_photometric.argtypes = [vp, vp, C.c_int, dp, dp, C.c_float, C.c_float, C.c_int, fp, C.POINTER(orc.Mode), fp, fp,
                                                dp, dp]
        L.orc_match_photometric.restype = C.c_int
        L.orc_match_photometric.argtypes = [vp, vp, C.POINTER(orc.Config), dp, dp, C.POINTER(orc.Mode), C.POINTER(orc.Result), dp,
                                            C.POINTER(orc.IterationStats), C.c_int, C.POINTER(C.c_int)]
        L.orc_ldlt_solve8.argtypes = [dp, dp, dp]
        L.orc_schur_pose.argtypes = [dp, dp]
        _lib = L
    return _lib


def _d(a):
    return np.ascontiguousarray(np.asarray(a, dtype=np.float64)).ctypes.data_as(C.POINTER(C.c_double))


class Pyramid:
    def __init__(self, intensity, depth, intrinsics, levels, mask=None):
        """mask (h, w; nonzero = usable): NaN depth at every unusable pixel of every level after the build, which is the
        engine's rule in both roles (tests/masked_oracle.py)"""
        I = np.ascontiguousarray(intensity, dtype=np.float32)
        Z = np.ascontiguousarray(depth, dtype=np.float32)
        h, w = I.shape
        fp = C.POINTER(C.c_float)
        self.h = lib().orc_pyramid_create(I.ctypes.data_as(fp), Z.ctypes.data_as(fp), w, h, *intrinsics, levels)
        if mask is not None:
            from masked_oracle import usable_by_footprint
            for l, usable in enumerate(usable_by_footprint(mask, levels)):
                lw, lh = self.level_info(l)
                z = np.ctypeslib.as_array(lib().orc_pyramid_plane(self.h, l, 1), shape=(lh, lw))
                z[~usable] = np.nan

    def __del__(self):
        if getattr(self, "h", None) and _lib is not None:
            _lib.orc_pyramid_destroy(self.h)

    def level_info(self, level):
        w, h, K = C.c_int(), C.c_int(), (C.c_float * 4)()
        lib().orc_pyramid_level_info(self.h, level, C.byref(w), C.byref(h), K)
        return w.value, h.value


def residual_image(ref, cur, level, T, ab, m):
    w, h = ref.level_info(level)
    out = np.empty((7, h, w), dtype=np.float32)
    T, ab = np.ascontiguousarray(T, dtype=np.float64), np.ascontiguousarray(ab, dtype=np.float64)
    n = lib().orc_residual_image_photometric(ref.h, cur.h, level, _d(T), _d(ab), 0.0, 0.0, C.byref(m),
                                             out.ctypes.data_as(C.POINTER(C.c_float)))
    return int(n), out


def linearize(ref, cur, level, T, ab, m, use_weights=False, prev_precision=None):
    T, ab = np.ascontiguousarray(T, dtype=np.float64), np.ascontiguousarray(ab, dtype=np.float64)
    pp = np.ascontiguousarray(prev_precision if prev_precision is not None else np.zeros(4), dtype=np.float32).reshape(4)
    P, ll, A, b = np.zeros(4, np.float32), C.c_float(), np.zeros(64), np.zeros(8)
    fp = C.POINTER(C.c_float)
    n = lib().orc_linearize_photometric(ref.h, cur.h, level, _d(T), _d(ab), 0.0, 0.0, int(use_weights), pp.ctypes.data_as(fp), C.byref(m),
                                        P.ctypes.data_as(fp), C.byref(ll), A.ctypes.data_as(C.POINTER(C.c_double)),
                                        b.ctypes.data_as(C.POINTER(C.c_double)))
    return {"n": int(n), "precision": P.reshape(2, 2), "ll": ll.value, "A": A.reshape(8, 8), "b": b}


def match(ref, cur, cfg, m, T_init=None, ab_init=None):
    T0 = np.ascontiguousarray(T_init if T_init is not None else np.eye(4), dtype=np.float64)
    res, ab = orc.Result(), np.zeros(2)
    its, n = (orc.IterationStats * 1024)(), C.c_int()
    lib().orc_match_photometric(ref.h, cur.h, C.byref(cfg), _d(T0), _d(ab_init) if ab_init is not None else None, C.byref(m),
                                C.byref(res), ab.ctypes.data_as(C.POINTER(C.c_double)), its, 1024, C.byref(n))
    return {"T": np.array(res.transformation).reshape(4, 4), "information": np.array(res.information).reshape(6, 6),
            "log_likelihood": res.log_likelihood, "ab": ab,
            "levels": [(res.levels[i].termination, res.levels[i].num_iterations) for i in range(res.num_levels)]}
