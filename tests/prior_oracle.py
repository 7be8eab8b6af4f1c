"""The motion prior on the CPU oracle (tests/native/prior_oracle.cpp), in the default and the photometric mode, built with
the oracle's flags once per process into a temporary directory that is removed as soon as the library is loaded.  Pyramids
are this library's own (the oracle's translation unit is part of it)."""
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
        tmp = tempfile.mkdtemp(prefix="dvo_prior_")
        try:
            out = os.path.join(tmp, "libprior_oracle.so")
            subprocess.check_call(["g++", "-std=c++17", "-O3", "-mavx2", "-mfma", "-msse3", "-ffp-contract=off", "-frounding-math",
                                   "-fPIC", "-Wall", "-Wno-subobject-linkage", "-shared", "-o", out,
                                   os.path.join(ROOT, "tests", "native", "prior_oracle.cpp")])
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
        L.orc_match.restype = C.c_int
        L.orc_match.argtypes = [vp, vp, C.POINTER(orc.Config), dp, C.POINTER(orc.Mode), C.POINTER(orc.Result),
                                C.POINTER(orc.IterationStats), C.c_int, C.POINTER(C.c_int)]
        L.orc_match_photometric.restype = C.c_int
        L.orc_match_photometric.argtypes = [vp, vp, C.POINTER(orc.Config), dp, dp, C.POINTER(orc.Mode), C.POINTER(orc.Result), dp,
                                            C.POINTER(orc.IterationStats), C.c_int, C.POINTER(C.c_int)]
        L.orc_match_prior.restype = C.c_int
        L.orc_match_prior.argtypes = [vp, vp, C.POINTER(orc.Config), dp, dp, dp, C.POINTER(orc.Mode), C.POINTER(orc.Result), dp,
                                      C.POINTER(orc.IterationStats), C.c_int, C.POINTER(C.c_int)]
        _lib = L
    return _lib


def _d(a):
    return np.ascontiguousarray(np.asarray(a, dtype=np.float64)).ctypes.data_as(C.POINTER(C.c_double))


class Pyramid:
    def __init__(self, intensity, depth, intrinsics, levels, mask=None):
        """mask: as photometric_oracle.Pyramid's (NaN depth at every unusable pixel of every level, both roles)"""
        I = np.ascontiguousarray(intensity, dtype=np.float32)
        Z = np.ascontiguousarray(depth, dtype=np.float32)
        h, w = I.shape
        fp = C.POINTER(C.c_float)
        self.h = lib().orc_pyramid_create(I.ctypes.data_as(fp), Z.ctypes.data_as(fp), w, h, *intrinsics, levels)
        if mask is not None:
            from masked_oracle import usable_by_footprint
            for l, usable in enumerate(usable_by_footprint(mask, levels)):
                lw, lh, K = C.c_int(), C.c_int(), (C.c_float * 4)()
                lib().orc_pyramid_level_info(self.h, l, C.byref(lw), C.byref(lh), K)
                z = np.ctypeslib.as_array(lib().orc_pyramid_plane(self.h, l, 1), shape=(lh.value, lw.value))
                z[~usable] = np.nan

    def __del__(self):
        if getattr(self, "h", None) and _lib is not None:
            _lib.orc_pyramid_destroy(self.h)


def _out(res, its, n, ab=None):
    iters = [{"level": its[k].level, "id": its[k].id, "n": its[k].valid_constraints, "nll": its[k].tdist_log_likelihood,
              "precision": np.array(its[k].tdist_precision), "prior": its[k].prior_log_likelihood,
              "x": np.array(its[k].increment), "A": np.array(its[k].information).reshape(6, 6)} for k in range(min(n, len(its)))]
    return {"T": np.array(res.transformation).reshape(4, 4), "information": np.array(res.information).reshape(6, 6),
            "log_likelihood": res.log_likelihood, "ab": ab, "iterations": iters,
            "levels": [(res.levels[i].termination, res.levels[i].num_iterations) for i in range(res.num_levels)]}


def match(ref, cur, cfg, m, T_init=None, prior=None, photometric=False, ab_init=None):
    """prior None: the oracle's own match with cfg.mu (orc_match / orc_match_photometric); else orc_match_prior with that
    6 x 6 prior information."""
    T0 = np.ascontiguousarray(T_init if T_init is not None else np.eye(4), dtype=np.float64)
    res, ab = orc.Result(), np.zeros(2)
    its, n = (orc.IterationStats * 1024)(), C.c_int()
    abp = ab.ctypes.data_as(C.POINTER(C.c_double)) if photometric else None
    ab0 = _d(ab_init) if ab_init is not None else None
    if prior is not None:
        lib().orc_match_prior(ref.h, cur.h, C.byref(cfg), _d(T0), _d(np.asarray(prior, dtype=np.float64).reshape(36)), ab0, C.byref(m),
                              C.byref(res), abp, its, 1024, C.byref(n))
    elif photometric:
        lib().orc_match_photometric(ref.h, cur.h, C.byref(cfg), _d(T0), ab0, C.byref(m), C.byref(res), abp, its, 1024, C.byref(n))
    else:
        lib().orc_match(ref.h, cur.h, C.byref(cfg), _d(T0), C.byref(m), C.byref(res), its, 1024, C.byref(n))
    return _out(res, its, n.value, ab if photometric else None)
