"""ctypes binding of the C ABI in include/dvo_b200.h (dvo_slam_b200/libdvo_b200.so).

This is the harness-side view used by tests/ and bench.py; the product is the CUDA library and the
C++ adapter (include/dvo_b200/).  There is no CPU fallback: if the shared library is missing or no
CUDA device is present, construction raises.
"""
from __future__ import annotations

import ctypes as C
import operator
import os
import weakref

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("DVO_B200_LIB", os.path.join(_HERE, "libdvo_b200.so"))   # env override: developer A/B builds
MAX_LEVELS = 8
MAX_HYPOTHESES = 64   # DVO_B200_MAX_HYPOTHESES

TERMINATION_NAMES = ["IterationsExceeded", "IncrementTooSmall", "LogLikelihoodDecreased", "TooFewConstraints"]

# every symbol include/dvo_b200.h declares (checked by tests/test_abi.py)
ABI_SYMBOLS = [
    "dvo_b200_abi_version", "dvo_b200_create", "dvo_b200_destroy", "dvo_b200_stream", "dvo_b200_synchronize",
    "dvo_b200_last_error", "dvo_b200_config_default", "dvo_b200_kernel_launches", "dvo_b200_h2d_bytes",
    "dvo_b200_d2h_bytes", "dvo_b200_pyramid_create", "dvo_b200_pyramid_create_batch", "dvo_b200_pyramid_create_raw",
    "dvo_b200_pyramid_create_raw_batch", "dvo_b200_pyramid_create_bgr_batch",
    "dvo_b200_pyramid_retain", "dvo_b200_pyramid_release", "dvo_b200_pyramid_num_levels", "dvo_b200_pyramid_level_info",
    "dvo_b200_pyramid_download", "dvo_b200_pyramid_select", "dvo_b200_match", "dvo_b200_match_batch",
    "dvo_b200_match_batch_device", "dvo_b200_residual_image", "dvo_b200_intensity_error_image", "dvo_b200_linearize", "dvo_b200_match_batch_photometric", "dvo_b200_residual_image_photometric",
    "dvo_b200_linearize_photometric", "dvo_b200_profile_enable",
    "dvo_b200_profile_read", "dvo_b200_pyramid_device", "dvo_b200_sharded_create", "dvo_b200_sharded_destroy",
    "dvo_b200_sharded_num_shards", "dvo_b200_sharded_ctx", "dvo_b200_sharded_last_error", "dvo_b200_shard_range",
    "dvo_b200_sharded_pyramid_create_batch", "dvo_b200_sharded_pyramid_create_raw_batch", "dvo_b200_match_batch_sharded",
    "dvo_b200_set_estimator", "dvo_b200_get_estimator", "dvo_b200_pyramid_create_masked_batch",
    "dvo_b200_pyramid_create_masked_batch_roles", "dvo_b200_pyramid_mask_roles", "dvo_b200_pyramid_create_device_batch",
    "dvo_b200_undistort_map", "dvo_b200_rectifier_create", "dvo_b200_rectifier_release", "dvo_b200_pyramid_create_rectified_batch",
    "dvo_b200_pyramid_create_rectified_device_batch", "dvo_b200_depth_rays", "dvo_b200_depth_registration_create",
    "dvo_b200_depth_registration_release", "dvo_b200_pyramid_create_registered_batch",
    "dvo_b200_pyramid_create_registered_device_batch", "dvo_b200_match_batch_prior", "dvo_b200_match_batch_maps",
    "dvo_b200_match_batch_hypotheses", "dvo_b200_match_batch_hypotheses_modes",
]

# dvo_b200_estimator
ESTIMATORS = {"reference": 0, "corrected": 1}

# dvo_b200_input_format (dvo_b200_pyramid_create_masked_batch)
INPUT_FORMATS = {"float32": 0, "grey8_depth16": 1, "bgr8_depth16": 2}

# dvo_b200_weight_maps.memory
MAPS_MEMORY = {"device": 0, "host": 1}

# role sets of a mask (DVO_B200_MASK_ROLE_*): "reference" = the selection only, "both" = also the current image's taps
MASK_ROLES = {"reference": 1, "both": 3}


class Config(C.Structure):
    """dvo_b200_config; defaults = DenseTracker::Config (dense_tracking_config.cpp:27-42)."""
    _fields_ = [("first_level", C.c_int32), ("last_level", C.c_int32), ("max_iterations_per_level", C.c_int32),
                ("use_initial_estimate", C.c_int32), ("precision", C.c_double), ("mu", C.c_double),
                ("intensity_derivative_threshold", C.c_float), ("depth_derivative_threshold", C.c_float)]

    def __init__(self, **kw):
        super().__init__()
        self.first_level, self.last_level, self.max_iterations_per_level, self.use_initial_estimate = 3, 1, 100, 0
        self.precision, self.mu = 5e-7, 0.0
        self.intensity_derivative_threshold = self.depth_derivative_threshold = 0.0
        for k, v in kw.items():
            if not hasattr(self, k):
                raise AttributeError(k)
            setattr(self, k, v)


class DevicePlane(C.Structure):
    """dvo_b200_device_plane: one plane of a batch of images in device memory"""
    _fields_ = [("data", C.c_void_p), ("row_bytes", C.c_int64), ("image_bytes", C.c_int64)]


def device_planes(image, depth, masks=None, depth_size=None):
    """The arguments of dvo_b200_pyramid_create_device_batch for torch tensors, from their shapes, dtypes and strides alone
    (nothing is copied, and the tensors may live on any device):
        float32 [n,h,w] image + float32 [n,h,w] depth   -> "float32"
        uint8 [n,h,w] grey + uint16 [n,h,w] raw depth   -> "grey8_depth16"
        uint8 [n,h,w,3] BGR + uint16 [n,h,w] raw depth  -> "bgr8_depth16" (pixel stride 3, channel stride 1)
    masks: None, or bool / uint8 [n,h,w] or [h,w] (nonzero = usable); a [h,w] mask, or one expanded along n, is one mask
    for the whole batch (image_bytes 0).  Strided views such as a crop big[:, y0:y0+h, x0:x0+w] become a plane with the
    larger image's row pitch.  Returns (format, (n, h, w), image, depth, masks) with each plane a (data_ptr, row_bytes,
    image_bytes) tuple, masks None without a mask.  A layout that one row pitch and one image stride per plane cannot
    express (a column stride other than one pixel, rows that overlap) raises ValueError.  depth_size = (dw, dh): the depth
    planes are [n, dh, dw], a depth camera of its own (dvo_b200_pyramid_create_registered_device_batch)."""
    import torch
    if image.dtype == torch.float32 and image.dim() == 3:
        fmt, depth_dtype, px = "float32", torch.float32, 1
    elif image.dtype == torch.uint8 and image.dim() == 3:
        fmt, depth_dtype, px = "grey8_depth16", torch.uint16, 1
    elif image.dtype == torch.uint8 and image.dim() == 4 and image.shape[3] == 3:
        fmt, depth_dtype, px = "bgr8_depth16", torch.uint16, 3
    else:
        raise ValueError(f"image: {image.dtype} {tuple(image.shape)} is none of float32 [n,h,w], uint8 [n,h,w] (grey) or "
                         "uint8 [n,h,w,3] (BGR)")
    n, h, w = (int(v) for v in image.shape[:3])
    dw, dh = (w, h) if depth_size is None else (int(depth_size[0]), int(depth_size[1]))
    if depth.dtype != depth_dtype or tuple(depth.shape) != (n, dh, dw):
        raise ValueError(f"depth: {depth.dtype} {tuple(depth.shape)}, want {depth_dtype} {(n, dh, dw)} with a {fmt} image")
    if px == 3 and image.stride(3) != 1:
        raise ValueError(f"image: BGR channel stride {image.stride(3)}, want 1 (interleaved pixels)")

    def plane(t, name, per_px, shared=False):
        h, w = t.shape[1:3] if t.dim() >= 3 else t.shape
        es = t.element_size()
        if w > 1 and t.stride(-1 if per_px == 1 else -2) != per_px:
            raise ValueError(f"{name}: column stride {t.stride(-1 if per_px == 1 else -2)} elements, want {per_px} (pixels packed "
                             "within a row)")
        row = t.stride(-2 if per_px == 1 else -3) if h > 1 else w * per_px
        if row < w * per_px:
            raise ValueError(f"{name}: row stride {row} elements is below the {w * per_px} of a row (rows overlap)")
        img = 0 if shared or n == 1 else t.stride(0)
        return (t.data_ptr(), row * es, img * es)

    pm = None
    if masks is not None:
        if masks.dtype not in (torch.bool, torch.uint8):
            raise ValueError(f"masks: {masks.dtype}, want bool or uint8")
        if tuple(masks.shape) == (h, w):
            pm = plane(masks, "masks", 1, shared=True)
        elif tuple(masks.shape) == (n, h, w):
            pm = plane(masks, "masks", 1)
        else:
            raise ValueError(f"masks: shape {tuple(masks.shape)}, want {(n, h, w)} or {(h, w)}")
    return fmt, (n, h, w), plane(image, "image", px), plane(depth, "depth", 1), pm


def _host_frames(image, depth, depth_size=None):
    """Host arrays of n frames -> (format, (n, h, w), image, depth) with C-contiguous arrays, the format from the dtypes:
        float32 [n,h,w] image + float32 depth, uint8 [n,h,w] grey + uint16 raw depth, uint8 [n,h,w,3] BGR + uint16 raw depth.
    depth: [n,h,w], or [n,dh,dw] with depth_size = (dw, dh).  Raises ValueError for anything else."""
    image, depth = np.asarray(image), np.asarray(depth)
    if image.dtype == np.float32 and image.ndim == 3 and depth.dtype == np.float32:
        fmt = "float32"
    elif image.dtype == np.uint8 and image.ndim == 3 and depth.dtype == np.uint16:
        fmt = "grey8_depth16"
    elif image.dtype == np.uint8 and image.ndim == 4 and image.shape[3] == 3 and depth.dtype == np.uint16:
        fmt = "bgr8_depth16"
    else:
        raise ValueError(f"image {image.dtype} {image.shape} with depth {depth.dtype}: want float32 [n,h,w] + float32, uint8 "
                         "[n,h,w] + uint16 or uint8 [n,h,w,3] + uint16")
    n, h, w = image.shape[:3]
    dw, dh = (w, h) if depth_size is None else depth_size
    if depth.shape != (n, dh, dw):
        raise ValueError(f"depth {depth.shape}, want {(n, dh, dw)}" + ("" if depth_size is None else " (the depth camera's size)"))
    return fmt, (n, h, w), np.ascontiguousarray(image), np.ascontiguousarray(depth)


def _depth_scale(fmt, depth_scale) -> float:
    """depth_scale as the creates take it: required with raw depth"""
    if fmt != "float32" and depth_scale is None:
        raise ValueError(f"{fmt}: depth_scale (metres per raw depth unit) is required")
    return float(depth_scale or 0.0)


def _host_masks(masks, n, h, w):
    """Host masks of n images of h x w -> (pointer, array): an int is a host pointer to n*h*w bytes (array None); an array
    of [h, w] is one mask for the whole batch; any other array must hold n*h*w values (nonzero = usable).  The array is the
    caller's own when it is C-contiguous uint8, else a converted copy that must outlive the create's upload."""
    if isinstance(masks, int):
        return masks, None
    M = np.asarray(masks)
    if M.size != n * h * w:
        if M.shape != (h, w):
            raise ValueError(f"masks {M.shape} for {n} images of {h}x{w}: want {(n, h, w)}, {(h, w)} or {n * h * w} values")
        M = np.broadcast_to(M, (n, h, w))
    M = np.ascontiguousarray(M if M.dtype == np.uint8 else M != 0, dtype=np.uint8)
    return M.ctypes.data, M


def _mask_roles(mask_roles) -> int:
    if mask_roles not in MASK_ROLES:
        raise ValueError(f"unknown mask_roles {mask_roles!r}: one of {sorted(MASK_ROLES)}")
    return MASK_ROLES[mask_roles]


_DP = C.POINTER(C.c_double)


def _ptr(a, ptype=_DP):
    """a numpy array as a C pointer, None as NULL"""
    return a.ctypes.data_as(ptype) if a is not None else None


def _rows(a, name, want, width):
    """An optional float64 input of shape want (per pair or per hypothesis) as C-contiguous rows of width values; None
    stays None.  Any other number of values raises ValueError."""
    if a is None:
        return None
    A = np.asarray(a, dtype=np.float64)
    if A.size != int(np.prod(want)):
        raise ValueError(f"{name} {A.shape}: want {list(want)}")
    return np.ascontiguousarray(A.reshape(-1, width))


def _photometric_init(photometric, photometric_init, want):
    """the (alpha, beta)_0 rows of the photometric mode, None = (1, 0); refused without the mode"""
    if photometric_init is not None and not photometric:
        raise ValueError("photometric_init without photometric=True")
    return _rows(photometric_init, "photometric_init", want, 2)


def _handles(pyramids, attr="handle"):
    """the C array of n pyramid handles: Pyramid.handle, or attr="value" for ShardedEngine's c_void_p handles"""
    return (C.c_void_p * len(pyramids))(*map(operator.attrgetter(attr), pyramids))


def _iteration_log(cfg, n, with_iterations):
    """(log, max_log): room for every iteration of levels cfg.first_level .. cfg.last_level per pair, or (None, 0)"""
    if not with_iterations:
        return None, 0
    max_log = (cfg.first_level - cfg.last_level + 1) * (cfg.max_iterations_per_level + 1)
    return (IterationStats * (n * max_log))(), max_log


class IterationStats(C.Structure):
    _fields_ = [("level", C.c_int32), ("id", C.c_int32), ("valid_constraints", C.c_int64),
                ("tdist_log_likelihood", C.c_double), ("tdist_precision", C.c_double * 4),
                ("prior_log_likelihood", C.c_double), ("increment", C.c_double * 6), ("information", C.c_double * 36)]


class LevelStats(C.Structure):
    _fields_ = [("id", C.c_int32), ("termination", C.c_int32), ("max_valid_pixels", C.c_int64),
                ("valid_pixels", C.c_int64), ("num_iterations", C.c_int32), ("has_iteration_with_increment", C.c_int32),
                ("last_valid_constraints", C.c_int64), ("last_increment_valid_constraints", C.c_int64),
                ("last_increment_log_likelihood", C.c_double)]


class MapPlane(C.Structure):
    """dvo_b200_map_plane: one output plane of dvo_b200_match_batch_maps (data NULL: not written)"""
    _fields_ = [("data", C.c_void_p), ("row_bytes", C.c_int64), ("image_bytes", C.c_int64)]


class WeightMaps(C.Structure):
    """dvo_b200_weight_maps: where dvo_b200_match_batch_maps writes each pair's maps"""
    _fields_ = [("memory", C.c_int32), ("weight", MapPlane), ("residual_i", MapPlane), ("residual_z", MapPlane), ("mask", MapPlane),
                ("mask_weight", C.c_float), ("estimate", C.POINTER(C.c_double)), ("precision", C.POINTER(C.c_float))]


class CResult(C.Structure):
    _fields_ = [("transformation", C.c_double * 16), ("information", C.c_double * 36), ("log_likelihood", C.c_double),
                ("num_levels", C.c_int32), ("num_iterations_total", C.c_int32), ("levels", LevelStats * MAX_LEVELS)]


class Result:
    """Python view of dvo_b200_result (dvo::DenseTracker::Result, dense_tracking.h:125-140)."""

    def __init__(self, c: CResult, iterations=None):
        self.transformation = np.array(c.transformation).reshape(4, 4)
        self.information = np.array(c.information).reshape(6, 6)
        self.log_likelihood = c.log_likelihood
        self.num_iterations_total = c.num_iterations_total
        self.levels = []
        for i in range(c.num_levels):
            l = c.levels[i]
            self.levels.append({"id": l.id, "termination": l.termination, "max_valid_pixels": l.max_valid_pixels,
                                "valid_pixels": l.valid_pixels, "num_iterations": l.num_iterations,
                                "has_iteration_with_increment": bool(l.has_iteration_with_increment),
                                "last_valid_constraints": l.last_valid_constraints,
                                "last_increment_valid_constraints": l.last_increment_valid_constraints,
                                "last_increment_log_likelihood": l.last_increment_log_likelihood})
        self.iterations = iterations or []

    def is_nan(self) -> bool:  # Result::isNaN (dense_tracking_config.cpp:96-99)
        return not (np.isfinite(self.transformation.sum()) and np.isfinite(self.information.sum()))


def prior_from_result(result: Result, scale: float = 1.0) -> np.ndarray:
    """A motion prior (Engine.match_batch(prior_information=...)) from an earlier alignment of the same motion:
    scale * Result.information / 0.008^2, in the units of the normal equations, made exactly symmetric (the photometric
    mode's Schur complement is symmetric only to rounding).  scale < 1 trusts the earlier alignment less."""
    lam = np.asarray(result.information, dtype=np.float64).reshape(6, 6) * (scale / 0.008 ** 2)
    return 0.5 * (lam + lam.T)


def _results(res, n, log=None, max_log=0) -> list[Result]:
    """Result views of n dvo_b200_result, with each pair's iterations when a log of max_log entries per pair is given"""
    out = []
    for i in range(n):
        its = []
        if log is not None:
            for k in range(res[i].num_iterations_total):
                s = log[i * max_log + k]
                its.append({"level": s.level, "id": s.id, "n": s.valid_constraints, "nll": s.tdist_log_likelihood,
                            "precision": np.array(s.tdist_precision).reshape(2, 2), "prior": s.prior_log_likelihood,
                            "x": np.array(s.increment), "A": np.array(s.information).reshape(6, 6)})
        out.append(Result(res[i], its))
    return out


_lib = None


def load_library():
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(f"{LIB_PATH} is missing: run `python __graft_entry__.py` (nvcc, sm_90a). "
                           "There is no CPU fallback for the engine.")
    L = C.CDLL(LIB_PATH)
    vp, fp, dp, i32, i64 = C.c_void_p, C.POINTER(C.c_float), C.POINTER(C.c_double), C.c_int32, C.c_int64
    L.dvo_b200_abi_version.restype = C.c_int
    L.dvo_b200_create.argtypes = [C.c_int, vp, C.POINTER(vp)]
    L.dvo_b200_destroy.argtypes = [vp]
    L.dvo_b200_stream.restype = vp
    L.dvo_b200_stream.argtypes = [vp]
    L.dvo_b200_synchronize.argtypes = [vp]
    L.dvo_b200_last_error.restype = C.c_char_p
    L.dvo_b200_last_error.argtypes = [vp]
    L.dvo_b200_config_default.argtypes = [C.POINTER(Config)]
    L.dvo_b200_config_default.restype = None
    for f in (L.dvo_b200_kernel_launches, L.dvo_b200_h2d_bytes, L.dvo_b200_d2h_bytes):
        f.restype = i64
        f.argtypes = [vp]
    L.dvo_b200_pyramid_create.argtypes = [vp, vp, vp, i32, i32, C.c_float, C.c_float, C.c_float, C.c_float, i32, C.POINTER(vp)]
    L.dvo_b200_pyramid_create_batch.argtypes = [vp, i32, vp, vp, i32, i32, C.c_float, C.c_float, C.c_float, C.c_float, i32, C.POINTER(vp)]
    L.dvo_b200_pyramid_create_raw.argtypes = [vp, vp, vp, C.c_float, i32, i32, C.c_float, C.c_float, C.c_float, C.c_float, i32, C.POINTER(vp)]
    L.dvo_b200_pyramid_create_raw_batch.argtypes = [vp, i32, vp, vp, C.c_float, i32, i32, C.c_float, C.c_float, C.c_float, C.c_float, i32, C.POINTER(vp)]
    L.dvo_b200_pyramid_create_bgr_batch.argtypes = [vp, i32, vp, vp, C.c_float, i32, i32, C.c_float, C.c_float, C.c_float, C.c_float, i32, C.POINTER(vp)]
    L.dvo_b200_pyramid_create_masked_batch.argtypes = [vp, i32, i32, vp, vp, C.c_float, vp, i32, i32, C.c_float, C.c_float, C.c_float,
                                                       C.c_float, i32, C.POINTER(vp)]
    L.dvo_b200_pyramid_create_masked_batch_roles.argtypes = [vp, i32, i32, vp, vp, C.c_float, vp, i32, i32, i32, C.c_float, C.c_float,
                                                             C.c_float, C.c_float, i32, C.POINTER(vp)]
    L.dvo_b200_pyramid_create_device_batch.argtypes = [vp, i32, i32, C.POINTER(DevicePlane), C.POINTER(DevicePlane), C.c_float,
                                                       C.POINTER(DevicePlane), i32, i32, i32, C.c_float, C.c_float, C.c_float,
                                                       C.c_float, i32, C.POINTER(vp)]
    L.dvo_b200_pyramid_mask_roles.argtypes = [vp]
    L.dvo_b200_undistort_map.argtypes = [i32, i32, dp, dp, dp, fp, fp]
    L.dvo_b200_rectifier_create.argtypes = [vp, i32, i32, i32, i32, fp, fp, fp, C.POINTER(vp)]
    L.dvo_b200_rectifier_release.argtypes = [vp]
    L.dvo_b200_pyramid_create_rectified_batch.argtypes = [vp, vp, i32, i32, vp, vp, C.c_float, vp, i32, i32, i32, i32, C.POINTER(vp)]
    L.dvo_b200_pyramid_create_rectified_device_batch.argtypes = [vp, vp, i32, i32, C.POINTER(DevicePlane), C.POINTER(DevicePlane),
                                                                 C.c_float, C.POINTER(DevicePlane), i32, i32, i32, i32, C.POINTER(vp)]
    L.dvo_b200_depth_rays.argtypes = [i32, i32, dp, dp, fp, fp, fp, fp]
    L.dvo_b200_depth_registration_create.argtypes = [vp, i32, i32, fp, fp, fp, fp, dp, i32, i32, fp, C.POINTER(vp)]
    L.dvo_b200_depth_registration_release.argtypes = [vp]
    L.dvo_b200_pyramid_create_registered_batch.argtypes = [vp, vp, vp, i32, i32, vp, vp, C.c_float, vp, i32, i32, i32, i32,
                                                           C.POINTER(vp)]
    L.dvo_b200_pyramid_create_registered_device_batch.argtypes = [vp, vp, vp, i32, i32, C.POINTER(DevicePlane), C.POINTER(DevicePlane),
                                                                  C.c_float, C.POINTER(DevicePlane), i32, i32, i32, i32, C.POINTER(vp)]
    L.dvo_b200_pyramid_device.argtypes = [vp]
    L.dvo_b200_sharded_create.argtypes = [i32, C.POINTER(i32), C.POINTER(vp)]
    L.dvo_b200_sharded_destroy.argtypes = [vp]
    L.dvo_b200_sharded_num_shards.argtypes = [vp]
    L.dvo_b200_sharded_ctx.restype = vp
    L.dvo_b200_sharded_ctx.argtypes = [vp, i32]
    L.dvo_b200_sharded_last_error.restype = C.c_char_p
    L.dvo_b200_sharded_last_error.argtypes = [vp]
    L.dvo_b200_shard_range.argtypes = [i64, i32, i32, C.POINTER(i64), C.POINTER(i64)]
    L.dvo_b200_sharded_pyramid_create_batch.argtypes = [vp, i32, vp, vp, i32, i32, C.c_float, C.c_float, C.c_float, C.c_float, i32, C.POINTER(vp)]
    L.dvo_b200_sharded_pyramid_create_raw_batch.argtypes = [vp, i32, vp, vp, C.c_float, i32, i32, C.c_float, C.c_float, C.c_float, C.c_float, i32,
                                                        C.POINTER(vp)]
    L.dvo_b200_match_batch_sharded.argtypes = [vp, C.POINTER(Config), i32, C.POINTER(vp), C.POINTER(vp), dp, C.POINTER(CResult),
                                               C.POINTER(IterationStats), i32]
    L.dvo_b200_pyramid_retain.argtypes = [vp]
    L.dvo_b200_pyramid_release.argtypes = [vp]
    L.dvo_b200_pyramid_num_levels.argtypes = [vp]
    L.dvo_b200_pyramid_level_info.argtypes = [vp, i32, C.POINTER(i32), C.POINTER(i32), fp]
    L.dvo_b200_pyramid_download.argtypes = [vp, vp, i32, fp]
    L.dvo_b200_pyramid_select.argtypes = [vp, vp, i32, C.c_float, C.c_float, C.POINTER(i64), C.POINTER(C.c_uint8)]
    L.dvo_b200_match.argtypes = [vp, C.POINTER(Config), vp, vp, dp, C.POINTER(CResult)]
    L.dvo_b200_match_batch.argtypes = [vp, C.POINTER(Config), i32, C.POINTER(vp), C.POINTER(vp), dp, C.POINTER(CResult),
                                       C.POINTER(IterationStats), i32]
    L.dvo_b200_match_batch_device.argtypes = [vp, C.POINTER(Config), i32, C.POINTER(vp), C.POINTER(vp), dp, vp]
    L.dvo_b200_residual_image.argtypes = [vp, C.POINTER(Config), vp, vp, i32, dp, fp, C.POINTER(i64)]
    L.dvo_b200_intensity_error_image.argtypes = [vp, C.POINTER(Config), vp, vp, i32, dp, fp, C.POINTER(i64)]
    L.dvo_b200_linearize.argtypes = [vp, C.POINTER(Config), vp, vp, i32, dp, i32, fp, C.POINTER(i64), fp, fp, dp, dp]
    L.dvo_b200_match_batch_photometric.argtypes = [vp, C.POINTER(Config), i32, C.POINTER(vp), C.POINTER(vp), dp, dp, C.POINTER(CResult),
                                                   dp, C.POINTER(IterationStats), i32]
    L.dvo_b200_match_batch_prior.argtypes = [vp, C.POINTER(Config), i32, C.POINTER(vp), C.POINTER(vp), dp, dp, dp, dp, C.POINTER(CResult),
                                             C.POINTER(IterationStats), i32]
    L.dvo_b200_match_batch_maps.argtypes = [vp, C.POINTER(Config), i32, C.POINTER(vp), C.POINTER(vp), dp, dp, dp, dp, C.POINTER(CResult),
                                            C.POINTER(IterationStats), i32, C.POINTER(WeightMaps)]
    L.dvo_b200_match_batch_hypotheses.argtypes = [vp, C.POINTER(Config), i32, C.POINTER(vp), C.POINTER(vp), i32, dp, i32, C.c_double,
                                                   C.POINTER(CResult), C.POINTER(i32), dp, C.POINTER(CResult), C.POINTER(IterationStats), i32]
    L.dvo_b200_match_batch_hypotheses_modes.argtypes = [vp, C.POINTER(Config), i32, C.POINTER(vp), C.POINTER(vp), i32, dp, i32, C.c_double,
                                                         dp, dp, dp, dp, C.POINTER(CResult), C.POINTER(i32), dp, C.POINTER(CResult),
                                                         C.POINTER(IterationStats), i32, C.POINTER(WeightMaps)]
    L.dvo_b200_residual_image_photometric.argtypes = [vp, C.POINTER(Config), vp, vp, i32, dp, dp, fp, C.POINTER(i64)]
    L.dvo_b200_linearize_photometric.argtypes = [vp, C.POINTER(Config), vp, vp, i32, dp, dp, i32, fp, C.POINTER(i64), fp, fp, dp, dp]
    L.dvo_b200_set_estimator.argtypes = [vp, i32]
    L.dvo_b200_get_estimator.argtypes = [vp]
    L.dvo_b200_profile_enable.argtypes = [vp, i32]
    L.dvo_b200_profile_read.argtypes = [vp, dp, C.POINTER(i64), i32]
    _lib = L
    return L


class Pyramid:
    """Owning handle of a dvo_b200_pyramid (device mirror of dvo::core::RgbdImagePyramid)."""

    def __init__(self, engine: "Engine", handle: int):
        self.engine, self.handle = engine, handle

    @property
    def num_levels(self) -> int:
        return load_library().dvo_b200_pyramid_num_levels(self.handle)

    def level_info(self, level: int):
        w, h = C.c_int32(), C.c_int32()
        K = (C.c_float * 4)()
        self.engine._check(load_library().dvo_b200_pyramid_level_info(self.handle, level, C.byref(w), C.byref(h), K))
        return w.value, h.value, tuple(K)

    @property
    def mask_roles(self) -> str | None:
        """None (no mask), "reference" or "both" (see Engine.pyramid)"""
        r = load_library().dvo_b200_pyramid_mask_roles(self.handle)
        self.engine._check(min(r, 0))
        return {0: None, 1: "reference", 3: "both"}[r]

    def download(self, level: int) -> np.ndarray:
        w, h, _ = self.level_info(level)
        out = np.empty((6, h, w), dtype=np.float32)
        self.engine._check(load_library().dvo_b200_pyramid_download(self.engine.ctx, self.handle, level,
                                                                    out.ctypes.data_as(C.POINTER(C.c_float))))
        return out

    def select(self, level: int, ti: float = 0.0, td: float = 0.0):
        w, h, _ = self.level_info(level)
        mask = np.zeros((h, w), dtype=np.uint8)
        cnt = C.c_int64()
        self.engine._check(load_library().dvo_b200_pyramid_select(self.engine.ctx, self.handle, level, ti, td, C.byref(cnt),
                                                                  mask.ctypes.data_as(C.POINTER(C.c_uint8))))
        return cnt.value, mask

    def release(self):
        if self.handle:
            load_library().dvo_b200_pyramid_release(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.release()
        except Exception:
            pass


def undistort_map(width: int, height: int, K, dist, K_new=None):
    """dvo_b200_undistort_map: (map_x, map_y), float32 [height, width] each, of OpenCV's plumb-bob model with R = I
    (cv2.initUndistortRectifyMap(K, dist, None, K_new, (width, height), cv2.CV_32FC1)).  K, K_new: (fx, fy, cx, cy), K_new
    defaults to K; dist: (k1, k2, p1, p2, k3).  Host only: no context and no GPU."""
    K = np.ascontiguousarray(K, dtype=np.float64).reshape(4)
    Kn = np.ascontiguousarray(K if K_new is None else K_new, dtype=np.float64).reshape(4)
    d = np.ascontiguousarray(dist, dtype=np.float64).reshape(5)
    mx, my = np.empty((height, width), np.float32), np.empty((height, width), np.float32)
    dp, fp = C.POINTER(C.c_double), C.POINTER(C.c_float)
    rc = load_library().dvo_b200_undistort_map(width, height, K.ctypes.data_as(dp), d.ctypes.data_as(dp), Kn.ctypes.data_as(dp),
                                               mx.ctypes.data_as(fp), my.ctypes.data_as(fp))
    if rc != 0:
        raise ValueError(f"dvo_b200_undistort_map: status {rc} (sizes {width}x{height}, K {K}, dist {d}, K_new {Kn})")
    return mx, my


class Rectifier:
    """Owning handle of a dvo_b200_rectifier: a remap of in_size = (w, h) frames to a pinhole camera K_new of size
    (w, h) = size.  Released with release(), when collected, or when its engine closes."""

    def __init__(self, engine: "Engine", handle: int, in_size, size, K_new):
        self.engine, self.handle = engine, handle
        self.in_size, self.size, self.K_new = tuple(in_size), tuple(size), tuple(K_new)

    def release(self):
        if self.handle:
            load_library().dvo_b200_rectifier_release(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.release()
        except Exception:
            pass


def depth_rays(size, K, dist=None):
    """dvo_b200_depth_rays: the ray tables (cx_ray, cy_ray, kx_ray, ky_ray) of a depth camera of size = (dw, dh) with
    intrinsics K = (fx, fy, cx, cy): float32 [dh, dw] rays through the pixel centres and [dh+1, dw+1] rays through the pixel
    corners (u - 0.5, v - 0.5), normalised to z = 1.  dist: None (pinhole) or plumb-bob (k1, k2, p1, p2, k3), inverted by
    Newton's method.  Host only: no context and no GPU."""
    dw, dh = (int(v) for v in size)
    Kd = np.ascontiguousarray(K, dtype=np.float64).reshape(4)
    d = None if dist is None else np.ascontiguousarray(dist, dtype=np.float64).reshape(5)
    cx, cy = np.empty((dh, dw), np.float32), np.empty((dh, dw), np.float32)
    kx, ky = np.empty((dh + 1, dw + 1), np.float32), np.empty((dh + 1, dw + 1), np.float32)
    dp, fp = C.POINTER(C.c_double), C.POINTER(C.c_float)
    rc = load_library().dvo_b200_depth_rays(dw, dh, Kd.ctypes.data_as(dp), None if d is None else d.ctypes.data_as(dp),
                                            *(a.ctypes.data_as(fp) for a in (cx, cy, kx, ky)))
    if rc != 0:
        raise ValueError(f"dvo_b200_depth_rays: status {rc} (size {dw}x{dh}, K {Kd}, dist {d})")
    return cx, cy, kx, ky


class DepthRegistration:
    """Owning handle of a dvo_b200_depth_registration: a depth camera of depth_size = (dw, dh) reprojected into a pinhole
    colour camera K of size = (w, h).  Released with release(), when collected, or when its engine closes."""

    def __init__(self, engine: "Engine", handle: int, depth_size, size, K):
        self.engine, self.handle = engine, handle
        self.depth_size, self.size, self.K = tuple(depth_size), tuple(size), tuple(K)

    def release(self):
        if self.handle:
            load_library().dvo_b200_depth_registration_release(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.release()
        except Exception:
            pass


class Engine:
    """One dvo_b200_ctx (one CUDA stream on one device).  estimator: "reference" (dvo::DenseTracker::match()'s numbers) or
    "corrected" (the same algorithm without the reference's scale-pairing, log-likelihood-tail and odd-point quirks; see
    dvo_b200_estimator in include/dvo_b200.h).  It applies to every later call on the engine."""

    def __init__(self, device: int = 0, stream: int | None = None, estimator: str = "reference"):
        self.lib = load_library()
        if estimator not in ESTIMATORS:
            raise ValueError(f"unknown estimator {estimator!r}: one of {sorted(ESTIMATORS)}")
        ctx = C.c_void_p()
        rc = self.lib.dvo_b200_create(device, C.c_void_p(stream) if stream else None, C.byref(ctx))
        if rc != 0:
            raise RuntimeError(f"dvo_b200_create(device={device}) failed with status {rc}: no usable CUDA device "
                               "(the engine has no CPU fallback)")
        self.ctx = ctx
        self.device = device
        self._rectifiers = weakref.WeakSet()
        self._registrations = weakref.WeakSet()
        self.set_estimator(estimator)

    def set_estimator(self, estimator: str):
        if estimator not in ESTIMATORS:
            raise ValueError(f"unknown estimator {estimator!r}: one of {sorted(ESTIMATORS)}")
        self._check(self.lib.dvo_b200_set_estimator(self.ctx, ESTIMATORS[estimator]))

    @property
    def estimator(self) -> str:
        e = self.lib.dvo_b200_get_estimator(self.ctx)
        self._check(min(e, 0))
        return {v: k for k, v in ESTIMATORS.items()}[e]

    def close(self):
        if getattr(self, "ctx", None):
            for r in list(getattr(self, "_rectifiers", ())):   # a rectifier is freed on its context's stream
                r.release()
            for r in list(getattr(self, "_registrations", ())):   # so is a depth registration
                r.release()
            self.lib.dvo_b200_destroy(self.ctx)
            self.ctx = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc: int):
        if rc != 0:
            raise RuntimeError(f"dvo_b200 status {rc}: {self.lib.dvo_b200_last_error(self.ctx).decode()}")

    @property
    def stream(self) -> int:
        return self.lib.dvo_b200_stream(self.ctx)

    def synchronize(self):
        self._check(self.lib.dvo_b200_synchronize(self.ctx))

    def kernel_launches(self) -> int:
        return self.lib.dvo_b200_kernel_launches(self.ctx)

    def h2d_bytes(self) -> int:
        return self.lib.dvo_b200_h2d_bytes(self.ctx)

    def d2h_bytes(self) -> int:
        return self.lib.dvo_b200_d2h_bytes(self.ctx)

    # ---- pyramids ----
    # mask= / masks=: reference masks (dvo_b200_pyramid_create_masked_batch): None, an array of n*h*w values (nonzero = usable
    # reference pixel; shape [n, h, w], or [h, w] for one mask of the whole batch) or, for the host-pointer forms, a host
    # pointer (int) to n*h*w bytes.
    # mask_roles="reference" (default): the mask keeps its pixels out of the point selection; "both": also out of the
    # bilinear taps when the pyramid is the current image of an alignment (dvo_b200_pyramid_create_masked_batch_roles).
    def _create_host(self, fmt, n, h, w, pI, pZ, depth_scale, masks, mask_roles, levels, intrinsics=None, remap=None, single=False,
                     sync=False) -> list[Pyramid]:
        """Every create from host memory: n images of h x w in format fmt at pI / pZ.  remap = (rectifier, registration):
        dvo_b200_pyramid_create_rectified_batch (registration None) or _registered_batch, which take the masks themselves.
        Otherwise masks -> dvo_b200_pyramid_create_masked_batch_roles, without masks the plain entry point of the format
        (single: the one-image form).  Synchronises when the masks were converted (except a remapped create) and, with
        sync, when the caller's staged arrays die with the call."""
        roles = _mask_roles(mask_roles) if masks is not None or remap is not None else None
        pM, M = _host_masks(masks, n, h, w) if masks is not None else (None, None)   # M: kept until the upload is done
        f = INPUT_FORMATS[fmt]
        out = (C.c_void_p * n)()
        if remap is not None:
            rect, reg = remap
            rh = rect.handle if rect is not None else None
            args = (n, f, pI, pZ, depth_scale, pM, roles, w, h, levels, out)
            if reg is None:
                rc = self.lib.dvo_b200_pyramid_create_rectified_batch(self.ctx, rh, *args)
            else:
                rc = self.lib.dvo_b200_pyramid_create_registered_batch(self.ctx, reg.handle, rh, *args)
        else:
            fx, fy, ox, oy = intrinsics
            if masks is not None:
                rc = self.lib.dvo_b200_pyramid_create_masked_batch_roles(self.ctx, n, f, pI, pZ, depth_scale, pM, roles, w, h, fx, fy,
                                                                         ox, oy, levels, out)
            else:
                entry = {("float32", True): "create", ("float32", False): "create_batch", ("grey8_depth16", True): "create_raw",
                         ("grey8_depth16", False): "create_raw_batch", ("bgr8_depth16", False): "create_bgr_batch"}[fmt, single]
                args = (() if single else (n,)) + (pI, pZ) + (() if fmt == "float32" else (depth_scale,))
                rc = getattr(self.lib, "dvo_b200_pyramid_" + entry)(self.ctx, *args, w, h, fx, fy, ox, oy, levels, out)
        self._check(rc)
        if M is not None and M is not masks and remap is None:
            self.synchronize()   # the converted masks die with this call
        if sync:
            self.synchronize()   # so may the caller's staged arrays
        return [Pyramid(self, out[i]) for i in range(n)]

    def pyramid(self, intensity, depth, intrinsics, levels: int, mask=None, mask_roles="reference") -> Pyramid:
        I = np.ascontiguousarray(intensity, dtype=np.float32)
        Z = np.ascontiguousarray(depth, dtype=np.float32)
        assert I.ndim == 2 and I.shape == Z.shape
        return self._create_host("float32", 1, *I.shape, I.ctypes.data, Z.ctypes.data, 0.0, mask, mask_roles, levels, intrinsics,
                                 single=True, sync=True)[0]

    def pyramid_batch(self, intensity, depth, intrinsics, levels: int, host_ptrs=None, masks=None, mask_roles="reference") -> list[Pyramid]:
        """intensity/depth: [n,h,w] float32 arrays, or (ptr_I, ptr_Z, n, h, w) raw host pointers via host_ptrs."""
        if host_ptrs is not None:
            pI, pZ, n, h, w = host_ptrs
        else:
            I = np.ascontiguousarray(intensity, dtype=np.float32)
            Z = np.ascontiguousarray(depth, dtype=np.float32)
            assert I.ndim == 3 and I.shape == Z.shape
            (n, h, w), pI, pZ = I.shape, I.ctypes.data, Z.ctypes.data
        return self._create_host("float32", n, h, w, pI, pZ, 0.0, masks, mask_roles, levels, intrinsics, sync=host_ptrs is None)

    def pyramid_raw_batch(self, host_ptrs, depth_scale, intrinsics, levels: int, masks=None, mask_roles="reference") -> list[Pyramid]:
        """host_ptrs = (ptr_grey_u8, ptr_depth_u16, n, h, w): n consecutive raw images in (pinned) host memory."""
        pG, pD, n, h, w = host_ptrs
        return self._create_host("grey8_depth16", n, h, w, pG, pD, depth_scale, masks, mask_roles, levels, intrinsics)

    def pyramid_bgr_batch(self, host_ptrs, depth_scale, intrinsics, levels: int, masks=None, mask_roles="reference") -> list[Pyramid]:
        """host_ptrs = (ptr_bgr_u8x3, ptr_depth_u16, n, h, w): n consecutive interleaved-BGR images and raw depth images
        in (pinned) host memory; grey conversion (OpenCV BGR2GRAY) and depth scaling run on the device."""
        pC, pD, n, h, w = host_ptrs
        return self._create_host("bgr8_depth16", n, h, w, pC, pD, depth_scale, masks, mask_roles, levels, intrinsics)

    def pyramid_batch_device(self, image, depth, intrinsics, levels: int, depth_scale=None, masks=None,
                             mask_roles="reference") -> list[Pyramid]:
        """Pyramids from torch CUDA tensors on the engine's device, read in place (dvo_b200_pyramid_create_device_batch): no
        host round trip and no host synchronisation.  The format follows from the dtypes and shapes (device_planes);
        depth_scale (metres per raw depth unit) is required for uint16 depth.  masks / mask_roles as in pyramid_batch.
        Ordered with torch: the engine's stream waits for the current stream before the build, and the current stream waits
        for the build after it, so the inputs may be produced and overwritten on the current stream."""
        roles = _mask_roles(mask_roles)
        fx, fy, ox, oy = intrinsics
        return self._create_device(image, depth, masks, depth_scale, None, lambda n, fmt, I, Z, scale, M, w, h, out:
                                   self.lib.dvo_b200_pyramid_create_device_batch(self.ctx, n, fmt, I, Z, scale, M, roles, w, h, fx, fy,
                                                                                 ox, oy, levels, out))

    def _create_device(self, image, depth, masks, depth_scale, depth_size, create) -> list[Pyramid]:
        """A device create from torch CUDA tensors (device_planes), ordered with torch's current stream: the engine's stream
        waits for it, the tensors' memory is kept until the build has read it, and the current stream waits for the build.
        create(n, format, image, depth, depth_scale, masks, w, h, out) calls the entry point with the planes."""
        import torch
        fmt, (n, h, w), pI, pZ, pM = device_planes(image, depth, masks, depth_size=depth_size)
        scale = _depth_scale(fmt, depth_scale)
        dev = torch.device("cuda", self.device)
        inputs = [t for t in (image, depth, masks) if t is not None]
        for t in inputs:
            if t.device != dev:
                raise ValueError(f"a tensor on {t.device}: the engine runs on {dev}")
        I, Z = DevicePlane(*pI), DevicePlane(*pZ)
        M = DevicePlane(*pM) if pM is not None else None
        out = (C.c_void_p * n)()
        current = torch.cuda.current_stream(dev)
        ext = torch.cuda.ExternalStream(self.stream, device=dev)
        ext.wait_stream(current)
        for t in inputs:
            t.record_stream(ext)     # the caching allocator keeps the memory until the build has read it
        rc = create(n, INPUT_FORMATS[fmt], C.byref(I), C.byref(Z), scale, C.byref(M) if M is not None else None, w, h, out)
        current.wait_stream(ext)
        self._check(rc)
        return [Pyramid(self, out[i]) for i in range(n)]

    # ---- distorted cameras ----
    undistort_map = staticmethod(undistort_map)

    def rectifier(self, in_size, map_x, map_y, K_new) -> Rectifier:
        """dvo_b200_rectifier_create: frames of in_size = (w, h) remapped through map_x / map_y (float32 [h', w'] input pixel
        coordinates, e.g. from undistort_map or cv2.initUndistortRectifyMap(..., cv2.CV_32FC1)) to a pinhole camera K_new =
        (fx, fy, cx, cy) of size (w', h').  The map is uploaded once."""
        mx = np.ascontiguousarray(map_x, dtype=np.float32)
        my = np.ascontiguousarray(map_y, dtype=np.float32)
        if mx.ndim != 2 or mx.shape != my.shape:
            raise ValueError(f"map_x {mx.shape} and map_y {my.shape}: want two [h, w] arrays")
        h, w = mx.shape
        K = (C.c_float * 4)(*[float(v) for v in K_new])
        out = C.c_void_p()
        fp = C.POINTER(C.c_float)
        self._check(self.lib.dvo_b200_rectifier_create(self.ctx, int(in_size[0]), int(in_size[1]), w, h, mx.ctypes.data_as(fp),
                                                       my.ctypes.data_as(fp), K, C.byref(out)))
        r = Rectifier(self, out.value, in_size, (w, h), tuple(K))
        self._rectifiers.add(r)
        return r

    def pyramid_rectified_batch(self, rect: Rectifier, image, depth, levels: int, depth_scale=None, masks=None,
                                mask_roles="reference") -> list[Pyramid]:
        """Pyramids of frames remapped through rect (dvo_b200_pyramid_create_rectified_batch): level 0 has rect's size and
        intrinsics.  Host arrays: float32 [n,h,w] image + float32 depth in metres, uint8 [n,h,w] grey + uint16 raw depth, or
        uint8 [n,h,w,3] BGR + uint16 raw depth, the format from the dtypes; synchronises before returning.  torch CUDA
        tensors: through device_planes and dvo_b200_pyramid_create_rectified_device_batch, ordered with torch's current
        stream as in pyramid_batch_device, without a host synchronisation.  depth_scale (metres per raw unit) is required
        with uint16 depth.  masks ([n,h,w] or [h,w], nonzero = usable, in the input geometry) / mask_roles as in
        pyramid_batch."""
        return self._create_remapped(rect, None, image, depth, levels, depth_scale, masks, mask_roles)

    def _create_remapped(self, rect, reg, image, depth, levels, depth_scale, masks, mask_roles) -> list[Pyramid]:
        """pyramid_rectified_batch (reg None) and pyramid_registered_batch (rect None or a Rectifier), from host arrays or
        torch CUDA tensors"""
        roles = _mask_roles(mask_roles)
        rh = rect.handle if rect is not None else None
        depth_size = reg.depth_size if reg is not None else None
        if not isinstance(image, np.ndarray) and hasattr(image, "is_cuda") and image.is_cuda:
            if reg is None:
                create = lambda n, fmt, I, Z, scale, M, w, h, out: self.lib.dvo_b200_pyramid_create_rectified_device_batch(
                    self.ctx, rh, n, fmt, I, Z, scale, M, roles, w, h, levels, out)
            else:
                create = lambda n, fmt, I, Z, scale, M, w, h, out: self.lib.dvo_b200_pyramid_create_registered_device_batch(
                    self.ctx, reg.handle, rh, n, fmt, I, Z, scale, M, roles, w, h, levels, out)
            return self._create_device(image, depth, masks, depth_scale, depth_size, create)
        fmt, (n, h, w), I, Z = _host_frames(image, depth, depth_size)
        return self._create_host(fmt, n, h, w, I.ctypes.data, Z.ctypes.data, _depth_scale(fmt, depth_scale), masks, mask_roles, levels,
                                 remap=(rect, reg), sync=True)

    # ---- unregistered depth ----
    depth_rays = staticmethod(depth_rays)

    def depth_registration(self, depth_size, rays, T_color_depth, size, K) -> DepthRegistration:
        """dvo_b200_depth_registration_create: a depth camera of depth_size = (dw, dh) given by rays = (cx_ray, cy_ray, kx_ray,
        ky_ray) as depth_rays returns them, at T_color_depth (4x4, p_color = T p_depth, metres) from a pinhole colour camera
        K = (fx, fy, cx, cy) of size = (w, h).  The tables are uploaded once."""
        dw, dh = (int(v) for v in depth_size)
        shapes = [(dh, dw), (dh, dw), (dh + 1, dw + 1), (dh + 1, dw + 1)]
        tabs = [np.ascontiguousarray(r, dtype=np.float32) for r in rays]
        if len(tabs) != 4 or [t.shape for t in tabs] != shapes:
            raise ValueError(f"rays {[t.shape for t in tabs]}: want {shapes}")
        T = np.ascontiguousarray(T_color_depth, dtype=np.float64).reshape(16)
        Kf = (C.c_float * 4)(*[float(v) for v in K])
        out = C.c_void_p()
        fp = C.POINTER(C.c_float)
        self._check(self.lib.dvo_b200_depth_registration_create(self.ctx, dw, dh, *(t.ctypes.data_as(fp) for t in tabs),
                                                                T.ctypes.data_as(C.POINTER(C.c_double)), int(size[0]), int(size[1]),
                                                                Kf, C.byref(out)))
        r = DepthRegistration(self, out.value, (dw, dh), size, tuple(Kf))
        self._registrations.add(r)
        return r

    def pyramid_registered_batch(self, reg: DepthRegistration, image, depth, levels: int, depth_scale=None, masks=None,
                                 mask_roles="reference", rectifier: Rectifier | None = None) -> list[Pyramid]:
        """Pyramids of colour frames with the depth of a separate depth camera reprojected into them
        (dvo_b200_pyramid_create_registered_batch): level 0 has reg's colour size and K.  image: the colour frames, [n,h,w]
        float32 or uint8 grey, or uint8 [n,h,w,3] BGR, of reg's size or, with a rectifier, of its input size; depth: [n,dh,dw]
        float32 metres (with float32 images) or uint16 raw (then depth_scale), in the depth camera's geometry.  masks
        ([n,h,w] or [h,w], nonzero = usable, in the colour frames' geometry) / mask_roles as in pyramid_batch.  numpy arrays:
        staged from the host, synchronises before returning.  torch CUDA tensors: through
        dvo_b200_pyramid_create_registered_device_batch, ordered with torch's current stream as in pyramid_batch_device,
        without a host synchronisation."""
        return self._create_remapped(rectifier, reg, image, depth, levels, depth_scale, masks, mask_roles)

    def pyramid_raw(self, grey_u8, depth_u16, depth_scale, intrinsics, levels: int, mask=None, mask_roles="reference") -> Pyramid:
        G = np.ascontiguousarray(grey_u8, dtype=np.uint8)
        D = np.ascontiguousarray(depth_u16, dtype=np.uint16)
        assert G.ndim == 2 and G.shape == D.shape
        return self._create_host("grey8_depth16", 1, *G.shape, G.ctypes.data, D.ctypes.data, depth_scale, mask, mask_roles, levels,
                                 intrinsics, single=True, sync=True)[0]

    # ---- alignment ----
    def match(self, ref: Pyramid, cur: Pyramid, cfg: Config, T_init=None, with_iterations: bool = False) -> Result:
        return self.match_batch([ref], [cur], cfg, None if T_init is None else [T_init], with_iterations)[0]

    def match_batch_photometric(self, refs, curs, cfg: Config, T_init=None, photometric_init=None, with_iterations: bool = False,
                                prior_information=None):
        """match_batch in the photometric mode (include/dvo_b200.h): the pose and an intensity gain and bias per pair.
        photometric_init: [n, 2] (alpha, beta) or None = (1, 0).  prior_information as in match_batch.  Returns (results,
        [n, 2] float64 final (alpha, beta))."""
        return self._match(refs, curs, cfg, T_init, with_iterations, prior_information, True, photometric_init)

    def _device_maps(self, refs, cfg: Config, mask_weight):
        """The torch CUDA tensors of match_batch_maps and the WeightMaps that points at them, with the engine's stream ordered
        after torch's current stream (the engine's stream writes memory that stream allocated; the call synchronises)."""
        import torch
        n = len(refs)
        L = cfg.last_level
        sizes = {tuple(r.level_info(L)[:2]) + tuple(r.level_info(0)[:2]) for r in refs}
        if len(sizes) != 1:
            raise ValueError(f"references of {len(sizes)} different sizes: match_batch_maps takes one size per call")
        w, h, w0, h0 = sizes.pop()
        dev = torch.device("cuda", self.device)
        maps = {k: torch.empty((n, h, w), dtype=torch.float32, device=dev) for k in ("weight", "residual_i", "residual_z")}
        maps["estimate"] = torch.empty((n, 4, 4), dtype=torch.float64, device=dev)
        maps["precision"] = torch.empty((n, 2, 2), dtype=torch.float32, device=dev)
        wm = WeightMaps()
        wm.memory = MAPS_MEMORY["device"]
        for k in ("weight", "residual_i", "residual_z"):
            setattr(wm, k, MapPlane(maps[k].data_ptr(), 4 * w, 4 * w * h))
        if mask_weight is not None:
            maps["mask"] = torch.empty((n, h0, w0), dtype=torch.uint8, device=dev)
            wm.mask = MapPlane(maps["mask"].data_ptr(), w0, w0 * h0)
            wm.mask_weight = float(mask_weight)
        wm.estimate = C.cast(maps["estimate"].data_ptr(), C.POINTER(C.c_double))
        wm.precision = C.cast(maps["precision"].data_ptr(), C.POINTER(C.c_float))
        current = torch.cuda.current_stream(dev)
        torch.cuda.ExternalStream(self.stream, device=dev).wait_stream(current)
        return maps, wm

    def match_batch_maps(self, refs, curs, cfg: Config, T_init=None, prior_information=None, photometric_init=None,
                         photometric: bool = False, mask_weight=None, with_iterations: bool = False):
        """An alignment and each pair's weight maps at its returned pose (dvo_b200_match_batch_maps; "weight maps" in
        include/dvo_b200.h).  The results (and (alpha, beta)) are those of match_batch / match_batch_photometric with the same
        arguments.  Returns (results, maps), or (results, maps, [n, 2] (alpha, beta)) when photometric.  maps holds torch CUDA
        tensors on the engine's device: "weight", "residual_i", "residual_z" [n, h_L, w_L] float32 at L = cfg.last_level (NaN
        where a pixel is not a constraint), "estimate" [n, 4, 4] float64 (the pose the maps are at, reference -> current),
        "precision" [n, 2, 2] float32 and, with mask_weight, "mask" [n, h, w] uint8 at level 0: 0 where the pixel's level-L
        parent is a constraint with weight < mask_weight, 1 elsewhere -- the masks= of pyramid_batch_device.  The pyramids of
        one call must share their size (ValueError otherwise)."""
        maps, wm = self._device_maps(refs, cfg, mask_weight)
        res, ab = self._match(refs, curs, cfg, T_init, with_iterations, prior_information, photometric, photometric_init, wm)
        return (res, maps, ab) if photometric else (res, maps)

    def match_batch(self, refs, curs, cfg: Config, T_init=None, with_iterations: bool = False, raw: bool = False, prior_information=None):
        """prior_information: [n, 6, 6] float64, a motion prior per pair in place of cfg.mu I (dvo_b200_match_batch_prior,
        which requires cfg.mu == 0); prior_from_result builds one from an earlier Result."""
        return self._match(refs, curs, cfg, T_init, with_iterations, prior_information, raw=raw)[0]

    def _match(self, refs, curs, cfg: Config, T_init, with_iterations, prior_information=None, photometric=False,
               photometric_init=None, maps=None, raw=False):
        """One n-pair alignment through dvo_b200_match_batch_maps (maps: a WeightMaps), _prior (prior_information),
        _photometric or dvo_b200_match_batch -> (results, or the CResult array with raw, and [n, 2] (alpha, beta) or None)"""
        n = len(refs)
        assert n == len(curs) and n > 0
        rh, ch = _handles(refs), _handles(curs)
        T = _rows(T_init, "T_init", (n, 4, 4), 16)
        ab0 = _photometric_init(photometric, photometric_init, (n, 2))
        ab = np.zeros((n, 2), dtype=np.float64) if photometric else None
        lam = _rows(prior_information, "prior_information", (n, 6, 6), 36)
        res = (CResult * n)()
        log, max_log = _iteration_log(cfg, n, with_iterations)
        head = (self.ctx, C.byref(cfg), n, rh, ch, _ptr(T))
        if maps is not None:
            rc = self.lib.dvo_b200_match_batch_maps(*head, _ptr(lam), _ptr(ab0), _ptr(ab), res, log, max_log, C.byref(maps))
        elif lam is not None:
            rc = self.lib.dvo_b200_match_batch_prior(*head, _ptr(lam), _ptr(ab0), _ptr(ab), res, log, max_log)
        elif photometric:
            rc = self.lib.dvo_b200_match_batch_photometric(*head, _ptr(ab0), res, _ptr(ab), log, max_log)
        else:
            rc = self.lib.dvo_b200_match_batch(*head, res, log, max_log)
        self._check(rc)
        return (res if raw else _results(res, n, log, max_log)), ab

    def match_batch_hypotheses(self, refs, curs, hypotheses, screen_level: int, min_constraint_ratio: float = 0.0,
                               cfg: Config | None = None, with_iterations: bool = False, screen_results: bool = False,
                               prior_information=None, photometric_init=None, photometric: bool = False, maps: bool = False,
                               mask_weight=None):
        """Multi-hypothesis alignment (dvo_b200_match_batch_hypotheses[_modes]): pair i starts from each of the k poses
        hypotheses[i] ([n, k, 4, 4], read as T_init) on levels cfg.first_level .. screen_level, and the one with the lowest
        per-constraint negative log-likelihood among those with a large enough constraint ratio continues to cfg.last_level.
        cfg: default Config(use_initial_estimate=1).  Returns (results, best [n] int32, scores [n, k] float64, NaN where a
        hypothesis was not eligible), and with screen_results=True also the screening results, a list of n lists of k.
        The modes, per hypothesis (include/dvo_b200.h, dvo_b200_match_batch_hypotheses_modes):
          prior_information  [n, k, 6, 6] float64: Lambda of each hypothesis, anchored at that hypothesis (cfg.mu must be 0).
          photometric        True: the photometric mode; photometric_init [n, k, 2] (alpha, beta)_0 per hypothesis, or None
                             = (1, 0).  Appends the final (alpha, beta) [n, 2] and, with screen_results, where each screening
                             run ended [n, k, 2].
          maps, mask_weight  True / a mask weight: the weight maps of the continued alignments, the dict of match_batch_maps
                             (mask only with mask_weight), appended last.
        The score is that of the data term alone whatever the mode."""
        if cfg is None:
            cfg = Config(use_initial_estimate=1)
        n = len(refs)
        assert n == len(curs) and n > 0
        H = np.asarray(hypotheses, dtype=np.float64)
        if H.ndim != 4 or H.shape[0] != n or H.shape[2:] != (4, 4):
            raise ValueError(f"hypotheses {H.shape}: want [{n}, k, 4, 4]")
        k = H.shape[1]
        H = _rows(H, "hypotheses", H.shape, 16)
        lam = _rows(prior_information, "prior_information", (n, k, 6, 6), 36)
        ab0 = _photometric_init(photometric, photometric_init, (n, k, 2))
        ab = np.zeros((n, 2), dtype=np.float64) if photometric else None
        screen_ab = np.zeros((n, k, 2), dtype=np.float64) if photometric and screen_results else None
        dmaps = wm = None
        if maps or mask_weight is not None:
            dmaps, wm = self._device_maps(refs, cfg, mask_weight)
        res = (CResult * n)()
        best = np.zeros(n, dtype=np.int32)
        scores = np.zeros((n, k), dtype=np.float64)
        screen = (CResult * (n * k))() if screen_results else None
        log, max_log = _iteration_log(cfg, n, with_iterations)
        self._check(self.lib.dvo_b200_match_batch_hypotheses_modes(
            self.ctx, C.byref(cfg), n, _handles(refs), _handles(curs), k, _ptr(H), int(screen_level), float(min_constraint_ratio),
            _ptr(lam), _ptr(ab0), _ptr(ab), _ptr(screen_ab), res, _ptr(best, C.POINTER(C.c_int32)), _ptr(scores), screen, log, max_log,
            C.byref(wm) if wm is not None else None))
        out = (_results(res, n, log, max_log), best, scores)
        if screen_results:
            flat = [Result(screen[i]) for i in range(n * k)]
            out += ([flat[i * k:(i + 1) * k] for i in range(n)],)
        if photometric:
            out += (ab,) + ((screen_ab,) if screen_results else ())
        if dmaps is not None:
            out += (dmaps,)
        return out

    def match_batch_device(self, refs, curs, cfg: Config, d_results_ptr: int, T_init=None):
        n = len(refs)
        self._check(self.lib.dvo_b200_match_batch_device(self.ctx, C.byref(cfg), n, _handles(refs), _handles(curs),
                                                         _ptr(_rows(T_init, "T_init", (n, 4, 4), 16)), C.c_void_p(d_results_ptr)))

    def residual_image(self, ref: Pyramid, cur: Pyramid, level: int, T, cfg: Config | None = None, ab=None):
        """ab = (alpha, beta): the photometric mode's hook at that brightness model (dvo_b200_residual_image_photometric)."""
        cfg = cfg or Config()
        w, h, _ = ref.level_info(level)
        out = np.empty((7, h, w), dtype=np.float32)
        cnt = C.c_int64()
        head = (self.ctx, C.byref(cfg), ref.handle, cur.handle, level, _ptr(_rows(T, "T", (4, 4), 16)))
        tail = (_ptr(out, C.POINTER(C.c_float)), C.byref(cnt))
        if ab is None:
            self._check(self.lib.dvo_b200_residual_image(*head, *tail))
        else:
            self._check(self.lib.dvo_b200_residual_image_photometric(*head, _ptr(_rows(ab, "ab", (2,), 2)), *tail))
        return cnt.value, out

    def intensity_error_image(self, ref: Pyramid, cur: Pyramid, level: int, T, cfg: Config | None = None):
        """DenseTracker::computeIntensityErrorImage (dense_tracking.cpp:378-444) -> (n_written, image[h, w])."""
        cfg = cfg or Config()
        w, h, _ = ref.level_info(level)
        out = np.empty((h, w), dtype=np.float32)
        cnt = C.c_int64()
        self._check(self.lib.dvo_b200_intensity_error_image(self.ctx, C.byref(cfg), ref.handle, cur.handle, level,
                                                            _ptr(_rows(T, "T", (4, 4), 16)), _ptr(out, C.POINTER(C.c_float)),
                                                            C.byref(cnt)))
        return int(cnt.value), out

    def linearize(self, ref: Pyramid, cur: Pyramid, level: int, T, use_weights=False, prev_precision=None, cfg: Config | None = None,
                  ab=None):
        """ab = (alpha, beta): the photometric mode's hook (dvo_b200_linearize_photometric); A is then 8 x 8 and b 8."""
        cfg = cfg or Config()
        pp = np.ascontiguousarray(np.asarray(prev_precision if prev_precision is not None else np.zeros(4), dtype=np.float32).reshape(4))
        P = np.zeros(4, dtype=np.float32)
        ll = C.c_float()
        k = 6 if ab is None else 8
        A = np.zeros(k * k)
        b = np.zeros(k)
        cnt = C.c_int64()
        fp = C.POINTER(C.c_float)
        head = (self.ctx, C.byref(cfg), ref.handle, cur.handle, level, _ptr(_rows(T, "T", (4, 4), 16)))
        tail = (int(use_weights), _ptr(pp, fp), C.byref(cnt), _ptr(P, fp), C.byref(ll), _ptr(A), _ptr(b))
        if ab is None:
            self._check(self.lib.dvo_b200_linearize(*head, *tail))
        else:
            self._check(self.lib.dvo_b200_linearize_photometric(*head, _ptr(_rows(ab, "ab", (2,), 2)), *tail))
        return {"n": cnt.value, "precision": P.reshape(2, 2), "ll": ll.value, "A": A.reshape(k, k), "b": b}

    # ---- profiling ----
    def profile_enable(self, on: bool = True):
        self._check(self.lib.dvo_b200_profile_enable(self.ctx, int(on)))

    def profile_read(self, reset: bool = True):
        ms = (C.c_double * 8)()
        ln = (C.c_int64 * 8)()
        self._check(self.lib.dvo_b200_profile_read(self.ctx, ms, ln, int(reset)))
        names = ["residual", "normal", "pair_step", "pyramid", "select"]
        return {names[i]: {"ms": ms[i], "launches": ln[i]} for i in range(len(names))}


class ShardedEngine:
    """dvo_b200_sharded: one process, one context + host thread per device, contiguous shards of pair indices
    (the C-ABI form of the multi-GPU path; the multi-process form is dvo_slam_b200/distributed.py)."""

    def __init__(self, devices):
        self.lib = load_library()
        devs = (C.c_int32 * len(devices))(*devices)
        h = C.c_void_p()
        rc = self.lib.dvo_b200_sharded_create(len(devices), devs, C.byref(h))
        if rc != 0:
            raise RuntimeError(f"dvo_b200_sharded_create({list(devices)}) failed with status {rc}: no usable CUDA device "
                               "(the engine has no CPU fallback)")
        self.h = h
        self.devices = list(devices)

    def close(self):
        if getattr(self, "h", None):
            self.lib.dvo_b200_sharded_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc):
        if rc != 0:
            raise RuntimeError(f"dvo_b200 sharded status {rc}: {self.lib.dvo_b200_sharded_last_error(self.h).decode()}")

    def set_estimator(self, estimator: str):
        """the estimator of every shard's context (see Engine)"""
        if estimator not in ESTIMATORS:
            raise ValueError(f"unknown estimator {estimator!r}: one of {sorted(ESTIMATORS)}")
        for k in range(len(self.devices)):
            ctx = self.lib.dvo_b200_sharded_ctx(self.h, k)
            self._check(self.lib.dvo_b200_set_estimator(ctx, ESTIMATORS[estimator]))

    def shard_range(self, total, shard):
        b, e = C.c_int64(), C.c_int64()
        self._check(self.lib.dvo_b200_shard_range(total, len(self.devices), shard, C.byref(b), C.byref(e)))
        return b.value, e.value

    def pyramid_batch(self, intensity, depth, intrinsics, levels):
        """intensity, depth: float32 arrays [n, h, w] on the host -> n pyramid handles (image i on its shard's device)."""
        I = np.ascontiguousarray(intensity, dtype=np.float32)
        Z = np.ascontiguousarray(depth, dtype=np.float32)
        n, h, w = I.shape
        out = (C.c_void_p * n)()
        fx, fy, ox, oy = [float(v) for v in intrinsics]
        self._check(self.lib.dvo_b200_sharded_pyramid_create_batch(self.h, n, I.ctypes.data, Z.ctypes.data, w, h, fx, fy, ox, oy, levels, out))
        return [C.c_void_p(v) for v in out]

    def release(self, handles):
        for p in handles:
            self.lib.dvo_b200_pyramid_release(p)

    def match_batch(self, refs, curs, cfg: Config, T_init=None):
        n = len(refs)
        res = (CResult * n)()
        self._check(self.lib.dvo_b200_match_batch_sharded(self.h, C.byref(cfg), n, _handles(refs, "value"), _handles(curs, "value"),
                                                          _ptr(_rows(T_init, "T_init", (n, 4, 4), 16)), res, None, 0))
        return res
