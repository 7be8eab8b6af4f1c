"""The weight maps without a GPU: the output checks of csrc/maps_args.h built for the host (with a fake in place of
cudaPointerGetAttributes), the mask's footprint rule, and the weight map as an outlier mask measured on the CPU oracle
(tests/weight_maps_model.py, the table of DESIGN §4.10)."""
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np
import pytest

import weight_maps_model as wmm
from dvo_slam_b200.engine import MAPS_MEMORY, MapPlane, WeightMaps

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# the fake's memory: device memory of devices 0 and 1, managed memory of device 0; everything else is host memory
DEV0, DEV1, MANAGED, HOST = 0x10000000, 0x30000000, 0x50000000, 0x70000000
REGION = 0x10000000
KIND_DEVICE, KIND_MANAGED = 1, 2
REGIONS = np.array([DEV0, DEV0 + REGION, KIND_DEVICE * 16 + 0, DEV1, DEV1 + REGION, KIND_DEVICE * 16 + 1,
                    MANAGED, MANAGED + REGION, KIND_MANAGED * 16 + 0], dtype=np.int64)
N, W, H, W0, H0 = 3, 80, 60, 641, 481   # level 3 of a 641 x 481 reference: 80 x 60


@pytest.fixture(scope="module")
def check():
    tmp = tempfile.mkdtemp(prefix="dvo_maps_args_")
    try:
        out = os.path.join(tmp, "libmaps_args.so")
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-Wall", "-fPIC", "-shared", "-I", os.path.join(ROOT, "dvo_slam_b200", "csrc"),
                               "-o", out, os.path.join(ROOT, "tests", "native", "maps_args.cpp")])
        L = C.CDLL(out)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    L.maps_check.argtypes = [C.POINTER(WeightMaps), C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_longlong),
                             C.c_int, C.c_char_p, C.c_int]

    def run(m, n=N, device=0):
        buf = C.create_string_buffer(512)
        L.maps_check(C.byref(m) if m is not None else None, n, W, H, W0, H0, device, REGIONS.ctypes.data_as(C.POINTER(C.c_longlong)),
                     len(REGIONS) // 3, buf, 512)
        return buf.value.decode()
    return run


def maps(memory="device", base=DEV0, planes=("weight",), mask_weight=0.3, estimate=False, precision=False):
    """outputs packed one after the other from `base`"""
    m = WeightMaps()
    m.memory = MAPS_MEMORY[memory] if isinstance(memory, str) else memory
    at = base
    for k in planes:
        row, h = (W0, H0) if k == "mask" else (4 * W, H)
        setattr(m, k, MapPlane(at, row, row * h))
        at += (N * row * h + 255) // 256 * 256 + 256
    m.mask_weight = mask_weight
    if estimate:
        m.estimate = C.cast(at, C.POINTER(C.c_double)); at += N * 128 + 256
    if precision:
        m.precision = C.cast(at, C.POINTER(C.c_float))
    return m


def test_accepted(check):
    assert check(maps(planes=("weight", "residual_i", "residual_z", "mask"), estimate=True, precision=True)) == ""
    assert check(maps(planes=(), estimate=True)) == ""
    assert check(maps(planes=(), precision=True)) == ""
    assert check(maps(base=MANAGED, planes=("mask",))) == ""                        # managed memory of the ctx's device
    assert check(maps(memory="host", base=HOST, planes=("weight", "mask"), estimate=True, precision=True)) == ""
    assert check(maps(memory="host", base=MANAGED, planes=("weight",))) == ""
    assert check(maps(base=DEV1, planes=("weight",)), device=1) == ""
    m = maps(planes=("weight",))
    m.weight.row_bytes, m.weight.image_bytes = 4 * W + 64, (4 * W + 64) * H + 12   # padded rows and images
    assert check(m) == ""
    m = maps(planes=("residual_z",), mask_weight=float("nan"))                       # mask_weight is read with a mask only
    assert check(m) == ""
    assert check(maps(planes=("mask",), mask_weight=1e-30)) == ""
    assert check(maps(base=HOST, planes=("weight",)), n=0) == ""                    # n <= 0: the batch checks refuse it


def test_refusals(check):
    def refused(m, what, **kw):
        msg = check(m, **kw)
        assert msg.startswith("match_batch_maps: ") and what in msg, (what, msg)

    refused(None, "maps is null")
    refused(maps(memory=2), "unknown memory 2")
    refused(maps(memory=-1), "unknown memory -1")
    refused(maps(planes=()), "no output requested")
    for mw in (0.0, -0.5, float("nan"), float("inf")):
        refused(maps(planes=("mask",), mask_weight=mw), "mask_weight")
    for k in ("weight", "residual_i", "residual_z", "mask"):
        elem, row_min, h = (1, W0, H0) if k == "mask" else (4, 4 * W, H)
        m = maps(planes=(k,)); getattr(m, k).row_bytes = row_min - elem
        refused(m, k + ".row_bytes")
        m = maps(planes=(k,)); getattr(m, k).image_bytes = row_min * h - 1
        refused(m, k + ".image_bytes")
        if elem > 1:
            m = maps(planes=(k,)); getattr(m, k).row_bytes = row_min + 2; getattr(m, k).image_bytes = (row_min + 2) * h
            refused(m, k + ".row_bytes")
            m = maps(planes=(k,)); getattr(m, k).image_bytes = row_min * h + 2
            refused(m, k + " is misaligned")
            m = maps(planes=(k,)); getattr(m, k).data = DEV0 + 2
            refused(m, k + " is misaligned")
        refused(maps(base=HOST, planes=(k,)), k + " is not device or managed memory of device 0")
        refused(maps(base=DEV1, planes=(k,)), k + " is not device or managed memory of device 0")
        refused(maps(memory="host", base=DEV0, planes=(k,)), k + " lies in device memory")
        # the first byte in place, the last one not: the extent of the last pair crosses out of the region
        end = N * (row_min * h)
        refused(maps(base=DEV0 + REGION - end + elem, planes=(k,)), k + " is not device or managed memory")
        refused(maps(memory="host", base=DEV0 - end + elem, planes=(k,)), k + " lies in device memory")
        assert check(maps(base=DEV0 + REGION - end, planes=(k,))) == ""
    m = maps(planes=(), estimate=True); m.estimate = C.cast(DEV0 + 4, C.POINTER(C.c_double))
    refused(m, "estimate is misaligned")
    m = maps(planes=(), precision=True); m.precision = C.cast(DEV0 + 2, C.POINTER(C.c_float))
    refused(m, "precision is misaligned")
    m = maps(planes=(), estimate=True); m.estimate = C.cast(DEV0 + REGION - N * 128 + 8, C.POINTER(C.c_double))
    refused(m, "estimate is not device")
    m = maps(planes=(), precision=True); m.precision = C.cast(HOST, C.POINTER(C.c_float))
    refused(m, "precision is not device")
    m = maps(memory="host", base=HOST, planes=(), precision=True); m.precision = C.cast(DEV1, C.POINTER(C.c_float))
    refused(m, "precision lies in device memory")


def _footprint_loop(weight, level, shape0, t):
    h0, w0 = shape0
    h, w = weight.shape
    out = np.ones(shape0, np.uint8)
    for y in range(h0):
        for x in range(w0):
            py, px = y >> level, x >> level
            if py < h and px < w and weight[py, px] == weight[py, px] and weight[py, px] < t:
                out[y, x] = 0
    return out


@pytest.mark.parametrize("level", [0, 1, 2, 3])
@pytest.mark.parametrize("shape0", [(48, 64), (37, 53)])
def test_footprint_rule(level, shape0):
    rng = np.random.default_rng(level * 100 + shape0[0])
    h, w = shape0[0] >> level, shape0[1] >> level                 # level sizes: the floor chain of the pyramid
    weight = rng.uniform(0.0, 1.4, (h, w)).astype(np.float32)
    weight[rng.random((h, w)) < 0.3] = np.nan                     # not constraints
    weight[0, 0], weight[0, 1] = 0.25, 0.3                        # at the threshold: not below it
    m = wmm.footprint_mask(weight, level, shape0, 0.3)
    assert m.dtype == np.uint8 and m.shape == shape0
    assert np.array_equal(m, _footprint_loop(weight, level, shape0, 0.3))
    s = 1 << level
    assert (m[:s, :s] == 0).all() and (m[:s, s:2 * s] == 1).all()
    assert (m[h * s:, :] == 1).all() and (m[:, w * s:] == 1).all()   # past an odd size: no parent, usable
    assert (m == 0).sum() == s * s * int((np.isfinite(weight) & (weight < 0.3)).sum())


def test_moving_object_table(oracle):
    """DESIGN §4.10: the kept iteration's weights on make_moving_object_pair (MIRROR), and a second alignment masked by
    w < MASK_WEIGHT.  Where the unmasked alignment is pulled away by the patch (seeds 0, 4, 6) the patch is mostly NOT
    down-weighted at the pose it converged to, so the mask recovers only part of the ground-truth mask's gain (seeds 0, 4)
    or none (seed 6); where it is not pulled away, the patch is marked almost entirely and the second pass stays as good."""
    rows = {r["seed"]: r for r in wmm.moving_object_table(oracle, mask_weight=wmm.MASK_WEIGHT)}
    t = wmm.MASK_WEIGHT
    for seed, r in rows.items():
        assert r["n"] == r["kept_n"], seed                                   # finite weights = the kept iteration's constraints
        assert r["other"][t] < 0.025, (seed, r["other"])                     # little of the static scene is marked
        assert r["weight_masked"][0] <= r["unmasked"][0] + 1e-3, (seed, r)   # a second pass never ends much worse
    for seed in (1, 2, 3, 5, 7):
        assert rows[seed]["patch"][t] > 0.9, (seed, rows[seed]["patch"])
    for seed in (0, 4):
        assert rows[seed]["weight_masked"][0] < 0.6 * rows[seed]["unmasked"][0], rows[seed]
        assert rows[seed]["weight_masked"][0] > 2 * rows[seed]["truth_masked"][0], rows[seed]   # well short of the truth's mask
    assert rows[6]["patch"][t] < 0.1 and rows[6]["weight_masked"][0] > 0.5 * rows[6]["unmasked"][0]
    for r in rows.values():
        print("seed %d: patch %s other %s | unmasked %.2e/%.2e  truth-masked %.2e/%.2e  weight-masked %.2e/%.2e" % (
            r["seed"], " ".join("%.3f" % r["patch"][k] for k in wmm.THRESHOLDS), " ".join("%.4f" % r["other"][k] for k in wmm.THRESHOLDS),
            *r["unmasked"], *r["truth_masked"], *r["weight_masked"]))
