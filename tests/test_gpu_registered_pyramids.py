"""Pyramids from unregistered depth on the H100 (dvo_b200_depth_registration, dvo_b200_pyramid_create_registered_batch and
its device form through Engine.depth_registration / Engine.pyramid_registered_batch): bit-for-bit equality with the float32
build of the numpy registration model (tests/registration_model.py) for every format, mask role set, input path and depth
camera, with and without a rectifier; the identity registration against the plain creates; repeatability of the atomic
depth test; the pose against MIRROR and the truth; traffic, stream order, early release and invalid arguments."""
import ctypes as C

import numpy as np
import pytest
import torch

import rectify_model as rm
import registration_model as rg
from helpers import pose_delta
from test_gpu_device_input import _to_device
from test_gpu_rectified_pyramids import _assert_same_pyramid, _records

pytestmark = pytest.mark.gpu

LEVELS = 5
SCALE = 1.0 / 5000.0
FORMATS = ["float32", "grey8_depth16", "bgr8_depth16"]
MASKS = [None, "reference", "both"]
CFG = dict(first_level=4, last_level=0, max_iterations_per_level=50, precision=1e-4)
FR1 = (517.3, 516.5, 318.6, 255.3)
# depth cameras: at the colour size with a baseline and a small rotation, a lower resolution (footprints above a pixel) and a
# higher one (footprints below a pixel, so many land on no colour pixel centre)
CAMERAS = {"baseline": ((640, 480), FR1), "low-res": ((320, 240), tuple(v / 2 for v in FR1)),
           "high-res": ((1280, 960), tuple(v * 2 for v in FR1))}


def _T():
    from dvo_slam_b200 import synth
    return synth.se3_exp(np.array([0.025, 0.003, -0.004, 0.004, -0.006, 0.002]))


_cache = {}


def _frames(camera, distorted=False):
    """three frames (a reference, its current frame, another reference) of colour in every host representation, depth from
    the depth camera (float metres and raw), a blob mask per frame, the ray tables and the transform"""
    key = (camera, distorted)
    if key in _cache:
        return _cache[key]
    from dvo_slam_b200 import synth
    size_d, K_d = CAMERAS[camera]
    T = _T()
    cfg = synth.SceneConfig(distortion=synth.FR1_DISTORTION if distorted else None, depth_camera=synth.DepthCamera(*size_d, K_d, T))
    p, q = synth.make_pair(21, cfg), synth.make_pair(22, cfg)
    I = np.stack([p["I_ref"].numpy(), p["I_cur"].numpy(), q["I_ref"].numpy()]).astype(np.float32)
    Z = np.stack([p["Z_ref"].numpy(), p["Z_cur"].numpy(), q["Z_ref"].numpy()]).astype(np.float32)
    n, h, w = I.shape
    rng = np.random.default_rng(11)
    yy, xx = np.ogrid[:h, :w]
    M = np.ones((n, h, w), np.uint8)
    for i in range(n):
        for _ in range(8):
            cy, cx, r = rng.integers(0, h), rng.integers(0, w), rng.integers(10, 70)
            M[i][(yy - cy) ** 2 + (xx - cx) ** 2 <= r * r] = 0
    f = {"float": (I, Z), "grey": np.clip(I, 0, 255).astype(np.uint8),
         "raw": np.where(np.isnan(Z), 0, np.round(Z * 5000.0)).astype(np.uint16),
         "bgr": rng.integers(0, 256, (n, h, w, 3), dtype=np.uint8), "masks": M, "T": T,
         "rays": rg.depth_rays(size_d, K_d)}
    if distorted:
        f["map"] = rm.undistort_map(w, h, FR1, synth.FR1_DISTORTION)
    _cache[key] = f
    return f


@pytest.fixture(scope="module")
def regs(engine):
    """one registration per depth camera"""
    out = {c: engine.depth_registration(CAMERAS[c][0], rg.depth_rays(*CAMERAS[c]), _T(), (640, 480), FR1) for c in CAMERAS}
    yield out
    for r in out.values():
        r.release()


def _inputs(f, fmt):
    image = {"float32": f["float"][0], "grey8_depth16": f["grey"], "bgr8_depth16": f["bgr"]}[fmt]
    depth = f["float"][1] if fmt == "float32" else f["raw"]
    return image, depth


def _mask_of(f, mask):
    """"reference": one mask per frame; "both": one mask shared by the batch (image_bytes 0 on the device path)"""
    return None if mask is None else f["masks"] if mask == "reference" else f["masks"][0]


def _model_build(engine, f, fmt, mask):
    """the float32 pyramids of the model's registered planes and mask, by the plain masked create"""
    image, depth = _inputs(f, fmt)
    I, Z, M = rg.register_batch(image, depth, f["rays"], f["T"], (640, 480), FR1, _mask_of(f, mask), SCALE, f.get("map"))
    kw = {} if mask is None else {"masks": M, "mask_roles": mask}
    return engine.pyramid_batch(I, Z, FR1, LEVELS, **kw)


def _registered_build(engine, reg, f, fmt, mask, path, rect=None):
    image, depth = _inputs(f, fmt)
    kw = {"depth_scale": None if fmt == "float32" else SCALE, "mask_roles": mask or "reference", "rectifier": rect}
    m = _mask_of(f, mask)
    if path == "host":
        return engine.pyramid_registered_batch(reg, image, depth, LEVELS, masks=m, **kw)
    fill_z = float("nan") if fmt == "float32" else 777
    dM = None if m is None else _to_device(m, "crop", torch.bool, fill=1) if m.ndim == 3 else torch.from_numpy(m).cuda()
    return engine.pyramid_registered_batch(reg, _to_device(image, "crop", fill=99), _to_device(depth, "crop", fill=fill_z), LEVELS,
                                           masks=dM, **kw)


def _check_equal(engine, R, H):
    assert [p.mask_roles for p in R] == [p.mask_roles for p in H]
    assert all(p.level_info(0) == (640, 480, tuple(np.float32(FR1))) for p in R)
    for p, q in zip(R, H):
        _assert_same_pyramid(p, q)
    assert _records(engine, [R[0], R[2], R[1]], [R[1], R[0], R[0]]) == _records(engine, [H[0], H[2], H[1]], [H[1], H[0], H[0]])


@pytest.mark.parametrize("camera", list(CAMERAS))
@pytest.mark.parametrize("path", ["host", "device"])
@pytest.mark.parametrize("mask", MASKS)
@pytest.mark.parametrize("fmt", FORMATS)
def test_registered_build_equals_the_model_build(engine, regs, fmt, mask, path, camera):
    f = _frames(camera)
    _check_equal(engine, _registered_build(engine, regs[camera], f, fmt, mask, path), _model_build(engine, f, fmt, mask))


@pytest.mark.parametrize("path", ["host", "device"])
@pytest.mark.parametrize("mask", MASKS)
@pytest.mark.parametrize("fmt", FORMATS)
def test_registered_build_through_a_rectifier_equals_the_model_build(engine, regs, fmt, mask, path):
    f = _frames("baseline", distorted=True)
    rect = engine.rectifier((640, 480), *f["map"], FR1)
    try:
        _check_equal(engine, _registered_build(engine, regs["baseline"], f, fmt, mask, path, rect), _model_build(engine, f, fmt, mask))
    finally:
        rect.release()


def test_model_planes_have_shadows_and_empty_footprints():
    """the cases above exercise what they claim: the baseline adds occlusion shadows to the depth holes, the
    low-resolution camera's footprints cover several colour pixels each, and most of the high-resolution camera's cover
    none"""
    for camera in CAMERAS:
        f = _frames(camera)
        d = f["float"][1][0]
        Z = rg.register(d, f["rays"], f["T"], (640, 480), FR1)
        valid, covered = np.isfinite(d).sum(), np.isfinite(Z).sum()
        if camera == "baseline":
            assert np.isnan(Z).mean() > np.isnan(d).mean() + 0.002
        elif camera == "low-res":
            assert covered > 3 * valid
        else:
            assert covered < 0.3 * valid


@pytest.mark.parametrize("fmt", FORMATS)
def test_identity_registration_gives_the_plain_pyramids(engine, fmt):
    """the pinhole rays of the colour camera with T = I: every colour pixel is covered by its own depth pixel alone, so the
    pyramids and the alignments are those of the unregistered create in the same format"""
    f = _frames("baseline")
    image = _inputs(f, fmt)[0]
    from dvo_slam_b200 import synth
    p = synth.make_pair(21)
    Zc = np.stack([p["Z_ref"].numpy(), p["Z_cur"].numpy(), p["Z_ref"].numpy()])
    depth = Zc if fmt == "float32" else np.where(np.isnan(Zc), 0, np.round(Zc * 5000.0)).astype(np.uint16)
    n, h, w = depth.shape
    reg = engine.depth_registration((w, h), rg.depth_rays((w, h), FR1), np.eye(4), (w, h), FR1)
    R = engine.pyramid_registered_batch(reg, image, depth, LEVELS, depth_scale=SCALE)
    image = np.ascontiguousarray(image)
    if fmt == "float32":
        P = engine.pyramid_batch(image, depth, FR1, LEVELS)
    else:
        build = engine.pyramid_raw_batch if fmt == "grey8_depth16" else engine.pyramid_bgr_batch
        P = build((image.ctypes.data, depth.ctypes.data, n, h, w), SCALE, FR1, LEVELS)
        engine.synchronize()
    for a, b in zip(R, P):
        _assert_same_pyramid(a, b)
    assert _records(engine, R[:2], R[1::-1]) == _records(engine, P[:2], P[1::-1])
    reg.release()


def test_two_builds_are_identical(engine, regs):
    """the atomic depth test does not depend on the order the threads run in: two builds of the same input, bit for bit"""
    f = _frames("low-res")
    I, Z = f["float"]
    A = engine.pyramid_registered_batch(regs["low-res"], I, Z, LEVELS)
    B = engine.pyramid_registered_batch(regs["low-res"], I, Z, LEVELS)
    for p, q in zip(A, B):
        for l in range(LEVELS):
            assert np.array_equal(p.download(l), q.download(l), equal_nan=True)


def test_pose_on_registered_pairs(engine, oracle):
    """depth 25 mm to the side of the colour camera: the registered alignment is within 1e-3 m / 5e-4 rad of MIRROR's on
    the model planes, or closer to the truth; and registering beats using the depth unregistered on the median (the CPU
    measurement of tests/test_registration_host.py, DESIGN.md section 4.7)"""
    from dvo_slam_b200 import synth
    from dvo_slam_b200.engine import Config
    T = synth.baseline(0.025)
    cfg = synth.SceneConfig(depth_camera=synth.DepthCamera(640, 480, FR1, T))
    rays = rg.depth_rays((640, 480), FR1)
    reg = engine.depth_registration((640, 480), rays, T, (640, 480), FR1)
    err_reg, err_un = [], []
    for seed in range(8):
        p = synth.make_pair(seed, cfg)
        truth = np.linalg.inv(p["T_true"])
        I = np.stack([p["I_ref"].numpy(), p["I_cur"].numpy()])
        Z = np.stack([p["Z_ref"].numpy(), p["Z_cur"].numpy()])
        R = engine.pyramid_registered_batch(reg, I, Z, LEVELS)
        g = engine.match(R[0], R[1], Config(**CFG)).transformation
        planes = [rg.register(Z[k], rays, T, (640, 480), FR1) for k in (0, 1)]
        o = oracle.match(*[oracle.Pyramid(I[k], planes[k], FR1, LEVELS) for k in (0, 1)], oracle.config(**CFG), oracle.mode("mirror"))["T"]
        dt, dr = pose_delta(o, g)
        et, er = pose_delta(truth, g)
        ot, orr = pose_delta(truth, o)
        assert (dt <= 1e-3 and dr <= 5e-4) or (et <= ot and er <= orr), (seed, dt, dr, et, ot)
        P = engine.pyramid_batch(I, Z, FR1, LEVELS)
        err_reg.append(et)
        err_un.append(pose_delta(truth, engine.match(P[0], P[1], Config(**CFG)).transformation)[0])
    assert np.median(err_reg) < np.median(err_un), (err_reg, err_un)
    reg.release()


@pytest.mark.parametrize("mask", [None, "both"])
@pytest.mark.parametrize("fmt", FORMATS)
def test_traffic(engine, regs, fmt, mask):
    f = _frames("low-res")
    image, depth = _inputs(f, fmt)
    m = f["masks"] if mask else None
    b0 = engine.h2d_bytes()
    engine.pyramid_registered_batch(regs["low-res"], image, depth, LEVELS, depth_scale=SCALE, masks=m, mask_roles=mask or "reference")
    assert engine.h2d_bytes() - b0 == image.nbytes + depth.nbytes + (m.nbytes if mask else 0)
    dI, dZ = _to_device(image, "packed"), _to_device(depth, "packed")
    dM = _to_device(m, "packed") if mask else None
    torch.cuda.synchronize()
    b0 = engine.h2d_bytes()
    engine.pyramid_registered_batch(regs["low-res"], dI, dZ, LEVELS, depth_scale=SCALE, masks=dM, mask_roles=mask or "reference")
    engine.synchronize()
    assert engine.h2d_bytes() == b0


def test_rays_are_uploaded_once(engine):
    rays = rg.depth_rays((320, 240), CAMERAS["low-res"][1])
    b0 = engine.h2d_bytes()
    r = engine.depth_registration((320, 240), rays, _T(), (640, 480), FR1)
    assert engine.h2d_bytes() - b0 == sum(a.nbytes for a in rays)
    r.release()


def test_stream_order_and_early_release(engine):
    f = _frames("baseline")
    I, Z = f["float"]
    r0 = engine.depth_registration((640, 480), f["rays"], f["T"], (640, 480), FR1)
    H = engine.pyramid_registered_batch(r0, I, Z, LEVELS, masks=f["masks"][0], mask_roles="both")
    r0.release()
    r = engine.depth_registration((640, 480), f["rays"], f["T"], (640, 480), FR1)
    src_I, src_Z = torch.from_numpy(I).cuda(), torch.from_numpy(Z).cuda()
    mask = torch.from_numpy(f["masks"][0]).cuda()
    dI, dZ = torch.full_like(src_I, float("nan")), torch.full_like(src_Z, float("nan"))
    torch.cuda.synchronize()
    torch.cuda._sleep(100_000_000)     # the inputs are written on the current stream behind a long kernel
    dI.copy_(src_I)
    dZ.copy_(src_Z)
    D = engine.pyramid_registered_batch(r, dI, dZ, LEVELS, masks=mask, mask_roles="both")
    r.release()                        # right after the call, with the registration still queued
    dI.fill_(0.0)                      # and the inputs overwritten on the current stream
    dZ.fill_(float("nan"))
    mask.zero_()
    for p, q in zip(D, H):
        _assert_same_pyramid(p, q)


def test_invalid_arguments_create_nothing(engine, regs):
    from dvo_slam_b200.engine import DevicePlane, Engine, load_library
    lib = load_library()
    f = _frames("low-res")
    I, Z = f["float"]
    h, w = 480, 640
    dI, dZ = torch.from_numpy(I[0]).cuda(), torch.from_numpy(Z[0]).cuda()
    big = torch.zeros(h * w + 2, device="cuda")
    torch.cuda.synchronize()
    other = Engine(device=0)
    foreign = other.depth_registration((320, 240), f["rays"], f["T"], (w, h), FR1)
    mx, my = rm.undistort_map(w, h, FR1, (0, 0, 0, 0, 0))
    foreign_rect = other.rectifier((w, h), mx, my, FR1)
    rect_other_K = engine.rectifier((w, h), mx, my, (FR1[0] + 1, FR1[1], FR1[2], FR1[3]))
    rect_other_size = engine.rectifier((w, h), mx[:, :-2], my[:, :-2], FR1)
    reg = regs["low-res"]
    good = DevicePlane(dI.data_ptr(), 4 * w, 4 * w * h)
    depth = DevicePlane(dZ.data_ptr(), 4 * 320, 4 * 320 * 240)
    b0, l0 = engine.h2d_bytes(), engine.kernel_launches()
    out = (C.c_void_p * 1)()
    try:
        cases = {
            "null registration": (None, None, good, depth, w, h),
            "another context's registration": (foreign.handle, None, good, depth, w, h),
            "colour size mismatch": (reg.handle, None, good, depth, w - 2, h),
            "another context's rectifier": (reg.handle, foreign_rect.handle, good, depth, w, h),
            "rectifier K_new differs": (reg.handle, rect_other_K.handle, good, depth, w, h),
            "rectifier output size differs": (reg.handle, rect_other_size.handle, good, depth, w, h),
            "depth plane smaller than dw x dh": (reg.handle, None, good, DevicePlane(dZ.data_ptr(), 4 * 300, 0), w, h),
            "misaligned image": (reg.handle, None, DevicePlane(big.data_ptr() + 2, 4 * w, 4 * w * h), depth, w, h),
        }
        for name, (rh, ch, plane, dplane, ww, hh) in cases.items():
            rc = lib.dvo_b200_pyramid_create_registered_device_batch(engine.ctx, rh, ch, 1, 0, C.byref(plane), C.byref(dplane), 0.0, None, 1,
                                                                     ww, hh, LEVELS, out)
            assert rc == -1 and not out[0], name
            assert lib.dvo_b200_last_error(engine.ctx).decode().startswith("pyramid_create_registered_device"), name
        for name, rh, ch, ww, fmt, roles in (("host size mismatch", reg.handle, None, w + 1, 0, 1), ("host foreign", foreign.handle, None, w, 0, 1),
                                             ("host foreign rectifier", reg.handle, foreign_rect.handle, w, 0, 1),
                                             ("host unknown format", reg.handle, None, w, 7, 1), ("host roles", reg.handle, None, w, 0, 2)):
            rc = lib.dvo_b200_pyramid_create_registered_batch(engine.ctx, rh, ch, 1, fmt, I[0].ctypes.data, Z[0].ctypes.data, 0.0, None,
                                                              roles, ww, h, LEVELS, out)
            assert rc == -1 and not out[0], name
        assert engine.h2d_bytes() == b0 and engine.kernel_launches() == l0
        rc = lib.dvo_b200_pyramid_create_registered_device_batch(engine.ctx, reg.handle, None, 1, 0, C.byref(good), C.byref(depth), 0.0,
                                                                 None, 1, w, h, LEVELS, out)
        assert rc == 0 and out[0]
        lib.dvo_b200_pyramid_release(out[0])
        # the registration's own checks
        rays = f["rays"]
        for name, T, K in (("non-rigid", np.diag([1.0, 1.0, 1.01, 1.0]), FR1), ("reflection", np.diag([1.0, 1.0, -1.0, 1.0]), FR1),
                           ("non-finite", np.full((4, 4), np.nan), FR1), ("focal", np.eye(4), (0.0, FR1[1], FR1[2], FR1[3]))):
            with pytest.raises(RuntimeError):
                engine.depth_registration((320, 240), rays, T, (w, h), K)
        bad = [a.copy() for a in rays]
        bad[2][5, 5] = np.inf
        with pytest.raises(RuntimeError):
            engine.depth_registration((320, 240), bad, np.eye(4), (w, h), FR1)
        assert engine.h2d_bytes() == b0
    finally:
        for x in (foreign, foreign_rect, rect_other_K, rect_other_size):
            x.release()
        other.close()
