"""Pyramids of distorted frames on the H100 (dvo_b200_rectifier, dvo_b200_pyramid_create_rectified_batch and its device
form through Engine.rectifier / Engine.pyramid_rectified_batch): bit-for-bit equality with the float32 build of the numpy
remap model (tests/rectify_model.py) for every format, mask role set and input path, the identity map, records against the
oracle with NaN-intensity borders, the pose against MIRROR and the truth on fr1-distorted pairs, traffic, stream order, early
release of the rectifier, invalid arguments and tum_replay --distortion."""
import ctypes as C
import json
import os
import subprocess

import numpy as np
import pytest
import torch

import rectify_model as rm
from helpers import nan_equal, pose_delta
from test_gpu_device_input import _to_device
from test_gpu_masked_pyramids import _same_result

pytestmark = pytest.mark.gpu

LEVELS = 5
SCALE = 1.0 / 5000.0
FORMATS = ["float32", "grey8_depth16", "bgr8_depth16"]
MASKS = [None, "reference", "both"]
CFG = dict(first_level=4, last_level=0, max_iterations_per_level=50, precision=1e-4)


@pytest.fixture(scope="module")
def frames():
    """Three fr1-distorted 640x480 frames (a reference, its current frame, another reference) in every host representation,
    a blob mask per frame, the fr1 map with K_new = K, and a pose between the first two."""
    from dvo_slam_b200 import synth
    cfg = synth.SceneConfig(distortion=synth.FR1_DISTORTION)
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
    K = p["intrinsics"]
    mx, my = rm.undistort_map(w, h, K, synth.FR1_DISTORTION)
    return {"float": (I, Z), "grey": np.clip(I, 0, 255).astype(np.uint8),
            "raw": np.where(np.isnan(Z), 0, np.round(Z * 5000.0)).astype(np.uint16),
            "bgr": rng.integers(0, 256, (n, h, w, 3), dtype=np.uint8), "masks": M, "K": K, "map": (mx, my),
            "T": np.linalg.inv(synth.se3_exp(p["xi"] * 0.7))}


@pytest.fixture(scope="module")
def rect(engine, frames):
    mx, my = frames["map"]
    r = engine.rectifier((640, 480), mx, my, frames["K"])
    yield r
    r.release()


def _inputs(frames, fmt):
    image = {"float32": frames["float"][0], "grey8_depth16": frames["grey"], "bgr8_depth16": frames["bgr"]}[fmt]
    depth = frames["float"][1] if fmt == "float32" else frames["raw"]
    return image, depth


def _model_build(engine, frames, fmt, mask, mx, my, K):
    """the float32 pyramids of the model's rectified planes and mask, by the plain masked create"""
    image, depth = _inputs(frames, fmt)
    I, Z, M = rm.remap_batch(image, depth, mx, my, frames["masks"] if mask else None, SCALE)
    kw = {} if mask is None else {"masks": M, "mask_roles": mask}
    return engine.pyramid_batch(I, Z, K, LEVELS, **kw)


def _rectified_build(engine, rect, frames, fmt, mask, path):
    image, depth = _inputs(frames, fmt)
    kw = {"depth_scale": None if fmt == "float32" else SCALE, "mask_roles": mask or "reference"}
    if path == "host":
        return engine.pyramid_rectified_batch(rect, image, depth, LEVELS, masks=frames["masks"] if mask else None, **kw)
    fill_z = float("nan") if fmt == "float32" else 777
    dM = _to_device(frames["masks"], "crop", torch.bool, fill=1) if mask else None
    return engine.pyramid_rectified_batch(rect, _to_device(image, "crop", fill=99), _to_device(depth, "crop", fill=fill_z), LEVELS,
                                          masks=dM, **kw)


def _assert_same_pyramid(p, q):
    for l in range(LEVELS):
        assert np.array_equal(p.download(l), q.download(l), equal_nan=True), l
        for ti, td in ((0.0, 0.0), (6.0, 0.02)):
            S0, m0 = p.select(l, ti, td)
            S1, m1 = q.select(l, ti, td)
            assert S0 == S1 and np.array_equal(m0, m1), (l, ti, td)


def _records(engine, refs, curs):
    """the whole result records of the alignments, as bytes"""
    from dvo_slam_b200.engine import Config
    res = engine.match_batch(refs, curs, Config(**CFG), raw=True)
    return bytes(res)


@pytest.mark.parametrize("path", ["host", "device"])
@pytest.mark.parametrize("mask", MASKS)
@pytest.mark.parametrize("fmt", FORMATS)
def test_rectified_build_equals_the_model_build(engine, rect, frames, fmt, mask, path):
    mx, my = frames["map"]
    H = _model_build(engine, frames, fmt, mask, mx, my, frames["K"])
    R = _rectified_build(engine, rect, frames, fmt, mask, path)
    assert [p.mask_roles for p in R] == [p.mask_roles for p in H]
    assert all(p.level_info(0) == (640, 480, tuple(np.float32(frames["K"]))) for p in R)
    for p, q in zip(R, H):
        _assert_same_pyramid(p, q)
    assert _records(engine, [R[0], R[2], R[1]], [R[1], R[0], R[0]]) == _records(engine, [H[0], H[2], H[1]], [H[1], H[0], H[0]])


@pytest.mark.parametrize("fmt", FORMATS)
def test_identity_map_gives_the_plain_pyramids(engine, frames, fmt):
    """integer coordinates with K_new = K: every output pixel reads its own input pixel, so the pyramids are those of the
    unrectified create in the same format"""
    h, w = 480, 640
    mx, my = rm.undistort_map(w, h, frames["K"], (0, 0, 0, 0, 0))
    assert np.array_equal(mx, np.broadcast_to(np.arange(w, dtype=np.float32), (h, w)))
    r = engine.rectifier((w, h), mx, my, frames["K"])
    image, depth = _inputs(frames, fmt)
    n = depth.shape[0]
    R = engine.pyramid_rectified_batch(r, image, depth, LEVELS, depth_scale=SCALE)
    if fmt == "float32":
        P = engine.pyramid_batch(image, depth, frames["K"], LEVELS)
    else:
        build = engine.pyramid_raw_batch if fmt == "grey8_depth16" else engine.pyramid_bgr_batch
        P = build((image.ctypes.data, depth.ctypes.data, n, h, w), SCALE, frames["K"], LEVELS)
        engine.synchronize()
    for p, q in zip(R, P):
        _assert_same_pyramid(p, q)
    assert _records(engine, R[:2], R[1::-1]) == _records(engine, P[:2], P[1::-1])
    r.release()


def test_records_with_nan_intensity_borders_match_mirror(engine, oracle, rect, frames):
    """The rectified pair has NaN intensities where the map leaves the frame.  Level 0 matches the bare oracle; every level
    matches the oracle under the engine's rule for NaN channels (rectify_model.oracle_pyramid)."""
    mx, my = frames["map"]
    I, Z = frames["float"]
    R = engine.pyramid_rectified_batch(rect, I[:2], Z[:2], LEVELS)
    planes = [rm.remap(I[k], Z[k], mx, my) for k in (0, 1)]
    assert np.isnan(planes[0][0]).mean() > 0.05
    mode, T = oracle.mode("mirror"), frames["T"]
    bare = [oracle.Pyramid(planes[k][0], planes[k][1], frames["K"], LEVELS) for k in (0, 1)]
    ruled = [rm.oracle_pyramid(oracle, planes[k][0], planes[k][1], frames["K"], LEVELS) for k in (0, 1)]
    n_g, img_g = engine.residual_image(R[0], R[1], 0, T)
    n_o, img_o = oracle.residual_image(bare[0], bare[1], 0, T, mode)
    assert n_g == n_o > 0 and nan_equal(img_g, img_o)
    for lvl in range(LEVELS):
        n_g, img_g = engine.residual_image(R[0], R[1], lvl, T)
        n_o, img_o = oracle.residual_image(ruled[0], ruled[1], lvl, T, mode)
        assert n_g == n_o > 0 and nan_equal(img_g, img_o), (lvl, n_g, n_o)
        ne_g, err_g = engine.intensity_error_image(R[0], R[1], lvl, T)
        ne_o, err_o = oracle.intensity_error_image(ruled[0], ruled[1], lvl, T, mode)
        assert ne_g == ne_o and np.array_equal(err_g, err_o), lvl


def test_pose_on_distorted_pairs(engine, oracle):
    """fr1-distorted pairs: the rectified alignment is within 1e-3 m / 5e-4 rad of MIRROR's on the model planes, or closer
    to the truth; and rectifying brings the median translation error below that of aligning the distorted frames as pinhole
    (the CPU measurement of tests/test_rectify_host.py, DESIGN.md section 4.6)"""
    from dvo_slam_b200 import synth
    from dvo_slam_b200.engine import Config
    cfg = synth.SceneConfig(distortion=synth.FR1_DISTORTION)
    K = cfg.intrinsics
    mx, my = rm.undistort_map(640, 480, K, synth.FR1_DISTORTION)
    r = engine.rectifier((640, 480), mx, my, K)
    err_rect, err_pin = [], []
    for seed in range(8):
        p = synth.make_pair(seed, cfg)
        truth = np.linalg.inv(p["T_true"])
        I = np.stack([p["I_ref"].numpy(), p["I_cur"].numpy()])
        Z = np.stack([p["Z_ref"].numpy(), p["Z_cur"].numpy()])
        R = engine.pyramid_rectified_batch(r, I, Z, LEVELS)
        g = engine.match(R[0], R[1], Config(**CFG)).transformation
        planes = [rm.remap(I[k], Z[k], mx, my) for k in (0, 1)]
        o = oracle.match(*[rm.oracle_pyramid(oracle, pl[0], pl[1], K, LEVELS) for pl in planes], oracle.config(**CFG),
                         oracle.mode("mirror"))["T"]
        dt, dr = pose_delta(o, g)
        et, er = pose_delta(truth, g)
        ot, orr = pose_delta(truth, o)
        assert (dt <= 1e-3 and dr <= 5e-4) or (et <= ot and er <= orr), (seed, dt, dr, et, ot)
        P = engine.pyramid_batch(I, Z, K, LEVELS)
        err_rect.append(et)
        err_pin.append(pose_delta(truth, engine.match(P[0], P[1], Config(**CFG)).transformation)[0])
    assert np.median(err_rect) < np.median(err_pin), (err_rect, err_pin)
    r.release()


@pytest.mark.parametrize("mask", [None, "both"])
@pytest.mark.parametrize("fmt", FORMATS)
def test_traffic(engine, rect, frames, fmt, mask):
    image, depth = _inputs(frames, fmt)
    b0 = engine.h2d_bytes()
    engine.pyramid_rectified_batch(rect, image, depth, LEVELS, depth_scale=SCALE, masks=frames["masks"] if mask else None,
                                   mask_roles=mask or "reference")
    assert engine.h2d_bytes() - b0 == image.nbytes + depth.nbytes + (frames["masks"].nbytes if mask else 0)
    dI, dZ = _to_device(image, "packed"), _to_device(depth, "packed")
    dM = _to_device(frames["masks"], "packed") if mask else None
    torch.cuda.synchronize()
    b0 = engine.h2d_bytes()
    engine.pyramid_rectified_batch(rect, dI, dZ, LEVELS, depth_scale=SCALE, masks=dM, mask_roles=mask or "reference")
    engine.synchronize()
    assert engine.h2d_bytes() == b0


def test_map_is_uploaded_once(engine, frames):
    mx, my = frames["map"]
    b0 = engine.h2d_bytes()
    r = engine.rectifier((640, 480), mx, my, frames["K"])
    assert engine.h2d_bytes() - b0 == mx.nbytes + my.nbytes
    r.release()


def test_stream_order_and_early_release(engine, frames):
    mx, my = frames["map"]
    I, Z = frames["float"]
    r0 = engine.rectifier((640, 480), mx, my, frames["K"])
    H = engine.pyramid_rectified_batch(r0, I, Z, LEVELS, masks=frames["masks"][0], mask_roles="both")
    r0.release()
    r = engine.rectifier((640, 480), mx, my, frames["K"])
    src_I, src_Z = torch.from_numpy(I).cuda(), torch.from_numpy(Z).cuda()
    mask = torch.from_numpy(frames["masks"][0]).cuda()
    dI, dZ = torch.full_like(src_I, float("nan")), torch.full_like(src_Z, float("nan"))
    torch.cuda.synchronize()
    torch.cuda._sleep(100_000_000)     # the inputs are written on the current stream behind a long kernel
    dI.copy_(src_I)
    dZ.copy_(src_Z)
    D = engine.pyramid_rectified_batch(r, dI, dZ, LEVELS, masks=mask, mask_roles="both")
    r.release()                        # right after the call, with the remap still queued
    dI.fill_(0.0)                      # and the inputs overwritten on the current stream
    dZ.fill_(float("nan"))
    mask.zero_()
    for p, q in zip(D, H):
        _assert_same_pyramid(p, q)


def test_invalid_arguments_create_nothing(engine, rect, frames):
    from dvo_slam_b200.engine import DevicePlane, Engine, load_library
    lib = load_library()
    I, Z = frames["float"]
    h, w = 480, 640
    dI, dZ = torch.from_numpy(I[0]).cuda(), torch.from_numpy(Z[0]).cuda()
    big = torch.zeros(h * w + 2, device="cuda")
    torch.cuda.synchronize()
    other = Engine(device=0)
    mx, my = frames["map"]
    foreign = other.rectifier((w, h), mx, my, frames["K"])
    good, depth = DevicePlane(dI.data_ptr(), 4 * w, 4 * w * h), DevicePlane(dZ.data_ptr(), 4 * w, 4 * w * h)
    b0, l0 = engine.h2d_bytes(), engine.kernel_launches()
    out = (C.c_void_p * 1)()
    try:
        cases = {
            "size mismatch": (rect.handle, good, w - 2, h),
            "another context's rectifier": (foreign.handle, good, w, h),
            "misaligned plane": (rect.handle, DevicePlane(big.data_ptr() + 2, 4 * w, 4 * w * h), w, h),
            "null rectifier": (None, good, w, h),
        }
        for name, (rh, plane, ww, hh) in cases.items():
            rc = lib.dvo_b200_pyramid_create_rectified_device_batch(engine.ctx, rh, 1, 0, C.byref(plane), C.byref(depth), 0.0, None, 1,
                                                                    ww, hh, LEVELS, out)
            assert rc == -1 and not out[0], name
            assert lib.dvo_b200_last_error(engine.ctx).decode().startswith("pyramid_create_rectified_device"), name
        for name, rh, ww in (("host size mismatch", rect.handle, w + 1), ("host foreign", foreign.handle, w)):
            rc = lib.dvo_b200_pyramid_create_rectified_batch(engine.ctx, rh, 1, 0, I[0].ctypes.data, Z[0].ctypes.data, 0.0, None, 1, ww, h,
                                                             LEVELS, out)
            assert rc == -1 and not out[0], name
        assert engine.h2d_bytes() == b0 and engine.kernel_launches() == l0
        rc = lib.dvo_b200_pyramid_create_rectified_device_batch(engine.ctx, rect.handle, 1, 0, C.byref(good), C.byref(depth), 0.0, None, 1,
                                                                w, h, LEVELS, out)
        assert rc == 0 and out[0]
        lib.dvo_b200_pyramid_release(out[0])
    finally:
        foreign.release()
        other.close()


def test_tum_replay_zero_distortion_is_the_plain_replay(tmp_path):
    import __graft_entry__ as ge
    from dvo_slam_b200 import synth
    from test_tum_replay import HOST, write_sequence
    ge.build_cuda()
    ge.build_host()
    cfg = synth.SceneConfig(width=320, height=240, intrinsics=tuple(v / 2 for v in synth.FR1_INTRINSICS))
    n = 6
    seq, poses = synth.make_sequence(5, n, cfg)
    rgb = [np.repeat(f[0].numpy().astype(np.uint8)[..., None], 3, axis=2) for f in seq]
    depth = [np.where(np.isnan(f[1].numpy()), 0, np.round(f[1].numpy() * 5000.0)).astype(np.uint16) for f in seq]
    assoc = write_sequence(str(tmp_path), rgb, depth, [100.0 + 0.033 * k for k in range(n)], poses)
    out = {}
    for name, extra in (("plain", []), ("zero", ["--distortion", "0", "0", "0", "0", "0"])):
        traj = str(tmp_path / f"{name}.txt")
        r = subprocess.run([os.path.join(HOST, "tum_replay"), "--assoc", assoc, "--out", traj, "--batch", "3", "--first", "2", "--last", "0",
                            "--intrinsics"] + [repr(float(v)) for v in cfg.intrinsics] + extra, capture_output=True, text=True, timeout=300)
        assert r.returncode == 0, r.stderr
        assert json.loads(r.stderr.strip().splitlines()[-1])["alignments"] == n - 1
        out[name] = open(traj).read()
    assert out["zero"] == out["plain"] and len(out["plain"].splitlines()) == n - 1
