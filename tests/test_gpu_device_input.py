"""Pyramids from device memory on the H100 (dvo_b200_pyramid_create_device_batch through Engine.pyramid_batch_device):
bit-for-bit parity with the host path for every input format, mask role set and plane layout (packed, a cropped view with
an odd base offset and a pitch above the width, an odd size, planes shared by the whole batch), no host-to-device traffic,
ordering with torch streams, pyramids shared with a second context, and invalid arguments that create nothing."""
import ctypes as C

import numpy as np
import pytest
import torch

from test_gpu_masked_pyramids import _same_result

pytestmark = pytest.mark.gpu

LEVELS = 5
SCALE = 1.0 / 5000.0
FORMATS = ["float32", "grey8_depth16", "bgr8_depth16"]
MASKS = [None, "reference", "both"]
LAYOUTS = ["packed", "crop", "odd", "shared"]
CFG = dict(first_level=4, last_level=0, max_iterations_per_level=50, precision=1e-4)


@pytest.fixture(scope="module")
def corrected(engine):
    from dvo_slam_b200.engine import Engine
    eng = Engine(device=0, estimator="corrected")
    yield eng
    eng.close()


@pytest.fixture(scope="module")
def frames():
    """Three 640x480 frames (a reference, its current frame, another reference) in every host representation, a blob mask per
    frame, the intrinsics and a pose between the first two."""
    from dvo_slam_b200 import synth
    p, q = synth.make_pair(21), synth.make_pair(22)
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
    return {"float": (I, Z), "grey": np.clip(I, 0, 255).astype(np.uint8),
            "raw": np.where(np.isnan(Z), 0, np.round(Z * 5000.0)).astype(np.uint16),
            "bgr": rng.integers(0, 256, (n, h, w, 3), dtype=np.uint8), "masks": M, "K": p["intrinsics"],
            "T": np.linalg.inv(synth.se3_exp(p["xi"] * 0.7))}


def _host_inputs(frames, fmt, layout):
    """(image, depth, masks) as packed host arrays with the values the device planes of `layout` hold"""
    image = {"float32": frames["float"][0], "grey8_depth16": frames["grey"], "bgr8_depth16": frames["bgr"]}[fmt]
    depth = frames["float"][1] if fmt == "float32" else frames["raw"]
    masks = frames["masks"]
    if layout == "odd":
        image, depth, masks = image[:, :479, :637], depth[:, :479, :637], masks[:, :479, :637]
    if layout == "shared":      # one depth plane and one mask for the whole batch
        depth, masks = np.broadcast_to(depth[:1], depth.shape), np.broadcast_to(masks[:1], masks.shape)
    return tuple(np.ascontiguousarray(a) for a in (image, depth, masks))


def _to_device(a, layout, dtype=None, fill=0):
    """a device tensor with a's values in the plane layout: packed, or a crop of a larger tensor whose other elements hold
    `fill` (the crop's first element sits at an odd element offset, its pitch above its width)"""
    u16 = a.dtype == np.uint16
    t = torch.from_numpy(a.view(np.int16) if u16 else a)     # 16-bit depth travels as int16 and is viewed as uint16 at the end
    if dtype is not None:
        t = t.to(dtype)
    t = t.cuda()
    if layout == "crop":
        n, h, w = t.shape[:3]
        big = torch.full((n, h + 3, w + 5) + tuple(t.shape[3:]), fill, dtype=t.dtype, device="cuda")
        big[:, 1:1 + h, 2:2 + w] = t      # element offset (w + 5) + 2: odd for w = 640
        t = big[:, 1:1 + h, 2:2 + w]
    return t.view(torch.uint16) if u16 else t


def _device_inputs(frames, fmt, layout, with_masks):
    image, depth, masks = _host_inputs(frames, fmt, layout)
    if layout == "shared":
        dI = _to_device(image, layout)
        dZ = _to_device(depth[:1], layout).expand(depth.shape)
        dM = _to_device(masks[0], layout, torch.bool) if with_masks else None
        return dI, dZ, dM
    fill_z = float("nan") if fmt == "float32" else 777
    dM = _to_device(masks, layout, torch.bool if layout == "crop" else None, fill=1) if with_masks else None
    return _to_device(image, layout, fill=99), _to_device(depth, layout, fill=fill_z), dM


def _host_build(engine, frames, fmt, layout, mask):
    image, depth, masks = _host_inputs(frames, fmt, layout)
    n, h, w = depth.shape
    kw = {} if mask is None else {"masks": masks, "mask_roles": mask}
    if fmt == "float32":
        return engine.pyramid_batch(image, depth, frames["K"], LEVELS, **kw)
    ptrs = (image.ctypes.data, depth.ctypes.data, n, h, w)
    build = engine.pyramid_raw_batch if fmt == "grey8_depth16" else engine.pyramid_bgr_batch
    out = build(ptrs, SCALE, frames["K"], LEVELS, **kw)
    engine.synchronize()        # the host arrays die with this frame
    return out


def _device_build(engine, frames, fmt, layout, mask):
    dI, dZ, dM = _device_inputs(frames, fmt, layout, mask is not None)
    return engine.pyramid_batch_device(dI, dZ, frames["K"], LEVELS, depth_scale=None if fmt == "float32" else SCALE, masks=dM,
                                       mask_roles=mask or "reference")


def _assert_same_pyramid(p, q):
    for l in range(LEVELS):
        assert np.array_equal(p.download(l), q.download(l), equal_nan=True), l
        for ti, td in ((0.0, 0.0), (6.0, 0.02)):
            S0, m0 = p.select(l, ti, td)
            S1, m1 = q.select(l, ti, td)
            assert S0 == S1 and np.array_equal(m0, m1), (l, ti, td)


@pytest.mark.parametrize("layout", LAYOUTS)
@pytest.mark.parametrize("mask", MASKS)
@pytest.mark.parametrize("fmt", FORMATS)
def test_device_build_equals_host_build(engine, corrected, frames, fmt, mask, layout):
    from dvo_slam_b200.engine import Config
    H = _host_build(engine, frames, fmt, layout, mask)
    D = _device_build(engine, frames, fmt, layout, mask)
    assert [p.mask_roles for p in D] == [p.mask_roles for p in H]
    for p, q in zip(D, H):
        _assert_same_pyramid(p, q)
    T = frames["T"]
    for l in range(LEVELS):       # the device pyramid in either role of an alignment
        n_h, r_h = engine.residual_image(H[0], H[1], l, T)
        for ref, cur in ((D[0], H[1]), (H[0], D[1])):
            n_d, r_d = engine.residual_image(ref, cur, l, T)
            assert n_d == n_h and np.array_equal(r_d, r_h, equal_nan=True), l
    cfg = Config(**CFG)
    for eng in (engine, corrected):       # one batch mixing device- and host-built pyramids
        r = eng.match_batch([D[0], H[0], D[1], H[1], D[2]], [D[1], H[1], H[0], D[0], H[0]], cfg)
        assert _same_result(r[0], r[1]) and _same_result(r[2], r[3]), eng.estimator
        assert _same_result(r[4], eng.match(H[2], H[0], cfg)), eng.estimator


@pytest.mark.parametrize("mask", MASKS)
@pytest.mark.parametrize("fmt", FORMATS)
def test_no_host_round_trip(engine, frames, fmt, mask):
    l0 = engine.kernel_launches()
    _host_build(engine, frames, fmt, "packed", mask)
    host_launches = engine.kernel_launches() - l0
    dI, dZ, dM = _device_inputs(frames, fmt, "packed", mask is not None)
    torch.cuda.synchronize()
    b0, l0 = engine.h2d_bytes(), engine.kernel_launches()
    engine.pyramid_batch_device(dI, dZ, frames["K"], LEVELS, depth_scale=SCALE, masks=dM, mask_roles=mask or "reference")
    assert engine.h2d_bytes() == b0
    assert engine.kernel_launches() - l0 == host_launches


def test_stream_order_with_torch_and_a_second_context(engine, frames):
    from dvo_slam_b200.engine import Config, Engine
    I, Z = frames["float"]
    n, h, w = I.shape
    H = engine.pyramid_batch(I, Z, frames["K"], LEVELS, masks=frames["masks"][:1].repeat(n, 0), mask_roles="both")
    src_I, src_Z = torch.from_numpy(I).cuda(), torch.from_numpy(Z).cuda()
    mask = torch.from_numpy(frames["masks"][0]).cuda()
    dI, dZ = torch.full_like(src_I, float("nan")), torch.full_like(src_Z, float("nan"))
    torch.cuda.synchronize()
    # the inputs are written on the current stream behind a long kernel; the build must wait for them
    torch.cuda._sleep(100_000_000)
    dI.copy_(src_I)
    dZ.copy_(src_Z)
    D = engine.pyramid_batch_device(dI, dZ, frames["K"], LEVELS, masks=mask, mask_roles="both")
    # and overwritten on the current stream right after the call, while the build may still be queued
    dI.fill_(0.0)
    dZ.fill_(float("nan"))
    mask.zero_()
    for p, q in zip(D, H):
        _assert_same_pyramid(p, q)
    other = Engine(device=0)
    try:
        cfg = Config(**CFG)
        assert _same_result(other.match(D[0], D[1], cfg), engine.match(H[0], H[1], cfg))
        for l in range(LEVELS):
            assert np.array_equal(other.residual_image(H[0], D[1], l, frames["T"])[1],
                                  engine.residual_image(H[0], H[1], l, frames["T"])[1], equal_nan=True)
    finally:
        for p in D:
            p.release()
        other.close()


def test_invalid_arguments_create_nothing(engine, frames):
    from dvo_slam_b200.engine import DevicePlane, load_library
    lib = load_library()
    I, Z = frames["float"]
    h, w = I.shape[1:]
    K = frames["K"]
    dI = torch.from_numpy(I[0]).cuda()
    dZ = torch.from_numpy(Z[0]).cuda()
    big = torch.zeros(h * w + 2, device="cuda")
    pageable = np.ascontiguousarray(I[0])
    pinned = torch.from_numpy(I[0]).pin_memory()
    row, img = 4 * w, 4 * w * h
    good = DevicePlane(dI.data_ptr(), row, img)
    depth = DevicePlane(dZ.data_ptr(), row, img)
    torch.cuda.synchronize()

    def create(image, fmt=0, roles=1, masks=None):
        out = (C.c_void_p * 1)()
        rc = lib.dvo_b200_pyramid_create_device_batch(engine.ctx, 1, fmt, C.byref(image), C.byref(depth), 0.0,
                                                      C.byref(masks) if masks is not None else None, roles, w, h, *K, LEVELS, out)
        return rc, out[0]

    cases = {
        "pageable host": (DevicePlane(pageable.ctypes.data, row, img), {}),
        "pinned host": (DevicePlane(pinned.data_ptr(), row, img), {}),
        "pinned host mask": (good, {"masks": DevicePlane(pinned.data_ptr(), w, w * h)}),
        "row_bytes too small": (DevicePlane(dI.data_ptr(), row - 4, img), {}),
        "row_bytes not a multiple of 4": (DevicePlane(dI.data_ptr(), row + 2, img), {}),
        "float pointer offset by 2 bytes": (DevicePlane(big.data_ptr() + 2, row, img), {}),
        "negative image stride": (DevicePlane(dI.data_ptr(), row, -img), {}),
        "null data": (DevicePlane(None, row, img), {}),
        "format 3": (good, {"fmt": 3}),
        "format -1": (good, {"fmt": -1}),
        "roles 2": (good, {"roles": 2}),
        "roles 0": (good, {"roles": 0}),
    }
    b0, l0 = engine.h2d_bytes(), engine.kernel_launches()
    for name, (plane, kw) in cases.items():
        rc, out = create(plane, **kw)
        assert rc == -1 and not out, (name, rc)
        assert lib.dvo_b200_last_error(engine.ctx).decode().startswith("pyramid_create_device"), name
    assert engine.h2d_bytes() == b0 and engine.kernel_launches() == l0
    rc, out = create(good)
    assert rc == 0 and out
    lib.dvo_b200_pyramid_release(out)


def test_memory_of_another_device_is_refused(engine, frames):
    from dvo_slam_b200.engine import DevicePlane, load_library
    if torch.cuda.device_count() < 2:
        pytest.skip("one GPU")
    lib = load_library()
    I, Z = frames["float"]
    h, w = I.shape[1:]
    dZ = torch.from_numpy(Z[0]).cuda()
    elsewhere = torch.from_numpy(I[0]).to("cuda:1")
    torch.cuda.synchronize(1)
    image, depth = DevicePlane(elsewhere.data_ptr(), 4 * w, 0), DevicePlane(dZ.data_ptr(), 4 * w, 0)
    out = (C.c_void_p * 1)()
    rc = lib.dvo_b200_pyramid_create_device_batch(engine.ctx, 1, 0, C.byref(image), C.byref(depth), 0.0, None, 1, w, h,
                                                  *frames["K"], LEVELS, out)
    assert rc == -1 and not out[0]
    assert "device 1" in lib.dvo_b200_last_error(engine.ctx).decode()
