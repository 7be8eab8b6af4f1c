"""Every pyramid create entry point through the refusals it can receive, on the H100: each returns
DVO_B200_ERR_INVALID_ARGUMENT with the entry point's prefix in dvo_b200_last_error, writes no handle, and leaves
dvo_b200_h2d_bytes and dvo_b200_kernel_launches where they were -- a bad level geometry included, which is refused before
the frames are uploaded or the BGR reduction is launched."""
import ctypes as C
from types import SimpleNamespace

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

W, H, LEVELS, SCALE = 64, 48, 3, 1.0 / 5000.0
K = (50.0, 50.0, 31.5, 23.5)
DEPTH_CAMERA = ((32, 24), (25.0, 25.0, 15.5, 11.5))

# entry point -> (prefix, host pointers or device planes, remap: None / "rect" / "reg", whether n, format and roles are arguments)
ENTRIES = {
    "dvo_b200_pyramid_create": ("pyramid_create", "host", None, False, False, False),
    "dvo_b200_pyramid_create_batch": ("pyramid_create", "host", None, True, False, False),
    "dvo_b200_pyramid_create_raw": ("pyramid_create_raw", "host", None, False, False, False),
    "dvo_b200_pyramid_create_raw_batch": ("pyramid_create_raw", "host", None, True, False, False),
    "dvo_b200_pyramid_create_bgr_batch": ("pyramid_create_bgr", "host", None, True, False, False),
    "dvo_b200_pyramid_create_masked_batch": ("pyramid_create_masked", "host", None, True, True, False),
    "dvo_b200_pyramid_create_masked_batch_roles": ("pyramid_create_masked_roles", "host", None, True, True, True),
    "dvo_b200_pyramid_create_device_batch": ("pyramid_create_device", "device", None, True, True, True),
    "dvo_b200_pyramid_create_rectified_batch": ("pyramid_create_rectified", "host", "rect", True, True, True),
    "dvo_b200_pyramid_create_rectified_device_batch": ("pyramid_create_rectified_device", "device", "rect", True, True, True),
    "dvo_b200_pyramid_create_registered_batch": ("pyramid_create_registered", "host", "reg", True, True, True),
    "dvo_b200_pyramid_create_registered_device_batch": ("pyramid_create_registered_device", "device", "reg", True, True, True),
}
FORMAT_OF = {"dvo_b200_pyramid_create_raw": 1, "dvo_b200_pyramid_create_raw_batch": 1, "dvo_b200_pyramid_create_bgr_batch": 2}


def _rows(entry):
    """(name, changes to the good call) of every refusal the entry point can receive"""
    _, _, remap, has_n, has_format, has_roles = ENTRIES[entry]
    rows = [("null image", dict(image=None)), ("null depth", dict(depth=None)), ("levels 0", dict(levels=0)),
            ("levels 9", dict(levels=9)), ("a level below 8x2", dict(levels=5))]
    rows += [("width 31", dict(width=31, levels=1))] if remap is None else []
    rows += [("n 0", dict(n=0)), ("n -1", dict(n=-1))] if has_n else []
    rows += [("format -1", dict(format=-1)), ("format 3", dict(format=3))] if has_format else []
    rows += [("width 31 from BGR", dict(format=2, width=31, levels=1))] if has_format and remap is None else []
    rows += [("roles 0", dict(roles=0)), ("roles 2", dict(roles=2))] if has_roles else []
    if remap == "rect":
        rows += [("null rectifier", dict(rect="none")), ("another context's rectifier", dict(rect="foreign")),
                 ("frames of another size", dict(width=W - 2)), ("a rectified width of 31", dict(rect="narrow", levels=1))]
    if remap == "reg":
        rows += [("null registration", dict(reg="none")), ("another context's registration", dict(reg="foreign")),
                 ("colour frames of another size", dict(width=W - 2)), ("a target width of 31", dict(reg="narrow", width=31, levels=1)),
                 ("another context's rectifier", dict(rect="foreign")), ("a rectifier of another output size", dict(rect="narrow")),
                 ("a rectifier of another K_new", dict(rect="other K"))]
    return rows


@pytest.fixture(scope="module")
def inputs(engine):
    from dvo_slam_b200.engine import DevicePlane, Engine
    rng = np.random.default_rng(5)
    (dw, dh), Kd = DEPTH_CAMERA
    host = {"float": rng.uniform(0, 255, (1, H, W)).astype(np.float32), "grey": rng.integers(0, 256, (1, H, W), dtype=np.uint8),
            "bgr": rng.integers(0, 256, (1, H, W, 3), dtype=np.uint8), "z": rng.uniform(0.5, 4, (1, H, W)).astype(np.float32),
            "raw": rng.integers(1, 20000, (1, H, W), dtype=np.uint16), "zd": rng.uniform(0.5, 4, (1, dh, dw)).astype(np.float32),
            "rawd": rng.integers(1, 20000, (1, dh, dw), dtype=np.uint16), "masks": np.ones((1, H, W), np.uint8)}
    dev = {k: torch.from_numpy(v).cuda() for k, v in host.items()}
    torch.cuda.synchronize()
    other = Engine(device=0)
    mx, my = engine.undistort_map(W, H, K, (0, 0, 0, 0, 0))
    rays = engine.depth_rays((dw, dh), Kd)
    Kn = (K[0] + 1, K[1], K[2], K[3])
    objs = {"rect": {"good": engine.rectifier((W, H), mx, my, K), "foreign": other.rectifier((W, H), mx, my, K),
                     "narrow": engine.rectifier((W, H), mx[:, :31], my[:, :31], K), "other K": engine.rectifier((W, H), mx, my, Kn)},
            "reg": {"good": engine.depth_registration((dw, dh), rays, np.eye(4), (W, H), K),
                    "foreign": other.depth_registration((dw, dh), rays, np.eye(4), (W, H), K),
                    "narrow": engine.depth_registration((dw, dh), rays, np.eye(4), (31, H), K)}}

    def plane(t, px=1):
        es = t.element_size()
        return DevicePlane(t.data_ptr(), t.shape[2] * px * es, t[0].numel() * es)

    yield SimpleNamespace(host=host, dev=dev, objs=objs, plane=plane)
    for group in objs.values():
        for o in group.values():
            o.release()
    other.close()


def _call(lib, engine, entry, a, out):
    _, form, remap, _, _, _ = ENTRIES[entry]
    fmt = a.format if a.format in (0, 1, 2) else 0
    depth_key = ("zd" if fmt == 0 else "rawd") if remap == "reg" else ("z" if fmt == 0 else "raw")
    image_key = ("float", "grey", "bgr")[fmt]
    if form == "host":
        image, depth = a.inputs.host[image_key].ctypes.data, a.inputs.host[depth_key].ctypes.data
    else:
        image = C.byref(a.inputs.plane(a.inputs.dev[image_key], 3 if fmt == 2 else 1))
        depth = C.byref(a.inputs.plane(a.inputs.dev[depth_key]))
    image, depth = (None if a.image is None else image), (None if a.depth is None else depth)
    f = getattr(lib, entry)
    if entry in ("dvo_b200_pyramid_create",):
        return f(engine.ctx, image, depth, a.width, H, *K, a.levels, out)
    if entry in ("dvo_b200_pyramid_create_raw",):
        return f(engine.ctx, image, depth, SCALE, a.width, H, *K, a.levels, out)
    if entry == "dvo_b200_pyramid_create_batch":
        return f(engine.ctx, a.n, image, depth, a.width, H, *K, a.levels, out)
    if entry in ("dvo_b200_pyramid_create_raw_batch", "dvo_b200_pyramid_create_bgr_batch"):
        return f(engine.ctx, a.n, image, depth, SCALE, a.width, H, *K, a.levels, out)
    if entry == "dvo_b200_pyramid_create_masked_batch":
        return f(engine.ctx, a.n, a.format, image, depth, SCALE, None, a.width, H, *K, a.levels, out)
    if entry == "dvo_b200_pyramid_create_masked_batch_roles":
        return f(engine.ctx, a.n, a.format, image, depth, SCALE, None, a.roles, a.width, H, *K, a.levels, out)
    if entry == "dvo_b200_pyramid_create_device_batch":
        return f(engine.ctx, a.n, a.format, image, depth, SCALE, None, a.roles, a.width, H, *K, a.levels, out)
    rect = a.inputs.objs["rect"].get(a.rect)
    rh = rect.handle if rect is not None else None
    if remap == "rect":
        return f(engine.ctx, rh, a.n, a.format, image, depth, SCALE, None, a.roles, a.width, H, a.levels, out)
    reg = a.inputs.objs["reg"].get(a.reg)
    return f(engine.ctx, reg.handle if reg is not None else None, rh, a.n, a.format, image, depth, SCALE, None, a.roles, a.width, H,
             a.levels, out)


@pytest.mark.parametrize("entry", list(ENTRIES))
def test_refusals_create_nothing(engine, inputs, entry):
    from dvo_slam_b200.engine import load_library
    lib = load_library()
    prefix, _, remap, _, _, _ = ENTRIES[entry]
    good = dict(n=1, format=FORMAT_OF.get(entry, 0), roles=1, width=W, levels=LEVELS, image=1, depth=1, inputs=inputs,
                rect="good" if remap == "rect" else "none", reg="good")
    out = (C.c_void_p * 1)()
    failed = []
    for name, change in _rows(entry):
        b0, l0 = engine.h2d_bytes(), engine.kernel_launches()
        rc = _call(lib, engine, entry, SimpleNamespace(**dict(good, **change)), out)
        msg = lib.dvo_b200_last_error(engine.ctx).decode()
        moved = (engine.h2d_bytes() - b0, engine.kernel_launches() - l0)
        if rc != -1 or out[0] or not msg.startswith(prefix + ": ") or moved != (0, 0):
            failed.append((name, rc, msg, moved))
        if out[0]:
            lib.dvo_b200_pyramid_release(out[0])
            out[0] = None
    assert not failed, failed
    # the good call itself is accepted
    assert _call(lib, engine, entry, SimpleNamespace(**good), out) == 0 and out[0]
    lib.dvo_b200_pyramid_release(out[0])
    engine.synchronize()
