"""CPU tests of pyramids from unregistered depth: dvo_b200_depth_rays against its numpy restatement and OpenCV, the
registration model (tests/registration_model.py) against an independent float64 reprojection, the entry points' answer to
NULL handles, the bindings' argument lists, synth's depth camera, and the accuracy gain of registering on the CPU oracle.
No GPU."""
import ctypes as C
import os
import re

import numpy as np
import pytest

import registration_model as rg
from helpers import digest, pose_delta

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FR1 = (517.3, 516.5, 318.6, 255.3)
FR1_DIST = (0.2624, -0.9531, -0.0054, 0.0026, 1.1633)
KV2 = (365.5, 365.5, 257.0, 206.0)                       # a Kinect-v2-like 512x424 time-of-flight camera
KV2_DIST = (0.0905, -0.2688, 0.0, 0.0, 0.0938)
CFG = dict(first_level=4, last_level=0, max_iterations_per_level=50, precision=1e-4)


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as ge
    ge.build_cuda()
    from dvo_slam_b200 import engine
    return engine.load_library()


def _T(tx=0.0, ty=0.0, tz=0.0, rx=0.0, ry=0.0, rz=0.0):
    from dvo_slam_b200 import synth
    return synth.se3_exp(np.array([tx, ty, tz, rx, ry, rz]))


RAY_CASES = [((640, 480), FR1, None), ((640, 480), FR1, FR1_DIST), ((512, 424), KV2, KV2_DIST), ((33, 7), (20.0, 21.0, 16.5, 3.0), None)]


@pytest.mark.parametrize("case", range(len(RAY_CASES)))
def test_depth_rays_equal_the_restatement(lib, case):
    from dvo_slam_b200.engine import depth_rays
    size, K, dist = RAY_CASES[case]
    got, want = depth_rays(size, K, dist), rg.depth_rays(size, K, dist)
    w, h = size
    assert [a.shape for a in got] == [(h, w), (h, w), (h + 1, w + 1), (h + 1, w + 1)]
    for a, b in zip(got, want):
        assert np.array_equal(a, b)


def test_pinhole_rays_are_the_pixel_coordinates(lib):
    from dvo_slam_b200.engine import depth_rays
    cx, cy, kx, ky = depth_rays((640, 480), FR1)
    u = np.arange(640, dtype=np.float64)
    assert np.array_equal(cx[5], ((u - FR1[2]) / FR1[0]).astype(np.float32))
    assert np.array_equal(kx[0], ((np.arange(641) - 0.5 - FR1[2]) / FR1[0]).astype(np.float32))
    assert np.array_equal(ky[:, 3], ((np.arange(481) - 0.5 - FR1[3]) / FR1[1]).astype(np.float32))


@pytest.mark.parametrize("size,K,dist", [((512, 424), KV2, KV2_DIST), ((640, 480), FR1, FR1_DIST)])
def test_depth_rays_agree_with_opencv(lib, size, K, dist):
    cv2 = pytest.importorskip("cv2")
    from dvo_slam_b200.engine import depth_rays
    cx, cy, kx, ky = depth_rays(size, K, dist)
    w, h = size
    M = np.array([[K[0], 0, K[2]], [0, K[1], K[3]], [0, 0, 1]])
    crit = (cv2.TERM_CRITERIA_COUNT | cv2.TERM_CRITERIA_EPS, 100, 1e-14)
    for (xs, ys), (rx, ry) in (((np.arange(w), np.arange(h)), (cx, cy)), ((np.arange(w + 1) - 0.5, np.arange(h + 1) - 0.5), (kx, ky))):
        uu, vv = np.meshgrid(xs.astype(np.float64), ys.astype(np.float64))
        pts = np.stack([uu.ravel(), vv.ravel()], -1)[:, None, :]
        und = cv2.undistortPointsIter(pts, M, np.array(dist), None, None, crit).reshape(uu.shape + (2,))
        assert np.abs(und[..., 0] - rx).max() <= 1e-6 and np.abs(und[..., 1] - ry).max() <= 1e-6


def test_depth_rays_reject_bad_arguments(lib):
    K = (C.c_double * 4)(*FR1)
    d = (C.c_double * 5)(*FR1_DIST)
    t = (C.c_float * 64)()
    assert lib.dvo_b200_depth_rays(4, 4, K, d, t, t, t, t) == 0
    assert lib.dvo_b200_depth_rays(4, 4, K, None, t, t, t, t) == 0
    assert lib.dvo_b200_depth_rays(1, 4, K, None, t, t, t, t) == -1
    assert lib.dvo_b200_depth_rays(4, 4, None, None, t, t, t, t) == -1
    assert lib.dvo_b200_depth_rays(4, 4, K, None, t, None, t, t) == -1
    assert lib.dvo_b200_depth_rays(4, 4, (C.c_double * 4)(float("nan"), 1, 1, 1), None, t, t, t, t) == -1
    assert lib.dvo_b200_depth_rays(4, 4, (C.c_double * 4)(-5.0, 5, 1, 1), None, t, t, t, t) == -1
    assert lib.dvo_b200_depth_rays(4, 4, K, (C.c_double * 5)(0.1, float("inf"), 0, 0, 0), t, t, t, t) == -1
    # a lens model that folds over: far corners have no preimage the iteration reaches
    assert lib.dvo_b200_depth_rays(4, 4, (C.c_double * 4)(1.0, 1.0, 0.0, 0.0), (C.c_double * 5)(-5.0, 0, 0, 0, 0), t, t, t, t) == -1


def _reproject64(depth, size_d, K_d, T, size, K):
    """float64 forward projection of every valid depth pixel: (Zc, x-extent, y-extent) of the pinhole depth camera"""
    dw, dh = size_d
    u, v = np.meshgrid(np.arange(dw, dtype=np.float64), np.arange(dh, dtype=np.float64))
    d = depth.astype(np.float64)

    def proj(uu, vv):
        P = np.stack([(uu - K_d[2]) / K_d[0] * d, (vv - K_d[3]) / K_d[1] * d, d], -1) @ T[:3, :3].T + T[:3, 3]
        return K[0] * P[..., 0] / P[..., 2] + K[2], K[1] * P[..., 1] / P[..., 2] + K[3], P[..., 2]

    zc = proj(u, v)[2]
    corners = [proj(u + a, v + b) for a in (-0.5, 0.5) for b in (-0.5, 0.5)]
    xs, ys = np.stack([c[0] for c in corners]), np.stack([c[1] for c in corners])
    return zc, (xs.min(0), xs.max(0)), (ys.min(0), ys.max(0))


@pytest.mark.parametrize("case", ["baseline", "low-res", "high-res", "rotated"])
def test_model_against_float64_reprojection(lib, case):
    """Every finite registered depth is the float64 Zc of a depth pixel whose footprint covers the colour pixel (to float
    rounding), and no depth pixel whose footprint surely covers it is nearer by more than rounding"""
    from dvo_slam_b200 import synth
    sizes = {"baseline": ((640, 480), FR1), "low-res": ((320, 240), tuple(v / 2 for v in FR1)),
             "high-res": ((1280, 960), tuple(v * 2 for v in FR1)), "rotated": ((640, 480), FR1)}
    size_d, K_d = sizes[case]
    T = _T(0.025, 0.004, -0.01, 0.01, -0.02, 0.005) if case == "rotated" else _T(0.025)
    cfg = synth.SceneConfig(depth_camera=synth.DepthCamera(*size_d, K_d, T))
    depth = synth.make_pair(4, cfg)["Z_ref"].numpy()
    Z = rg.register(depth, rg.depth_rays(size_d, K_d), T, (640, 480), FR1)
    zc, (x0, x1), (y0, y1) = _reproject64(depth, size_d, K_d, T, (640, 480), FR1)
    ok = np.isfinite(depth) & (depth > 0)
    x0, y0 = np.where(ok, x0, 0), np.where(ok, y0, 0)
    eps, rel = 1e-3, 2e-6
    lo = np.full((480, 640), np.inf)       # nearest candidate whose footprint surely covers the pixel
    found = np.zeros((480, 640), bool)     # the output is some loosely covering candidate's depth
    for oy in range(rg.MAX_FOOTPRINT + 1):
        for ox in range(rg.MAX_FOOTPRINT + 1):
            xx, yy = np.ceil(x0 - eps).astype(np.int64) + ox, np.ceil(y0 - eps).astype(np.int64) + oy
            inside = ok & (xx >= 0) & (xx < 640) & (yy >= 0) & (yy < 480) & (x1 - x0 < rg.MAX_FOOTPRINT - 0.01) & (y1 - y0 < rg.MAX_FOOTPRINT - 0.01)
            loose = inside & (xx < x1 + eps) & (yy < y1 + eps)
            tight = inside & (xx >= x0 + eps) & (xx < x1 - eps) & (yy >= y0 + eps) & (yy < y1 - eps)
            np.minimum.at(lo, (yy[tight], xx[tight]), zc[tight])
            zo = Z[yy[loose], xx[loose]]
            hit = np.abs(zo - zc[loose]) <= rel * zc[loose]
            found[yy[loose][hit], xx[loose][hit]] = True
    fin = np.isfinite(Z)
    assert fin.mean() > 0.8
    assert found[fin].all()
    assert (Z[fin] <= lo[fin] * (1 + rel)).all()
    assert not np.isfinite(lo[~fin]).any()         # every surely covered pixel holds a depth
    if case == "low-res":                           # footprints above a pixel
        assert ((x1 - x0)[ok] > 1).all()
    if case == "high-res":                          # footprints below a pixel: many land on no pixel centre
        assert ((x1 - x0)[ok] < 1).all()


def test_identity_registration_returns_the_input_depth(lib):
    from dvo_slam_b200 import synth
    for seed in (3, 5):
        p = synth.make_pair(seed)
        for fmt in ("float", "raw"):
            z = p["Z_cur"].numpy()
            d = z if fmt == "float" else np.where(np.isnan(z), 0, np.round(z * 5000)).astype(np.uint16)
            Z = rg.register(d, rg.depth_rays((640, 480), FR1), np.eye(4), (640, 480), FR1, depth_scale=1 / 5000)
            assert np.array_equal(Z, rg.depth_metres(d, 1 / 5000), equal_nan=True)


def test_model_rules():
    """the z-test keeps the nearest, invalid depth and points behind the colour camera are skipped, an oversized
    footprint is skipped"""
    K = (10.0, 10.0, 4.0, 4.0)
    rays = rg.depth_rays((8, 8), K)
    d = np.full((8, 8), 2.0, np.float32)
    d[3, 3] = 1.0
    d[0, 0] = np.nan
    d[0, 1] = 0.0
    d[0, 2] = -1.0
    Z = rg.register(d, rays, np.eye(4), (8, 8), K)
    assert Z[3, 3] == 1.0 and np.isnan(Z[0, :3]).all() and Z[5, 5] == 2.0
    T = _T(-0.2)      # 20 cm to the side: the far surface moves 1 px, the near pixel 2 px and leaves a shadow behind it
    Z = rg.register(d, rays, T, (8, 8), K)
    assert Z[3, 1] == 1.0 and np.isnan(Z[3, 2]) and Z[3, 3] == 2.0 and np.isnan(Z[:, 7]).all()
    near = np.full((8, 8), 0.01, np.float32)        # a 1 cm surface: footprints of 10 px > DVO_B200_REGISTRATION_MAX_FOOTPRINT
    assert np.isnan(rg.register(near, rays, T, (8, 8), K)).all()


def test_null_handles_are_invalid_arguments(lib):
    from dvo_slam_b200.engine import DevicePlane
    t = (C.c_float * 64)()
    T = (C.c_double * 16)(*np.eye(4).ravel())
    K = (C.c_float * 4)(*FR1)
    out = C.c_void_p()
    assert lib.dvo_b200_depth_registration_create(None, 4, 4, t, t, t, t, T, 4, 4, K, C.byref(out)) == -1 and not out.value
    assert lib.dvo_b200_depth_registration_release(None) == -1
    outs = (C.c_void_p * 1)()
    img = np.zeros((48, 64), np.float32)
    assert lib.dvo_b200_pyramid_create_registered_batch(None, None, None, 1, 0, img.ctypes.data, img.ctypes.data, 0.0, None, 1, 64, 48,
                                                        3, outs) == -1
    p = DevicePlane(1 << 20, 256, 256 * 48)
    assert lib.dvo_b200_pyramid_create_registered_device_batch(None, None, None, 1, 0, C.byref(p), C.byref(p), 0.0, None, 1, 64, 48, 3,
                                                               outs) == -1
    assert not outs[0]


def test_bindings_match_the_header(lib):
    """every new entry point's ctypes argument list has the header's length"""
    header = open(os.path.join(ROOT, "include", "dvo_b200.h")).read()
    for name in ("dvo_b200_depth_rays", "dvo_b200_depth_registration_create", "dvo_b200_depth_registration_release",
                 "dvo_b200_pyramid_create_registered_batch", "dvo_b200_pyramid_create_registered_device_batch"):
        decl = re.search(r"int " + name + r"\(([^;]*)\);", header).group(1)
        decl = re.sub(r"/\*.*?\*/", "", decl, flags=re.S)
        assert len(getattr(lib, name).argtypes) == len(decl.split(",")), name


def test_synth_default_frames_are_unchanged():
    """the digests of the frames before SceneConfig.depth_camera existed"""
    from dvo_slam_b200 import synth
    want = {3: ("b524827ca294e0d9ccf96fd16b4a1ca59907505abdbf0772671091024f47271e", "eee1c1e80b1799319736e27eb4dd8fb54351b17072fe3dccac04b46d77668329",
                "441a365f48768e7d92a03d5b191eb36ad33ffe2b9310fa614d4baa57fad37f38", "7ea085d68b09d992e69af8a19791473000fcbd10ea9d49a41491bd782d87fdf3"),
            4: ("747cc850bd64b1d9c3acc9cb5c07563fd0a83ae5e365eab84dd2efc267578141", "84d1f768c128de97712e03057e89768ccfc9bb326ee7dc49893dbb3b433a1085",
                "0c918d9be04b57158f0dd93f25d2a4e7c103e5af559e414179aae871f11a378e", "b82b587fae58751994cb7707159e0b7b04887d55f4083f90c23602a9e3895b7c")}
    for seed, cfg in ((3, synth.SceneConfig()), (4, synth.SceneConfig().scaled(2))):
        p = synth.make_pair(seed, cfg)
        assert tuple(digest(p[k].numpy()) for k in ("I_ref", "Z_ref", "I_cur", "Z_cur")) == want[seed], seed


def test_synth_depth_camera():
    """intensity and the colour camera's own depth are the default frames; the depth is rendered in the depth camera's
    geometry, and a depth camera at the colour camera's place renders the colour camera's depth"""
    from dvo_slam_b200 import synth
    q = synth.make_pair(6)
    p = synth.make_pair(6, synth.SceneConfig(depth_camera=synth.DepthCamera(320, 240, tuple(v / 2 for v in FR1), synth.baseline(0.025))))
    assert p["Z_ref"].shape == (240, 320) and p["I_ref"].shape == (480, 640)
    for k in ("I_ref", "I_cur"):
        assert np.array_equal(p[k].numpy(), q[k].numpy())
    assert np.array_equal(p["Z_ref_color"].numpy(), q["Z_ref"].numpy(), equal_nan=True)
    s = synth.make_pair(6, synth.SceneConfig(depth_camera=synth.DepthCamera(640, 480, FR1, np.eye(4))))
    zs, zq = s["Z_cur"].numpy(), q["Z_cur"].numpy()
    both = np.isfinite(zs) & np.isfinite(zq)          # the hole blocks are drawn anew for the depth camera
    assert both.mean() > 0.9 and np.array_equal(zs[both], zq[both])


def registration_errors(oracle, modes=("faithful", "mirror"), seeds=range(16), baseline_m=0.025):
    """per mode and arm, the (translation, rotation) pose errors against the truth on pairs whose depth comes from a
    640x480 fr1-intrinsics depth camera baseline_m to the side of the colour camera: "unregistered" uses that depth as if
    it were registered, "registered" the model's registration of it, "color" the colour camera's own depth render"""
    from dvo_slam_b200 import synth
    T = synth.baseline(baseline_m)
    cfg = synth.SceneConfig(depth_camera=synth.DepthCamera(640, 480, FR1, T))
    rays = rg.depth_rays((640, 480), FR1)
    err = {m: {"unregistered": [], "registered": [], "color": []} for m in modes}
    for seed in seeds:
        p = synth.make_pair(seed, cfg)
        truth = np.linalg.inv(p["T_true"])
        I0, I1 = p["I_ref"].numpy(), p["I_cur"].numpy()
        depth = {"unregistered": (p["Z_ref"].numpy(), p["Z_cur"].numpy()),
                 "registered": tuple(rg.register(p[k].numpy(), rays, T, (640, 480), FR1) for k in ("Z_ref", "Z_cur")),
                 "color": (p["Z_ref_color"].numpy(), p["Z_cur_color"].numpy())}
        for name, (z0, z1) in depth.items():
            ref, cur = oracle.Pyramid(I0, z0, FR1, 5), oracle.Pyramid(I1, z1, FR1, 5)
            for m in modes:
                err[m][name].append(pose_delta(truth, oracle.match(ref, cur, oracle.config(**CFG), oracle.mode(m))["T"]))
    return {m: {k: np.array(v) for k, v in e.items()} for m, e in err.items()}


def test_registering_brings_the_pose_closer(oracle):
    """DESIGN.md section 4.7, measured: registering cuts the median translation error to 0.79x (FAITHFUL) and 0.58x
    (MIRROR) of using the depth unregistered, to the level of the colour camera's own depth, and the median rotation
    error to 0.79x / 0.66x.  The p90 and the worst case do not improve: they stay at the method's own accuracy.  The
    bounds below leave a margin around those figures."""
    err = registration_errors(oracle)
    for m, e in err.items():
        un, reg, col = e["unregistered"], e["registered"], e["color"]
        for k in (0, 1):
            assert np.median(reg[:, k]) < 0.9 * np.median(un[:, k]), (m, k, np.median(reg[:, k]), np.median(un[:, k]))
        assert np.median(reg[:, 0]) < 1.25 * np.median(col[:, 0]), m
        assert np.percentile(reg[:, 0], 90) < 3e-3 and np.percentile(reg[:, 1], 90) < 1e-3, m
        assert reg[:, 0].max() < 3.5e-3 and reg[:, 1].max() < 1.2e-3, m          # no divergence
