"""CPU tests of pyramids from distorted cameras: dvo_b200_undistort_map against its numpy restatement and OpenCV, the remap
model (tests/rectify_model.py) against cv2.remap, the entry points' answer to NULL handles, the bindings' argument lists,
tum_replay --distortion parsing, synth's distorted frames, and the accuracy gain of rectifying on the CPU oracle.  No GPU."""
import ctypes as C
import json
import os
import re
import subprocess

import numpy as np
import pytest

import rectify_model as rm
from helpers import digest, pose_delta

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FR1 = (517.3, 516.5, 318.6, 255.3)
FR1_DIST = (0.2624, -0.9531, -0.0054, 0.0026, 1.1633)
CFG = dict(first_level=4, last_level=0, max_iterations_per_level=50, precision=1e-4)


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as ge
    ge.build_cuda()
    from dvo_slam_b200 import engine
    return engine.load_library()


CASES = [(640, 480, FR1, FR1_DIST, None),
         (640, 480, FR1, FR1_DIST, (430.0, 431.5, 320.25, 240.75)),
         (321, 77, (300.0, 290.0, 150.5, 40.0), (-0.3, 0.1, 0.001, -0.002, 0.0), (280.0, 270.0, 161.0, 38.5))]


@pytest.mark.parametrize("case", range(len(CASES)))
def test_undistort_map_equals_the_restatement(lib, case):
    from dvo_slam_b200.engine import undistort_map
    w, h, K, d, Kn = CASES[case]
    mx, my = undistort_map(w, h, K, d, Kn)
    ex, ey = rm.undistort_map(w, h, K, d, Kn)
    assert mx.shape == (h, w) and np.array_equal(mx, ex) and np.array_equal(my, ey)


@pytest.mark.parametrize("case", range(len(CASES)))
def test_undistort_map_agrees_with_opencv(lib, case):
    cv2 = pytest.importorskip("cv2")
    from dvo_slam_b200.engine import undistort_map
    w, h, K, d, Kn = CASES[case]
    mx, my = undistort_map(w, h, K, d, Kn)
    M = lambda k: np.array([[k[0], 0, k[2]], [0, k[1], k[3]], [0, 0, 1]])
    cx, cy = cv2.initUndistortRectifyMap(M(K), np.array(d), None, M(Kn or K), (w, h), cv2.CV_32FC1)
    assert np.abs(cx - mx).max() <= 1e-3 and np.abs(cy - my).max() <= 1e-3


def test_fr1_map_displacement(lib):
    """the figures DESIGN.md quotes: fr1 moves pixels up to ~37 px, and ~6 % of the rectified pixels have no source"""
    from dvo_slam_b200.engine import undistort_map
    mx, my = undistort_map(640, 480, FR1, FR1_DIST)
    u, v = np.meshgrid(np.arange(640), np.arange(480))
    disp = np.hypot(mx - u, my - v)
    assert 36 < disp.max() < 38
    outside = (mx < 0) | (mx > 639) | (my < 0) | (my > 479)
    assert 0.05 < outside.mean() < 0.07


def test_zero_distortion_gives_integer_coordinates(lib):
    from dvo_slam_b200.engine import undistort_map
    for w, h, K in ((640, 480, FR1), (1280, 960, tuple(2 * v for v in FR1)), (321, 77, (300.0, 290.0, 150.5, 40.0))):
        mx, my = undistort_map(w, h, K, (0, 0, 0, 0, 0))
        assert np.array_equal(mx, np.broadcast_to(np.arange(w, dtype=np.float32), (h, w)))
        assert np.array_equal(my, np.broadcast_to(np.arange(h, dtype=np.float32)[:, None], (h, w)))


def test_undistort_map_rejects_bad_arguments(lib):
    d = (C.c_double * 5)(*FR1_DIST)
    K = (C.c_double * 4)(*FR1)
    m = (C.c_float * 16)()
    assert lib.dvo_b200_undistort_map(4, 4, K, d, K, m, m) == 0
    assert lib.dvo_b200_undistort_map(0, 4, K, d, K, m, m) == -1
    assert lib.dvo_b200_undistort_map(4, 4, None, d, K, m, m) == -1
    assert lib.dvo_b200_undistort_map(4, 4, K, d, K, None, m) == -1
    bad = (C.c_double * 5)(*FR1_DIST[:4], float("nan"))
    assert lib.dvo_b200_undistort_map(4, 4, K, bad, K, m, m) == -1


def _smooth_image(h, w, seed):
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    img = np.zeros((h, w))
    for _ in range(10):
        kx, ky = rng.uniform(-0.3, 0.3, 2)
        img += rng.uniform(5, 20) * np.sin(kx * xx + ky * yy + rng.uniform(0, 6.3))
    return (128 + img).astype(np.float32)


def test_remap_model_agrees_with_opencv(lib):
    """cv2.remap (INTER_LINEAR, float32 maps) rounds coordinates to 1/32 px: on maps already on that grid the model and
    OpenCV agree to float32 rounding, which also pins the pixel-centre convention (integer coordinates are pixel centres);
    on arbitrary maps they differ by at most what a 1/64 px shift per axis explains"""
    cv2 = pytest.importorskip("cv2")
    h, w = 60, 80
    img = _smooth_image(h, w, 1)
    depth = np.ones((h, w), np.float32)
    rng = np.random.default_rng(2)
    mx = rng.uniform(0, w - 1, (50, 70)).astype(np.float32)
    my = rng.uniform(0, h - 1, (50, 70)).astype(np.float32)
    qx, qy = (np.round(mx * 32) / 32).astype(np.float32), (np.round(my * 32) / 32).astype(np.float32)
    model_q = rm.remap(img, depth, qx, qy)[0]
    cv_q = cv2.remap(img, qx, qy, cv2.INTER_LINEAR, borderMode=cv2.BORDER_REPLICATE)
    assert np.abs(model_q - cv_q).max() <= 1e-3
    gx, gy = np.abs(np.diff(img, axis=1)).max(), np.abs(np.diff(img, axis=0)).max()
    model = rm.remap(img, depth, mx, my)[0]
    cv_full = cv2.remap(img, mx, my, cv2.INTER_LINEAR, borderMode=cv2.BORDER_REPLICATE)
    assert np.abs(model - cv_full).max() <= (gx + gy) / 64 + 1e-3
    # pixel centres: integer coordinates read the pixel itself, half-way reads the mean of two
    ix = np.broadcast_to(np.arange(w, dtype=np.float32), (h, w))
    iy = np.broadcast_to(np.arange(h, dtype=np.float32)[:, None], (h, w))
    assert np.array_equal(rm.remap(img, depth, ix, iy)[0], img)
    half = rm.remap(img, depth, (ix[:, :-1] + 0.5).astype(np.float32), iy[:, :-1])[0]
    assert np.allclose(half, (img[:, :-1] + img[:, 1:]) / 2, rtol=0, atol=1e-4)


def test_remap_model_rules():
    """invalid outside [0, w-1] x [0, h-1] (NaN / NaN, unusable), nearest-tap depth, raw depth 0 -> NaN, the four-tap mask"""
    img = np.arange(20, dtype=np.float32).reshape(4, 5)
    raw = (np.arange(20, dtype=np.uint16).reshape(4, 5) + 1) * 100
    raw[2, 3] = 0
    mask = np.ones((4, 5), np.uint8)
    mask[0, 0] = 0
    mx = np.array([[-0.01, 0.0, 4.0, 4.01, 2.49, 2.5, 3.2, float("nan"), 0.5]], np.float32)
    my = np.array([[1.0, 0.0, 3.0, 1.0, 1.51, 1.49, 2.0, 1.0, 0.5]], np.float32)
    I, Z, M = rm.remap(img, raw, mx, my, mask, 0.001)
    assert np.isnan(I[0, [0, 3, 7]]).all() and np.isnan(Z[0, [0, 3, 7]]).all() and not M[0, [0, 3, 7]].any()
    assert I[0, 1] == 0 and I[0, 2] == 19 and Z[0, 2] == np.float32(2000) * np.float32(0.001)
    assert Z[0, 4] == np.float32(raw[2, 2]) * np.float32(0.001) and Z[0, 5] == np.float32(raw[1, 3]) * np.float32(0.001)
    assert np.isnan(Z[0, 6])              # nearest tap (3, 2) holds raw depth 0
    assert M[0, 1] == 0 and M[0, 8] == 0 and M[0, 2] == 1 and M[0, 4] == 1


def test_null_handles_are_invalid_arguments(lib):
    from dvo_slam_b200.engine import DevicePlane
    m = (C.c_float * 16)()
    K = (C.c_float * 4)(*FR1)
    out = C.c_void_p()
    assert lib.dvo_b200_rectifier_create(None, 4, 4, 4, 4, m, m, K, C.byref(out)) == -1 and not out.value
    assert lib.dvo_b200_rectifier_release(None) == -1
    outs = (C.c_void_p * 1)()
    img = np.zeros((48, 64), np.float32)
    assert lib.dvo_b200_pyramid_create_rectified_batch(None, None, 1, 0, img.ctypes.data, img.ctypes.data, 0.0, None, 1, 64, 48, 3,
                                                       outs) == -1
    p = DevicePlane(1 << 20, 256, 256 * 48)
    assert lib.dvo_b200_pyramid_create_rectified_device_batch(None, None, 1, 0, C.byref(p), C.byref(p), 0.0, None, 1, 64, 48, 3,
                                                              outs) == -1
    assert not outs[0]


def test_bindings_match_the_header(lib):
    """every new entry point's ctypes argument list has the header's length"""
    header = open(os.path.join(ROOT, "include", "dvo_b200.h")).read()
    for name in ("dvo_b200_undistort_map", "dvo_b200_rectifier_create", "dvo_b200_rectifier_release",
                 "dvo_b200_pyramid_create_rectified_batch", "dvo_b200_pyramid_create_rectified_device_batch"):
        decl = re.search(r"int " + name + r"\(([^;]*)\);", header).group(1)
        decl = re.sub(r"/\*.*?\*/", "", decl, flags=re.S)
        assert len(getattr(lib, name).argtypes) == len(decl.split(",")), name


def test_tum_replay_parses_distortion(tmp_path):
    import __graft_entry__ as ge
    from test_tum_replay import HOST, write_sequence
    ge.build_cuda()
    ge.build_host()
    rng = np.random.default_rng(3)
    h, w = 48, 64
    rgb = [rng.integers(0, 256, size=(h, w, 3), dtype=np.uint8) for _ in range(2)]
    depth = [rng.integers(1, 40000, size=(h, w), dtype=np.uint16) for _ in range(2)]
    assoc = write_sequence(str(tmp_path), rgb, depth, [10.0, 10.03])
    exe = os.path.join(HOST, "tum_replay")
    r = subprocess.run([exe, "--assoc", assoc, "--parse-only", "--distortion", "0.2624", "-0.9531", "-0.0054", "0.0026", "1.1633"],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    assert np.allclose(json.loads(r.stdout)["distortion"], FR1_DIST)
    assert "distortion" not in json.loads(subprocess.run([exe, "--assoc", assoc, "--parse-only"], capture_output=True, text=True).stdout)
    for bad in (["0.1", "0.2", "0", "0"], ["0.1", "0.2", "0", "0", "x"], ["0.1", "0.2", "0", "0", "0", "7"]):
        r = subprocess.run([exe, "--assoc", assoc, "--parse-only", "--distortion"] + bad, capture_output=True, text=True)
        assert r.returncode == 2, bad


def test_synth_default_frames_are_unchanged():
    """the digests of the frames before SceneConfig.distortion existed"""
    from dvo_slam_b200 import synth
    want = {3: ("b524827ca294e0d9ccf96fd16b4a1ca59907505abdbf0772671091024f47271e", "eee1c1e80b1799319736e27eb4dd8fb54351b17072fe3dccac04b46d77668329",
                "441a365f48768e7d92a03d5b191eb36ad33ffe2b9310fa614d4baa57fad37f38", "7ea085d68b09d992e69af8a19791473000fcbd10ea9d49a41491bd782d87fdf3"),
            4: ("747cc850bd64b1d9c3acc9cb5c07563fd0a83ae5e365eab84dd2efc267578141", "84d1f768c128de97712e03057e89768ccfc9bb326ee7dc49893dbb3b433a1085",
                "0c918d9be04b57158f0dd93f25d2a4e7c103e5af559e414179aae871f11a378e", "b82b587fae58751994cb7707159e0b7b04887d55f4083f90c23602a9e3895b7c")}
    for seed, cfg in ((3, synth.SceneConfig()), (4, synth.SceneConfig().scaled(2))):
        p = synth.make_pair(seed, cfg)
        assert tuple(digest(p[k].numpy()) for k in ("I_ref", "Z_ref", "I_cur", "Z_cur")) == want[seed], seed


def test_synth_distorted_rays():
    """distorting the undistorted points gives back the pixel grid, and scaled() keeps the lens"""
    import torch
    from dvo_slam_b200 import synth
    cfg = synth.SceneConfig(distortion=FR1_DIST)
    assert cfg.scaled(2).distortion == FR1_DIST
    fx, fy, ox, oy = cfg.intrinsics
    xd = ((torch.arange(640, dtype=torch.float64) - ox) / fx)[None, :].expand(480, 640).contiguous()
    yd = ((torch.arange(480, dtype=torch.float64) - oy) / fy)[:, None].expand(480, 640).contiguous()
    x, y = synth.undistort_points(xd, yd, FR1_DIST)
    k1, k2, p1, p2, k3 = FR1_DIST
    r2 = x * x + y * y
    R = 1 + k1 * r2 + k2 * r2 ** 2 + k3 * r2 ** 3
    assert float((x * R + 2 * p1 * x * y + p2 * (r2 + 2 * x * x) - xd).abs().max()) < 1e-12
    assert float((y * R + p1 * (r2 + 2 * y * y) + 2 * p2 * x * y - yd).abs().max()) < 1e-12
    p, q = synth.make_pair(5, cfg), synth.make_pair(5)
    assert not torch.equal(p["I_ref"], q["I_ref"]) and np.allclose(p["T_true"], q["T_true"])


def distortion_errors(oracle, modes=("faithful", "mirror"), seeds=range(16)):
    """per mode and arm, the (translation, rotation) pose errors against the truth: "pinhole" aligns the fr1-distorted
    frames as if they were pinhole, "rectified" aligns them after the model remap (K_new = K, under the engine's rule for
    NaN channels), "floor" aligns an undistorted render of the same scene and motion"""
    from dvo_slam_b200 import synth
    mx, my = rm.undistort_map(640, 480, FR1, FR1_DIST)
    err = {m: {"pinhole": [], "rectified": [], "floor": []} for m in modes}
    for seed in seeds:
        d = synth.make_pair(seed, synth.SceneConfig(distortion=FR1_DIST))
        f = synth.make_pair(seed)
        truth = np.linalg.inv(d["T_true"])
        a = [d[k].numpy() for k in ("I_ref", "Z_ref", "I_cur", "Z_cur")]
        r0, r1 = rm.remap(a[0], a[1], mx, my), rm.remap(a[2], a[3], mx, my)
        arms = {"pinhole": (oracle.Pyramid(a[0], a[1], FR1, 5), oracle.Pyramid(a[2], a[3], FR1, 5)),
                "rectified": (rm.oracle_pyramid(oracle, r0[0], r0[1], FR1, 5), rm.oracle_pyramid(oracle, r1[0], r1[1], FR1, 5)),
                "floor": tuple(oracle.Pyramid(f[i].numpy(), f[z].numpy(), FR1, 5) for i, z in (("I_ref", "Z_ref"), ("I_cur", "Z_cur")))}
        for name, (ref, cur) in arms.items():
            for m in modes:
                err[m][name].append(pose_delta(truth, oracle.match(ref, cur, oracle.config(**CFG), oracle.mode(m))["T"]))
    return {m: {k: np.array(v) for k, v in e.items()} for m, e in err.items()}


def test_rectifying_brings_the_pose_closer(oracle):
    """DESIGN.md section 4.6: rectifying cuts the median translation error about two- to fivefold and the median rotation
    error about fivefold at the benchmark's motion; the worst case is of the order of the method's own accuracy on both
    inputs, so only the medians and the rotation p90 are asserted"""
    err = distortion_errors(oracle)
    for m, e in err.items():
        pin, rect = e["pinhole"], e["rectified"]
        assert np.median(rect[:, 0]) <= 0.6 * np.median(pin[:, 0]), (m, np.median(rect[:, 0]), np.median(pin[:, 0]))
        assert np.median(rect[:, 1]) <= 0.3 * np.median(pin[:, 1]), (m, np.median(rect[:, 1]), np.median(pin[:, 1]))
        assert np.percentile(rect[:, 1], 90) < np.percentile(pin[:, 1], 90), m
        assert rect[:, 0].max() < 5e-3 and rect[:, 1].max() < 2e-3, m          # no divergence
