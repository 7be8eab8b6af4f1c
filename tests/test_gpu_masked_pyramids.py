"""Reference masks on the H100 (dvo_b200_pyramid_create_masked_batch): selections at every level and for non-default
thresholds against the oracle, residual records bit-exact against MIRROR with both estimators, the all-ones mask equal to
no mask for every input format, the current role untouched, mixed and shared batches, whole matches, the moving-object use
case, invalid arguments and the C++ adapter's setReferenceMask."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from helpers import POSE_TOL_R, POSE_TOL_T, nan_equal, pose_delta
from test_corrected_estimator import corrected_mode
from masked_oracle import masked_pyramid
from test_masked_selection import MOVING_CFG, MOVING_SEEDS

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LEVELS = 4
PP = np.array([[2000.0, -30.0], [-30.0, 9000.0]], dtype=np.float32)


@pytest.fixture(scope="module")
def corrected(engine):
    from dvo_slam_b200.engine import Engine
    eng = Engine(device=0, estimator="corrected")
    yield eng
    eng.close()


def _band_for_odd_last(oracle, I, Z, K, base):
    """base mask plus a bottom/right band (a vignetted border) of the first width 4..39 that leaves an odd level-0 selection
    whose last point is a valid constraint of the identity alignment against the unmasked frame itself"""
    cur = oracle.Pyramid(I, Z, K, 1)
    for band in range(4, 40):
        m = base.copy()
        m[-band:, :] = 0
        m[:, -band:] = 0
        ref = masked_pyramid(oracle, I, Z, K, 1, m)
        S, sel = oracle.select(ref, 0, 0.0, 0.0, None)
        last = np.flatnonzero(sel.reshape(-1))[-1]
        _, planes = oracle.residual_image(ref, cur, 0, np.eye(4), oracle.mode("exact"))
        if S % 2 == 1 and not np.isnan(planes[0].reshape(-1)[last]):
            return m
    raise AssertionError("no band width gave an odd selection with a valid last point")


@pytest.fixture(scope="module")
def scene(oracle):
    from dvo_slam_b200 import synth
    p = synth.make_pair(21)
    a = {k: p[k].numpy() for k in ("I_ref", "Z_ref", "I_cur", "Z_cur")}
    a["K"], a["xi"] = p["intrinsics"], p["xi"]
    h, w = a["I_ref"].shape
    rng = np.random.default_rng(5)
    yy, xx = np.ogrid[:h, :w]
    blobs = np.ones((h, w), np.uint8)
    for _ in range(10):
        cy, cx, r = rng.integers(0, h), rng.integers(0, w), rng.integers(5, 60)
        blobs[(yy - cy) ** 2 + (xx - cx) ** 2 <= r * r] = 0
    border = np.ones((h, w), np.uint8)
    border[:24, :] = 0
    border[:, :9] = 0
    single = np.ones((h, w), np.uint8)
    single[237, 411] = 0                  # off the subsample grid of every coarse level
    a["masks"] = {"blobs": blobs, "border": border, "single": single,
                  "odd": _band_for_odd_last(oracle, a["I_ref"], a["Z_ref"], a["K"], blobs)}
    return a


def test_selection_equals_oracle_at_every_level_and_threshold(engine, oracle, scene):
    a = scene
    parities = set()
    for name, m in a["masks"].items():
        g = engine.pyramid(a["I_ref"], a["Z_ref"], a["K"], LEVELS, mask=m)
        o = masked_pyramid(oracle, a["I_ref"], a["Z_ref"], a["K"], LEVELS, m)
        for ti, td in ((0.0, 0.0), (6.0, 0.02), (0.0, 0.0)):      # default, the k_reselect path, and back
            for l in range(LEVELS):
                S_g, sel_g = g.select(l, ti, td)
                S_o, sel_o = oracle.select(o, l, ti, td, None)
                assert S_g == S_o and np.array_equal(sel_g, sel_o), (name, l, ti, td, S_g, S_o)
                parities.add(S_o % 2)
        # a mask only removes points
        u = engine.pyramid(a["I_ref"], a["Z_ref"], a["K"], LEVELS)
        for l in range(LEVELS):
            assert not (g.select(l)[1] & ~u.select(l)[1].astype(bool)).any()
    assert parities == {0, 1}


def _check_records(eng, oracle, m, gref, gcur, oref, ocur, lvl, T):
    n_g, img_g = eng.residual_image(gref, gcur, lvl, T)
    n_o, img_o = oracle.residual_image(oref, ocur, lvl, T, m)
    assert n_g == n_o and n_g > 0 and nan_equal(img_g, img_o), (lvl, n_g, n_o)
    for uw in (False, True):
        lg = eng.linearize(gref, gcur, lvl, T, uw, PP)
        lo = oracle.linearize(oref, ocur, lvl, T, m, uw, PP)
        assert lg["n"] == lo["n"] == n_o
        assert np.allclose(lg["precision"], lo["precision"], rtol=2e-6), (lvl, uw)
        assert abs(lg["ll"] - lo["ll"]) <= 2e-6 * abs(lo["ll"]) + 0.5, (lvl, uw, lg["ll"], lo["ll"])
        assert np.allclose(lg["A"], lo["A"], rtol=0, atol=2e-6 * np.abs(lo["A"]).max())
        assert np.allclose(lg["b"], lo["b"], rtol=0, atol=2e-6 * np.abs(lo["b"]).max())
    return img_g


@pytest.mark.parametrize("name", ["blobs", "odd"])
def test_records_bit_exact_against_mirror_both_estimators(engine, corrected, oracle, scene, name):
    from dvo_slam_b200 import synth
    a, m = scene, scene["masks"][name]
    gref = engine.pyramid(a["I_ref"], a["Z_ref"], a["K"], LEVELS, mask=m)
    gcur = engine.pyramid(a["I_cur"], a["Z_cur"], a["K"], LEVELS)
    oref = masked_pyramid(oracle, a["I_ref"], a["Z_ref"], a["K"], LEVELS, m)
    ocur = oracle.Pyramid(a["I_cur"], a["Z_cur"], a["K"], LEVELS)
    T = np.linalg.inv(synth.se3_exp(a["xi"] * 0.7))
    for lvl in range(LEVELS):
        _check_records(engine, oracle, oracle.mode("mirror"), gref, gcur, oref, ocur, lvl, T)
        _check_records(corrected, oracle, corrected_mode(oracle), gref, gcur, oref, ocur, lvl, T)
    if name == "odd":
        # identity alignment against the unmasked frame itself: the odd last point of the MASKED selection is dropped by the
        # reference estimator and is a constraint of the corrected one
        gself = engine.pyramid(a["I_ref"], a["Z_ref"], a["K"], LEVELS)
        oself = oracle.Pyramid(a["I_ref"], a["Z_ref"], a["K"], LEVELS)
        S, sel = gref.select(0)
        assert S % 2 == 1
        last = np.flatnonzero(sel.reshape(-1))[-1]
        img_r = _check_records(engine, oracle, oracle.mode("mirror"), gref, gself, oref, oself, 0, np.eye(4))
        img_c = _check_records(corrected, oracle, corrected_mode(oracle), gref, gself, oref, oself, 0, np.eye(4))
        assert np.isnan(img_r[0].reshape(-1)[last]) and not np.isnan(img_c[0].reshape(-1)[last])


def _raw_inputs(a):
    grey = np.ascontiguousarray(a["I_ref"], dtype=np.uint8)[None]
    depth = np.ascontiguousarray(np.where(np.isnan(a["Z_ref"]), 0, np.round(a["Z_ref"] * 5000.0)), dtype=np.uint16)[None]
    bgr = np.ascontiguousarray(np.random.default_rng(2).integers(0, 256, grey.shape + (3,), dtype=np.uint8))
    return grey, depth, bgr


def _same_result(r0, r1):
    return (np.array_equal(r0.transformation, r1.transformation) and np.array_equal(r0.information, r1.information, equal_nan=True)
            and (r0.log_likelihood == r1.log_likelihood or (np.isnan(r0.log_likelihood) and np.isnan(r1.log_likelihood)))
            and len(r0.levels) == len(r1.levels)
            and all(a.keys() == b.keys() and all(a[k] == b[k] or (a[k] != a[k] and b[k] != b[k]) for k in a) for a, b in zip(r0.levels, r1.levels)))


def _dump_equal(p, q):
    for l in range(LEVELS):
        assert np.array_equal(p.download(l), q.download(l), equal_nan=True), l
        S0, m0 = p.select(l)
        S1, m1 = q.select(l)
        assert S0 == S1 and np.array_equal(m0, m1), l


def test_all_ones_mask_equals_no_mask_for_every_input_format(engine, scene):
    from dvo_slam_b200.engine import Config
    a = scene
    K = a["K"]
    h, w = a["I_ref"].shape
    ones = np.full((1, h, w), 7, np.uint8)
    grey, depth, bgr = _raw_inputs(a)
    cur = engine.pyramid(a["I_cur"], a["Z_cur"], K, LEVELS)
    cfg = Config(first_level=3, last_level=0, max_iterations_per_level=50, precision=1e-4)
    pairs = {"float32": (engine.pyramid(a["I_ref"], a["Z_ref"], K, LEVELS), engine.pyramid(a["I_ref"], a["Z_ref"], K, LEVELS, mask=ones[0]))}
    g_ptrs = (grey.ctypes.data, depth.ctypes.data, 1, h, w)
    c_ptrs = (bgr.ctypes.data, depth.ctypes.data, 1, h, w)
    pairs["grey8_depth16"] = (engine.pyramid_raw_batch(g_ptrs, 1 / 5000.0, K, LEVELS)[0],
                              engine.pyramid_raw_batch(g_ptrs, 1 / 5000.0, K, LEVELS, masks=ones)[0])
    pairs["bgr8_depth16"] = (engine.pyramid_bgr_batch(c_ptrs, 1 / 5000.0, K, LEVELS)[0],
                             engine.pyramid_bgr_batch(c_ptrs, 1 / 5000.0, K, LEVELS, masks=ones)[0])
    engine.synchronize()
    for fmt, (p, q) in pairs.items():
        _dump_equal(p, q)
        r = engine.match_batch([p, q], [cur, cur], cfg)
        assert _same_result(r[0], r[1]), fmt
    # the H2D bytes of a masked build: one byte per pixel more
    b0 = engine.h2d_bytes()
    engine.pyramid_raw_batch(g_ptrs, 1 / 5000.0, K, LEVELS, masks=ones)
    engine.synchronize()
    assert engine.h2d_bytes() - b0 == 4 * h * w


def test_mask_does_not_touch_the_current_role(engine, scene):
    from dvo_slam_b200.engine import Config
    a = scene
    ref = engine.pyramid(a["I_ref"], a["Z_ref"], a["K"], LEVELS)
    cur = engine.pyramid(a["I_cur"], a["Z_cur"], a["K"], LEVELS)
    cur_m = engine.pyramid(a["I_cur"], a["Z_cur"], a["K"], LEVELS, mask=a["masks"]["blobs"])
    for l in range(LEVELS):
        assert np.array_equal(cur.download(l), cur_m.download(l), equal_nan=True)
    cfg = Config(first_level=3, last_level=0, max_iterations_per_level=50, precision=1e-4)
    r = engine.match_batch([ref, ref], [cur, cur_m], cfg)
    assert _same_result(r[0], r[1])
    T = np.eye(4)
    T[:3, 3] = (0.01, 0.0, -0.01)
    n0, i0 = engine.residual_image(ref, cur, 1, T)
    n1, i1 = engine.residual_image(ref, cur_m, 1, T)
    assert n0 == n1 and nan_equal(i0, i1)


def test_mixed_batches_and_shared_masked_pyramids(engine, corrected, scene):
    from dvo_slam_b200 import synth
    from dvo_slam_b200.engine import Config
    a = scene
    K = a["K"]
    refs, curs = [], []
    for k, name in enumerate((None, "blobs", None, "border", "odd", "single")):
        p = synth.make_pair(40 + k)
        refs.append(engine.pyramid(p["I_ref"].numpy(), p["Z_ref"].numpy(), K, LEVELS, mask=None if name is None else a["masks"][name]))
        curs.append(engine.pyramid(p["I_cur"].numpy(), p["Z_cur"].numpy(), K, LEVELS))
    cfg = Config(first_level=3, last_level=0, max_iterations_per_level=50, precision=1e-4)
    batch = engine.match_batch(refs, curs, cfg)
    rev = engine.match_batch(refs[::-1], curs[::-1], cfg)[::-1]
    for i in range(len(refs)):
        single = engine.match(refs[i], curs[i], cfg)
        assert _same_result(batch[i], single) and _same_result(rev[i], single), i
    # one masked pyramid, two contexts, two estimators, interleaved: each equals its context's answer on its own pyramid
    own_c = corrected.pyramid(a["I_ref"], a["Z_ref"], K, LEVELS, mask=a["masks"]["odd"])
    shared = engine.pyramid(a["I_ref"], a["Z_ref"], K, LEVELS, mask=a["masks"]["odd"])
    cur = engine.pyramid(a["I_cur"], a["Z_cur"], K, LEVELS)
    cur_c = corrected.pyramid(a["I_cur"], a["Z_cur"], K, LEVELS)
    r_ref = engine.match(shared, cur, cfg)
    r_cor = corrected.match(shared, cur, cfg)
    assert _same_result(corrected.match(own_c, cur_c, cfg), r_cor)
    assert _same_result(engine.match(shared, cur, cfg), r_ref)
    assert not np.array_equal(r_ref.transformation, r_cor.transformation)


@pytest.mark.parametrize("name", ["blobs", "border", "odd"])
def test_match_within_tolerance_of_faithful(engine, oracle, scene, name):
    from dvo_slam_b200.engine import Config
    a, m = scene, scene["masks"][name]
    g = engine.match(engine.pyramid(a["I_ref"], a["Z_ref"], a["K"], 5, mask=m), engine.pyramid(a["I_cur"], a["Z_cur"], a["K"], 5),
                     Config(first_level=4, last_level=0, max_iterations_per_level=50, precision=1e-4))
    o = oracle.match(masked_pyramid(oracle, a["I_ref"], a["Z_ref"], a["K"], 5, m), oracle.Pyramid(a["I_cur"], a["Z_cur"], a["K"], 5),
                     oracle.config(first_level=4, last_level=0, max_iterations_per_level=50, precision=1e-4), oracle.mode("faithful"))
    dt, dr = pose_delta(o["T"], g.transformation)
    assert dt < POSE_TOL_T and dr < POSE_TOL_R, (dt, dr)
    assert [l["valid_pixels"] for l in g.levels] == [l["valid_pixels"] for l in o["levels"]]


@pytest.mark.parametrize("seed", MOVING_SEEDS)
def test_masking_a_moving_object(engine, oracle, seed):
    """The GPU's masked alignment is at least as close to the truth as oracle MIRROR's masked one, within 1e-3 m / 5e-4 rad
    (half the stated GPU-vs-reference tolerance; the CPU measurement in test_masked_selection.py shows masking gains
    1.5e-2 .. 3e-2 m on these seeds), and at least 5x closer than the GPU's unmasked alignment."""
    from dvo_slam_b200 import synth
    from dvo_slam_b200.engine import Config
    p = synth.make_moving_object_pair(seed)
    K = p["intrinsics"]
    truth = np.linalg.inv(p["T_true"])
    cur = engine.pyramid(p["I_cur"], p["Z_cur"], K, 5)
    cfg = Config(**MOVING_CFG)
    g_un = pose_delta(truth, engine.match(engine.pyramid(p["I_ref"], p["Z_ref"], K, 5), cur, cfg).transformation)
    g_m = pose_delta(truth, engine.match(engine.pyramid(p["I_ref"], p["Z_ref"], K, 5, mask=p["mask"]), cur, cfg).transformation)
    o_m = pose_delta(truth, oracle.match(masked_pyramid(oracle, p["I_ref"], p["Z_ref"], K, 5, p["mask"]), oracle.Pyramid(p["I_cur"], p["Z_cur"], K, 5),
                                         oracle.config(**MOVING_CFG), oracle.mode("mirror"))["T"])
    print("moving object seed %d: GPU unmasked %.2e m / %.2e rad, masked %.2e / %.2e; MIRROR masked %.2e / %.2e" % (seed, *g_un, *g_m, *o_m))
    assert g_m[0] <= o_m[0] + 1e-3 and g_m[1] <= o_m[1] + 5e-4
    assert g_m[0] * 5 < g_un[0] and g_m[1] * 5 < g_un[1]


def test_invalid_arguments_create_nothing(engine, scene):
    from dvo_slam_b200.engine import load_library
    lib = load_library()
    a = scene
    h, w = a["I_ref"].shape
    I = np.ascontiguousarray(a["I_ref"])
    Z = np.ascontiguousarray(a["Z_ref"])
    m = np.ones((h, w), np.uint8)
    for fmt, pI, pZ in ((3, I.ctypes.data, Z.ctypes.data), (-1, I.ctypes.data, Z.ctypes.data), (0, None, Z.ctypes.data),
                        (0, I.ctypes.data, None), (1, None, None)):
        out = (C.c_void_p * 1)()
        rc = lib.dvo_b200_pyramid_create_masked_batch(engine.ctx, 1, fmt, pI, pZ, 0.0, m.ctypes.data, w, h, *a["K"], LEVELS, out)
        assert rc == -1 and not out[0], (fmt, rc)
        if fmt in (3, -1):
            assert "unknown input format" in lib.dvo_b200_last_error(engine.ctx).decode()


ADAPTER_DRIVER = r"""
#include <cstdio>
#include <cstdlib>
#include <fstream>
#include "dvo/dense_tracking.h"
static cv::Mat plane(std::ifstream& f, int w, int h, int type, size_t bytes) {
  cv::Mat m(h, w, type);
  f.read(reinterpret_cast<char*>(m.ptr<unsigned char>()), bytes * size_t(w) * h);
  return m;
}
int main(int argc, char** argv) {
  const int w = 640, h = 480;
  std::ifstream f(argv[1], std::ios::binary);
  cv::Mat Ir = plane(f, w, h, CV_32FC1, 4), Zr = plane(f, w, h, CV_32FC1, 4), Ic = plane(f, w, h, CV_32FC1, 4),
          Zc = plane(f, w, h, CV_32FC1, 4), M = plane(f, w, h, CV_8UC1, 1);
  dvo::core::IntrinsicMatrix K = dvo::core::IntrinsicMatrix::create(float(std::atof(argv[2])), float(std::atof(argv[3])),
                                                                    float(std::atof(argv[4])), float(std::atof(argv[5])));
  dvo::core::RgbdCameraPyramid camera(w, h, K);
  dvo::core::RgbdImagePyramidPtr reference = camera.create(Ir, Zr), current = camera.create(Ic, Zc);
  const int wrong_size = reference->setReferenceMask(cv::Mat(h / 2, w, CV_8UC1));
  const int wrong_type = reference->setReferenceMask(cv::Mat(h, w, CV_32FC1));
  const int ok = reference->setReferenceMask(M);
  dvo::DenseTracker::Config cfg = dvo::DenseTracker::getDefaultConfig();
  cfg.FirstLevel = 3; cfg.LastLevel = 0; cfg.MaxIterationsPerLevel = 50; cfg.Precision = 1e-4;
  dvo::DenseTracker tracker(cfg);
  dvo::DenseTracker::Result result;
  tracker.match(*reference, *current, result);
  const int after = reference->setReferenceMask(M);
  std::printf("%d %d %d %d", wrong_size, wrong_type, ok, after);
  for (int i = 0; i < 4; ++i) for (int j = 0; j < 4; ++j) std::printf(" %.17g", result.Transformation.matrix()(i, j));
  std::printf("\n");
  return 0;
}
"""


def test_adapter_set_reference_mask(engine, scene, tmp_path):
    import __graft_entry__ as ge
    from dvo_slam_b200.engine import Config
    ge.build_cuda()
    ge.build_host()
    a, m = scene, scene["masks"]["blobs"]
    src = tmp_path / "masked_driver.cpp"
    src.write_text(ADAPTER_DRIVER)
    exe = tmp_path / "masked_driver"
    libdir = os.path.join(ROOT, "dvo_slam_b200")
    subprocess.check_call([os.environ.get("CXX", "g++"), "-std=c++17", "-O2", "-I" + os.path.join(ROOT, "include"), str(src), "-o", str(exe),
                           "-L" + libdir, "-ldvo_core_b200", "-ldvo_b200", "-Wl,-rpath," + libdir])
    data = tmp_path / "pair_mask.bin"
    with open(data, "wb") as f:
        for k in ("I_ref", "Z_ref", "I_cur", "Z_cur"):
            f.write(np.ascontiguousarray(a[k], dtype=np.float32).tobytes())
        f.write(np.ascontiguousarray(m, dtype=np.uint8).tobytes())
    r = subprocess.run([str(exe), str(data)] + [repr(float(v)) for v in a["K"]], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    vals = r.stdout.split()
    assert [int(v) for v in vals[:4]] == [0, 0, 1, 0]       # wrong size, wrong type, accepted, refused after the first match
    T = np.array([float(v) for v in vals[4:]]).reshape(4, 4)
    cfg = Config(first_level=3, last_level=0, max_iterations_per_level=50, precision=1e-4)
    g = engine.match(engine.pyramid(a["I_ref"], a["Z_ref"], a["K"], 4, mask=m), engine.pyramid(a["I_cur"], a["Z_cur"], a["K"], 4), cfg)
    assert np.array_equal(T, g.transformation)
