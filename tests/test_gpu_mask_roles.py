"""Masks in both roles on the H100 (dvo_b200_pyramid_create_masked_batch_roles with REFERENCE | CURRENT): residual records,
error images and linearisations against oracle MIRROR with both estimators at levels 0..3, the tile paths of stage B
forced one by one, the all-ones mask, mixed batches against single alignments under every launch-plan override, whole
alignments against FAITHFUL, the overlay use case, the API and the C++ adapter's setMask(m, true).

The oracle model is tests/masked_oracle.masked_pyramid: NaN in the depth plane of every unusable pixel after the build.
Used as the current image it rejects a warped point iff one of its four bilinear taps is unusable (the oracle blends all
six channels and rejects any NaN lane; the gradients were built before the NaNs were written), so it models a "both"
pyramid in either role."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from helpers import POSE_TOL_R, POSE_TOL_T, nan_equal, pose_delta
from masked_oracle import masked_pyramid, usable_by_footprint
from test_corrected_estimator import corrected_mode
from test_mask_roles_accuracy import CFG as OVERLAY_CFG
from test_mask_roles_accuracy import SEEDS as OVERLAY_SEEDS
from tile_geometry import TILE_W, assert_partial_band

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LEVELS = 4
PP = np.array([[2000.0, -30.0], [-30.0, 9000.0]], dtype=np.float32)
MATCH_CFG = dict(first_level=3, last_level=0, max_iterations_per_level=50, precision=1e-4)


def _rot_z(deg):
    a = np.deg2rad(deg)
    T = np.eye(4)
    T[:2, :2] = [[np.cos(a), -np.sin(a)], [np.sin(a), np.cos(a)]]
    return T


def _shift_z(dz):
    T = np.eye(4)
    T[2, 3] = dz
    return T


@pytest.fixture(scope="module")
def corrected(engine):
    from dvo_slam_b200.engine import Engine
    eng = Engine(device=0, estimator="corrected")
    yield eng
    eng.close()


@pytest.fixture(scope="module")
def scene(oracle):
    """synth pair 21 and masks of the kinds test_gpu_masked_pyramids builds: blobs, a border, and blobs plus a bottom/right band"""
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
    odd = blobs.copy()
    odd[-13:, :] = 0
    odd[:, -13:] = 0
    a["masks"] = {"blobs": blobs, "border": border, "odd": odd}
    return a


def _pyrs(eng, oracle, I, Z, K, m, roles, levels=LEVELS):
    """(GPU pyramid, oracle model) for mask m (None: unmasked) in the given role set"""
    if m is None:
        return eng.pyramid(I, Z, K, levels), oracle.Pyramid(I, Z, K, levels)
    return eng.pyramid(I, Z, K, levels, mask=m, mask_roles=roles), masked_pyramid(oracle, I, Z, K, levels, m)


def _check_records(eng, oracle, mode, gref, gcur, oref, ocur, lvl, T):
    n_g, img_g = eng.residual_image(gref, gcur, lvl, T)
    n_o, img_o = oracle.residual_image(oref, ocur, lvl, T, mode)
    assert n_g == n_o and n_g > 0 and nan_equal(img_g, img_o), (lvl, n_g, n_o)
    ne_g, err_g = eng.intensity_error_image(gref, gcur, lvl, T)
    ne_o, err_o = oracle.intensity_error_image(oref, ocur, lvl, T, mode)
    assert ne_g == ne_o and np.array_equal(err_g, err_o), lvl
    for uw in (False, True):
        lg = eng.linearize(gref, gcur, lvl, T, uw, PP)
        lo = oracle.linearize(oref, ocur, lvl, T, mode, uw, PP)
        assert lg["n"] == lo["n"] == n_o
        # relative to the matrix, as A and b: an off-diagonal entry of P can nearly cancel (0.308 against a diagonal of 433
        # at level 3 with the blob mask in the current role), and the two sum orders then differ by 3e-6 of that entry,
        # 1e-9 of the matrix
        assert np.allclose(lg["precision"], lo["precision"], rtol=2e-6, atol=2e-6 * np.abs(lo["precision"]).max()), (lvl, uw)
        assert abs(lg["ll"] - lo["ll"]) <= 2e-6 * abs(lo["ll"]) + 0.5, (lvl, uw, lg["ll"], lo["ll"])
        assert np.allclose(lg["A"], lo["A"], rtol=0, atol=2e-6 * np.abs(lo["A"]).max())
        assert np.allclose(lg["b"], lo["b"], rtol=0, atol=2e-6 * np.abs(lo["b"]).max())
    return n_g, img_g


def _both_estimators(engine, corrected, oracle, gref, gcur, oref, ocur, lvl, T):
    _check_records(engine, oracle, oracle.mode("mirror"), gref, gcur, oref, ocur, lvl, T)
    _check_records(corrected, oracle, corrected_mode(oracle), gref, gcur, oref, ocur, lvl, T)


@pytest.mark.parametrize("name", ["blobs", "border", "odd"])
@pytest.mark.parametrize("ref_masked", [True, False])
def test_records_against_mirror_both_estimators(engine, corrected, oracle, scene, name, ref_masked):
    from dvo_slam_b200 import synth
    a, m = scene, scene["masks"][name]
    gref, oref = _pyrs(engine, oracle, a["I_ref"], a["Z_ref"], a["K"], m if ref_masked else None, "both")
    gcur, ocur = _pyrs(engine, oracle, a["I_cur"], a["Z_cur"], a["K"], m, "both")
    T = np.linalg.inv(synth.se3_exp(a["xi"] * 0.7))
    plain = engine.pyramid(a["I_cur"], a["Z_cur"], a["K"], LEVELS)
    for lvl in range(LEVELS):
        _both_estimators(engine, corrected, oracle, gref, gcur, oref, ocur, lvl, T)
        # the mask in the current role really removes points here
        assert engine.residual_image(gref, gcur, lvl, T)[0] < engine.residual_image(gref, plain, lvl, T)[0], lvl


def _blob_at(h, w, cx, cy, r):
    m = np.ones((h, w), np.uint8)
    yy, xx = np.ogrid[:h, :w]
    m[(yy - cy) ** 2 + (xx - cx) ** 2 <= r * r] = 0
    return m


@pytest.fixture(scope="module")
def pair0(engine, oracle):
    from dvo_slam_b200 import synth
    p = synth.make_pair(0)
    a = {k: p[k].numpy() for k in ("I_ref", "Z_ref", "I_cur", "Z_cur")}
    a["K"] = p["intrinsics"]
    return a


@pytest.mark.parametrize("case", ["clean_exact", "dirty_exact", "inexact", "no_window", "partial_band"])
def test_forced_tile_paths(engine, corrected, oracle, pair0, case):
    """clean_exact: a mask in one corner, a small motion -- most tiles have an exact window that misses it, a few (near the
    corner) a dirty one; dirty_exact: many small blobs, every exact window touches one; inexact: a 20 degree roll (no
    160-pixel tile row fits the window); no_window: the camera moved past the median depth (tile corners behind it);
    partial_band: levels 1 and 2 of the 720 x 540 scene of test_gpu_generic_tiles (full 160-column bands and a partial one),
    with the mask inside the partial band."""
    from test_gpu_generic_tiles import partial_pair, partial_pose
    a = partial_pair(0) if case == "partial_band" else pair0
    h, w = a["I_ref"].shape
    if case == "clean_exact":
        m, T, lvls = _blob_at(h, w, 40, 40, 25), _rot_z(0.5) @ _shift_z(0.01), [0]
    elif case == "dirty_exact":
        m = np.ones((h, w), np.uint8)
        m[4::32, 4::32] = 0
        T, lvls = _rot_z(0.5) @ _shift_z(0.01), [0]
    elif case == "inexact":
        m, T, lvls = _blob_at(h, w, 320, 240, 60), _rot_z(20.0), [0]
    elif case == "no_window":
        m, T, lvls = _blob_at(h, w, 320, 240, 60), _shift_z(-float(np.nanmedian(a["Z_ref"]))), [0]
    else:
        m, T, lvls = _blob_at(h, w, 680, 270, 30), partial_pose(), [1, 2]
        for lvl in lvls:
            assert_partial_band(w >> lvl)
            x0 = ((w >> lvl) // TILE_W * TILE_W) << lvl         # the level-0 column where the level's partial band starts
            assert (m[:, x0:] == 0).any() and (m[:, :x0] != 0).all()
    gref, oref = _pyrs(engine, oracle, a["I_ref"], a["Z_ref"], a["K"], None, "both", 5)
    gcur, ocur = _pyrs(engine, oracle, a["I_cur"], a["Z_cur"], a["K"], m, "both", 5)
    for lvl in lvls:
        _both_estimators(engine, corrected, oracle, gref, gcur, oref, ocur, lvl, T)


def _same_result(r0, r1):
    return (np.array_equal(r0.transformation, r1.transformation) and np.array_equal(r0.information, r1.information, equal_nan=True)
            and (r0.log_likelihood == r1.log_likelihood or (np.isnan(r0.log_likelihood) and np.isnan(r1.log_likelihood)))
            and len(r0.levels) == len(r1.levels)
            and all(a.keys() == b.keys() and all(a[k] == b[k] or (a[k] != a[k] and b[k] != b[k]) for k in a) for a, b in zip(r0.levels, r1.levels)))


def test_all_ones_mask_equals_no_mask(engine, scene):
    from dvo_slam_b200.engine import Config
    a = scene
    h, w = a["I_ref"].shape
    ones = np.full((h, w), 3, np.uint8)
    ref = engine.pyramid(a["I_ref"], a["Z_ref"], a["K"], LEVELS)
    ref1 = engine.pyramid(a["I_ref"], a["Z_ref"], a["K"], LEVELS, mask=ones, mask_roles="both")
    cur = engine.pyramid(a["I_cur"], a["Z_cur"], a["K"], LEVELS)
    cur1 = engine.pyramid(a["I_cur"], a["Z_cur"], a["K"], LEVELS, mask=ones, mask_roles="both")
    for p, q in ((ref, ref1), (cur, cur1)):
        for l in range(LEVELS):
            assert np.array_equal(p.download(l), q.download(l), equal_nan=True), l
    cfg = Config(**MATCH_CFG)
    r = engine.match_batch([ref, ref1, ref, ref1], [cur, cur, cur1, cur1], cfg)
    for k in (1, 2, 3):
        assert _same_result(r[0], r[k]), k


def test_download_and_roles(engine, scene):
    a, m = scene, scene["masks"]["blobs"]
    plain = engine.pyramid(a["I_cur"], a["Z_cur"], a["K"], LEVELS)
    ref_only = engine.pyramid(a["I_cur"], a["Z_cur"], a["K"], LEVELS, mask=m)
    both = engine.pyramid(a["I_cur"], a["Z_cur"], a["K"], LEVELS, mask=m, mask_roles="both")
    assert (plain.mask_roles, ref_only.mask_roles, both.mask_roles) == (None, "reference", "both")
    for l, usable in enumerate(usable_by_footprint(m, LEVELS)):
        d0, d1, d2 = plain.download(l), ref_only.download(l), both.download(l)
        assert np.array_equal(d0, d1, equal_nan=True)
        expect = np.where(usable, d0[1], np.nan)
        assert np.array_equal(d2[1], expect, equal_nan=True) and (~usable).any(), l
        assert np.array_equal(np.delete(d2, 1, axis=0), np.delete(d0, 1, axis=0), equal_nan=True), l
        assert np.array_equal(both.select(l)[1], ref_only.select(l)[1]) and both.select(l)[0] == ref_only.select(l)[0]


def test_invalid_arguments_create_nothing(engine, scene):
    from dvo_slam_b200.engine import load_library
    lib = load_library()
    a = scene
    h, w = a["I_ref"].shape
    I, Z = np.ascontiguousarray(a["I_ref"]), np.ascontiguousarray(a["Z_ref"])
    m = np.ones((h, w), np.uint8)
    cases = [(0, I.ctypes.data, Z.ctypes.data, r) for r in (0, 2, 4, 5, 7, -1)]
    cases += [(3, I.ctypes.data, Z.ctypes.data, 3), (0, None, Z.ctypes.data, 3), (0, I.ctypes.data, None, 3)]
    for fmt, pI, pZ, roles in cases:
        out = (C.c_void_p * 1)()
        rc = lib.dvo_b200_pyramid_create_masked_batch_roles(engine.ctx, 1, fmt, pI, pZ, 0.0, m.ctypes.data, roles, w, h, *a["K"], LEVELS, out)
        assert rc == -1 and not out[0], (fmt, roles, rc)
    out = (C.c_void_p * 1)()
    rc = lib.dvo_b200_pyramid_create_masked_batch_roles(engine.ctx, 1, 0, I.ctypes.data, Z.ctypes.data, 0.0, m.ctypes.data, 3, w, h,
                                                        *a["K"], LEVELS, None)
    assert rc == -1
    assert lib.dvo_b200_pyramid_mask_roles(None) == -1
    # masks == NULL: the unmasked pyramid whatever the roles
    rc = lib.dvo_b200_pyramid_create_masked_batch_roles(engine.ctx, 1, 0, I.ctypes.data, Z.ctypes.data, 0.0, None, 3, w, h, *a["K"], LEVELS, out)
    assert rc == 0 and out[0]
    engine.synchronize()
    assert lib.dvo_b200_pyramid_mask_roles(out[0]) == 0
    lib.dvo_b200_pyramid_release(out[0])


def _mixed_batch(engine, scene):
    from dvo_slam_b200 import synth
    a = scene
    K = a["K"]
    kinds = ((None, None), ("blobs", "both"), ("border", "reference"), (None, None), ("odd", "both"), ("blobs", "reference"))
    refs, curs, plain_curs = [], [], []
    for k, (name, roles) in enumerate(kinds):
        p = synth.make_pair(40 + k)
        m = None if name is None else a["masks"][name]
        refs.append(engine.pyramid(p["I_ref"].numpy(), p["Z_ref"].numpy(), K, LEVELS, mask=m, mask_roles=roles or "reference"))
        curs.append(engine.pyramid(p["I_cur"].numpy(), p["Z_cur"].numpy(), K, LEVELS, mask=m, mask_roles=roles or "reference"))
        plain_curs.append(roles != "both")
    return refs, curs, plain_curs


def test_mixed_batch_equals_single_alignments_under_every_plan(engine, scene, monkeypatch):
    from dvo_slam_b200.engine import Config
    refs, curs, plain = _mixed_batch(engine, scene)
    cfg = Config(**MATCH_CFG)
    single = [engine.match(refs[i], curs[i], cfg) for i in range(len(refs))]
    batch = engine.match_batch(refs, curs, cfg)
    rev = engine.match_batch(refs[::-1], curs[::-1], cfg)[::-1]
    for i in range(len(refs)):
        assert _same_result(batch[i], single[i]) and _same_result(rev[i], single[i]), i
    # the pairs without a "both" current give the bits of a batch in which no pyramid has one (the default instance)
    idx = [i for i in range(len(refs)) if plain[i]]
    plain_batch = engine.match_batch([refs[i] for i in idx], [curs[i] for i in idx], cfg)
    for j, i in enumerate(idx):
        assert _same_result(plain_batch[j], batch[i]), i
    # a bigger batch, so that the fused launch and its slices exist, under the plan overrides
    big_r, big_c = refs * 6, curs * 6
    big_single = single * 6
    for knob, value in (("DVO_B200_FINE_G", "2"), ("DVO_B200_FINE_G", "4"), ("DVO_B200_TAIL", "6,6"), ("DVO_B200_COARSE_TILES", "0"),
                        ("DVO_B200_COARSE_TILES", "1000000"), ("DVO_B200_NO_FUSE", "1")):
        monkeypatch.setenv(knob, value)
        r = engine.match_batch(big_r, big_c, cfg)
        monkeypatch.delenv(knob)
        for i in range(len(big_r)):
            assert _same_result(r[i], big_single[i]), (knob, value, i)


def test_shared_both_pyramid_two_contexts(engine, corrected, scene):
    from dvo_slam_b200.engine import Config
    a, m = scene, scene["masks"]["odd"]
    K = a["K"]
    cfg = Config(**MATCH_CFG)
    ref = engine.pyramid(a["I_ref"], a["Z_ref"], K, LEVELS, mask=m, mask_roles="both")
    shared = engine.pyramid(a["I_cur"], a["Z_cur"], K, LEVELS, mask=m, mask_roles="both")
    own_c = corrected.pyramid(a["I_cur"], a["Z_cur"], K, LEVELS, mask=m, mask_roles="both")
    ref_c = corrected.pyramid(a["I_ref"], a["Z_ref"], K, LEVELS, mask=m, mask_roles="both")
    r_ref = engine.match(ref, shared, cfg)
    r_cor = corrected.match(ref, shared, cfg)
    assert _same_result(corrected.match(ref_c, own_c, cfg), r_cor)
    assert _same_result(engine.match(ref, shared, cfg), r_ref)
    assert not np.array_equal(r_ref.transformation, r_cor.transformation)


@pytest.mark.parametrize("name", ["blobs", "border", "odd"])
def test_match_within_tolerance_of_faithful(engine, oracle, scene, name):
    from dvo_slam_b200.engine import Config
    a, m = scene, scene["masks"][name]
    kw = dict(first_level=4, last_level=0, max_iterations_per_level=50, precision=1e-4)
    g = engine.match(engine.pyramid(a["I_ref"], a["Z_ref"], a["K"], 5, mask=m, mask_roles="both"),
                     engine.pyramid(a["I_cur"], a["Z_cur"], a["K"], 5, mask=m, mask_roles="both"), Config(**kw))
    o = oracle.match(masked_pyramid(oracle, a["I_ref"], a["Z_ref"], a["K"], 5, m), masked_pyramid(oracle, a["I_cur"], a["Z_cur"], a["K"], 5, m),
                     oracle.config(**kw), oracle.mode("faithful"))
    dt, dr = pose_delta(o["T"], g.transformation)
    assert dt < POSE_TOL_T and dr < POSE_TOL_R, (dt, dr)
    assert [l["valid_pixels"] for l in g.levels] == [l["valid_pixels"] for l in o["levels"]]


def test_overlay_accuracy(engine, oracle):
    """Per seed, the GPU's both-roles pose is within 1e-3 m / 5e-4 rad of MIRROR's both-roles pose or closer to the truth;
    over the seeds it meets the bounds tests/test_mask_roles_accuracy.py asserts on the oracle."""
    from dvo_slam_b200 import synth
    from dvo_slam_b200.engine import Config
    cfg = Config(**OVERLAY_CFG)
    e_ref, e_both = [], []
    for seed in OVERLAY_SEEDS:
        p = synth.make_overlay_pair(seed)
        K, m = p["intrinsics"], p["mask"]
        truth = np.linalg.inv(p["T_true"])
        ref = engine.pyramid(p["I_ref"], p["Z_ref"], K, 5, mask=m, mask_roles="both")
        cur = engine.pyramid(p["I_cur"], p["Z_cur"], K, 5, mask=m, mask_roles="both")
        cur_plain = engine.pyramid(p["I_cur"], p["Z_cur"], K, 5)
        g_both = engine.match(ref, cur, cfg).transformation
        e_both.append(pose_delta(truth, g_both)[0])
        e_ref.append(pose_delta(truth, engine.match(ref, cur_plain, cfg).transformation)[0])
        o_both = oracle.match(masked_pyramid(oracle, p["I_ref"], p["Z_ref"], K, 5, m), masked_pyramid(oracle, p["I_cur"], p["Z_cur"], K, 5, m),
                              oracle.config(**OVERLAY_CFG), oracle.mode("mirror"))["T"]
        dt, dr = pose_delta(o_both, g_both)
        closer = pose_delta(truth, g_both)[0] <= pose_delta(truth, o_both)[0]
        assert (dt <= 1e-3 and dr <= 5e-4) or closer, (seed, dt, dr)
    e_ref, e_both = np.array(e_ref), np.array(e_both)
    print("overlay GPU: reference-only median %.2e max %.2e; both median %.2e max %.2e m" % (np.median(e_ref), e_ref.max(), np.median(e_both), e_both.max()))
    assert np.median(e_both) <= 0.85 * np.median(e_ref)
    assert e_both.max() <= 0.6 * e_ref.max()


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
  const int wrong_size = current->setMask(cv::Mat(h / 2, w, CV_8UC1), true);
  const int wrong_type = current->setMask(cv::Mat(h, w, CV_32FC1), true);
  const int ok = reference->setMask(M, true) && current->setMask(M, true);
  dvo::DenseTracker::Config cfg = dvo::DenseTracker::getDefaultConfig();
  cfg.FirstLevel = 3; cfg.LastLevel = 0; cfg.MaxIterationsPerLevel = 50; cfg.Precision = 1e-4;
  dvo::DenseTracker tracker(cfg);
  std::vector<dvo::core::RgbdImagePyramid*> both;
  both.push_back(reference.get()); both.push_back(current.get());
  std::vector<dvo_b200_pyramid*> handles;
  dvo_b200_ctx* upload = nullptr;   // pyramids are shared objects: the tracker's context aligns what this one built
  if (dvo_b200_create(0, nullptr, &upload) != 0) return 1;
  dvo::core::RgbdImagePyramid::deviceBatch(upload, both, 4, handles);   // one create call, one synchronisation
  dvo::DenseTracker::Result result;
  tracker.match(*reference, *current, result);
  const int after = current->setMask(M, true);
  std::printf("%d %d %d %d %d %d", wrong_size, wrong_type, ok, after, dvo_b200_pyramid_mask_roles(handles[0]),
              dvo_b200_pyramid_mask_roles(handles[1]));
  for (int i = 0; i < 4; ++i) for (int j = 0; j < 4; ++j) std::printf(" %.17g", result.Transformation.matrix()(i, j));
  std::printf("\n");
  dvo_b200_destroy(upload);
  return 0;
}
"""


def test_adapter_set_mask_both_roles(engine, scene, tmp_path):
    import __graft_entry__ as ge
    from dvo_slam_b200.engine import Config
    ge.build_cuda()
    ge.build_host()
    a, m = scene, scene["masks"]["blobs"]
    src = tmp_path / "mask_roles_driver.cpp"
    src.write_text(ADAPTER_DRIVER)
    exe = tmp_path / "mask_roles_driver"
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
    assert [int(v) for v in vals[:6]] == [0, 0, 1, 0, 3, 3]     # wrong size, wrong type, accepted, refused after the match; roles
    T = np.array([float(v) for v in vals[6:]]).reshape(4, 4)
    cfg = Config(**MATCH_CFG)
    g = engine.match(engine.pyramid(a["I_ref"], a["Z_ref"], a["K"], 4, mask=m, mask_roles="both"),
                     engine.pyramid(a["I_cur"], a["Z_cur"], a["K"], 4, mask=m, mask_roles="both"), cfg)
    assert np.array_equal(T, g.transformation)
