"""Reference masks on the CPU side: the masked oracle model (tests/masked_oracle.py) against the footprint rule stated as
the level-by-level 2x2 AND chain, its selection = isPointOk AND usable, a mask excluding everything, the moving-object use
case, and the declarations of the C ABI entry and the adapter extension.  No GPU."""
import os
import re

import numpy as np
import pytest

from helpers import TERM_INCREMENT_TOO_SMALL, pose_delta
from masked_oracle import masked_pyramid, usable_by_footprint

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MODES = ("faithful", "exact", "mirror")


def usable_by_chain(mask, levels):
    """the same rule as the engine builds it: level 0 = mask != 0, level l = AND of each 2x2 block of level l-1"""
    out = [np.asarray(mask) != 0]
    for _ in range(1, levels):
        u = out[-1]
        h, w = u.shape[0] // 2, u.shape[1] // 2
        out.append(u[0:2 * h:2, 0:2 * w:2] & u[0:2 * h:2, 1:2 * w:2] & u[1:2 * h:2, 0:2 * w:2] & u[1:2 * h:2, 1:2 * w:2])
    return out


def dense_scene(h, w, seed):
    """every pixel valid (no NaN depth), textured: with negative thresholds isPointOk holds everywhere, so the selection of
    a masked pyramid IS its usable set"""
    rng = np.random.default_rng(seed)
    I = np.round(rng.uniform(0, 255, (h, w))).astype(np.float32)
    Z = (1.5 + 0.001 * rng.integers(0, 400, (h, w))).astype(np.float32)
    return I, Z


def _masks(h, w, seed):
    rng = np.random.default_rng(seed)
    masks = {"single_odd": np.ones((h, w), np.uint8), "blobs": np.ones((h, w), np.uint8), "border": np.ones((h, w), np.uint8)}
    masks["single_odd"][201, 317] = 0
    yy, xx = np.ogrid[:h, :w]
    for _ in range(12):
        cy, cx, r = rng.integers(0, h), rng.integers(0, w), rng.integers(3, 40)
        masks["blobs"][(yy - cy) ** 2 + (xx - cx) ** 2 <= r * r] = 0
    masks["border"][:13, :] = 0
    masks["border"][:, -7:] = 0
    masks["border"][-1, :] = 0            # the last row of an odd height: outside every coarse footprint but level 0's
    return masks


def test_footprint_rule_at_odd_sizes(oracle):
    h, w, levels = 481, 643, 5
    I, Z = dense_scene(h, w, 1)
    K = (517.3, 516.5, 318.6, 255.3)
    rng = np.random.default_rng(7)
    full = oracle.Pyramid(I, Z, K, levels)
    for name, m in _masks(h, w, 7).items():
        pm = masked_pyramid(oracle, I, Z, K, levels, (m * rng.integers(1, 256, m.shape)).astype(np.uint8))   # nonzero = usable
        chain = usable_by_chain(m, levels)
        for l in range(levels):
            assert np.array_equal(usable_by_footprint(m, levels)[l], chain[l]), (name, l)
            S0, sel0 = oracle.select(full, l, -1.0, -1.0, None)
            S, sel = oracle.select(pm, l, -1.0, -1.0, None)
            assert S0 == sel0.size, "every pixel is selected without a mask"
            assert np.array_equal(sel.astype(bool), chain[l]), (name, l)
            assert S == int(chain[l].sum())
            # only the depth of unusable pixels differs from the unmasked pyramid: no neighbour loses its gradients
            pf, pp = full.planes(l), pm.planes(l)
            assert np.array_equal(np.delete(pp, 1, 0), np.delete(pf, 1, 0)) and np.array_equal(pp[1][chain[l]], pf[1][chain[l]])
    # the single excluded pixel at odd coordinates removes exactly its containing pixel at every level
    pm = masked_pyramid(oracle, I, Z, K, levels, _masks(h, w, 7)["single_odd"])
    for l in range(levels):
        _, sel = oracle.select(pm, l, -1.0, -1.0, None)
        assert np.argwhere(sel == 0).tolist() == [[201 >> l, 317 >> l]], l


def _pair(small_scene):
    from dvo_slam_b200 import synth
    p = synth.make_pair(3, small_scene)
    return {k: p[k].numpy() for k in ("I_ref", "Z_ref", "I_cur", "Z_cur")}


@pytest.mark.parametrize("mode", MODES)
def test_selection_is_point_ok_and_usable(oracle, small_scene, mode):
    """the masked oracle's selection, for default and non-default thresholds at every level, is the unmasked selection
    AND usable; the residual records of the selected points are those of the unmasked pyramid"""
    a = _pair(small_scene)
    K = small_scene.intrinsics
    h, w = a["I_ref"].shape
    m = _masks(481, 643, 3)["blobs"][:h, :w]
    ref = oracle.Pyramid(a["I_ref"], a["Z_ref"], K, 3)
    pm = masked_pyramid(oracle, a["I_ref"], a["Z_ref"], K, 3, m)
    cur = oracle.Pyramid(a["I_cur"], a["Z_cur"], K, 3)
    usable = usable_by_chain(m, 3)
    T = np.eye(4)
    T[:3, 3] = (0.01, -0.005, 0.004)
    md = oracle.mode(mode)
    for l in range(3):
        for ti, td in ((0.0, 0.0), (3.0, 0.02)):
            S0, sel0 = oracle.select(ref, l, ti, td, None)
            S, sel = oracle.select(pm, l, ti, td, None)
            assert np.array_equal(sel.astype(bool), sel0.astype(bool) & usable[l]) and S == int(sel.sum()) <= S0
            _, r0 = oracle.residual_image(ref, cur, l, T, md, ti, td)
            _, r1 = oracle.residual_image(pm, cur, l, T, md, ti, td)
            valid = ~np.isnan(r1[0])
            both = valid & ~np.isnan(r0[0])
            assert valid.any() and not (valid & ~usable[l]).any() and np.array_equal(r1[:, both], r0[:, both])
            assert (valid & ~both).sum() <= (1 if md.drop_odd_point else 0)   # the unmasked selection's dropped odd last point


@pytest.mark.parametrize("mode", MODES)
def test_mask_excluding_everything_selects_nothing(oracle, small_scene, mode):
    """S = 0 at every level: the single iteration of each level has n = 0 < 6 constraints (TooFewConstraints), which the
    reference's increment test then reports as IncrementTooSmall (dense_tracking.cpp:359: the increment is still zero);
    the pose stays the identity and the information is NaN, so Result::isNaN() holds."""
    a = _pair(small_scene)
    K = small_scene.intrinsics
    ref = masked_pyramid(oracle, a["I_ref"], a["Z_ref"], K, 3, np.zeros(a["I_ref"].shape, np.uint8))
    cur = oracle.Pyramid(a["I_cur"], a["Z_cur"], K, 3)
    for l in range(3):
        S, sel = oracle.select(ref, l, 0.0, 0.0, None)
        assert S == 0 and not sel.any()
    r = oracle.match(ref, cur, oracle.config(first_level=2, last_level=0), oracle.mode(mode))
    assert [l["valid_pixels"] for l in r["levels"]] == [0, 0, 0]
    assert [l["termination"] for l in r["levels"]] == [TERM_INCREMENT_TOO_SMALL] * 3
    assert [it["n"] for it in r["iterations"]] == [0, 0, 0]
    assert np.array_equal(r["T"], np.eye(4)) and np.isnan(r["information"]).all()


# Moving object (synth.make_moving_object_pair, 640x480, 5 levels, levels 4..0): a 150x120 textured patch at ~0.9 m moves
# (24, 10) px between the frames on its own, and the reference mask excludes it with an 8 px margin.  Camera pose error
# against the truth (max translation / rotation component), measured with this oracle on seeds 0..7:
#   seed                      0                  4                  6
#   FAITHFUL unmasked   2.77e-2 / 8.9e-3   1.67e-2 / 5.6e-3   3.09e-2 / 1.08e-2   m / rad
#   FAITHFUL masked     8.8e-4 / 3.4e-4    2.24e-3 / 4.9e-4   1.25e-3 / 4.2e-4
#   MIRROR   unmasked   2.76e-2 / 8.9e-3   1.70e-2 / 5.9e-3   3.10e-2 / 1.08e-2
#   MIRROR   masked     1.11e-3 / 4.0e-4   1.42e-3 / 5.0e-4   1.32e-3 / 4.6e-4
# On the other five seeds the patch barely pulls the unmasked estimate (all errors 3e-4 .. 2.3e-3 m either way).  On these
# three masking brings the pose 7.5x (seed 4, translation) to 31x closer (DESIGN.md §4.5).
MOVING_SEEDS = (0, 4, 6)
MOVING_CFG = dict(first_level=4, last_level=0, max_iterations_per_level=50, precision=1e-4)


@pytest.mark.parametrize("seed", MOVING_SEEDS)
def test_masking_a_moving_object_brings_the_pose_closer(oracle, seed):
    from dvo_slam_b200 import synth
    p = synth.make_moving_object_pair(seed)
    K = p["intrinsics"]
    truth = np.linalg.inv(p["T_true"])          # what match() returns for the camera motion
    cur = oracle.Pyramid(p["I_cur"], p["Z_cur"], K, 5)
    for mode in ("faithful", "mirror"):
        err = {}
        for name, m in (("unmasked", None), ("masked", p["mask"])):
            ref = masked_pyramid(oracle, p["I_ref"], p["Z_ref"], K, 5, m)
            err[name] = pose_delta(truth, oracle.match(ref, cur, oracle.config(**MOVING_CFG), oracle.mode(mode))["T"])
        assert err["masked"][0] < 2.5e-3 and err["masked"][1] < 1e-3, (mode, err)
        assert err["masked"][0] * 5 < err["unmasked"][0] and err["masked"][1] * 5 < err["unmasked"][1], (mode, err)


def test_masked_create_is_declared_and_exported():
    hdr = open(os.path.join(ROOT, "include", "dvo_b200.h")).read()
    assert re.search(r"int dvo_b200_pyramid_create_masked_batch\(", hdr)
    for name in ("DVO_B200_INPUT_FLOAT32 = 0", "DVO_B200_INPUT_GREY8_DEPTH16 = 1", "DVO_B200_INPUT_BGR8_DEPTH16 = 2"):
        assert name in hdr
    assert "#define DVO_B200_ABI_VERSION 1" in hdr
    from dvo_slam_b200 import engine
    assert "dvo_b200_pyramid_create_masked_batch" in engine.ABI_SYMBOLS
    lib = os.path.join(ROOT, "dvo_slam_b200", "libdvo_b200.so")
    if os.path.exists(lib):
        import subprocess
        syms = subprocess.run(["nm", "-D", "--defined-only", lib], capture_output=True, text=True).stdout
        assert " dvo_b200_pyramid_create_masked_batch" in syms
    img = open(os.path.join(ROOT, "include", "dvo", "core", "rgbd_image.h")).read()
    assert "bool setReferenceMask(const cv::Mat& mask);" in img
