"""Masks in both roles on the CPU oracle: a textured overlay fixed in the image (synth.make_overlay_pair) pulls the
alignment through the current frame's taps as well as through the reference points, and masking the current frame too
brings the pose closer to the truth than masking the reference alone.  No GPU.

tests/masked_oracle.masked_pyramid writes NaN into the depth plane of every unusable pixel after the build.  The oracle's
residual pass blends all six channels of the four taps and rejects any NaN lane, and the gradient planes were built before
the NaNs were written, so the same model pyramid used as the CURRENT image rejects a warped point iff one of its bilinear
taps is unusable -- the rule of a pyramid created with DVO_B200_MASK_ROLE_REFERENCE | DVO_B200_MASK_ROLE_CURRENT.  As the
reference it is the reference-mask model.  So here it models a "both" pyramid in either role."""
import numpy as np
import pytest

from helpers import pose_delta
from masked_oracle import masked_pyramid

SEEDS = tuple(range(16))
CFG = dict(first_level=4, last_level=0, max_iterations_per_level=50, precision=1e-4)


def overlay_errors(oracle, mode="mirror", seeds=SEEDS, **kw):
    """per arm ("none", "reference", "both"): the (translation, rotation) pose errors against the truth, one per seed"""
    from dvo_slam_b200 import synth
    err = {"none": [], "reference": [], "both": []}
    for seed in seeds:
        p = synth.make_overlay_pair(seed, **kw)
        K, m = p["intrinsics"], p["mask"]
        truth = np.linalg.inv(p["T_true"])          # what match() returns for the camera motion
        cur_plain = oracle.Pyramid(p["I_cur"], p["Z_cur"], K, 5)
        arms = {"none": (oracle.Pyramid(p["I_ref"], p["Z_ref"], K, 5), cur_plain),
                "reference": (masked_pyramid(oracle, p["I_ref"], p["Z_ref"], K, 5, m), cur_plain),
                "both": (masked_pyramid(oracle, p["I_ref"], p["Z_ref"], K, 5, m), masked_pyramid(oracle, p["I_cur"], p["Z_cur"], K, 5, m))}
        for name, (ref, cur) in arms.items():
            err[name].append(pose_delta(truth, oracle.match(ref, cur, oracle.config(**CFG), oracle.mode(mode))["T"]))
    return {k: np.array(v) for k, v in err.items()}


def test_overlay_pair_shape_and_mask():
    from dvo_slam_b200 import synth
    p = synth.make_overlay_pair(3)
    q = synth.make_pair(3)
    m = p["mask"]
    assert m.dtype == np.uint8 and m.shape == p["I_ref"].shape
    assert (m == 0).sum() == (160 + 16) * (120 + 16)
    assert np.array_equal(p["Z_ref"], q["Z_ref"].numpy(), equal_nan=True)      # depth stays the scene's
    assert np.array_equal(p["Z_cur"], q["Z_cur"].numpy(), equal_nan=True)
    assert np.array_equal(p["I_ref"][300:420, 420:580], p["I_cur"][300:420, 420:580])   # the same overlay in both frames
    assert np.array_equal(p["I_ref"][m != 0], q["I_ref"].numpy()[m != 0])
    assert np.array_equal(p["I_cur"][m != 0], q["I_cur"].numpy()[m != 0])


@pytest.mark.parametrize("mode", ["mirror"])
def test_masking_the_current_frame_too_brings_the_pose_closer(oracle, mode):
    err = overlay_errors(oracle, mode)
    t_ref, t_both = err["reference"][:, 0], err["both"][:, 0]
    assert np.median(t_both) <= 0.85 * np.median(t_ref), (np.median(t_both), np.median(t_ref))
    assert t_both.max() <= 0.6 * t_ref.max(), (t_both.max(), t_ref.max())
    assert np.median(err["reference"][:, 0]) < np.median(err["none"][:, 0])    # masking the reference does most of the work
