"""The weight maps (dvo_b200_match_batch_maps) restated in numpy, and their use as an outlier mask measured on the CPU oracle.

footprint_mask is the mask rule of include/dvo_b200.h: a level-0 pixel is 0 iff its level-L parent (x >> L, y >> L) is a
constraint (finite weight) with weight < t.  moving_object_table runs, on synth.make_moving_object_pair, the unmasked
alignment in MIRROR, takes its kept iteration (the last accepted entry of the last level: its precision, and the returned
pose), the oracle's residual image there and the Student-t weights (student_weights), and measures how well `w < t` finds the moving
patch and what a second alignment masked by it achieves."""
import numpy as np

from helpers import pose_delta
from masked_oracle import masked_pyramid

CFG = dict(first_level=4, last_level=0, max_iterations_per_level=50, precision=1e-4)
SEEDS = tuple(range(8))
THRESHOLDS = (0.1, 0.2, 0.3, 0.5)
MASK_WEIGHT = 0.3                                   # the documented threshold (DESIGN §4.10): the best second pass of 0.2, 0.3, 0.5
PATCH = dict(corner=(250, 200), patch=(150, 120))   # make_moving_object_pair's defaults: where the patch lies in the reference


def footprint_mask(weight, level, shape0, t):
    """uint8 [h0, w0]: 0 where the level-`level` parent is a constraint with weight < t, 1 elsewhere"""
    h0, w0 = shape0
    h, w = weight.shape
    out = np.ones((h0, w0), np.uint8)
    bad = np.isfinite(weight) & (weight < t)
    ys, xs = np.mgrid[0:h0, 0:w0]
    py, px = ys >> level, xs >> level
    inside = (py < h) & (px < w)
    out[inside] = np.where(bad[py[inside], px[inside]], 0, 1)
    return out


def _fma32(a, b, c):
    """fp32 fma: the fp64 product of two floats is exact"""
    return (a.astype(np.float64) * b + c).astype(np.float32)


def student_denominator(ei, ez, P):
    """5 + r^T P r in float32 with the level kernel's operation sequence (stages.cuh, student_weight):
    q = (fma(ez, P10, ei P00), fma(ez, P11, ei P01)), d = fma(q0, ei, q1 ez), 5 + d"""
    P = np.asarray(P, dtype=np.float32).reshape(4)
    ei, ez = np.asarray(ei, np.float32), np.asarray(ez, np.float32)
    q0 = _fma32(ez, P[2], (ei * P[0]).astype(np.float32))
    q1 = _fma32(ez, P[3], (ei * P[1]).astype(np.float32))
    d = _fma32(q0, ei, (q1 * ez).astype(np.float32))
    return (np.float32(5.0) + d).astype(np.float32)


def student_weights(ei, ez, P):
    """7 / (5 + r^T P r) in fp64 over the kernel's float32 denominator: the kernel's weight up to its rcp.approx and the
    final multiply (a few ulp), NaN where the residual is"""
    return 7.0 / student_denominator(ei, ez, P).astype(np.float64)


def patch_region(shape):
    m = np.zeros(shape, bool)
    (x0, y0), (pw, ph) = PATCH["corner"], PATCH["patch"]
    m[y0:y0 + ph, x0:x0 + pw] = True
    return m


def kept_iteration(result, last_level):
    """the last accepted (finite-increment) entry of the last level's log"""
    its = [e for e in result["iterations"] if e["level"] == last_level and np.isfinite(e["x"]).all()]
    return its[-1]


def moving_object_table(orc, seeds=SEEDS, thresholds=THRESHOLDS, mask_weight=None):
    """per seed: the unmasked alignment's pose "T", kept precision and weight map, the fractions of selected patch / other pixels
    with w < t for each t, and the pose errors (translation, rotation) against the truth of the unmasked alignment, of the one masked by the ground-truth mask and, with mask_weight,
    of the one masked by the weight map's own mask at that threshold"""
    from dvo_slam_b200 import synth
    rows = []
    m = orc.mode("mirror")
    cfg = orc.config(**CFG)
    for seed in seeds:
        p = synth.make_moving_object_pair(seed)
        K = p["intrinsics"]
        truth = np.linalg.inv(p["T_true"])
        ref = orc.Pyramid(p["I_ref"], p["Z_ref"], K, 5)
        cur = orc.Pyramid(p["I_cur"], p["Z_cur"], K, 5)
        res = orc.match(ref, cur, cfg, m)
        kept = kept_iteration(res, CFG["last_level"])
        n, planes = orc.residual_image(ref, cur, CFG["last_level"], np.linalg.inv(res["T"]), m)
        w = student_weights(planes[0], planes[1], kept["precision"])
        valid = np.isfinite(w)
        patch = patch_region(w.shape)
        row = {"seed": seed, "n": int(valid.sum()), "kept_n": kept["n"], "T": res["T"], "precision": kept["precision"], "weight": w,
               "patch": {t: float((w[valid & patch] < t).mean()) for t in thresholds},
               "other": {t: float((w[valid & ~patch] < t).mean()) for t in thresholds},
               "unmasked": pose_delta(truth, res["T"])}
        gt = masked_pyramid(orc, p["I_ref"], p["Z_ref"], K, 5, p["mask"])
        row["truth_masked"] = pose_delta(truth, orc.match(gt, cur, cfg, m)["T"])
        if mask_weight is not None:
            own = masked_pyramid(orc, p["I_ref"], p["Z_ref"], K, 5, footprint_mask(w, CFG["last_level"], w.shape, mask_weight))
            row["weight_masked_T"] = orc.match(own, cur, cfg, m)["T"]
            row["weight_masked"] = pose_delta(truth, row["weight_masked_T"])
        rows.append(row)
    return rows
