import os

import numpy as np

GOLDEN_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
GOLDEN_SEEDS = (11, 12, 13)
GOLDEN_LEVELS = 3

# Stated SE(3) tolerance of the path (DESIGN.md "Parity").  Measured with scripts/oracle_spread.py over 96
# seeded 640x480 pairs: the reference's own numerical noise (_mm_rcp_ps, round-toward-zero, fp32 serial
# sums; FAITHFUL vs MIRROR oracle) moves the converged pose by median 1.3e-4 m / 3.0e-5 rad,
# p90 6.2e-4 m / 7.6e-5 rad, max 1.06e-3 m / 3.4e-4 rad -- the same order as the method's accuracy on
# this data (FAITHFUL vs ground truth: median 9.7e-4 m, max 2.3e-3 m).  Tolerance = ~2x the max spread.
POSE_TOL_T = 2e-3   # metres
POSE_TOL_R = 1e-3   # radians


def load_golden(seed):
    g = dict(np.load(os.path.join(GOLDEN_DIR, f"pair_{seed}.npz")))
    g["K"] = tuple(float(v) for v in g["intrinsics"])
    return g


def golden_images(g, orc):
    """float32 intensity/depth exactly as benchmark_slam.cpp:46-93 would hand them to the tracker."""
    out = {}
    for k in ("ref", "cur"):
        out[f"I_{k}"] = g[f"grey_{k}"].astype(np.float32)
        out[f"Z_{k}"] = orc.convert_raw_depth(g[f"depth_{k}"], 1.0 / 5000.0)
    return out


def pose_delta(Ta, Tb):
    """(max |translation|, max |rotation|) components of log(Ta^-1 Tb)."""
    from dvo_slam_b200 import synth
    d = synth.se3_log(np.linalg.inv(Ta) @ Tb)
    return float(np.abs(d[:3]).max()), float(np.abs(d[3:]).max())


def nan_equal(a, b):
    return np.array_equal(np.isnan(a), np.isnan(b)) and np.array_equal(a[~np.isnan(a)], b[~np.isnan(b)])


# ---- the pin against the original project's object code (tests/test_reference_pin.py, tests/golden/make_reference_pin.py) ----
O3_SAMPLE = 128     # valid points per (pair, level) at which the -O3 build's records are stored


def load_reference_pin():
    return dict(np.load(os.path.join(GOLDEN_DIR, "reference_pin.npz")))


def digest(a):
    """sha256 of an array's shape, dtype and values, with every NaN and -0 made canonical: two arrays have the same digest
    iff they are equal in the sense of nan_equal (NaN where the other has NaN, the same bits elsewhere up to the sign of 0)."""
    import hashlib
    a = np.ascontiguousarray(a)
    if a.dtype.kind == "f":
        a = np.where(np.isnan(a), np.array(np.nan, a.dtype), a + a.dtype.type(0))
    h = hashlib.sha256(f"{a.shape}{a.dtype.str}".encode())
    h.update(a.tobytes())
    return h.hexdigest()


def dense_records(r, h, w):
    """scatter the reference's compacted records {point (4), i, z, idx, idy, zdx, zdy, -, -} into seven h*w planes"""
    d = np.full((7, h * w), np.nan, np.float32)
    d[0:6, r["index"]] = r["records"][:, 4:10].T
    d[6, r["index"]] = r["records"][:, 2]
    return d


def o3_sample_index(d, seed, lvl):
    """a fixed seeded sample of the valid points (columns) of a seven-plane record image"""
    valid = np.flatnonzero(~np.isnan(d[0]))
    rng = np.random.default_rng(1000 * seed + lvl)
    return np.sort(rng.choice(valid, size=min(O3_SAMPLE, valid.size), replace=False))


def match_cases(orc):
    """(I_ref, Z_ref, I_cur, Z_cur, K, levels, config, T_init) of the whole-alignment pin: the golden pairs at 160x120,
    and two seeded 640x480 pairs with 5 levels (BASELINE configs[0]), the second with mu and an initial estimate"""
    from dvo_slam_b200 import synth
    cases = []
    for seed in GOLDEN_SEEDS:
        g = load_golden(seed)
        im = golden_images(g, orc)
        cases.append((im["I_ref"], im["Z_ref"], im["I_cur"], im["Z_cur"], g["K"], GOLDEN_LEVELS,
                      dict(first_level=2, last_level=0, max_iterations_per_level=50, precision=1e-4), None))
    for seed, extra in ((3, {}), (5, dict(mu=0.05, use_initial_estimate=1))):
        p = synth.make_pair(seed)
        a = {k: p[k].numpy() for k in ("I_ref", "Z_ref", "I_cur", "Z_cur")}
        cfg = dict(first_level=4, last_level=0, max_iterations_per_level=50, precision=1e-4)
        cfg.update(extra)
        T0 = synth.se3_exp(p["xi"] * 0.8) if extra else None
        cases.append((a["I_ref"], a["Z_ref"], a["I_cur"], a["Z_cur"], p["intrinsics"], 5, cfg, T0))
    return cases


def odd_point_margin(orc):
    """The odd-point drop made visible: reference = the first golden frame with its bottom/right margin made invalid,
    current = the same frame unmasked, identity transform -> every selected point maps onto itself and is valid, so the only
    selected pixel the intensity error image may leave at 0 is the odd last one.  Returns the first margin (4..39) that
    gives an odd selection count whose last point is valid on its own, with its images and one-level pyramids."""
    g = load_golden(GOLDEN_SEEDS[0])
    im = golden_images(g, orc)
    for margin in range(4, 40):
        Z = im["Z_ref"].copy()
        Z[-margin:, :] = np.nan
        Z[:, -margin:] = np.nan
        oref = orc.Pyramid(im["I_ref"], Z, g["K"], 1)
        ocur = orc.Pyramid(im["I_ref"], im["Z_ref"], g["K"], 1)
        S, mask = orc.select(oref, 0, 0.0, 0.0, None)
        last = np.flatnonzero(mask.reshape(-1))[-1]
        _, planes_exact = orc.residual_image(oref, ocur, 0, np.eye(4), orc.mode("exact"))
        if S % 2 == 0 or np.isnan(planes_exact[0].reshape(-1)[last]):   # need: odd count, last point valid by itself
            continue
        return margin, im, oref, ocur
    raise AssertionError("no margin gave an odd selection count with a valid last point")
