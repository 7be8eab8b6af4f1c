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


def corrected_mode(orc, fused=1):
    """the corrected estimator's oracle definition: MIRROR with the reference's four structural quirks off -- the scale's
    pair bug, the dropped log-likelihood tail, the dropped odd point, and the log-likelihood as logs of 50-point products
    (which overflow to -inf where the per-point sum the kernel computes is finite)"""
    m = orc.mode("mirror")
    m.scale_pair_bug = 0
    m.ll_drop_tail = 0
    m.drop_odd_point = 0
    m.ll_group_product = 0
    m.fused_pixel_math = fused
    return m


# TerminationCriteria (dense_tracking.h:62-78), as dvo_b200_termination and the oracle number them
TERM_ITERATIONS_EXCEEDED, TERM_INCREMENT_TOO_SMALL, TERM_LOG_LIKELIHOOD_DECREASED, TERM_TOO_FEW_CONSTRAINTS = 0, 1, 2, 3


def split_levels(result):
    """a match result's iteration log (dicts with "n", "nll", ...) cut into one list per level, in level order"""
    its, out, k = result["iterations"] if isinstance(result, dict) else result.iterations, [], 0
    for l in (result["levels"] if isinstance(result, dict) else result.levels):
        out.append(its[k:k + l["num_iterations"]])
        k += l["num_iterations"]
    assert k == len(its)
    return out


def level_fields(iterations, termination):
    """LevelStats::HasIterationWithIncrement / LastIterationWithIncrement (dense_tracking_config.cpp:138-155) over one
    level's iteration log, as the fields of dvo_b200_level_stats: the picked iteration is Iterations[size-2] after
    LogLikelihoodDecreased and Iterations.back() after every other termination, TooFewConstraints included."""
    need = 2 if termination in (TERM_LOG_LIKELIHOOD_DECREASED, TERM_TOO_FEW_CONSTRAINTS) else 1
    has = len(iterations) >= need
    out = {"has_iteration_with_increment": has, "last_valid_constraints": iterations[-1]["n"] if iterations else 0,
           "last_increment_valid_constraints": -1, "last_increment_log_likelihood": float("nan")}
    if has:
        e = iterations[-2] if termination == TERM_LOG_LIKELIHOOD_DECREASED else iterations[-1]
        out["last_increment_valid_constraints"] = e["n"]
        out["last_increment_log_likelihood"] = e["nll"]
    return out


# ---- the named alignment cases of tests/test_gpu_statistics.py and tests/test_step_replay_host.py -------------------
# Every termination path is reached by one of them (asserted from the oracle in test_gpu_statistics.py): IncrementTooSmall,
# IterationsExceeded (max_iterations_per_level 1 and 0), LogLikelihoodDecreased, TooFewConstraints on the first iteration of
# the last level, TooFewConstraints on the first iteration turned into IncrementTooSmall by the post-loop check, and
# TooFewConstraints after an accepted iteration on the last level.  All 160x120, 3 levels.
STATISTICS_CFG = dict(first_level=2, last_level=0, max_iterations_per_level=50, precision=1e-4)
STATISTICS_CASES = ["golden11", "golden12", "golden13", "iterations_1", "iterations_0", "increment_too_small", "initial_estimate",
                    "tfc_first_iteration", "tfc_overridden", "tfc_after_accept"]


def golden_case(seed, **cfg):
    """a golden pair as a case dict (images, K, levels, cfg, T_init), STATISTICS_CFG updated by cfg"""
    from oracle import oracle_py as orc
    g = load_golden(seed)
    im = golden_images(g, orc)
    c = dict(STATISTICS_CFG)
    c.update(cfg)
    return dict(I_ref=im["I_ref"], Z_ref=im["Z_ref"], I_cur=im["I_cur"], Z_cur=im["Z_cur"], K=g["K"], levels=GOLDEN_LEVELS,
                cfg=c, T_init=None)


def statistics_case(name):
    """(images, intrinsics, levels, config, T_init) of a named case of STATISTICS_CASES"""
    if name.startswith("golden"):
        return golden_case(int(name[6:]))
    if name == "iterations_1":
        return golden_case(12, max_iterations_per_level=1)
    if name == "iterations_0":
        return golden_case(12, max_iterations_per_level=0)
    if name == "increment_too_small":
        return golden_case(13, precision=2e-3)
    if name == "initial_estimate":
        c = golden_case(11, use_initial_estimate=1, mu=0.05)
        c["T_init"] = load_golden(11)["kat_T"]
        return c
    if name == "tfc_first_iteration":
        # level-0 depth of the current frame NaN on every odd row and column: no 2x2 bilinear footprint is valid there, the
        # coarser levels (which subsample the even pixels) keep their depth -> TooFewConstraints on the first iteration of
        # the last level, with the increment of level 1 still large
        c = golden_case(11)
        Z = c["Z_cur"].copy()
        Z[1::2, :] = np.nan
        Z[:, 1::2] = np.nan
        c["Z_cur"] = Z
        return c
    if name == "tfc_overridden":
        # no valid current depth: TooFewConstraints on the first iteration of every level, with the initial increment 0 ->
        # the post-loop check makes it IncrementTooSmall, and LastIterationWithIncrement() is that one entry
        c = golden_case(12)
        c["Z_cur"] = np.full_like(c["Z_cur"], np.nan)
        return c
    if name == "tfc_after_accept":
        # found by a seeded search over large-motion 160x120 scenes: the one accepted iteration of level 0 moves the camera
        # off the overlap and the next finds no constraint; FAITHFUL and MIRROR agree on every level's flow
        from dvo_slam_b200 import synth
        scfg = synth.SceneConfig(width=160, height=120, intrinsics=tuple(v / 4 for v in synth.FR1_INTRINSICS),
                                 max_translation=0.3, max_rotation=0.2)
        p = synth.make_pair(26, scfg)
        return dict(I_ref=p["I_ref"].numpy(), Z_ref=p["Z_ref"].numpy(), I_cur=p["I_cur"].numpy(), Z_cur=p["Z_cur"].numpy(),
                    K=p["intrinsics"], levels=3, cfg=dict(STATISTICS_CFG), T_init=None)
    raise KeyError(name)


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
