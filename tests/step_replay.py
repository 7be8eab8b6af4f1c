"""An fp64 replay of the level kernel's end step (pair_end_cta in dvo_slam_b200/csrc/tracker.cu) from an alignment's own
iteration log, in plain numpy / scipy.

Teacher forcing: the log holds every increment x the end step computed.  From those, and from the accept decisions the
logged log-likelihoods imply, the replay rebuilds in fp64 the pose (and in the photometric mode the brightness (alpha,
beta)) every iteration linearised at, following DenseTracker::match as oracle/dvo_oracle.cpp:865-1034 writes it out:

  inc = T0 (use_initial_estimate, else I); initial = inc; estimate = I           dvo_oracle.cpp:875-878
  every level: x = log(inc)                                                      :912  (dense_tracking.cpp:238)
    every iteration: inc = exp(x); initial <- inc^-1 initial; estimate <- inc estimate   :923-925 (259-261)
      n < 6: revert initial and estimate, TooFewConstraints                      :942-948
      accept iff nll < the previous entry's nll of the level (first: always)     :972-974
      rejected: revert, LogLikelihoodDecreased                                   :975-981
      accepted: x = the logged increment; iteration += 1                         :995-1004
    while accepted, linf(x) > precision and iteration < max_iterations           :1005
    then linf(x) <= precision -> IncrementTooSmall; iteration >= max -> IterationsExceeded   :1007-1008

So the level start applies again the last `inc` of the previous level, whether that increment was kept or reverted; the last
increment a level computes is never applied.  The photometric mode (dvo_oracle.cpp:879-882, 913-1002) adds
(alpha, beta) to the Revertable state: the top of an iteration adds the (alpha, beta) part dab of the previous accepted
solve of the same level (0 at a level start), a revert restores them, and they carry over between levels.  The log does
not hold dab, so the replay takes it from the reference's own 8 x 8 solve at the replayed pose and brightness.  Each dab
so carries the relative error of a system known to 2e-6, and the replayed (alpha, beta) drift from the kernel's by up to
~1e-6 of the path they travel; near convergence that moves the intensity residuals enough to show in P (PHOTOMETRIC).

At every entry the reference linearises at the replayed state (weighted by the kernel's own logged precision of the
previous entry, unweighted on a level's first), and the entry's numbers are checked against it:

  n           the reference's constraint count, +-bounds.n (a pixel exactly on a validity bound)
  precision   max |dP| / max |P|
  nll         -ll, |d| <= bounds.rel |nll| + bounds.nll_abs; +inf on one side only fails
  prior       mu |li|^2 or li^T Lambda li with li = log(initial), |d| / s <= bounds.prior_rel with
              s = max(|prior| + 2 |Lambda li|_inf |li|_inf, prior_abs / prior_rel): the form's sensitivity to li, since a
              stiff prior holds its direction of li near 0 and the value cancels there
  A           the information: A + mu I (+ Lambda), or the Schur complement of the 8 x 8 with the prior on its pose block;
              max |dA| / max |A|
  x           backward error in the reference system M x = c: |M x_g - c|_inf / (|M|_inf |x_g|_inf + |c|_inf) <= bounds.tau
              (a forward error would depend on A's condition number, translation against rotation)
  decision    the increment is finite exactly on accepted entries, and each level's length and termination are what the
              loop above gives on the logged numbers
  pose        Result.transformation against inverse(replayed estimate), max abs over the 4 x 4
  ab          the returned (alpha, beta) against the replayed ones, relative to max(1, the path travelled) (ab_error)

SE(3) is scipy.linalg.expm / logm of the 4 x 4 twist matrix (twist order [v; omega]), independent of the closed forms in
se3.cuh and the oracle.
"""
from dataclasses import dataclass, field

import numpy as np
import scipy.linalg

from helpers import (TERM_INCREMENT_TOO_SMALL, TERM_ITERATIONS_EXCEEDED, TERM_LOG_LIKELIHOOD_DECREASED,
                     TERM_TOO_FEW_CONSTRAINTS)

QUANTITIES = ("n", "precision", "nll", "prior", "A", "x", "pose", "ab")

# variants of the model that each break one rule of the end step; tests/test_step_replay_host.py shows that the checks
# tell every one of them from the rule itself
MUTATIONS = ("no_level_start_reapply",      # the next level starts from inc = I instead of exp(log(inc))
             "li_from_estimate",            # the prior's li = log(estimate) instead of log(initial)
             "information_without_prior",   # A (default mode) without mu I / Lambda
             "ab_not_reverted",             # a reject keeps (alpha, beta) + dab
             "schur_without_prior",         # the Schur complement of the 8 x 8 without Lambda / mu I on its pose block
             "flip_accept")                 # one accept decision flipped (the entry index in Mutation.entry)


@dataclass
class Bounds:
    """what the kernel is held to.  P, nll and A: the suite's bounds for the same quantities at a given pose (measured
    maxima 8.2e-7, 2.0e-7, 8.7e-7).  The others from the largest values measured over every case on an H100 (80 GB HBM3,
    tests/test_gpu_step_replay.py prints them), with margin: n 0 (the kernel's pose and the replayed one differ by ~1e-15,
    and no pixel flipped), prior 2.8e-13, x 2.3e-7, pose 1.7e-15, ab 6.6e-7."""
    n: int = 0
    P: float = 2e-6            # precision, relative to max |P|
    rel: float = 2e-6          # nll, relative
    nll_abs: float = 0.5
    prior_rel: float = 2e-12
    prior_abs: float = 2e-15
    A: float = 2e-6            # relative to max |A|
    tau: float = 2e-6          # backward error of x
    pose: float = 1e-14
    ab: float = 5e-6           # relative to max(1, the path (alpha, beta) travelled), per component


# the same arithmetic replayed (the oracle's own logs): everything but the fp64 summation order of A + Lambda, the solve and
# the SE(3) closed forms is bit for bit.  Measured maxima over every case: prior 6.5e-14, A 1.9e-16, x 7.1e-13, pose 7.8e-16,
# ab 2.6e-13 (scipy / LAPACK against the oracle's closed forms and LDL^T).
TIGHT = Bounds(n=0, P=0.0, rel=0.0, nll_abs=0.0, prior_rel=1e-12, prior_abs=1e-15, A=1e-15, tau=2e-12, pose=1e-14, ab=1e-12)

# the photometric mode, where the replayed (alpha, beta) are the reference's, not the kernel's (see above): P measured to 7.9e-6
# and A to 2.0e-6 of their maxima on an H100, against 8.5e-7 and 8.7e-7 in every other mode
PHOTOMETRIC = Bounds(P=2e-5, A=5e-6)


@dataclass
class Mutation:
    name: str
    entry: int = -1            # flip_accept: the log index of the entry whose decision is flipped


@dataclass
class Report:
    maxima: dict = field(default_factory=lambda: {q: 0.0 for q in QUANTITIES})
    failures: list = field(default_factory=list)      # (quantity, entry index or -1, detail)
    states: list = field(default_factory=list)        # per entry: (estimate, ab, path of ab) after its decision
    T: np.ndarray = None                              # inverse(replayed estimate)
    ab: np.ndarray = None

    @property
    def failed(self):
        return {f[0] for f in self.failures}

    def note(self, quantity, value, bound, entry, detail=""):
        if not value <= self.maxima[quantity]:
            self.maxima[quantity] = value
        if not value <= bound:
            self.failures.append((quantity, entry, f"{value:.3e} > {bound:.3e} {detail}"))


# ---- SE(3) through the matrix exponential -------------------------------------------------------------------------------
def hat(xi):
    v, w = xi[:3], xi[3:]
    return np.array([[0.0, -w[2], w[1], v[0]], [w[2], 0.0, -w[0], v[1]], [-w[1], w[0], 0.0, v[2]], [0.0, 0.0, 0.0, 0.0]])


def se3_exp(xi):
    return scipy.linalg.expm(hat(np.asarray(xi, dtype=np.float64)))


def se3_log(T):
    M = np.real(scipy.linalg.logm(np.asarray(T, dtype=np.float64)))
    return np.array([M[0, 3], M[1, 3], M[2, 3], 0.5 * (M[2, 1] - M[1, 2]), 0.5 * (M[0, 2] - M[2, 0]), 0.5 * (M[1, 0] - M[0, 1])])


def se3_inv(T):
    R, t = T[:3, :3], T[:3, 3]
    out = np.eye(4)
    out[:3, :3] = R.T
    out[:3, 3] = -R.T @ t
    return out


def ab_error(ab_kernel, ab, path):
    """max over (alpha, beta) of |kernel - replayed| / max(1, path travelled): each applied dab carries the relative error of
    the system it solves (measured on an H100: 3e-7 of a one-step move of beta by 26 intensity levels), so the error grows
    with the path"""
    return float((np.abs(np.asarray(ab_kernel) - ab) / np.maximum(path, 1.0)).max())


# ---- the log of an alignment, from the engine or either oracle --------------------------------------------------------
@dataclass
class Log:
    iterations: list
    levels: list        # [(termination, num_iterations)] in level order
    T: np.ndarray       # Result.transformation
    ab: np.ndarray = None


def as_log(result, ab=None):
    """an engine Result (with_iterations=True) with its final (alpha, beta), or an oracle match dict (orc.match)"""
    if isinstance(result, dict):
        lv = [(l["termination"], l["num_iterations"]) for l in result["levels"]]
        return Log(result["iterations"], lv, np.asarray(result["T"]), result.get("ab") if ab is None else ab)
    return Log(result.iterations, [(l["termination"], l["num_iterations"]) for l in result.levels], result.transformation, ab)


# ---- the replay ---------------------------------------------------------------------------------------------------------
def _system(r, li, lam, photometric, mutation):
    """(M, c, information, dab) of the reference linearisation r with the prior lam on the pose block"""
    if not photometric:
        M, c = r["A"] + lam, r["b"] + lam @ li
        info = r["A"] if mutation == "information_without_prior" else M
        return M, c, info, None
    M8, c8 = r["A"].copy(), r["b"].copy()
    M8[:6, :6] += lam
    c8[:6] += lam @ li
    G = np.linalg.solve(M8[6:, 6:], M8[6:, :6])          # A_pp^-1 A_px
    S = M8[:6, :6] - M8[:6, 6:] @ G
    c_red = c8[:6] - G.T @ c8[6:]
    info = S - lam if mutation == "schur_without_prior" else S
    return S, c_red, info, np.linalg.solve(M8, c8)[6:]


def replay(log, cfg, linearize, T0=None, mu=0.0, prior=None, photometric=False, ab0=None, bounds=Bounds(), mutation=None):
    """Replay `log` (as_log) of an alignment with config `cfg` (a dict of Config fields).  linearize(level, T, ab,
    use_weights, prev_precision) -> {"n", "precision", "ll", "A", "b"}: the reference at that pose and brightness (ab is
    None outside the photometric mode).  T0: the initial estimate (used iff cfg["use_initial_estimate"]).  prior: a 6 x 6
    Lambda in place of mu I."""
    rep = Report()
    mut = mutation.name if mutation else None
    precision = cfg.get("precision", 1e-4)
    max_it = cfg.get("max_iterations_per_level", 50)
    lam = np.asarray(prior, dtype=np.float64) if prior is not None else mu * np.eye(6)
    inc = np.asarray(T0, dtype=np.float64) if (T0 is not None and cfg.get("use_initial_estimate", 0)) else np.eye(4)
    initial, estimate = inc.copy(), np.eye(4)
    ab = np.array(ab0 if ab0 is not None else (1.0, 0.0), dtype=np.float64) if photometric else None
    path = np.zeros(2)      # sum of |dab| applied: the scale of the ab error, a sum of per-step relative errors
    k0 = 0
    level_ids = list(range(cfg["first_level"], cfg["last_level"] - 1, -1))
    if len(log.levels) != len(level_ids) or sum(c for _, c in log.levels) != len(log.iterations):
        rep.failures.append(("decision", -1, f"levels {log.levels} for {len(log.iterations)} entries"))
        return rep
    for li_, (level, (term, count)) in enumerate(zip(level_ids, log.levels)):
        entries = log.iterations[k0:k0 + count]
        x = np.zeros(6) if (mut == "no_level_start_reapply" and li_ > 0) else se3_log(inc)     # dvo_oracle.cpp:912
        dab = np.zeros(2)
        prev_nll, prev_P = np.inf, None
        iteration, ended, model_term = 0, False, -1
        for j, e in enumerate(entries):
            idx = k0 + j
            if ended:
                rep.failures.append(("decision", idx, "an entry after the level's loop ended"))
                break
            if e["level"] != level or e["id"] != j:
                rep.failures.append(("decision", idx, f"entry ({e['level']}, {e['id']}) at ({level}, {j})"))
            inc = se3_exp(x)                                                                     # :923-925
            saved = (initial, estimate, None if ab is None else ab.copy(), path.copy())
            initial, estimate = se3_inv(inc) @ initial, inc @ estimate
            if photometric:
                ab, path = ab + dab, path + np.abs(dab)
            r = linearize(level, estimate, ab, j > 0, prev_P)
            rep.note("n", abs(int(e["n"]) - int(r["n"])), bounds.n, idx)
            if e["n"] < 6:                                                                       # :942-948
                if np.isfinite(e["x"]).any():
                    rep.failures.append(("decision", idx, "an increment on an entry with n < 6"))
                initial, estimate, sab, spath = saved
                if photometric and mut != "ab_not_reverted":
                    ab, path = sab, spath
                model_term, ended = TERM_TOO_FEW_CONSTRAINTS, True
                rep.states.append((estimate, None if ab is None else ab.copy(), path.copy()))
                continue
            if r["n"] < 6:
                rep.failures.append(("n", idx, f"kernel n = {e['n']}, reference n = {r['n']}"))
                break
            Pr = np.asarray(r["precision"], dtype=np.float64).reshape(2, 2)
            Pg = np.asarray(e["precision"], dtype=np.float64).reshape(2, 2)
            rep.note("precision", np.abs(Pg - Pr).max() / np.abs(Pr).max(), bounds.P, idx)
            nll_r = -float(r["ll"])
            # an infinite -ll on both sides is equal; on one side only it fails (the reference's 50-point products
            # overflowing where the kernel's per-point sum does not: an accept / reject split)
            d = 0.0 if e["nll"] == nll_r else abs(e["nll"] - nll_r)
            rep.note("nll", d / abs(nll_r), bounds.rel + bounds.nll_abs / abs(nll_r), idx, f"({e['nll']} vs {nll_r})")
            li = se3_log(estimate if mut == "li_from_estimate" else initial)
            prior_r = float(li @ lam @ li)
            # relative to |prior| + 2 |Lambda li| |li|, the quadratic form's first-order sensitivity to li: a stiff prior holds
            # its direction of li near 0, and there the fp64 rounding of li alone moves the value far more than |prior| says.
            # The scale has the floor prior_abs / prior_rel, so that the reported value is measured against prior_rel.
            s = max(abs(prior_r) + 2.0 * np.abs(lam @ li).max() * np.abs(li).max(), bounds.prior_abs / bounds.prior_rel)
            rep.note("prior", abs(e["prior"] - prior_r) / s, bounds.prior_rel, idx, f"({e['prior']} vs {prior_r})")
            accept = e["nll"] < prev_nll                                                         # :972-974
            if mut == "flip_accept" and idx == mutation.entry:
                accept = not accept
            if np.isfinite(e["x"]).all() != accept or np.isfinite(e["A"]).all() != accept:
                rep.failures.append(("decision", idx, f"accept = {accept}, increment {e['x']}"))
            if not accept:                                                                       # :975-981
                initial, estimate, sab, spath = saved
                if photometric and mut != "ab_not_reverted":
                    ab, path = sab, spath
                model_term, ended = TERM_LOG_LIKELIHOOD_DECREASED, True
                rep.states.append((estimate, None if ab is None else ab.copy(), path.copy()))
                continue
            xg = np.asarray(e["x"], dtype=np.float64)
            M, c, info, dab_r = _system(r, li, lam, photometric, mut)
            if np.isfinite(e["A"]).all():
                rep.note("A", np.abs(e["A"] - info).max() / np.abs(info).max(), bounds.A, idx)
            if np.isfinite(xg).all():
                eta = np.abs(M @ xg - c).max() / (np.abs(M).sum(axis=1).max() * np.abs(xg).max() + np.abs(c).max())
                rep.note("x", eta, bounds.tau, idx)
                x = xg                                                                            # :995-996
            if photometric:
                dab = dab_r
            prev_nll, prev_P = e["nll"], Pg
            iteration += 1                                                                        # :1004
            rep.states.append((estimate, None if ab is None else ab.copy(), path.copy()))
            if not (np.abs(x).max() > precision and iteration < max_it):                         # :1005
                ended = True
        if not ended:
            rep.failures.append(("decision", k0 + count - 1, f"level {level}: the loop goes on after {count} entries"))
        if np.abs(x).max() <= precision:                                                         # :1007
            model_term = TERM_INCREMENT_TOO_SMALL
        if iteration >= max_it:                                                                  # :1008
            model_term = TERM_ITERATIONS_EXCEEDED
        if model_term != term:
            rep.failures.append(("decision", k0 + count - 1, f"level {level}: termination {term}, replayed {model_term}"))
        k0 += count
    rep.T = se3_inv(estimate)
    rep.note("pose", np.abs(rep.T - np.asarray(log.T)).max(), bounds.pose, -1)
    if photometric:
        rep.ab = ab
        if log.ab is not None:
            rep.note("ab", ab_error(log.ab, ab, path), bounds.ab, -1, f"({log.ab} vs {ab}, path {path})")
    return rep


# ---- the cases both test files replay -----------------------------------------------------------------------------------
# name -> builder; every case is a dict: images, K, levels, cfg (Config fields), T_init, estimator ("reference" or
# "corrected"), photometric, ab0 (photometric_init or None), prior (6 x 6 or None), mask (both roles, or None)
PHOTOMETRIC_SCENE = dict(width=320, height=240, scale=2)
EXPOSURES = [(1.1, 0.0), (0.9, 5.0), (1.2, -15.0), (1.0, 0.0)]      # tests/test_gpu_photometric.py
PRIOR_DELTA = np.array([4e-3, -3e-3, 2e-3, -2e-3, 3e-3, 1e-3])       # tests/test_gpu_prior.py
PRIOR_MU = 1e8   # Lambda = mu I: ~1e-3 of A's diagonal at level 0, so that the information tells it from A alone


def _base(**kw):
    c = dict(T_init=None, estimator="reference", photometric=False, ab0=None, prior=None, mask=None)
    c.update(kw)
    return c


def _synth_case(seed, scfg, levels, cfg, **kw):
    from dvo_slam_b200 import synth
    p = synth.make_pair(seed, scfg)
    return _base(I_ref=p["I_ref"].numpy(), Z_ref=p["Z_ref"].numpy(), I_cur=p["I_cur"].numpy(), Z_cur=p["Z_cur"].numpy(),
                 K=p["intrinsics"], levels=levels, cfg=cfg, pair=p, **kw)


def _scene320():
    from dvo_slam_b200 import synth
    return synth.SceneConfig(width=320, height=240, intrinsics=tuple(v / 2 for v in synth.FR1_INTRINSICS))


def _photometric(k, estimator, mask=False, ab0=None):
    from dvo_slam_b200 import synth
    c = _synth_case(k, _scene320(), 3, dict(first_level=2, last_level=0, max_iterations_per_level=50, precision=1e-4),
                    estimator=estimator, photometric=True, ab0=ab0)
    c["I_cur"] = synth.exposure(c["I_cur"], *EXPOSURES[k])
    if mask:
        m = np.ones((240, 320), np.uint8)
        m[50:120, 60:150] = 0
        m[170:200, 200:300] = 0
        c["mask"] = m
    return c


def _prior(k, lam, photometric=False):
    from dvo_slam_b200 import synth
    c = _synth_case(60 + k, _scene320(), 3, dict(first_level=2, last_level=0, max_iterations_per_level=50, precision=1e-4,
                                                  use_initial_estimate=1), photometric=photometric, prior=lam)
    c["T_init"] = synth.se3_exp(PRIOR_DELTA * (1 + 0.3 * k)) @ c["pair"]["T_true"]
    return c


def _spd(seed, scale):
    M = np.random.default_rng(seed).standard_normal((6, 6))
    S = (M @ M.T + 0.5 * np.eye(6)) * scale
    return 0.5 * (S + S.T)


def _rank_one(scale):
    e = np.array([1.0, -0.5, 0.25, 0.02, -0.01, 0.03])
    e /= np.linalg.norm(e)
    return scale * np.outer(e, e)


def _statistics(name, estimator):
    from helpers import statistics_case
    c = _base(**statistics_case(name))
    c["estimator"] = estimator
    return c


def _thresholds():
    from helpers import golden_case
    c = _base(**golden_case(11, intensity_derivative_threshold=4.0, depth_derivative_threshold=0.02))   # "moderate"
    return c


def _bench640():
    return _synth_case(3, None, 5, dict(first_level=4, last_level=0, max_iterations_per_level=50, precision=1e-4))


def _bench1280():
    from dvo_slam_b200 import synth
    return _synth_case(41, synth.SceneConfig().scaled(2), 6,
                       dict(first_level=5, last_level=0, max_iterations_per_level=50, precision=1e-4, mu=0.05))


def _cases():
    from helpers import STATISTICS_CASES
    out = {}
    for est in ("reference", "corrected"):
        for name in STATISTICS_CASES:
            out[f"{est}/{name}"] = (lambda n=name, e=est: _statistics(n, e))
    out["reference/thresholds"] = _thresholds
    for est in ("reference", "corrected"):
        for k in range(4):
            out[f"photometric-{est}/exposure{k}"] = (lambda k=k, e=est: _photometric(k, e, mask=(k == 1),
                                                                                     ab0=(1.15, -12.0) if k == 2 else None))
    out["prior/spd1e9"] = lambda: _prior(0, _spd(3, 1e9))
    out["prior/rank_one1e12"] = lambda: _prior(2, _rank_one(1e12))
    out["prior/mu"] = lambda: _prior(3, PRIOR_MU * np.eye(6))
    out["prior-photometric/spd1e9"] = lambda: _prior(0, _spd(3, 1e9), photometric=True)
    out["prior-photometric/mu"] = lambda: _prior(3, PRIOR_MU * np.eye(6), photometric=True)
    out["reference/bench640"] = _bench640
    out["reference/bench1280"] = _bench1280
    return out


CASES = _cases()


def case(name):
    return CASES[name]()


def mode_of(c):
    """the reference's mode for the case's estimator: MIRROR, or helpers.corrected_mode"""
    from helpers import corrected_mode
    from oracle import oracle_py as orc
    return orc.mode("mirror") if c["estimator"] == "reference" else corrected_mode(orc)


def _oracle_pyramids(c):
    """the oracle's pyramids of case c, its mask (if any) in both roles"""
    from masked_oracle import masked_pyramid
    from oracle import oracle_py as orc
    return (masked_pyramid(orc, c["I_ref"], c["Z_ref"], c["K"], c["levels"], c["mask"]),
            masked_pyramid(orc, c["I_cur"], c["Z_cur"], c["K"], c["levels"], c["mask"]))


def oracle_linearize(c):
    """the reference linearisation callback of replay() for case c (ab is None outside the photometric mode)"""
    from oracle import oracle_py as orc
    m = mode_of(c)
    ti = float(c["cfg"].get("intensity_derivative_threshold", 0.0))
    td = float(c["cfg"].get("depth_derivative_threshold", 0.0))
    oref, ocur = _oracle_pyramids(c)
    return lambda level, T, ab, uw, pp: orc.linearize(oref, ocur, level, T, m, uw, pp, ti, td, ab=ab)


def oracle_log(c):
    """the oracle's own match of case c, with its iteration log"""
    from oracle import oracle_py as orc
    oref, ocur = _oracle_pyramids(c)
    return as_log(orc.match(oref, ocur, orc.config(**c["cfg"]), mode_of(c), T_init=c["T_init"], prior=c["prior"],
                            photometric=c["photometric"], ab_init=c["ab0"]))


def replay_case(c, log, bounds=Bounds(), mutation=None, linearize=None):
    return replay(log, c["cfg"], linearize or oracle_linearize(c), T0=c["T_init"], mu=c["cfg"].get("mu", 0.0), prior=c["prior"],
                  photometric=c["photometric"], ab0=c["ab0"], bounds=bounds, mutation=mutation)
