"""Cost of multi-hypothesis alignment in the photometric mode and with a motion prior (dvo_b200_match_batch_hypotheses_modes)
at the workload of scripts/bench_hypotheses.py: 512 pairs of 640x480 frames, levels 4..0, 50 iterations, precision 1e-4,
pyramids resident, the current frames under an exposure change (gain 1.1, bias -6).  Pair p is started from k hypotheses: the
identity and k - 1 small random twists around it, each with (alpha, beta)_0 = (1, 0) in the photometric arms and a full
(dense, positive definite) Lambda in the prior arms, screened on levels 4..s and continued from the best.  Arms, alternated
round by round in one session, each timed with a host clock around the call (which ends in a device synchronisation):
  photometric       match_batch_photometric from the identity, and the photometric hypotheses for k in {1, 2, 4, 8}, s in {4, 3};
  prior             match_batch_prior from the identity with the first Lambda, and the prior hypotheses likewise;
  maps              the photometric + prior hypotheses at k = 4, s = 3, without and with the weight maps (device memory, with the
                    mask) of the continuation, and match_batch_maps against match_batch_prior in the same mode.
Prints the card's name, power limit and maximum SM clock, then one JSON line per arm: ms per call (median over rounds),
alignments/s, and the time relative to the single-start call of its mode."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from dvo_slam_b200 import synth  # noqa: E402
from dvo_slam_b200.engine import Config, Engine  # noqa: E402

KS = (1, 2, 4, 8)
SCREEN_LEVELS = (4, 3)


def _card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, check=True).stdout.strip()
    except (OSError, subprocess.CalledProcessError):
        import torch
        return torch.cuda.get_device_name(0)


def _lambda(rng):
    """a dense symmetric positive definite 6 x 6 of the order of an alignment's normal equations at level 0"""
    M = rng.normal(size=(6, 6)) * np.sqrt(np.r_[[2e4] * 3, [2e5] * 3])[:, None]
    L = M @ M.T + np.diag(np.r_[[1e3] * 3, [1e4] * 3])
    return 0.5 * (L + L.T)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=512)
    ap.add_argument("--distinct", type=int, default=64, help="distinct seeded pairs, repeated to fill the batch")
    ap.add_argument("--rounds", type=int, default=5, help="timed rounds after one warm-up round")
    ap.add_argument("--out", default=None, help="also write the JSON lines to this file")
    args = ap.parse_args()
    rng = np.random.default_rng(0)
    eng = Engine(device=0)
    K = synth.FR1_INTRINSICS
    refs, curs = [], []
    for s in range(args.distinct):
        p = synth.make_pair(s)
        refs.append(eng.pyramid(p["I_ref"].numpy(), p["Z_ref"].numpy(), K, 5))
        curs.append(eng.pyramid(synth.exposure(p["I_cur"].numpy(), 1.1, -6.0), p["Z_cur"].numpy(), K, 5))
    idx = [i % args.distinct for i in range(args.pairs)]
    R, Cu = [refs[i] for i in idx], [curs[i] for i in idx]
    n, kmax = args.pairs, max(KS)
    twists = rng.normal(0, [0.01] * 3 + [0.01] * 3, size=(n, kmax, 6))
    H = np.stack([np.stack([np.eye(4)] + [synth.se3_exp(twists[p, j]) for j in range(1, kmax)]) for p in range(n)])
    lam = np.stack([np.stack([_lambda(rng) for _ in range(kmax)]) for _ in range(n)])
    cfg = Config(first_level=4, last_level=0, max_iterations_per_level=50, precision=1e-4, use_initial_estimate=1)
    T0 = H[:, 0]

    def run(arm):
        mode, k, s = arm
        if mode == "photometric_single":
            return eng.match_batch_photometric(R, Cu, cfg, T0)[0]
        if mode == "prior_single":
            return eng.match_batch(R, Cu, cfg, T0, prior_information=lam[:, 0])
        if mode == "maps_single":
            return eng.match_batch_maps(R, Cu, cfg, T0, prior_information=lam[:, 0], photometric=True, mask_weight=0.3)[0]
        if mode == "prior_photometric_single":
            return eng.match_batch_photometric(R, Cu, cfg, T0, prior_information=lam[:, 0])[0]
        photometric = mode in ("photometric", "both", "both_maps")
        prior = lam[:, :k] if mode in ("prior", "both", "both_maps") else None
        maps = mode == "both_maps"
        return eng.match_batch_hypotheses(R, Cu, H[:, :k], s, 0.0, cfg, prior_information=prior, photometric=photometric, maps=maps,
                                          mask_weight=0.3 if maps else None)[0]

    arms = [("photometric_single", None, None), ("prior_single", None, None)]
    arms += [(m, k, s) for m in ("photometric", "prior") for s in SCREEN_LEVELS for k in KS]
    arms += [("prior_photometric_single", None, None), ("maps_single", None, None), ("both", 4, 3), ("both_maps", 4, 3)]
    times = {a: [] for a in arms}
    for rnd in range(args.rounds + 1):
        single = {}
        for a in arms:
            eng.synchronize()
            t0 = time.perf_counter()
            res = run(a)
            t1 = time.perf_counter()
            mode, k, _ = a
            if mode.endswith("_single"):
                single[mode] = res
            elif k == 1:   # one hypothesis is the single-start call of its mode
                want = single["photometric_single" if mode == "photometric" else "prior_single"]
                assert all(np.array_equal(x.transformation, y.transformation) for x, y in zip(res, want)), f"k = 1 differs: {a}"
            if rnd > 0:    # round 0 warms every shape up
                times[a].append(t1 - t0)
    lines = [{"card": _card(), "workload": f"{n} pairs ({args.distinct} distinct) 640x480, exposure (1.1, -6), levels 4..0, "
              "50 iterations, precision 1e-4", "rounds": args.rounds}]
    med = {a: float(np.median(times[a])) for a in arms}
    base = {"photometric": med[arms[0]], "prior": med[arms[1]], "both": med[("prior_photometric_single", None, None)],
            "both_maps": med[("prior_photometric_single", None, None)], "maps_single": med[("prior_photometric_single", None, None)]}
    for a in arms:
        mode, k, s = a
        line = {"arm": mode, "k": k, "screen_level": s, "ms": round(1e3 * med[a], 3), "alignments_per_s": round(n / med[a], 1),
                "ms_all": [round(1e3 * x, 3) for x in times[a]]}
        if mode in base:
            line["relative_to_single_start"] = round(med[a] / base[mode], 4)
        lines.append(line)
    for line in lines:
        print(json.dumps(line))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write("".join(json.dumps(line) + "\n" for line in lines))


if __name__ == "__main__":
    main()
