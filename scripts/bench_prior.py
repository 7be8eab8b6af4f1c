"""Cost of the motion prior (dvo_b200_match_batch_prior) at bench.py's workload: 512 pairs of 640x480 frames, levels 4..0, 50
iterations, precision 1e-4, initial estimates perturbed from the truth.  Arms, alternated round by round and timed with CUDA
events: match_batch with mu = 0.05; the prior entry with Lambda = 0.05 I (its results are checked to equal the first arm's);
the prior entry with a full SPD Lambda per pair; and the photometric twins of the three.  Prints the card's name and power
limit, then one JSON line per arm: ms per step (median over rounds) and iterations per alignment."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from dvo_slam_b200 import synth  # noqa: E402
from dvo_slam_b200.engine import Config, Engine  # noqa: E402


def _card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, check=True).stdout.strip()
    except (OSError, subprocess.CalledProcessError):
        return torch.cuda.get_device_name(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=512)
    ap.add_argument("--distinct", type=int, default=64)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    rng = np.random.default_rng(0)
    eng = Engine(device=0)
    K = synth.FR1_INTRINSICS
    refs, curs, T0 = [], [], []
    for s in range(args.distinct):
        p = synth.make_pair(s)
        refs.append(eng.pyramid(p["I_ref"].numpy(), p["Z_ref"].numpy(), K, 5))
        curs.append(eng.pyramid(p["I_cur"].numpy(), p["Z_cur"].numpy(), K, 5))
        T0.append(synth.se3_exp(rng.normal(0, [5e-3] * 3 + [3e-3] * 3)) @ p["T_true"])
    idx = [i % args.distinct for i in range(args.pairs)]
    R, C_, T = [refs[i] for i in idx], [curs[i] for i in idx], [T0[i] for i in idx]
    full = []
    for _ in range(args.distinct):
        M = rng.standard_normal((6, 6))
        S = (M @ M.T + 0.5 * np.eye(6)) * 1e8
        full.append(0.5 * (S + S.T))
    full = np.stack([full[i] for i in idx])
    scalar = np.stack([0.05 * np.eye(6)] * args.pairs)
    mu_cfg = Config(first_level=4, last_level=0, max_iterations_per_level=50, precision=1e-4, use_initial_estimate=1, mu=0.05)
    cfg = Config(first_level=4, last_level=0, max_iterations_per_level=50, precision=1e-4, use_initial_estimate=1)

    def run(photometric, c, prior):
        if photometric:
            return eng.match_batch_photometric(R, C_, c, T, prior_information=prior)[0]
        return eng.match_batch(R, C_, c, T, prior_information=prior)

    arms = {(m, a): [] for m in ("default", "photometric") for a in ("mu=0.05", "Lambda=0.05I", "Lambda full SPD")}
    its = {}
    for rnd in range(args.rounds + 1):
        last = {}
        for (m, a) in arms:
            ph = m == "photometric"
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record()
            res = run(ph, mu_cfg, None) if a == "mu=0.05" else run(ph, cfg, scalar if a == "Lambda=0.05I" else full)
            e1.record()
            torch.cuda.synchronize()
            last[(m, a)] = res
            if a == "Lambda=0.05I":
                base = last[(m, "mu=0.05")]
                assert all(np.array_equal(x.transformation, y.transformation) and np.array_equal(x.information, y.information)
                           for x, y in zip(res, base)), "Lambda = mu I differs from the mu path"
            if rnd == 0:
                continue   # warm-up round
            arms[(m, a)].append(e0.elapsed_time(e1))
            its[(m, a)] = float(np.mean([r.num_iterations_total for r in res]))
    print(json.dumps({"card": _card()}))
    for (m, a), ms in arms.items():
        print(json.dumps({"mode": m, "arm": a, "ms_per_step": float(np.median(ms)), "ms_all": [round(x, 3) for x in ms],
                          "iterations_per_alignment": its[(m, a)]}))


if __name__ == "__main__":
    main()
