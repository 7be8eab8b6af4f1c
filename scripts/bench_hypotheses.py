"""Cost of multi-hypothesis alignment (dvo_b200_match_batch_hypotheses) at bench.py's workload: 512 pairs of 640x480 frames,
levels 4..0, 50 iterations, precision 1e-4, mu 0, pyramids resident.  Pair p is started from k hypotheses: the identity (what
bench.py starts from) and k - 1 small random twists around it, screened on levels 4..s and continued from the best.  Arms,
alternated round by round in one session, each timed with a host clock around the call (which ends in a device
synchronisation): dvo_b200_match_batch from the identity, and the hypotheses entry for every k in {1, 2, 4, 8, 16} and
s in {4, 3}.  Prints the card's name, power limit and maximum SM clock, then one JSON line per arm: ms per call (median over
rounds), alignments/s (pairs / median), the time relative to match_batch, and for k > 1 the measured cost of one more
hypothesis as a share of the match_batch time, (t_k - t_1) / (k - 1) / t_match_batch."""
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

KS = (1, 2, 4, 8, 16)
SCREEN_LEVELS = (4, 3)


def _card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, check=True).stdout.strip()
    except (OSError, subprocess.CalledProcessError):
        import torch
        return torch.cuda.get_device_name(0)


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
        curs.append(eng.pyramid(p["I_cur"].numpy(), p["Z_cur"].numpy(), K, 5))
    idx = [i % args.distinct for i in range(args.pairs)]
    R, Cu = [refs[i] for i in idx], [curs[i] for i in idx]
    n = args.pairs
    twists = rng.normal(0, [0.01] * 3 + [0.01] * 3, size=(n, max(KS), 6))
    H = np.stack([np.stack([np.eye(4)] + [synth.se3_exp(twists[p, j]) for j in range(1, max(KS))]) for p in range(n)])
    cfg = Config(first_level=4, last_level=0, max_iterations_per_level=50, precision=1e-4, use_initial_estimate=1)
    T0 = H[:, 0]

    arms = [("match_batch", None, None)] + [("hypotheses", k, s) for s in SCREEN_LEVELS for k in KS]
    times = {a: [] for a in arms}
    for rnd in range(args.rounds + 1):
        base = None
        for a in arms:
            name, k, s = a
            eng.synchronize()
            t0 = time.perf_counter()
            if name == "match_batch":
                res = eng.match_batch(R, Cu, cfg, T0)
            else:
                res, best, _ = eng.match_batch_hypotheses(R, Cu, H[:, :k], s, 0.0, cfg)
            t1 = time.perf_counter()
            if name == "match_batch":
                base = res
            elif k == 1:   # one hypothesis is match_batch from it
                assert all(np.array_equal(x.transformation, y.transformation) for x, y in zip(res, base)), "k = 1 differs"
            if rnd > 0:    # round 0 warms every shape up
                times[a].append(t1 - t0)
    lines = [{"card": _card(), "workload": f"{n} pairs ({args.distinct} distinct) 640x480, levels 4..0, 50 iterations, precision 1e-4",
              "rounds": args.rounds}]
    t_base = float(np.median(times[arms[0]]))
    t_one = {s: float(np.median(times[("hypotheses", 1, s)])) for s in SCREEN_LEVELS}
    for a in arms:
        name, k, s = a
        t = float(np.median(times[a]))
        line = {"arm": name, "k": k, "screen_level": s, "ms": round(1e3 * t, 3), "alignments_per_s": round(n / t, 1),
                "relative_to_match_batch": round(t / t_base, 4), "ms_all": [round(1e3 * x, 3) for x in times[a]]}
        if name == "hypotheses" and k > 1:
            line["extra_hypothesis_share"] = round((t - t_one[s]) / (k - 1) / t_base, 4)
        lines.append(line)
    for line in lines:
        print(json.dumps(line))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write("".join(json.dumps(line) + "\n" for line in lines))


if __name__ == "__main__":
    main()
