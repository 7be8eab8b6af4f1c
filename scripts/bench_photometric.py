"""Cost and accuracy of the photometric mode (include/dvo_b200.h) at bench.py's workload: 512 pairs of 640x480 frames, levels
4..0, 50 iterations, precision 1e-4.  Every current frame gets an exposure change (gain in [0.85, 1.15], bias in [-15, 15]).
Arms: the default mode and the photometric mode, on the changed and the unchanged frames, alternated round by round and timed
with CUDA events.  Prints one JSON line per arm: ms per step, iterations per alignment, ns per pixel-iteration (the kernel time
over the sum, over pairs and levels, of the level's pixels times the pair's iterations on it), and the median / max pose error
against the truth.  --label names the build in the output (the occupancy of the photometric instances is a build setting,
DVO_AFFINE_CTAS_PER_SM in csrc/tracker.cu)."""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from dvo_slam_b200 import synth  # noqa: E402
from dvo_slam_b200.engine import Config, Engine  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=512)
    ap.add_argument("--distinct", type=int, default=64)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--label", default="")
    args = ap.parse_args()
    rng = np.random.default_rng(0)
    eng = Engine(device=0)
    K = synth.FR1_INTRINSICS
    refs, cur_same, cur_exp, truth = [], [], [], []
    for s in range(args.distinct):
        p = synth.make_pair(s)
        g, b = rng.uniform(0.85, 1.15), rng.uniform(-15, 15)
        refs.append(eng.pyramid(p["I_ref"].numpy(), p["Z_ref"].numpy(), K, 5))
        cur_same.append(eng.pyramid(p["I_cur"].numpy(), p["Z_cur"].numpy(), K, 5))
        cur_exp.append(eng.pyramid(synth.exposure(p["I_cur"].numpy(), g, b), p["Z_cur"].numpy(), K, 5))
        truth.append(p["T_true"])
    idx = [i % args.distinct for i in range(args.pairs)]
    R = [refs[i] for i in idx]
    cfg = Config(first_level=4, last_level=0, max_iterations_per_level=50, precision=1e-4)
    arms = {(m, f): [] for m in ("default", "photometric") for f in ("unchanged", "changed")}
    out = {}
    for rnd in range(args.rounds + 1):
        for (m, f) in arms:
            C_ = [(cur_exp if f == "changed" else cur_same)[i] for i in idx]
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record()
            res = eng.match_batch(R, C_, cfg) if m == "default" else eng.match_batch_photometric(R, C_, cfg)[0]
            e1.record()
            torch.cuda.synchronize()
            if rnd == 0:
                continue   # warm-up round
            arms[(m, f)].append(e0.elapsed_time(e1))
            its = np.mean([r.num_iterations_total for r in res])
            pix_its = sum((640 >> lv["id"]) * (480 >> lv["id"]) * lv["num_iterations"] for r in res for lv in r.levels)
            errs = []
            for r, i in zip(res, idx):
                d = synth.se3_log(truth[i] @ r.transformation)
                errs.append((np.abs(d[:3]).max(), np.abs(d[3:]).max()))
            errs = np.array(errs)
            out[(m, f)] = {"iterations_per_alignment": float(its), "pixel_iterations": int(pix_its), "dt_median": float(np.median(errs[:, 0])),
                           "dt_max": float(errs[:, 0].max()), "dr_median": float(np.median(errs[:, 1])), "dr_max": float(errs[:, 1].max())}
    for (m, f), ms in arms.items():
        o = out[(m, f)]
        o.update({"label": args.label, "mode": m, "frames": f, "ms_per_step": float(np.median(ms)), "ms_all": [round(x, 3) for x in ms],
                  "ns_per_pixel_iteration": float(np.median(ms)) * 1e6 / o["pixel_iterations"]})
        print(json.dumps(o))


if __name__ == "__main__":
    main()
