"""Every alignment mode with device outputs and over several GPUs: 512 pairs of 640x480 frames, levels 4..0, 50 iterations,
precision 1e-4, pyramids resident, the current frames under an exposure change (gain 1.1, bias -6).  Modes: photometric,
prior (a dense positive definite Lambda per pair), maps (photometric + prior with the weight maps and mask) and the
multi-hypothesis alignment at k = 4, s = 3.  Arms, alternated round by round, each timed with a host clock around work that
ends in a device synchronisation:
  one process (default)  on GPU 0, the host-output call of each mode against dvo_b200_match_batch_modes_device into
                         preallocated torch tensors; then dvo_b200_match_batch_modes_sharded over every visible GPU against
                         one shard on GPU 0.
  --distributed          under torchrun, one rank per GPU: each rank runs its shard (distributed.shard_range) through
                         match_batch_modes_device and all-gathers the results, (alpha, beta), best and scores with NCCL,
                         inside the timed region.
Prints the card's name, power limit and maximum SM clock with every JSON line: ms per call (median over rounds) and
alignments/s."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from dvo_slam_b200 import synth  # noqa: E402
from dvo_slam_b200.engine import Config, Engine, ShardedEngine  # noqa: E402

MODES = ("photometric", "prior", "maps", "hypotheses")
K, S = 4, 3


def _card(device=0):
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(device), "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, check=True).stdout.strip()
        return out
    except (OSError, subprocess.CalledProcessError):
        import torch
        return torch.cuda.get_device_name(device) + ", power limit not read"


def _lambda(rng):
    M = rng.normal(size=(6, 6)) * np.sqrt(np.r_[[2e4] * 3, [2e5] * 3])[:, None]
    L = M @ M.T + np.diag(np.r_[[1e3] * 3, [1e4] * 3])
    return 0.5 * (L + L.T)


def _workload(n, seed=0):
    rng = np.random.default_rng(seed)
    twists = rng.normal(0, 0.01, size=(n, K, 6))
    H = np.stack([np.stack([np.eye(4)] + [synth.se3_exp(twists[p, j]) for j in range(1, K)]) for p in range(n)])
    lam = np.stack([_lambda(rng) for _ in range(n)])
    cfg = Config(first_level=4, last_level=0, max_iterations_per_level=50, precision=1e-4, use_initial_estimate=1)
    return H, lam, cfg


def _pyramids(eng, distinct):
    refs, curs = [], []
    for s in range(distinct):
        p = synth.make_pair(s)
        refs.append(eng.pyramid(p["I_ref"].numpy(), p["Z_ref"].numpy(), synth.FR1_INTRINSICS, 5))
        curs.append(eng.pyramid(synth.exposure(p["I_cur"].numpy(), 1.1, -6.0), p["Z_cur"].numpy(), synth.FR1_INTRINSICS, 5))
    return refs, curs


def _kwargs(mode, H, lam):
    """ShardedEngine.match_batch_modes / the modes arguments of one mode"""
    if mode == "hypotheses":
        return dict(hypotheses=H, screen_level=S)
    kw = dict(T_init=H[:, 0])
    if mode in ("photometric", "maps"):
        kw["photometric"] = True
    if mode in ("prior", "maps"):
        kw["prior_information"] = lam
    if mode == "maps":
        kw["mask_weight"] = 0.3
    return kw


def _host_call(eng, R, Cu, cfg, mode, H, lam):
    if mode == "hypotheses":
        return eng.match_batch_hypotheses(R, Cu, H, S, 0.0, cfg)
    if mode == "maps":
        return eng.match_batch_maps(R, Cu, cfg, H[:, 0], prior_information=lam, photometric=True, mask_weight=0.3)
    if mode == "prior":
        return eng.match_batch(R, Cu, cfg, H[:, 0], prior_information=lam)
    return eng.match_batch_photometric(R, Cu, cfg, H[:, 0])


def _device_call(eng, R, Cu, cfg, mode, H, lam, out):
    kw = _kwargs(mode, H, lam)
    kw.pop("photometric", None)
    kw.pop("mask_weight", None)
    eng.match_batch_modes_device(R, Cu, cfg, out, min_constraint_ratio=0.0, **kw)


def _outputs(eng, R, cfg, mode):
    return eng.device_outputs(R, cfg, K if mode == "hypotheses" else 0, photometric=mode in ("photometric", "maps"),
                              mask_weight=0.3 if mode == "maps" else None)


def _timed(arms, rounds, sync):
    times = {a: [] for a in arms}
    for rnd in range(rounds + 1):
        for a, fn in arms.items():
            sync()
            t0 = time.perf_counter()
            fn()
            sync()
            if rnd > 0:   # round 0 warms every shape up
                times[a].append(time.perf_counter() - t0)
    return {a: float(np.median(v)) for a, v in times.items()}, times


def one_process(args):
    import torch
    ndev = torch.cuda.device_count()
    H, lam, cfg = _workload(args.pairs)
    n = args.pairs
    engines = [Engine(device=d) for d in range(ndev)]
    pyr = [_pyramids(e, args.distinct) for e in engines]
    idx = [i % args.distinct for i in range(n)]
    eng = engines[0]
    R, Cu = [pyr[0][0][i] for i in idx], [pyr[0][1][i] for i in idx]
    outs = {m: _outputs(eng, R, cfg, m) for m in MODES}
    many, one = ShardedEngine(list(range(ndev))), ShardedEngine([0])
    # the sharded arm over every GPU: pair i from the pyramids of the device of the shard that owns it
    owner = [next(s for s in range(ndev) if many.shard_range(n, s)[0] <= i < many.shard_range(n, s)[1]) for i in range(n)]
    Rm, Cm = [pyr[owner[i]][0][idx[i]] for i in range(n)], [pyr[owner[i]][1][idx[i]] for i in range(n)]
    arms = {}
    for m in MODES:
        arms[("host", m)] = lambda m=m: _host_call(eng, R, Cu, cfg, m, H, lam)
        arms[("device", m)] = lambda m=m: (_device_call(eng, R, Cu, cfg, m, H, lam, outs[m]), eng.synchronize())
        if ndev > 1:
            arms[(f"sharded_{ndev}", m)] = lambda m=m: many.match_batch_modes(Rm, Cm, cfg, **_kwargs(m, H, lam))
        arms[("sharded_1", m)] = lambda m=m: one.match_batch_modes(R, Cu, cfg, **_kwargs(m, H, lam))
    med, times = _timed(arms, args.rounds, lambda: [e.synchronize() for e in engines])
    card = [_card(d) for d in range(ndev)]
    lines = []
    for (arm, m), t in med.items():
        lines.append({"arm": arm, "mode": m, "gpus": int(arm.split("_")[1]) if arm.startswith("sharded") else 1, "pairs": n,
                      "ms": round(1e3 * t, 3), "alignments_per_s": round(n / t, 1),
                      "ms_all": [round(1e3 * x, 3) for x in times[(arm, m)]], "card": card})
    return lines


def distributed(args):
    import torch
    import torch.distributed as dist
    from dvo_slam_b200.distributed import all_gather_results, shard_range
    dist.init_process_group("nccl")
    rank, ws = dist.get_rank(), dist.get_world_size()
    torch.cuda.set_device(rank)
    H, lam, cfg = _workload(args.pairs)
    b, e = shard_range(args.pairs, ws, rank)
    eng = Engine(device=rank)
    refs, curs = _pyramids(eng, args.distinct)
    idx = [i % args.distinct for i in range(b, e)]
    R, Cu = [refs[i] for i in idx], [curs[i] for i in idx]
    lines = []
    for m in MODES:
        out = _outputs(eng, R, cfg, m)

        def step():   # the all-gathers run on torch's current stream, which the device call orders after its work
            _device_call(eng, R, Cu, cfg, m, H[b:e], lam[b:e], out)
            gathered = [all_gather_results(out["results"], args.pairs)]
            if "photometric" in out:
                gathered.append(all_gather_results(out["photometric"], args.pairs))
            if "best" in out:
                gathered.append(all_gather_results(out["best"].view(-1, 1), args.pairs))
                gathered.append(all_gather_results(out["scores"], args.pairs))
            torch.cuda.synchronize()
            return gathered

        med, times = _timed({m: step}, args.rounds, lambda: (eng.synchronize(), dist.barrier()))
        lines.append({"arm": "distributed_device_allgather", "mode": m, "gpus": ws, "rank": rank, "pairs": args.pairs,
                      "ms": round(1e3 * med[m], 3), "alignments_per_s": round(args.pairs / med[m], 1),
                      "ms_all": [round(1e3 * x, 3) for x in times[m]], "card": _card(rank)})
    dist.destroy_process_group()
    return lines if rank == 0 else []


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=512)
    ap.add_argument("--distinct", type=int, default=64, help="distinct seeded pairs, repeated to fill the batch")
    ap.add_argument("--rounds", type=int, default=5, help="timed rounds after one warm-up round")
    ap.add_argument("--distributed", action="store_true", help="one rank per GPU under torchrun")
    ap.add_argument("--out", default=None, help="also write the JSON lines to this file")
    args = ap.parse_args()
    lines = distributed(args) if args.distributed else one_process(args)
    for line in lines:
        print(json.dumps(line))
    if args.out and lines:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write("".join(json.dumps(line) + "\n" for line in lines))


if __name__ == "__main__":
    main()
