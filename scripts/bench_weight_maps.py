"""Cost of the weight maps (dvo_b200_match_batch_maps) at bench.py's workload: 512 pairs of 640x480 frames, levels 4..0, 50
iterations, precision 1e-4, initial estimates perturbed from the truth.  Three arms, alternated round by round and timed with
CUDA events: match_batch; match_batch_maps writing the weight map only; and match_batch_maps writing every output and the mask.
Then, in a separate profiled call per maps arm, k_weight_maps's own time (torch.profiler) and its achieved bytes/s from the
bytes it must move, counted here.  Prints the card's name and power limit, then one JSON line per arm."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from dvo_slam_b200 import synth  # noqa: E402
from dvo_slam_b200.engine import MAPS_MEMORY, CResult, Config, Engine, MapPlane, WeightMaps  # noqa: E402

W, H = 640, 480


def _card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, check=True).stdout.strip()
    except (OSError, subprocess.CalledProcessError):
        return torch.cuda.get_device_name(0)


def compulsory_bytes(n, full):
    """what k_weight_maps must move at level 0: per pixel the reference's (I, Zsel) record cell (8 B) and the current P0 (8 B,
    each tap read once), then the float32 planes it writes (4 B each) and with the mask one byte"""
    px = n * W * H
    return px * (8 + 8 + (12 + 1 if full else 4))


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
    n = args.pairs
    idx = [i % args.distinct for i in range(n)]
    R, C_, T = [refs[i] for i in idx], [curs[i] for i in idx], [T0[i] for i in idx]
    cfg = Config(first_level=4, last_level=0, max_iterations_per_level=50, precision=1e-4, use_initial_estimate=1)
    planes = {k: torch.empty((n, H, W), dtype=torch.float32, device="cuda") for k in ("weight", "residual_i", "residual_z")}
    mask = torch.empty((n, H, W), dtype=torch.uint8, device="cuda")
    est, prec = torch.empty((n, 16), dtype=torch.float64, device="cuda"), torch.empty((n, 4), dtype=torch.float32, device="cuda")

    def maps(full):
        m = WeightMaps()
        m.memory = MAPS_MEMORY["device"]
        m.weight = MapPlane(planes["weight"].data_ptr(), 4 * W, 4 * W * H)
        if full:
            m.residual_i = MapPlane(planes["residual_i"].data_ptr(), 4 * W, 4 * W * H)
            m.residual_z = MapPlane(planes["residual_z"].data_ptr(), 4 * W, 4 * W * H)
            m.mask = MapPlane(mask.data_ptr(), W, W * H)
            m.mask_weight = 0.3
            m.estimate = C.cast(est.data_ptr(), C.POINTER(C.c_double))
            m.precision = C.cast(prec.data_ptr(), C.POINTER(C.c_float))
        return m

    rh = (C.c_void_p * n)(*[p.handle for p in R])
    ch = (C.c_void_p * n)(*[p.handle for p in C_])
    Tn = np.ascontiguousarray(np.asarray(T, dtype=np.float64).reshape(n, 16))
    res = (CResult * n)()
    dp = C.POINTER(C.c_double)

    def run(arm):
        if arm == "match_batch":
            rc = eng.lib.dvo_b200_match_batch(eng.ctx, C.byref(cfg), n, rh, ch, Tn.ctypes.data_as(dp), res, None, 0)
        else:
            rc = eng.lib.dvo_b200_match_batch_maps(eng.ctx, C.byref(cfg), n, rh, ch, Tn.ctypes.data_as(dp), None, None, None, res, None, 0,
                                                   C.byref(maps(arm == "maps: every output + mask")))
        assert rc == 0, rc
        return [bytes(r) for r in res]

    arms = {a: [] for a in ("match_batch", "maps: weight", "maps: every output + mask")}
    for rnd in range(args.rounds + 1):
        out = {}
        for a in arms:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record()
            out[a] = run(a)
            e1.record()
            torch.cuda.synchronize()
            if rnd > 0:   # round 0 warms up
                arms[a].append(e0.elapsed_time(e1))
        assert out["maps: weight"] == out["match_batch"] == out["maps: every output + mask"], "results differ between arms"
    kernel_ms = {}
    for a, full in (("maps: weight", False), ("maps: every output + mask", True)):
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            run(a)
            torch.cuda.synchronize()
        kernel_ms[a] = sum(e.device_time_total for e in prof.key_averages() if "k_weight_maps" in e.key) / 1e3
    print(json.dumps({"card": _card(), "pairs": n, "size": [W, H]}))
    for a, ms in arms.items():
        line = {"arm": a, "ms_per_step": float(np.median(ms)), "ms_all": [round(x, 3) for x in ms]}
        if a in kernel_ms:
            b = compulsory_bytes(n, a.startswith("maps: every"))
            line.update({"k_weight_maps_ms": kernel_ms[a], "compulsory_bytes": b, "achieved_GBps": b / (kernel_ms[a] * 1e-3) / 1e9,
                         "bytes_bound_ms_at_3.35TBps": b / 3.35e12 * 1e3})
        print(json.dumps(line))


if __name__ == "__main__":
    main()
