"""Resident throughput of one estimator (dvo_b200_estimator) at bench.py's workload, on one GPU.

    python scripts/bench_estimator.py --estimator corrected --steps 20 --warmup 3
    python scripts/bench_estimator.py --estimator reference --config 5 --dump-outputs /tmp/out

The same seeded pairs, configuration and timing as bench.py's resident `value` (CUDA events on the engine's stream, 512
pyramids resident in HBM, one dvo_b200_match_batch per step), on a context set to the chosen estimator.  Prints one JSON
line: alignments/s, ms per step, k_level_persistent time per step, mean iterations per alignment, pixel-iterations per step,
ns per pixel-iteration, the roofline fraction as bench.py defines it (against the 3 350 GB/s data-sheet peak), and the
sampled SM clock.  Writes nothing except the
--dump-outputs directory (bench.py's format)."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (bench.py: workload constants, scene, clock sampler, output dump)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--estimator", default="corrected", choices=["reference", "corrected"])
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--batch", type=int, default=0, help="frame pairs (0 = bench.py's default for the workload)")
    ap.add_argument("--config", type=int, default=2, help="bench.py --config: 2 = 640x480x5 (default), 5 = 1280x960x6 mu=0.05")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None)
    args = ap.parse_args()
    if args.steps < 1 or args.warmup < 0:
        ap.error("--steps must be >= 1 and --warmup >= 0")
    bench.select_workload(args.config)

    import torch
    from dvo_slam_b200 import synth
    from dvo_slam_b200.engine import Config, Engine

    if not torch.cuda.is_available():
        raise SystemExit("bench_estimator.py needs a CUDA device (no CPU fallback)")
    dev = torch.device("cuda", 0)
    B = args.batch or bench.DEFAULT_BATCH
    W, H, L = bench.W, bench.H, bench.LEVELS
    eng = Engine(device=0, estimator=args.estimator)
    stream = torch.cuda.ExternalStream(eng.stream, device=dev)
    cfg = Config(first_level=bench.FIRST_LEVEL, last_level=bench.LAST_LEVEL, max_iterations_per_level=bench.MAX_IT,
                 precision=bench.PRECISION, mu=bench.MU)
    scfg = bench.scene_config()
    hI = torch.empty((2 * B, H, W), dtype=torch.float32).pin_memory()
    hZ = torch.empty((2 * B, H, W), dtype=torch.float32).pin_memory()
    for i in range(B):                              # bench.py's seeds (rank 0)
        p = synth.make_pair(i, scfg, device=dev)
        hI[i].copy_(p["I_ref"]); hZ[i].copy_(p["Z_ref"])
        hI[B + i].copy_(p["I_cur"]); hZ[B + i].copy_(p["Z_cur"])
    torch.cuda.synchronize()
    # float32 depth as bench.py feeds its resident leg: quantised to 1/5000 m like the raw images it derives from
    raw = torch.where(torch.isnan(hZ), torch.zeros_like(hZ), torch.round(hZ * 5000.0)).to(torch.int32)
    hZ.copy_(torch.where(raw == 0, torch.full_like(hZ, float("nan")), raw.to(torch.float32) * torch.tensor(1.0 / 5000.0, dtype=torch.float32)))
    del raw
    pyrs = eng.pyramid_batch(None, None, scfg.intrinsics, L, host_ptrs=(hI.data_ptr(), hZ.data_ptr(), 2 * B, H, W))
    refs, curs = pyrs[:B], pyrs[B:]
    eng.synchronize()

    last = {}

    def step():
        last["res"] = eng.match_batch(refs, curs, cfg, raw=True)

    for _ in range(args.warmup):
        step()
    eng.profile_read(reset=True)
    eng.profile_enable(True)
    sampler = bench.ClockSampler(0)
    sampler.start()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for _ in range(args.steps):
        step()
    e1.record(stream)
    torch.cuda.synchronize()
    clocks = sampler.stop()
    prof = eng.profile_read(reset=True)
    eng.profile_enable(False)
    ms_per_step = e0.elapsed_time(e1) / args.steps
    res = last["res"]
    pix_iters, iters = 0, 0
    for i in range(B):
        for l in range(res[i].num_levels):
            ls = res[i].levels[l]
            pix_iters += bench.LEVEL_PIXELS[ls.id] * ls.num_iterations
            iters += ls.num_iterations
    kernel_ms = (prof["residual"]["ms"] + prof["normal"]["ms"]) / args.steps
    achieved = bench.ALGO_BYTES_PER_PIXEL_ITERATION * pix_iters / (kernel_ms * 1e-3) / 1e9 if kernel_ms > 0 else 0.0
    if args.dump_outputs:
        bench.dump_outputs(args.dump_outputs, res)
    print(json.dumps({"estimator": args.estimator, "workload": f"batch={B} {W}x{H}x{L}", "steps": args.steps,
                      "value": B / (ms_per_step * 1e-3), "unit": "alignments/s", "ms_per_step": ms_per_step,
                      "kernel_ms_per_step": kernel_ms, "iterations_per_alignment_mean": iters / B,
                      "pixel_iterations_per_step": pix_iters,
                      "ns_per_pixel_iteration": kernel_ms * 1e6 / pix_iters if pix_iters else None,
                      "roofline_frac": achieved / bench.H100_HBM_GBS, "clocks": clocks}))


if __name__ == "__main__":
    main()
