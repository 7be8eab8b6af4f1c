"""Cost of masks in both roles: bench.py's flagship workload (512 pairs, 640x480, 5 levels) with no masks, with reference-role
masks and with masks in both roles (dvo_b200_pyramid_create_masked_batch_roles).  Every frame gets a seeded blob mask over a
few percent of the image, as scripts/bench_masked_build.py makes them.  The three arms alternate step by step.  Reports per
arm the level-kernel time per step (CUDA events of the profile), the event time of the whole step, the iterations per
alignment, ns per pixel-iteration, and the build time of the 2 x 512 masked frames per role set; with the card's name, power
limit and the SM clock sampled during the timed steps.  One JSON line on stdout; writes nothing else.

    python scripts/bench_current_mask.py [--steps 20] [--warmup 3]

For the share of stage-B tiles that took the generic loop because of the mask (cmask tiles), run it against a library built
with -DDVO_PIPE_TIMING (scripts/build_variant.sh timing -DDVO_PIPE_TIMING, then DVO_B200_LIB=dvo_slam_b200/variants/timing.so)
and DVO_B200_TIMING=1: dvo_b200_profile_read then prints the tile counts of each level-slot to stderr after every arm's steps.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402  (bench.py: workload constants, scene, clock sampler)
from scripts.bench_masked_build import card  # noqa: E402


def blob_masks(n, h, w, seed=0):
    rng = np.random.default_rng(seed)
    yy, xx = np.ogrid[:h, :w]
    out = np.ones((n, h, w), np.uint8)
    for i in range(n):
        for _ in range(4):   # a few blobs: a segmentation mask of people / a mount, glare
            cy, cx, r = rng.integers(0, h), rng.integers(0, w), rng.integers(15, 60)
            out[i][(yy - cy) ** 2 + (xx - cx) ** 2 <= r * r] = 0
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--build-reps", type=int, default=5)
    args = ap.parse_args()
    bench.select_workload(2)
    import torch
    from dvo_slam_b200 import synth
    from dvo_slam_b200.engine import Config, Engine

    if not torch.cuda.is_available():
        raise SystemExit("bench_current_mask.py needs a CUDA device (no CPU fallback)")
    dev = torch.device("cuda", 0)
    B, W, H, L = bench.DEFAULT_BATCH, bench.W, bench.H, bench.LEVELS
    eng = Engine(device=0)
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
    masks = torch.from_numpy(blob_masks(2 * B, H, W)).pin_memory()
    coverage = float(1.0 - masks.float().mean())
    ptrs = (hI.data_ptr(), hZ.data_ptr(), 2 * B, H, W)

    # build time of the masked batch per role set (event time of the create call: H2D copies + kernels)
    build_ms = {"reference": [], "both": []}
    for rep in range(1 + args.build_reps):
        for roles in build_ms:
            eng.synchronize()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(stream)
            pyrs = eng.pyramid_batch(None, None, scfg.intrinsics, L, host_ptrs=ptrs, masks=masks.data_ptr(), mask_roles=roles)
            b.record(stream)
            b.synchronize()
            if rep:
                build_ms[roles].append(a.elapsed_time(b))
            for p in pyrs:
                p.release()

    arms = {"none": eng.pyramid_batch(None, None, scfg.intrinsics, L, host_ptrs=ptrs),
            "reference": eng.pyramid_batch(None, None, scfg.intrinsics, L, host_ptrs=ptrs, masks=masks.data_ptr(), mask_roles="reference"),
            "both": eng.pyramid_batch(None, None, scfg.intrinsics, L, host_ptrs=ptrs, masks=masks.data_ptr(), mask_roles="both")}
    eng.synchronize()
    kernel_ms = {k: [] for k in arms}
    step_ms = {k: [] for k in arms}
    last = {}
    sampler = bench.ClockSampler(0)
    for s in range(args.warmup + args.steps):
        if s == args.warmup:
            sampler.start()
        for name, pyrs in arms.items():
            eng.synchronize()
            eng.profile_read(reset=True)
            eng.profile_enable(True)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            last[name] = eng.match_batch(pyrs[:B], pyrs[B:], cfg, raw=True)
            e1.record(stream)
            e1.synchronize()
            prof = eng.profile_read(reset=True)
            eng.profile_enable(False)
            if s >= args.warmup:
                kernel_ms[name].append(prof["residual"]["ms"] + prof["normal"]["ms"])
                step_ms[name].append(e0.elapsed_time(e1))
    clocks = sampler.stop()
    out = {"card": card(), "workload": f"batch={B} {W}x{H}x{L}", "steps": args.steps, "mask_coverage": coverage, "clocks": clocks,
           "build_ms_median": {k: float(np.median(v)) for k, v in build_ms.items()}}
    for name in arms:
        res = last[name]
        pix_iters, iters = 0, 0
        for i in range(B):
            for l in range(res[i].num_levels):
                ls = res[i].levels[l]
                pix_iters += bench.LEVEL_PIXELS[ls.id] * ls.num_iterations
                iters += ls.num_iterations
        km = np.asarray(kernel_ms[name])
        out[name] = {"kernel_ms_median": float(np.median(km)), "kernel_ms_min": float(km.min()), "kernel_ms_max": float(km.max()),
                     "step_ms_median": float(np.median(step_ms[name])), "iterations_per_alignment": iters / B,
                     "ns_per_pixel_iteration": float(np.median(km)) * 1e6 / pix_iters if pix_iters else None}
    for p in [q for v in arms.values() for q in v]:
        p.release()
    eng.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
