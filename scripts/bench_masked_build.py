"""Cost of a reference mask in the pyramid build: 512 raw 640x480 frames (8-bit grey + 16-bit depth, pinned host memory),
5 levels, built with dvo_b200_pyramid_create_raw_batch and with dvo_b200_pyramid_create_masked_batch (random blob masks),
alternating.  Reports the CUDA-event time of one whole build (H2D copies + kernels) and its pyramid kernels alone, and the
H2D bytes per pixel, with the card's name and power limit.  One JSON line on stdout; writes nothing else.

    python scripts/bench_masked_build.py [--frames 512] [--reps 20] [--warmup 3]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=512)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--levels", type=int, default=5)
    args = ap.parse_args()
    import torch
    from dvo_slam_b200 import synth
    from dvo_slam_b200.engine import Engine

    n, h, w = args.frames, 480, 640
    K = synth.FR1_INTRINSICS
    rng = np.random.default_rng(0)
    grey = torch.empty((n, h, w), dtype=torch.uint8).pin_memory()
    depth = torch.empty((n, h, w), dtype=torch.int16).pin_memory()     # the bits of uint16 raw depth
    masks = torch.ones((n, h, w), dtype=torch.uint8).pin_memory()
    base = [synth.make_pair(s) for s in range(8)]
    yy, xx = np.ogrid[:h, :w]
    for i in range(n):
        p = base[i % 8]
        grey[i] = torch.from_numpy(p["I_ref"].numpy().astype(np.uint8))
        z = p["Z_ref"].numpy()
        depth[i] = torch.from_numpy(np.where(np.isnan(z), 0, np.round(z * 5000.0)).astype(np.uint16).view(np.int16))
        m = np.ones((h, w), np.uint8)
        for _ in range(6):   # a few blobs: a segmentation mask of people / a mount
            cy, cx, r = rng.integers(0, h), rng.integers(0, w), rng.integers(20, 90)
            m[(yy - cy) ** 2 + (xx - cx) ** 2 <= r * r] = 0
        masks[i] = torch.from_numpy(m)

    stream = torch.cuda.Stream()
    eng = Engine(device=0, stream=stream.cuda_stream)
    ptrs = (grey.data_ptr(), depth.data_ptr(), n, h, w)
    variants = {"unmasked": None, "masked": masks.data_ptr()}
    times = {k: [] for k in variants}
    kernel_ms = {k: [] for k in variants}
    h2d = {}
    for rep in range(args.warmup + args.reps):
        for name, pm in variants.items():
            eng.synchronize()
            eng.profile_enable(True)
            eng.profile_read(reset=True)
            b0 = eng.h2d_bytes()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(stream)
            pyrs = eng.pyramid_raw_batch(ptrs, 1.0 / 5000.0, K, args.levels, masks=pm)
            b.record(stream)
            b.synchronize()
            prof = eng.profile_read(reset=True)
            eng.profile_enable(False)
            h2d[name] = eng.h2d_bytes() - b0
            if rep >= args.warmup:
                times[name].append(a.elapsed_time(b))
                kernel_ms[name].append(prof["pyramid"]["ms"])
            for p in pyrs:
                p.release()
    eng.close()

    def stats(v):
        v = np.asarray(v)
        return {"median_ms": float(np.median(v)), "min_ms": float(v.min()), "max_ms": float(v.max())}

    out = {"card": card(), "frames": n, "size": [w, h], "levels": args.levels, "reps": args.reps,
           "build": {k: stats(v) for k, v in times.items()}, "pyramid_kernels": {k: stats(v) for k, v in kernel_ms.items()},
           "h2d_bytes_per_pixel": {k: h2d[k] / (n * h * w) for k in variants}}
    out["masked_over_unmasked"] = out["build"]["masked"]["median_ms"] / out["build"]["unmasked"]["median_ms"]
    print(json.dumps(out))


if __name__ == "__main__":
    main()
