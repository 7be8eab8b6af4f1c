"""The cost of rectifying in the pyramid build: 512 raw 640x480 frames (8-bit grey + 16-bit depth), 5 levels, built with and
without the fr1 undistortion remap (dvo_b200_pyramid_create_rectified_batch / _rectified_device_batch against
dvo_b200_pyramid_create_raw_batch / _device_batch), from pinned host memory and from device memory, each without masks and
with both-role masks (random blobs, one per frame): eight arms, alternating.  Reports the CUDA-event time of one whole build
(copies + kernels) and of its pyramid kernels alone (profiling class 3, the remap included), median (min-max), the H2D bytes
per pixel, the card's name and power limit, and checks that the rectified host and device arms built the same pyramids in
this run.  One JSON line on stdout; writes nothing else.

    python scripts/bench_rectified_build.py [--frames 512] [--reps 20] [--warmup 3]
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
    import ctypes as C
    from dvo_slam_b200.engine import INPUT_FORMATS, MASK_ROLES, Engine, Pyramid, undistort_map

    n, h, w = args.frames, 480, 640
    K = synth.FR1_INTRINSICS
    scale = 1.0 / 5000.0
    rng = np.random.default_rng(0)
    grey = torch.empty((n, h, w), dtype=torch.uint8).pin_memory()
    depth = torch.empty((n, h, w), dtype=torch.int16).pin_memory()     # the bits of uint16 raw depth
    masks = torch.ones((n, h, w), dtype=torch.uint8).pin_memory()
    base = [synth.make_pair(s) for s in range(8)]
    yy, xx = np.ogrid[:h, :w]
    for i in range(n):
        p = base[i % 8]
        grey[i] = torch.from_numpy(np.clip(p["I_ref"].numpy(), 0, 255).astype(np.uint8))
        z = p["Z_ref"].numpy()
        depth[i] = torch.from_numpy(np.where(np.isnan(z), 0, np.round(z * 5000.0)).astype(np.uint16).view(np.int16))
        m = np.ones((h, w), np.uint8)
        for _ in range(6):   # a few blobs: a segmentation mask of people / a mount
            cy, cx, r = rng.integers(0, h), rng.integers(0, w), rng.integers(20, 90)
            m[(yy - cy) ** 2 + (xx - cx) ** 2 <= r * r] = 0
        masks[i] = torch.from_numpy(m)
    d_grey, d_depth, d_masks = grey.cuda(), depth.cuda().view(torch.uint16), masks.cuda()
    torch.cuda.synchronize()

    stream = torch.cuda.Stream()
    eng = Engine(device=0, stream=stream.cuda_stream)
    ptrs = (grey.data_ptr(), depth.data_ptr(), n, h, w)
    rect = eng.rectifier((w, h), *undistort_map(w, h, K, synth.FR1_DISTORTION), K)

    def host_rectified(m):   # the C call itself: Engine.pyramid_rectified_batch would add a host synchronisation
        out = (C.c_void_p * n)()
        eng._check(eng.lib.dvo_b200_pyramid_create_rectified_batch(eng.ctx, rect.handle, n, INPUT_FORMATS["grey8_depth16"], grey.data_ptr(),
                                                                   depth.data_ptr(), scale, m, MASK_ROLES["both"], w, h, args.levels, out))
        return [Pyramid(eng, out[i]) for i in range(n)]

    arms = {
        "host": lambda: eng.pyramid_raw_batch(ptrs, scale, K, args.levels),
        "host_rectified": lambda: host_rectified(None),
        "device": lambda: eng.pyramid_batch_device(d_grey, d_depth, K, args.levels, depth_scale=scale),
        "device_rectified": lambda: eng.pyramid_rectified_batch(rect, d_grey, d_depth, args.levels, depth_scale=scale),
        "host_masked": lambda: eng.pyramid_raw_batch(ptrs, scale, K, args.levels, masks=masks.data_ptr(), mask_roles="both"),
        "host_masked_rectified": lambda: host_rectified(masks.data_ptr()),
        "device_masked": lambda: eng.pyramid_batch_device(d_grey, d_depth, K, args.levels, depth_scale=scale, masks=d_masks,
                                                          mask_roles="both"),
        "device_masked_rectified": lambda: eng.pyramid_rectified_batch(rect, d_grey, d_depth, args.levels, depth_scale=scale,
                                                                       masks=d_masks, mask_roles="both"),
    }
    times = {k: [] for k in arms}
    kernel_ms = {k: [] for k in arms}
    h2d = {}
    with torch.cuda.stream(stream):
        for rep in range(args.warmup + args.reps):
            for name, build in arms.items():
                eng.synchronize()
                eng.profile_enable(True)
                eng.profile_read(reset=True)
                b0 = eng.h2d_bytes()
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record(stream)
                pyrs = build()
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

        # the rectified host and device arms build the same pyramids: every plane, the selection and S at every level of a sample
        equal = {}
        for host, dev in (("host_rectified", "device_rectified"), ("host_masked_rectified", "device_masked_rectified")):
            P, Q = arms[host](), arms[dev]()
            ok = True
            for i in sorted({0, 1, n // 3, n - 1}):
                for l in range(args.levels):
                    ok &= bool(np.array_equal(P[i].download(l), Q[i].download(l), equal_nan=True))
                    (s0, m0), (s1, m1) = P[i].select(l), Q[i].select(l)
                    ok &= s0 == s1 and bool(np.array_equal(m0, m1))
            equal[dev] = ok
            for p in P + Q:
                p.release()
    rect.release()
    eng.close()

    def stats(v):
        v = np.asarray(v)
        return {"median_ms": float(np.median(v)), "min_ms": float(v.min()), "max_ms": float(v.max())}

    out = {"card": card(), "frames": n, "size": [w, h], "levels": args.levels, "reps": args.reps,
           "build": {k: stats(v) for k, v in times.items()}, "pyramid_kernels": {k: stats(v) for k, v in kernel_ms.items()},
           "h2d_bytes_per_pixel": {k: h2d[k] / (n * h * w) for k in arms}, "device_equals_host": equal}
    print(json.dumps(out))
    if not all(equal.values()):
        sys.exit(1)


if __name__ == "__main__":
    main()
