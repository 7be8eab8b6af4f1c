"""The cost of depth registration in the pyramid build: 512 raw 640x480 colour frames (8-bit grey) at 5 levels, built with
the depth used as registered (dvo_b200_pyramid_create_raw_batch / _device_batch) and with the depth of a separate camera
registered into them (dvo_b200_pyramid_create_registered_batch / _registered_device_batch): a 640x480 depth camera 25 mm to
the side ("registered") and a 320x240 one ("registered_lowres"), from pinned host memory and from device memory: six arms,
alternating.  Reports the CUDA-event time of one whole build (copies + kernels) and of its pyramid kernels alone (profiling
class 3, the registration included), median (min-max), the H2D bytes per colour pixel, the card's name and power limit,
and checks that the registered host and device arms built the same pyramids in this run.  One JSON line on stdout; writes
nothing else.

    python scripts/bench_registered_build.py [--frames 512] [--reps 20] [--warmup 3]
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
    from dvo_slam_b200.engine import INPUT_FORMATS, MASK_ROLES, Engine, Pyramid, depth_rays

    n, h, w = args.frames, 480, 640
    K = synth.FR1_INTRINSICS
    K_low = tuple(v / 2 for v in K)
    T = synth.baseline(0.025)
    scale = 1.0 / 5000.0
    grey = torch.empty((n, h, w), dtype=torch.uint8).pin_memory()
    depth = torch.empty((n, h, w), dtype=torch.int16).pin_memory()     # the bits of uint16 raw depth
    depth_low = torch.empty((n, h // 2, w // 2), dtype=torch.int16).pin_memory()
    cams = {"full": synth.DepthCamera(w, h, K, T), "low": synth.DepthCamera(w // 2, h // 2, K_low, T)}
    base = [(synth.make_pair(s, synth.SceneConfig(depth_camera=cams["full"])),
             synth.make_pair(s, synth.SceneConfig(depth_camera=cams["low"]))) for s in range(8)]
    raw = lambda z: torch.from_numpy(np.where(np.isnan(z), 0, np.round(z * 5000.0)).astype(np.uint16).view(np.int16))
    for i in range(n):
        p, q = base[i % 8]
        grey[i] = torch.from_numpy(np.clip(p["I_ref"].numpy(), 0, 255).astype(np.uint8))
        depth[i] = raw(p["Z_ref"].numpy())
        depth_low[i] = raw(q["Z_ref"].numpy())
    d_grey, d_depth, d_depth_low = grey.cuda(), depth.cuda().view(torch.uint16), depth_low.cuda().view(torch.uint16)
    torch.cuda.synchronize()

    stream = torch.cuda.Stream()
    eng = Engine(device=0, stream=stream.cuda_stream)
    ptrs = (grey.data_ptr(), depth.data_ptr(), n, h, w)
    reg = eng.depth_registration((w, h), depth_rays((w, h), K), T, (w, h), K)
    reg_low = eng.depth_registration((w // 2, h // 2), depth_rays((w // 2, h // 2), K_low), T, (w, h), K)

    def host_registered(r, z):   # the C call itself: Engine.pyramid_registered_batch would add a host synchronisation
        out = (C.c_void_p * n)()
        eng._check(eng.lib.dvo_b200_pyramid_create_registered_batch(eng.ctx, r.handle, None, n, INPUT_FORMATS["grey8_depth16"],
                                                                    grey.data_ptr(), z.data_ptr(), scale, None, MASK_ROLES["reference"],
                                                                    w, h, args.levels, out))
        return [Pyramid(eng, out[i]) for i in range(n)]

    arms = {
        "host": lambda: eng.pyramid_raw_batch(ptrs, scale, K, args.levels),
        "host_registered": lambda: host_registered(reg, depth),
        "host_registered_lowres": lambda: host_registered(reg_low, depth_low),
        "device": lambda: eng.pyramid_batch_device(d_grey, d_depth, K, args.levels, depth_scale=scale),
        "device_registered": lambda: eng.pyramid_registered_batch(reg, d_grey, d_depth, args.levels, depth_scale=scale),
        "device_registered_lowres": lambda: eng.pyramid_registered_batch(reg_low, d_grey, d_depth_low, args.levels, depth_scale=scale),
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

        # the registered host and device arms build the same pyramids: every plane, the selection and S at every level of a sample
        equal = {}
        for host, dev in (("host_registered", "device_registered"), ("host_registered_lowres", "device_registered_lowres")):
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
    reg.release()
    reg_low.release()
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
