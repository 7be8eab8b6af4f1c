"""The launch plan of the level kernel, compiled for the host from csrc/launch_plan.h (tests/native/launch_plan.cpp), equals
the Python restatement of launch_plan_model.py segment for segment and field for field: every batch size up to 1077 on
four grids and five level ranges and geometries, and every developer override."""
import json
import os
import shutil
import subprocess

import pytest

from launch_plan_model import OVERRIDES, level_geometry, plan

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GRIDS = (264, 228, 132, 16)
RANGES = [((640, 480, 5), 4, 0), ((640, 480, 5), 3, 1), ((640, 480, 5), 0, 0), ((1280, 960, 6), 5, 0),
          ((641, 479, 5), 4, 0)]


def _cases():
    """(geometry, first, last, grid, pairs, overrides)"""
    out = []
    for size, first, last in RANGES:
        geom = level_geometry(*size)
        out += [(geom, first, last, grid, n, {}) for grid in GRIDS for n in range(1, 1078)]
    geom = level_geometry(640, 480, 5)
    out += [(geom, 4, 0, grid, n, {f"DVO_B200_{k}": v}) for k, v in OVERRIDES for grid in GRIDS for n in (24, 512)]
    return out


def test_launch_plan_equals_the_restatement(tmp_path):
    gxx = shutil.which("g++")
    if not gxx:
        pytest.skip("g++ not available")
    exe = str(tmp_path / "launch_plan")
    r = subprocess.run([gxx, "-std=c++17", "-O1", "-Wall", "-Werror", "-I", os.path.join(ROOT, "dvo_slam_b200", "csrc"),
                        "-o", exe, os.path.join(ROOT, "tests", "native", "launch_plan.cpp")],
                       capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    assert [nb for _, nb, _ in level_geometry(640, 480, 5)] == [4, 2, 1, 1, 1]      # the kernel's 160-column bands
    cases = _cases()
    lines = []
    for geom, first, last, grid, n, env in cases:
        shape = " ".join(f"{h} {nbands} {nstrips}" for nstrips, nbands, h in geom)
        lines.append(f"{grid} {n} {first} {last} {len(geom)} {shape}" + "".join(f" {k}={v}" for k, v in env.items()))
    r = subprocess.run([exe], input="\n".join(lines) + "\n", capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    got = r.stdout.splitlines()
    assert len(got) == len(cases)
    bad = []
    for (geom, first, last, grid, n, env), line in zip(cases, got):
        want = plan(geom, first, last, grid, n, env)["segments"]
        if json.loads(line) != want:
            bad.append((geom[0], first, last, grid, n, env, line, want))
    assert not bad, f"{len(bad)} of {len(cases)} plans differ, first: {bad[:2]}"
