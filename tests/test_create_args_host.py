"""The checks every pyramid create passes before any upload or launch (csrc/create_args.h, built for the host with
tests/native/create_args.cpp): every entry point's prefix against every refusal it can receive -- null pointers and sizes,
format, roles, the rectifier, the depth registration and the level geometry -- the order in which several faults are
reported, and the accepted cases at each boundary."""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# entry-point prefix -> (remap, device, format, whether format and roles are arguments); remap 0 none, 1 rectify, 2 register
ENTRIES = {
    "pyramid_create": (0, 0, 0, False, False),
    "pyramid_create_raw": (0, 0, 1, False, False),
    "pyramid_create_bgr": (0, 0, 2, False, False),
    "pyramid_create_masked": (0, 0, 0, True, False),
    "pyramid_create_masked_roles": (0, 0, 0, True, True),
    "pyramid_create_device": (0, 1, 0, True, True),
    "pyramid_create_rectified": (1, 0, 0, True, True),
    "pyramid_create_rectified_device": (1, 1, 0, True, True),
    "pyramid_create_registered": (2, 0, 0, True, True),
    "pyramid_create_registered_device": (2, 1, 0, True, True),
}
FIELDS = ["remap", "device", "ctx", "out", "image", "depth", "n", "format", "roles", "width", "height", "levels", "rect", "rect_in_w",
          "rect_in_h", "rect_w", "rect_h", "rect_fx", "reg", "reg_w", "reg_h", "reg_fx"]

NULL = "null/invalid argument"
FORMAT = "unknown input format"
ROLES = "unsupported role set"
GEOMETRY_LEVELS, GEOMETRY_WIDTH, GEOMETRY_LEVEL, GEOMETRY_LARGE = "levels ", "below 32 wide", "below 8x2", "2^30 pixels"


def _good(fn, with_rect=False):
    remap, device, fmt, _, _ = ENTRIES[fn]
    c = dict(remap=remap, device=device, ctx=1, out=1, image=1, depth=1, n=2, format=fmt, roles=1, width=640, height=480, levels=5,
             rect=0, rect_in_w=640, rect_in_h=480, rect_w=640, rect_h=480, rect_fx=500, reg=0, reg_w=640, reg_h=480, reg_fx=500)
    if remap == 1 or with_rect:
        c["rect"] = 1
    if remap == 2:
        c["reg"] = 1
    return c


def _level0(c, w, h):
    """the changes that make level 0 of the build w x h"""
    if c["reg"]:
        return dict(reg_w=w, reg_h=h, rect_w=w, rect_h=h) if c["rect"] else dict(reg_w=w, reg_h=h, width=w, height=h)
    if c["rect"]:
        return dict(rect_w=w, rect_h=h)
    return dict(width=w, height=h)


def _cases():
    """(prefix, case, expected: None = accepted, else a part of the refusal)"""
    out = []
    variants = [(fn, False) for fn in ENTRIES] + [("pyramid_create_registered", True), ("pyramid_create_registered_device", True)]
    for fn, with_rect in variants:
        remap, _, _, has_format, has_roles = ENTRIES[fn]
        base = _good(fn, with_rect)
        rows = [({}, None), (dict(n=1), None),
                (dict(ctx=0), NULL), (dict(out=0), NULL), (dict(image=0), NULL), (dict(depth=0), NULL),
                (dict(n=0), NULL), (dict(n=-1), NULL), (dict(width=0), NULL), (dict(height=-1), NULL),
                (dict(levels=0), GEOMETRY_LEVELS), (dict(levels=9), GEOMETRY_LEVELS), (dict(levels=1), None),
                (dict(_level0(base, 31, 480), levels=1), GEOMETRY_WIDTH), (dict(_level0(base, 32, 480), levels=3), None),
                (dict(_level0(base, 64, 1), levels=1), GEOMETRY_WIDTH), (dict(_level0(base, 64, 2), levels=1), None),
                (dict(_level0(base, 64, 48), levels=4), None), (dict(_level0(base, 64, 48), levels=5), GEOMETRY_LEVEL),
                (dict(_level0(base, 640, 8), levels=3), None), (dict(_level0(base, 640, 8), levels=4), GEOMETRY_LEVEL),
                (dict(_level0(base, 1024, 256), levels=8), None),
                (dict(_level0(base, 32768, 32768), levels=1), GEOMETRY_LARGE),
                (dict(_level0(base, 32768, 32767), levels=1), None)]
        if has_format:
            rows += [(dict(format=-1), FORMAT), (dict(format=3), FORMAT), (dict(format=1), None), (dict(format=2), None)]
        if has_roles:
            rows += [(dict(roles=0), ROLES), (dict(roles=2), ROLES), (dict(roles=3), None)]
        if remap == 1 or with_rect:
            rows += [(dict(rect=0), "null rectifier" if remap == 1 else None), (dict(rect=2), "the rectifier belongs to another context"),
                     (dict(width=320), "the rectifier takes"), (dict(height=479), "the rectifier takes"),
                     (dict(width=800, height=600, rect_in_w=800, rect_in_h=600), None)]
        if remap == 2:
            rows += [(dict(reg=0), "null depth registration"), (dict(reg=2), "the depth registration belongs to another context")]
            if with_rect:
                rows += [(dict(rect_w=320), "the rectifier's output is not the registration's target"),
                         (dict(rect_fx=501), "the rectifier's K_new is not the registration's K")]
            else:
                rows += [(dict(width=320), "the registration's target is"), (dict(height=479), "the registration's target is")]
        # several faults: the first in the order of the checks decides
        rows += [(dict(n=0, levels=9), NULL), (dict(levels=9, **_level0(base, 31, 480)), GEOMETRY_LEVELS)]
        if has_format and has_roles:
            rows += [(dict(format=3, roles=0, levels=9), FORMAT), (dict(roles=0, levels=9), ROLES)]
        if remap:
            rows += [(dict(roles=2, reg=2 if remap == 2 else 0, rect=2 if remap == 1 or with_rect else 0), ROLES)]
        if remap == 2 and with_rect:
            rows += [(dict(rect=2, reg=2), "the rectifier belongs to another context")]
        out += [(fn, dict(base, **change), want) for change, want in rows]
    return out


def test_every_entry_point_against_every_refusal(tmp_path):
    gxx = shutil.which("g++")
    if not gxx:
        pytest.skip("g++ not available")
    exe = str(tmp_path / "create_args")
    r = subprocess.run([gxx, "-std=c++17", "-O1", "-Wall", "-Werror", "-I", os.path.join(ROOT, "dvo_slam_b200", "csrc"), "-o", exe,
                        os.path.join(ROOT, "tests", "native", "create_args.cpp")], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    cases = _cases()
    lines = [" ".join([fn] + [str(c[k]) for k in FIELDS]) for fn, c, _ in cases]
    r = subprocess.run([exe], input="\n".join(lines) + "\n", capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    got = r.stdout.splitlines()
    assert len(got) == len(cases)
    bad = []
    for (fn, c, want), line in zip(cases, got):
        ok = line == "ok" if want is None else line.startswith(fn + ": ") and want in line
        if not ok:
            bad.append((fn, {k: v for k, v in c.items() if v != _good(fn, bool(c["rect"]))[k]}, want, line))
    assert not bad, f"{len(bad)} of {len(cases)} cases differ, first: {bad[:4]}"
    assert {fn for fn, _, _ in cases} == set(ENTRIES)


def test_host_masks_take_every_accepted_shape():
    """the binding's one normaliser of host masks: a host pointer, [h, w] for the whole batch, or any n*h*w values; the
    caller's C-contiguous uint8 array is passed as it is, anything else as a 0/1 copy; other shapes raise ValueError"""
    import numpy as np
    from dvo_slam_b200.engine import _host_masks
    n, h, w = 3, 4, 5
    assert _host_masks(12345, n, h, w) == (12345, None)
    one = (np.arange(h * w).reshape(h, w) % 3).astype(np.uint8)
    p, M = _host_masks(one, n, h, w)
    assert M.shape == (n, h, w) and M.flags.c_contiguous and (M == one).all() and p == M.ctypes.data
    mine = np.ones((n, h, w), np.uint8)
    assert _host_masks(mine, n, h, w)[1] is mine
    flat = np.zeros(n * h * w, bool)
    flat[7] = True
    M = _host_masks(flat, n, h, w)[1]
    assert M.dtype == np.uint8 and M.sum() == 1 and M.reshape(-1)[7] == 1
    for bad in (np.ones((h, w + 1)), np.ones((n + 1, h, w)), np.ones(7)):
        with pytest.raises(ValueError):
            _host_masks(bad, n, h, w)
