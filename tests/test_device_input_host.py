"""CPU tests of pyramids from device memory (dvo_b200_pyramid_create_device_batch): the layout of dvo_b200_device_plane
against the header, the planes engine.device_planes derives from torch tensors (packed, cropped, shared masks, BGR and the
layouts it must refuse), and the entry point's answer to a NULL context.  No GPU: the tensors live on the CPU."""
import ctypes as C
import os
import subprocess

import pytest
import torch

from dvo_slam_b200.engine import DevicePlane, device_planes

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as ge
    ge.build_cuda()
    from dvo_slam_b200 import engine
    return engine.load_library()


def test_device_plane_layout_matches_header(lib, tmp_path):
    prog = tmp_path / "plane_layout.c"
    prog.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "dvo_b200.h"\nint main(){printf("%zu %zu %zu %zu\\n",'
                    'sizeof(dvo_b200_device_plane),offsetof(dvo_b200_device_plane,data),offsetof(dvo_b200_device_plane,row_bytes),'
                    'offsetof(dvo_b200_device_plane,image_bytes));return 0;}\n')
    exe = tmp_path / "plane_layout"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(prog), "-o", str(exe)])
    got = [int(v) for v in subprocess.check_output([str(exe)]).split()]
    assert got == [C.sizeof(DevicePlane), DevicePlane.data.offset, DevicePlane.row_bytes.offset, DevicePlane.image_bytes.offset]


def test_packed_planes():
    n, h, w = 3, 48, 64
    I, Z = torch.zeros(n, h, w), torch.zeros(n, h, w)
    M = torch.ones(n, h, w, dtype=torch.bool)
    fmt, shape, pI, pZ, pM = device_planes(I, Z, M)
    assert fmt == "float32" and shape == (n, h, w)
    assert pI == (I.data_ptr(), 4 * w, 4 * w * h) and pZ == (Z.data_ptr(), 4 * w, 4 * w * h)
    assert pM == (M.data_ptr(), w, w * h)
    G, R = torch.zeros(n, h, w, dtype=torch.uint8), torch.zeros(n, h, w, dtype=torch.uint16)
    fmt, _, pG, pR, pM = device_planes(G, R)
    assert fmt == "grey8_depth16" and pM is None
    assert pG == (G.data_ptr(), w, w * h) and pR == (R.data_ptr(), 2 * w, 2 * w * h)


def test_cropped_views_keep_the_larger_pitch():
    n, H, W, h, w, y0, x0 = 2, 60, 81, 48, 64, 5, 3
    big = torch.zeros(n, H, W)
    bigz = torch.zeros(n, H, W, dtype=torch.float32)
    I, Z = big[:, y0:y0 + h, x0:x0 + w], bigz[:, y0:y0 + h, x0:x0 + w]
    fmt, shape, pI, pZ, _ = device_planes(I, Z)
    assert shape == (n, h, w)
    assert pI == (big.data_ptr() + 4 * (y0 * W + x0), 4 * W, 4 * W * H)
    assert pZ == (bigz.data_ptr() + 4 * (y0 * W + x0), 4 * W, 4 * W * H)
    # every other frame of a sequence: a larger image stride
    seq = torch.zeros(2 * n, h, w)
    _, _, pS, _, _ = device_planes(seq[::2], torch.zeros(n, h, w))
    assert pS == (seq.data_ptr(), 4 * w, 2 * 4 * w * h)


def test_shared_masks_have_no_image_stride():
    n, h, w = 4, 48, 64
    I, Z = torch.zeros(n, h, w), torch.zeros(n, h, w)
    one = torch.ones(h, w, dtype=torch.uint8)
    _, _, _, _, p2 = device_planes(I, Z, one)
    _, _, _, _, pe = device_planes(I, Z, one.expand(n, h, w))
    assert p2 == pe == (one.data_ptr(), w, 0)
    big = torch.ones(h + 8, w + 8, dtype=torch.bool)
    _, _, _, _, pc = device_planes(I, Z, big[2:2 + h, 4:4 + w].expand(n, h, w))
    assert pc == (big.data_ptr() + 2 * (w + 8) + 4, w + 8, 0)


def test_bgr_planes():
    n, h, w = 2, 48, 64
    C3 = torch.zeros(n, h, w, 3, dtype=torch.uint8)
    R = torch.zeros(n, h, w, dtype=torch.uint16)
    fmt, _, pC, _, _ = device_planes(C3, R)
    assert fmt == "bgr8_depth16" and pC == (C3.data_ptr(), 3 * w, 3 * w * h)
    big = torch.zeros(n, h + 2, w + 5, 3, dtype=torch.uint8)
    fmt, _, pC, _, _ = device_planes(big[:, 1:1 + h, 2:2 + w], R)
    assert pC == (big.data_ptr() + 3 * ((w + 5) + 2), 3 * (w + 5), 3 * (w + 5) * (h + 2))


def test_rejected_layouts():
    n, h, w = 2, 48, 64
    I, Z = torch.zeros(n, h, w), torch.zeros(n, h, w)
    G, R = torch.zeros(n, h, w, dtype=torch.uint8), torch.zeros(n, h, w, dtype=torch.uint16)
    bad = {
        "transposed image": (torch.zeros(n, w, h).transpose(1, 2), Z, None),
        "every other column": (torch.zeros(n, h, 2 * w)[:, :, ::2], Z, None),
        "rows expanded": (torch.zeros(n, 1, w).expand(n, h, w), Z, None),
        "planar BGR": (torch.zeros(n, 3, h, w, dtype=torch.uint8).permute(0, 2, 3, 1), R, None),
        "BGRA view": (torch.zeros(n, h, w, 4, dtype=torch.uint8)[..., :3], R, None),
        "float64 image": (I.double(), Z, None),
        "int16 depth": (G, R.view(torch.int16), None),
        "float depth with grey": (G, Z, None),
        "depth shape": (I, Z[:, :-1], None),
        "2-D image": (I[0], Z[0], None),
        "float mask": (I, Z, torch.ones(n, h, w)),
        "mask shape": (I, Z, torch.ones(n, h, w + 1, dtype=torch.uint8)),
        "transposed mask": (I, Z, torch.ones(w, h, dtype=torch.uint8).t()),
    }
    for name, (a, b, m) in bad.items():
        with pytest.raises(ValueError):
            device_planes(a, b, m)
            pytest.fail(name)


def test_null_context_is_an_invalid_argument(lib):
    p = DevicePlane(1 << 20, 256, 256 * 64)
    out = (C.c_void_p * 1)()
    rc = lib.dvo_b200_pyramid_create_device_batch(None, 1, 0, C.byref(p), C.byref(p), 0.0, None, 1, 64, 48, 500.0, 500.0, 32.0, 24.0,
                                                  3, out)
    assert rc == -1 and not out[0]
