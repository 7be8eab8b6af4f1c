"""The drop-in boundary with the REAL type spellings (SURVEY.md 8b): the adapter sources are compiled with
-DDVO_B200_WITH_EIGEN_OPENCV -- the branch a dvo_slam checkout uses -- against header-only Eigen / OpenCV / Boost
look-alikes that are spelled as the real include paths (oracle/ref_shim/, the same stand-ins that let the reference's own SSE
translation units compile for the pin).  Nothing is executed (no GPU needed)."""
import os
import shutil
import subprocess
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STUBS = os.path.join(ROOT, "oracle", "ref_shim")
INC = os.path.join(ROOT, "include")
HOST = os.path.join(ROOT, "dvo_slam_b200", "host")
FLAGS = ["-std=c++17", "-O1", "-fPIC", "-DDVO_B200_WITH_EIGEN_OPENCV", "-I" + STUBS, "-I" + INC]


def _cxx():
    return os.environ.get("CXX") or shutil.which("g++") or "g++"


def _compile(src, obj):
    res = subprocess.run([_cxx()] + FLAGS + ["-c", src, "-o", obj], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-4000:]


def test_adapter_compiles_with_real_type_spellings():
    lib = os.path.join(ROOT, "dvo_slam_b200", "libdvo_b200.so")
    with tempfile.TemporaryDirectory() as tmp:
        objs = {}
        for name in ("dvo_core_b200", "selftest", "tum_replay"):
            objs[name] = os.path.join(tmp, name + ".o")
            _compile(os.path.join(HOST, name + ".cpp"), objs[name])
        if os.path.exists(lib):   # the adapter + its self-test link against the C-ABI library (undefined symbols would show)
            for exe in ("selftest", "tum_replay"):
                res = subprocess.run([_cxx(), "-o", os.path.join(tmp, exe), objs[exe], objs["dvo_core_b200"], lib, "-lz", "-lpthread",
                                      "-Wl,-rpath," + os.path.dirname(lib), "-Wl,--allow-shlib-undefined"], capture_output=True, text=True)
                assert res.returncode == 0, res.stderr[-4000:]
