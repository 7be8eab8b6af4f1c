"""Masks in both roles, CPU side: the C ABI declares and exports the role-set create call and the role query, the Python
binding knows them, and the C++ adapter's setMask compiles against the real type spellings (the Eigen / OpenCV / Boost
look-alikes of oracle/ref_shim/, as tests/test_boundary_real_types.py compiles the rest of the surface).  No GPU."""
import os
import re
import shutil
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "dvo_slam_b200", "libdvo_b200.so")
NEW = ("dvo_b200_pyramid_create_masked_batch_roles", "dvo_b200_pyramid_mask_roles")


def _header():
    return open(os.path.join(ROOT, "include", "dvo_b200.h")).read()


def test_header_declares_roles():
    hdr = _header()
    assert "#define DVO_B200_MASK_ROLE_REFERENCE 1" in hdr and "#define DVO_B200_MASK_ROLE_CURRENT 2" in hdr
    assert "#define DVO_B200_ABI_VERSION 1" in hdr
    assert re.search(r"int dvo_b200_pyramid_create_masked_batch_roles\(dvo_b200_ctx\* ctx, int32_t n, int32_t format, const void\* image,"
                     r"\s+const void\* depth, float depth_scale, const uint8_t\* masks, int32_t roles,", hdr)
    assert re.search(r"int dvo_b200_pyramid_mask_roles\(const dvo_b200_pyramid\* p\);", hdr)


def test_library_exports_and_binding():
    from dvo_slam_b200 import engine
    for s in NEW:
        assert s in engine.ABI_SYMBOLS
    assert engine.MASK_ROLES == {"reference": 1, "both": 3}
    if os.path.exists(LIB):
        syms = subprocess.run(["nm", "-D", "--defined-only", LIB], capture_output=True, text=True).stdout
        for s in NEW:
            assert " " + s + "\n" in syms, s
        L = engine.load_library()
        assert L.dvo_b200_pyramid_mask_roles(None) == -1      # no device needed for a null handle


def test_prototypes_compile_as_c(tmp_path):
    src = tmp_path / "roles.c"
    src.write_text('#include "dvo_b200.h"\n'
                   "int (*f)(dvo_b200_ctx*, int32_t, int32_t, const void*, const void*, float, const uint8_t*, int32_t, int32_t, int32_t,\n"
                   "         float, float, float, float, int32_t, dvo_b200_pyramid**) = dvo_b200_pyramid_create_masked_batch_roles;\n"
                   "int (*g)(const dvo_b200_pyramid*) = dvo_b200_pyramid_mask_roles;\n"
                   "int roles = DVO_B200_MASK_ROLE_REFERENCE | DVO_B200_MASK_ROLE_CURRENT;\n")
    cc = os.environ.get("CC") or shutil.which("gcc") or "gcc"
    res = subprocess.run([cc, "-std=c99", "-Wall", "-Werror", "-I" + os.path.join(ROOT, "include"), "-c", str(src), "-o", str(tmp_path / "roles.o")],
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stderr


def test_adapter_set_mask_compiles_with_real_type_spellings(tmp_path):
    img = open(os.path.join(ROOT, "include", "dvo", "core", "rgbd_image.h")).read()
    assert "bool setMask(const cv::Mat& mask, bool current_role_too);" in img
    assert "bool setReferenceMask(const cv::Mat& mask);" in img
    src = tmp_path / "set_mask.cpp"
    src.write_text('#include "dvo/core/rgbd_image.h"\n'
                   "bool use(dvo::core::RgbdImagePyramid& p, const cv::Mat& m) { return p.setMask(m, true) && p.setReferenceMask(m); }\n")
    cxx = os.environ.get("CXX") or shutil.which("g++") or "g++"
    flags = ["-std=c++17", "-O1", "-fPIC", "-DDVO_B200_WITH_EIGEN_OPENCV", "-I" + os.path.join(ROOT, "oracle", "ref_shim"),
             "-I" + os.path.join(ROOT, "include")]
    for f, o in ((str(src), "set_mask.o"), (os.path.join(ROOT, "dvo_slam_b200", "host", "dvo_core_b200.cpp"), "adapter.o")):
        res = subprocess.run([cxx] + flags + ["-c", f, "-o", str(tmp_path / o)], capture_output=True, text=True)
        assert res.returncode == 0, res.stderr[-4000:]
    nm = subprocess.run(["nm", "-C", "--defined-only", str(tmp_path / "adapter.o")], capture_output=True, text=True).stdout
    assert "RgbdImagePyramid::setMask(" in nm
