"""Generates tests/golden/reference_pin.npz: what the ORIGINAL project's own object code computes on the golden pairs.

oracle/_ref/libdvo_ref*.so are dvo_core/src/{dense_tracking_impl,core/math_sse,core/intrinsic_matrix}.cpp of a dvo_slam
checkout compiled unmodified (oracle/Makefile target `ref`; build with DVO_REFERENCE=<checkout> python -c "import
__graft_entry__ as g; g.build()").  Run from the repo root:  python tests/golden/make_reference_pin.py

tests/test_reference_pin.py compares the oracle's FAITHFUL mode against these numbers, so the pin holds in any checkout.
Arrays the tests compare bit for bit are stored as digests (helpers.digest: sha256 with NaN and -0 made canonical); the
-O3 build, which the tests compare to a tolerance, keeps its values at a fixed seeded sample of the valid points.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))
from helpers import (GOLDEN_LEVELS, GOLDEN_SEEDS, dense_records, digest, golden_images,  # noqa: E402
                     load_golden, match_cases, odd_point_margin, o3_sample_index)
from oracle import oracle_py as orc  # noqa: E402


def main():
    for v in ("", "_O3"):
        if not orc.ref_available(v):
            raise SystemExit(f"oracle/_ref/libdvo_ref{v}.so missing: build with DVO_REFERENCE=<dvo_slam checkout>")
    orc.build()
    out = {k: [] for k in ("lin_counts", "lin_records", "lin_P", "lin_ll", "lin_A", "lin_b", "o3_n", "o3_valid", "o3_sample",
                           "o3_P", "o3_A", "o3_b", "iei_n", "iei_img", "thr_counts", "thr_P", "thr_ll", "thr_A", "thr_b",
                           "match_levels", "match_T", "match_information", "match_ll")}
    for seed in GOLDEN_SEEDS:                      # lin_* [seed, level, use_weights], o3_* [seed, level], iei_* [seed, level, thresholds]
        g = load_golden(seed)
        im = golden_images(g, orc)
        oref = orc.Pyramid(im["I_ref"], im["Z_ref"], g["K"], GOLDEN_LEVELS)
        ocur = orc.Pyramid(im["I_cur"], im["Z_cur"], g["K"], GOLDEN_LEVELS)
        rref, rcur = orc.RefPyramid(oref), orc.RefPyramid(ocur)
        for lvl in range(GOLDEN_LEVELS):
            w, h, K = oref.level_info(lvl)
            for uw in (False, True):
                r = orc.ref_linearize(oref.planes(lvl), ocur.planes(lvl), K, g["kat_T"], uw, g["kat_prev_precision"])
                out["lin_counts"].append([r["n_selected"], r["n"]])
                out["lin_records"].append(digest(dense_records(r, h, w)))
                for k in ("P", "ll", "A", "b"):
                    out["lin_" + k].append(r["precision" if k == "P" else k])
            r = orc.ref_linearize(oref.planes(lvl), ocur.planes(lvl), K, g["kat_T"], True, g["kat_prev_precision"], variant="_O3")
            d = dense_records(r, h, w)
            out["o3_n"].append(r["n"])
            out["o3_valid"].append(digest(np.isnan(d)))
            out["o3_sample"].append(d[:, o3_sample_index(d, seed, lvl)])
            for k in ("P", "A", "b"):
                out["o3_" + k].append(r["precision" if k == "P" else k])
            for ti, td in ((0.0, 0.0), (2.0, 0.02)):
                n, img = orc.ref_intensity_error_image(rref, rcur, lvl, g["kat_T"], ti, td)
                out["iei_n"].append(n)
                out["iei_img"].append(digest(img))
        if seed == 12:                             # thr_* [case]: non-default thresholds and a second transform, level 1
            w, h, K = oref.level_info(1)
            for T, ti, td in ((np.eye(4), 0.0, 0.0), (g["kat_T"], 4.0, 0.02)):
                r = orc.ref_linearize(oref.planes(1), ocur.planes(1), K, T, True, g["kat_prev_precision"], ti, td)
                out["thr_counts"].append([r["n_selected"], r["n"]])
                for k in ("P", "ll", "A", "b"):
                    out["thr_" + k].append(r["precision" if k == "P" else k])
    for Ir, Zr, Ic, Zc, K, levels, cfg, T0 in match_cases(orc):     # match_* [case]; levels: (termination, iterations, valid)
        oref, ocur = orc.Pyramid(Ir, Zr, K, levels), orc.Pyramid(Ic, Zc, K, levels)
        r = orc.ref_match(orc.RefPyramid(oref), orc.RefPyramid(ocur), orc.config(**cfg), T_init=T0)
        out["match_levels"].append(np.full((5, 3), -1, dtype=np.int64))
        out["match_levels"][-1][:len(r["levels"])] = [[l["termination"], l["num_iterations"], l["valid_pixels"]] for l in r["levels"]]
        out["match_T"].append(r["T"]); out["match_information"].append(r["information"]); out["match_ll"].append(r["log_likelihood"])
    shape = {"lin": (len(GOLDEN_SEEDS), GOLDEN_LEVELS, 2), "o3": (len(GOLDEN_SEEDS), GOLDEN_LEVELS),
             "iei": (len(GOLDEN_SEEDS), GOLDEN_LEVELS, 2)}
    arrays = {}
    for k, v in out.items():
        a = np.array(v)
        if k.split("_")[0] in shape:
            a = a.reshape(shape[k.split("_")[0]] + a.shape[1:])
        arrays[k] = a
    margin, im, oref, ocur = odd_point_margin(orc)
    n, img = orc.ref_intensity_error_image(orc.RefPyramid(oref), orc.RefPyramid(ocur), 0, np.eye(4))
    arrays["odd"] = np.array([margin, n], dtype=np.int64)
    arrays["odd_img"] = np.array(digest(img))
    np.savez_compressed(os.path.join(HERE, "reference_pin.npz"), **arrays)
    print("wrote", {k: (a.shape, a.dtype.str) for k, a in arrays.items()})


if __name__ == "__main__":
    main()
