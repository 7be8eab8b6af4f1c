"""The level kernel's 160-column bands.

Tiles are 160 x 7 reference pixels, so the 640-, 320- and 160-pixel-wide levels of a 640 x 480 pyramid are whole bands and
their tiles take the exact pixel loops (which end with an odd fifth stage-A round).  A partial band now needs a width that
is not a multiple of 160: 400 x 300 has bands of 160, 160 and 80 columns at level 0 and of 160 and 40 at level 1, so each
level has both full bands (exact loops) and a partial band (generic loop).  That case is checked here as the other
generic-loop cases are: residual records bit-exact against the oracle's MIRROR mode (and the corrected estimator's
definition), and a batch returning the bits of single alignments, for both estimators.  On the host: the shared-memory
layout still leaves room for two CTAs per SM, and every geometry the launch-plan tests run keeps the launch count that
their 128-column restatement of the plan predicts.
"""
import os
import shutil
import subprocess

import numpy as np
import pytest

import launch_plan_model as lpm

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TILE_W, TILE_H = 160, 7
W, H, LEVELS = 400, 300, 4
CARVEOUT, SMEM_RESERVED_PER_CTA = 196 * 1024, 1024     # of an H100 SM's 256 KB: 60 KB stay L1; 1 KB per resident CTA
LARGEST_TAIL = 5696      # sizeof(LevelTailOf<true, true>) (photometric, motion prior) in tracker.cu under nvcc 12.9


def _bands(w):
    return [min(TILE_W, w - x0) for x0 in range(0, w, TILE_W)]


# ---- host ----
@pytest.fixture(scope="module")
def layout(tmp_path_factory):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    exe = str(tmp_path_factory.mktemp("tile_budget") / "tile_budget")
    r = subprocess.run([nvcc, "-std=c++17", "--expt-relaxed-constexpr", "-w", "-I", os.path.join(ROOT, "dvo_slam_b200", "csrc"),
                        "-I", os.path.join(ROOT, "include"), "-o", exe, os.path.join(ROOT, "tests", "native", "tile_budget.cu")],
                       capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    r = subprocess.run([exe], capture_output=True, text=True, timeout=60)
    assert r.returncode == 0, r.stdout[-2000:]
    return {k: int(v) for k, v in (line.split() for line in r.stdout.splitlines())}


def test_tile_geometry(layout):
    """160 x 7 tiles; the window holds the tile's columns plus 24, in 19 rows; the record is 2 320 float2, of which stage A
    copies the first 1 200; every bulk copy is a multiple of 16 bytes"""
    L = layout
    assert (L["tile_w"], L["tile_h"], L["win_cols"], L["win_rows"], L["stages"]) == (TILE_W, TILE_H, TILE_W + 24, 19, 2)
    assert L["rec_bytes"] == 8 * (2 * TILE_H * TILE_W + TILE_W // 2) == 18560
    assert L["rec_stage_a_bytes"] == 8 * (TILE_H * TILE_W + TILE_W // 2) == 9600
    assert L["rec_bytes"] % 16 == 0 and L["rec_stage_a_bytes"] % 16 == 0 and (8 * L["win_cols"]) % 16 == 0
    assert L["win_cols"] < 256                                  # produce_tiles packs the window width into 8 bits
    assert _bands(640) == [160] * 4 and _bands(320) == [160] * 2 and _bands(160) == [160]
    assert _bands(W) == [160, 160, 80] and _bands(W // 2) == [160, 40]


def test_shared_memory_leaves_two_ctas_per_sm(layout):
    """Two stage buffers (record + window, 128-byte aligned) and the barriers fill 93 312 bytes; with the largest tail of
    shared state after the pipeline, two CTAs fit in the 196 KB shared-memory carveout, which leaves 60 KB of L1 (tracker.cu
    asserts two CTAs per SM of every instance at build time)."""
    L = layout
    assert L["stage_buf"] == (L["rec_bytes"] + 8 * L["win_rows"] * L["win_cols"] + 127) // 128 * 128 == 46592
    assert L["tile_pipe"] == 93312
    assert L["seg_combine"] < LARGEST_TAIL           # the tail holds the strip combine's scratch and the end step's state
    assert 2 * (L["tile_pipe"] + LARGEST_TAIL + SMEM_RESERVED_PER_CTA) <= CARVEOUT


@pytest.mark.parametrize("geom,first,last", [((640, 480, 5), 4, 0), ((640, 480, 5), 3, 1), ((640, 480, 5), 0, 0),
                                             ((1280, 960, 6), 5, 0)], ids=["640-4..0", "640-3..1", "640-0..0", "1280-5..0"])
def test_launch_counts_do_not_depend_on_the_band_width(monkeypatch, geom, first, last):
    """The ranges test_gpu_launch_plans.py runs, at every batch size up to 1077 and with every override: 160-column bands
    give the same coarse / fine split and the same number of persistent launches as the 128-column restatement."""
    grid = 264
    envs = [{}] + [{f"DVO_B200_{k}": v} for k, v in lpm.OVERRIDES]

    def plans(tile_w):
        monkeypatch.setattr(lpm, "TILE_W", tile_w)
        g = lpm.level_geometry(*geom)
        return [(p["launches"], p["fused"], [(G["first_li"], G["nlev"]) for G in p["groups"]])
                for env in envs for n in range(1, 1078) for p in [lpm.plan(g, first, last, grid, n, env)]]

    assert plans(128) == plans(TILE_W)


# ---- GPU ----
def _K():
    from dvo_slam_b200 import synth
    return tuple(v * W / 640 for v in synth.FR1_INTRINSICS)


def _pair(seed):
    from dvo_slam_b200 import synth
    p = synth.make_pair(seed, synth.SceneConfig(width=W, height=H, intrinsics=_K()))
    return {k: p[k].numpy() for k in ("I_ref", "Z_ref", "I_cur", "Z_cur")}


@pytest.fixture(scope="module")
def corrected():
    from dvo_slam_b200.engine import Engine
    eng = Engine(device=0, estimator="corrected")
    yield eng
    eng.close()


@pytest.fixture(scope="module")
def pair400(engine, oracle):
    a = _pair(3)
    a["gref"] = engine.pyramid(a["I_ref"], a["Z_ref"], _K(), LEVELS)
    a["gcur"] = engine.pyramid(a["I_cur"], a["Z_cur"], _K(), LEVELS)
    a["oref"] = oracle.Pyramid(a["I_ref"], a["Z_ref"], _K(), LEVELS)
    a["ocur"] = oracle.Pyramid(a["I_cur"], a["Z_cur"], _K(), LEVELS)
    return a


POSES = ["identity", "rot3"]


def _pose(name):
    from test_gpu_generic_tiles import _rot_z, _shift_z
    return np.eye(4) if name == "identity" else _rot_z(3.0) @ _shift_z(0.02)


@pytest.mark.gpu
@pytest.mark.parametrize("pose", POSES)
@pytest.mark.parametrize("lvl", [0, 1])
def test_records_reference_estimator(engine, oracle, pair400, lvl, pose):
    """full bands and a partial band in every strip: records bit-exact against MIRROR, counts exact, P / LL / A / b to 2e-6"""
    from test_gpu_generic_tiles import _check_level
    assert len(_bands(W >> lvl)) >= 2 and _bands(W >> lvl)[-1] < TILE_W
    _check_level(engine, oracle, pair400, lvl, _pose(pose))


@pytest.mark.gpu
@pytest.mark.parametrize("pose", POSES)
@pytest.mark.parametrize("lvl", [0, 1])
def test_records_corrected_estimator(corrected, oracle, pair400, lvl, pose):
    """the same under the corrected estimator (its oracle definition: MIRROR without the reference's quirks)"""
    from test_gpu_corrected_estimator import _check_level
    _check_level(corrected, oracle, pair400, lvl, _pose(pose))


NPAIRS = 72      # at least grid / 4 on 132 SMs: the walking plan, level 0 fine (129 tiles), levels 1..3 coarse


@pytest.fixture(scope="module")
def batch400(engine, corrected):
    imgs = [_pair(100 + i) for i in range(NPAIRS)]
    out = {}
    for name, eng in (("reference", engine), ("corrected", corrected)):
        out[name] = [(eng.pyramid(a["I_ref"], a["Z_ref"], _K(), LEVELS), eng.pyramid(a["I_cur"], a["Z_cur"], _K(), LEVELS))
                     for a in imgs]
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("est", ["reference", "corrected"])
def test_batch_equals_single_alignments(engine, corrected, batch400, est):
    """a 72-pair batch (fused walking launch) returns, pair for pair, the bits of the pair's single alignment"""
    from dvo_slam_b200.engine import Config
    from test_gpu_mixed_batch import _same
    assert (H // TILE_H + 1) * len(_bands(W)) > lpm.COARSE_TILES >= (H // 2 // TILE_H + 1) * len(_bands(W // 2))
    eng = engine if est == "reference" else corrected
    cfg = Config(first_level=LEVELS - 1, last_level=0, max_iterations_per_level=50, precision=1e-4)
    pairs = batch400[est]
    res = eng.match_batch([p[0] for p in pairs], [p[1] for p in pairs], cfg)
    for k, (r, c) in enumerate(pairs):
        single = eng.match(r, c, cfg)
        assert not single.is_nan(), k
        assert _same(res[k], single), k
