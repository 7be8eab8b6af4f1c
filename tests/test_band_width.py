"""The level kernel's 160-column bands.

Tiles are 160 x 7 reference pixels, so the 640-, 320- and 160-pixel-wide levels of a 640 x 480 pyramid are whole bands and
their tiles take the exact pixel loops (which end with an odd fifth stage-A round).  A partial band now needs a width that
is not a multiple of 160: 400 x 300 has bands of 160, 160 and 80 columns at level 0 and of 160 and 40 at level 1, so each
level has both full bands (exact loops) and a partial band (generic loop).  That case is checked here as the other
generic-loop cases are: residual records bit-exact against the oracle's MIRROR mode (and the corrected estimator's
definition), and a batch returning the bits of single alignments, for both estimators.  On the host: the compiled tile
geometry is the one the suite computes with (tests/tile_geometry.py), and the shared-memory layout still leaves room for
two CTAs per SM.
"""
import os
import shutil
import subprocess

import numpy as np
import pytest

import launch_plan_model as lpm
import tile_geometry as tg
from tile_geometry import TILE_H, TILE_W, assert_partial_band, bands

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
W, H, LEVELS = 400, 300, 4
CARVEOUT, SMEM_RESERVED_PER_CTA = 196 * 1024, 1024     # of an H100 SM's 256 KB: 60 KB stay L1; 1 KB per resident CTA
LARGEST_TAIL = 5696      # sizeof(LevelTailOf<true, true>) (photometric, motion prior) in tracker.cu under nvcc 12.9


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
    copies the first 1 200; every bulk copy is a multiple of 16 bytes.  The suite's geometry (tests/tile_geometry.py) is the
    compiled one."""
    L = layout
    assert (L["tile_w"], L["tile_h"], L["win_cols"], L["win_rows"]) == (tg.TILE_W, tg.TILE_H, tg.WIN_COLS, tg.WIN_ROWS)
    assert (L["tile_w"], L["tile_h"], L["win_cols"], L["win_rows"], L["stages"]) == (160, 7, 160 + 24, 19, 2)
    assert lpm.TILE_W == tg.TILE_W and lpm.TILE_H == tg.TILE_H
    assert L["rec_bytes"] == 8 * (2 * TILE_H * TILE_W + TILE_W // 2) == 18560
    assert L["rec_stage_a_bytes"] == 8 * (TILE_H * TILE_W + TILE_W // 2) == 9600
    assert L["rec_bytes"] % 16 == 0 and L["rec_stage_a_bytes"] % 16 == 0 and (8 * L["win_cols"]) % 16 == 0
    assert L["win_cols"] < 256                                  # produce_tiles packs the window width into 8 bits
    assert bands(640) == [160] * 4 and bands(320) == [160] * 2 and bands(160) == [160]
    assert bands(W) == [160, 160, 80] and bands(W // 2) == [160, 40]


def test_partial_band_helper():
    """the helper the partial-band cases assert their geometry with: full bands followed by a partial one, nothing else"""
    assert assert_partial_band(W) == [160, 160, 80] and assert_partial_band(W // 2) == [160, 40]
    assert assert_partial_band(161) == [160, 1] and assert_partial_band(319) == [160, 159]
    for w in (640, 320, 160, 80, 40, 128, 1280):
        with pytest.raises(AssertionError):
            assert_partial_band(w)
    assert tg.in_partial_band(160, 161) and not tg.in_partial_band(159, 161) and not tg.in_partial_band(319, 320)
    assert tg.level_shapes(640, 480, 5) == [(640, 480), (320, 240), (160, 120), (80, 60), (40, 30)]
    assert tg.strips(480) == [7] * 68 + [4] and tg.strips(14) == [7, 7]


def test_tile_edge_sizes_state_their_case():
    """every size of test_gpu_geometry reaches the case it states on 160-column bands; the sizes chosen for 128-column
    bands (a 1-, 33- and 63-column band at 129, 161 and 191, whole bands at 256) are refused"""
    from test_gpu_geometry import SIZES, _assert_reason
    for w, h, levels in SIZES:
        _assert_reason(w, h, levels)
    partial = sorted(bands(w)[-1] for w, _, _ in SIZES if len(bands(w)) >= 2 and bands(w)[-1] < TILE_W)
    assert {1, 33, 63, 128, 159} <= set(partial), partial
    for w, h, levels in ((129, 50, 3), (161, 55, 3), (191, 49, 3), (256, 96, 3)):
        with pytest.raises(AssertionError):
            _assert_reason(w, h, levels)


def test_shared_memory_leaves_two_ctas_per_sm(layout):
    """Two stage buffers (record + window, 128-byte aligned) and the barriers fill 93 312 bytes; with the largest tail of
    shared state after the pipeline, two CTAs fit in the 196 KB shared-memory carveout, which leaves 60 KB of L1 (tracker.cu
    asserts two CTAs per SM of every instance at build time)."""
    L = layout
    assert L["stage_buf"] == (L["rec_bytes"] + 8 * L["win_rows"] * L["win_cols"] + 127) // 128 * 128 == 46592
    assert L["tile_pipe"] == 93312
    assert L["seg_combine"] < LARGEST_TAIL           # the tail holds the strip combine's scratch and the end step's state
    assert 2 * (L["tile_pipe"] + LARGEST_TAIL + SMEM_RESERVED_PER_CTA) <= CARVEOUT


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
    assert_partial_band(W >> lvl)
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
    assert (H // TILE_H + 1) * len(bands(W)) > lpm.COARSE_TILES >= (H // 2 // TILE_H + 1) * len(bands(W // 2))
    eng = engine if est == "reference" else corrected
    cfg = Config(first_level=LEVELS - 1, last_level=0, max_iterations_per_level=50, precision=1e-4)
    pairs = batch400[est]
    res = eng.match_batch([p[0] for p in pairs], [p[1] for p in pairs], cfg)
    for k, (r, c) in enumerate(pairs):
        single = eng.match(r, c, cfg)
        assert not single.is_nan(), k
        assert _same(res[k], single), k
