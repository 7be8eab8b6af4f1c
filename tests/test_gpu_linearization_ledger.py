"""Every entry of the level kernel's linearisation against the fp64 ledger of its own residual records
(tests/linearization_ledger.py), at each entry's own scale.

The kernel's residual_image and linearize go into the ledger at one pose; n must be exact, and every entry of P, the
log-likelihood, A and b within its derived bound gamma_k M + E.  Cases: both estimators, use_weights 0 and 1 (with the
suite's prev_precision and with the P of the unweighted run), 640x480 levels 0-4, 1280x960 levels 0 and 5, the tile-edge
sizes of test_gpu_geometry, the generic-loop poses of test_gpu_generic_tiles, reference masks and masks in both roles,
non-default selection thresholds, and the photometric mode.  At the module's end one line gives the largest
|kernel - ledger| / bound per mode and quantity.
"""
import json

import numpy as np
import pytest

import linearization_ledger as L
from test_gpu_generic_tiles import _rot_z, _shift_z, partial_pair, partial_pose
from test_gpu_geometry import SIZES, _scene, _small_motion
from tile_geometry import assert_partial_band, level_shapes

pytestmark = pytest.mark.gpu

PP = np.array([[2000.0, -30.0], [-30.0, 9000.0]], dtype=np.float32)
ABS = [(1.0, 0.0), (1.1, -7.5), (0.85, 12.0)]                           # tests/test_gpu_photometric.py
THRESHOLDS = (4.0, 0.02)


@pytest.fixture(scope="module")
def maxima(request):
    found = {}
    yield found
    line = "linearisation ledger maxima (|kernel - ledger| / bound): " + json.dumps(
        {m: {k: float("%.3g" % v) for k, v in d.items()} for m, d in sorted(found.items())})
    cap = request.config.pluginmanager.getplugin("capturemanager")
    if cap is None:
        print("\n" + line)
    else:
        with cap.global_and_fixture_disabled():
            print("\n" + line)


@pytest.fixture(scope="module")
def engines(engine):
    from dvo_slam_b200.engine import Engine
    corrected = Engine(device=0, estimator="corrected")
    yield {"reference": engine, "corrected": corrected}
    corrected.close()


def _check(engines, maxima, mode, estimator, gref, gcur, level, T, K, ab=None, cfg=None):
    """residual_image + linearize of the kernel against the ledger, use_weights 0 and 1 (PP, and the unweighted run's P)"""
    eng = engines[estimator]
    n, rec = eng.residual_image(gref, gcur, level, T, cfg, ab)
    Ir = gref.download(level)[0] if ab is not None else None
    runs = [(False, PP)]
    first = eng.linearize(gref, gcur, level, T, False, PP, cfg, ab)
    runs.append((True, PP))
    if first["n"] >= 6:
        runs.append((True, np.asarray(first["precision"], np.float32)))
    for uw, pp in runs:
        out = first if not uw else eng.linearize(gref, gcur, level, T, uw, pp, cfg, ab)
        led = L.ledger(rec, K, level, out["precision"], estimator, uw, pp, I_ref=Ir)
        assert led.n == n == out["n"], (led.n, n, out["n"])
        rep = L.compare(led, out)
        d = maxima.setdefault(f"{mode}/{estimator}", {})
        for q, v in rep.maxima.items():
            d[q] = max(d.get(q, 0.0), v)
        assert not rep.failures, (mode, estimator, level, uw, rep.failures[:8])
    return n


# ---- sizes ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def bench640(engine):
    from dvo_slam_b200 import synth
    p = synth.make_pair(3)
    a = {k: p[k].numpy() for k in ("I_ref", "Z_ref", "I_cur", "Z_cur")}
    a["K"], a["T_true"], a["xi"] = p["intrinsics"], p["T_true"], p["xi"]
    a["gref"] = engine.pyramid(a["I_ref"], a["Z_ref"], a["K"], 5)
    a["gcur"] = engine.pyramid(a["I_cur"], a["Z_cur"], a["K"], 5)
    return a


def _poses(a):
    from dvo_slam_b200 import synth
    return {"true": a["T_true"], "perturbed": synth.se3_exp(a["xi"] * 0.9)}


@pytest.mark.parametrize("estimator", ["reference", "corrected"])
@pytest.mark.parametrize("level", [0, 1, 2, 3, 4])
def test_640x480(engines, maxima, bench640, level, estimator):
    a = bench640
    for T in _poses(a).values():
        _check(engines, maxima, "640x480", estimator, a["gref"], a["gcur"], level, T, a["K"])


@pytest.mark.parametrize("estimator", ["reference", "corrected"])
@pytest.mark.parametrize("level", [0, 5])
def test_1280x960(engine, engines, maxima, level, estimator):
    """bench.py --config 5: level 0 has 8 bands and 40 rounds of 32 pixels per row, the longest lane chains"""
    from dvo_slam_b200 import synth
    p = synth.make_pair(41, synth.SceneConfig().scaled(2))
    K = p["intrinsics"]
    gref = engine.pyramid(p["I_ref"].numpy(), p["Z_ref"].numpy(), K, 6)
    gcur = engine.pyramid(p["I_cur"].numpy(), p["Z_cur"].numpy(), K, 6)
    assert L.nbands(gref.level_info(0)[0]) == 8 and L.rounds(gref.level_info(0)[0]) == 40
    for T in (p["T_true"], synth.se3_exp(p["xi"] * 0.9)):
        _check(engines, maxima, "1280x960", estimator, gref, gcur, level, T, K)


@pytest.mark.parametrize("estimator", ["reference", "corrected"])
@pytest.mark.parametrize("w,h,levels", SIZES, ids=[f"{w}x{h}" for w, h, _ in SIZES])
def test_tile_edge_sizes(engine, engines, maxima, w, h, levels, estimator):
    a = _scene(w, h)
    gref = engine.pyramid(a["I_ref"], a["Z_ref"], a["K"], levels)
    gcur = engine.pyramid(a["I_cur"], a["Z_cur"], a["K"], levels)
    for lvl in range(len(level_shapes(w, h, levels))):
        _check(engines, maxima, "sizes", estimator, gref, gcur, lvl, _small_motion(), a["K"])


# ---- tile paths, masks, selection ------------------------------------------------------------------------------------------
GENERIC = {"roll20": (0, lambda a: _rot_z(20.0)),
           "corner_behind": (0, lambda a: _shift_z(-float(np.nanmedian(a["Z_ref"])))),
           "partial_band_l1": (1, lambda a: partial_pose()),        # on the 720 x 540 scene of test_gpu_generic_tiles
           "partial_band_l2": (2, lambda a: partial_pose())}


@pytest.fixture(scope="module")
def pair0(engine):
    """the scene of test_gpu_generic_tiles"""
    from dvo_slam_b200 import synth
    p = synth.make_pair(0)
    a = {k: p[k].numpy() for k in ("I_ref", "Z_ref", "I_cur", "Z_cur")}
    a["K"] = p["intrinsics"]
    a["gref"] = engine.pyramid(a["I_ref"], a["Z_ref"], a["K"], 5)
    a["gcur"] = engine.pyramid(a["I_cur"], a["Z_cur"], a["K"], 5)
    return a


@pytest.fixture(scope="module")
def pair720(engine):
    """the partial-band scene of test_gpu_generic_tiles"""
    a = partial_pair(0)
    a["gref"] = engine.pyramid(a["I_ref"], a["Z_ref"], a["K"], 5)
    a["gcur"] = engine.pyramid(a["I_cur"], a["Z_cur"], a["K"], 5)
    return a


@pytest.mark.parametrize("estimator", ["reference", "corrected"])
@pytest.mark.parametrize("case", list(GENERIC))
def test_generic_tile_paths(engines, maxima, pair0, pair720, case, estimator):
    level, pose = GENERIC[case]
    a = pair720 if case.startswith("partial_band") else pair0
    if a is pair720:
        assert_partial_band(a["gref"].level_info(level)[0])
    _check(engines, maxima, "generic", estimator, a["gref"], a["gcur"], level, pose(a), a["K"])


@pytest.fixture(scope="module")
def mask_scene():
    """synth pair 21 and the blob / border masks of test_gpu_mask_roles"""
    from dvo_slam_b200 import synth
    p = synth.make_pair(21)
    a = {k: p[k].numpy() for k in ("I_ref", "Z_ref", "I_cur", "Z_cur")}
    a["K"], a["xi"] = p["intrinsics"], p["xi"]
    h, w = a["I_ref"].shape
    rng = np.random.default_rng(5)
    yy, xx = np.ogrid[:h, :w]
    blobs = np.ones((h, w), np.uint8)
    for _ in range(10):
        cy, cx, r = rng.integers(0, h), rng.integers(0, w), rng.integers(5, 60)
        blobs[(yy - cy) ** 2 + (xx - cx) ** 2 <= r * r] = 0
    border = np.ones((h, w), np.uint8)
    border[:24, :] = 0
    border[:, :9] = 0
    a["masks"] = {"blobs": blobs, "border": border}
    return a


@pytest.mark.parametrize("estimator", ["reference", "corrected"])
@pytest.mark.parametrize("roles", ["reference", "both"])
@pytest.mark.parametrize("name", ["blobs", "border"])
def test_masks(engine, engines, maxima, mask_scene, name, roles, estimator):
    """a reference mask, and a mask in both roles on both images (the current image's taps take the cmask path)"""
    from dvo_slam_b200 import synth
    a, m = mask_scene, mask_scene["masks"][name]
    gref = engine.pyramid(a["I_ref"], a["Z_ref"], a["K"], 4, mask=m, mask_roles=roles)
    gcur = engine.pyramid(a["I_cur"], a["Z_cur"], a["K"], 4, mask=m, mask_roles=roles) if roles == "both" else \
        engine.pyramid(a["I_cur"], a["Z_cur"], a["K"], 4)
    T = np.linalg.inv(synth.se3_exp(a["xi"] * 0.7))
    for lvl in range(4):
        _check(engines, maxima, f"mask-{roles}", estimator, gref, gcur, lvl, T, a["K"])


@pytest.mark.parametrize("estimator", ["reference", "corrected"])
def test_selection_thresholds(engines, maxima, bench640, estimator):
    from dvo_slam_b200.engine import Config
    a = bench640
    cfg = Config(intensity_derivative_threshold=THRESHOLDS[0], depth_derivative_threshold=THRESHOLDS[1])
    for lvl in (0, 2, 4):
        n = _check(engines, maxima, "thresholds", estimator, a["gref"], a["gcur"], lvl, a["T_true"], a["K"], cfg=cfg)
        assert n < engines[estimator].residual_image(a["gref"], a["gcur"], lvl, a["T_true"])[0]


# ---- the photometric mode ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def photometric_pair(engine):
    """pair 3 of the 320 x 240 scene with the current frame's exposure changed"""
    import step_replay
    from dvo_slam_b200 import synth
    p = synth.make_pair(3, step_replay._scene320())
    a = {k: p[k].numpy() for k in ("I_ref", "Z_ref", "I_cur", "Z_cur")}
    a["I_cur"] = synth.exposure(a["I_cur"], 1.1, -7.5)
    a["K"], a["T_true"], a["xi"] = p["intrinsics"], p["T_true"], p["xi"]
    a["gref"] = engine.pyramid(a["I_ref"], a["Z_ref"], a["K"], 3)
    a["gcur"] = engine.pyramid(a["I_cur"], a["Z_cur"], a["K"], 3)
    return a


@pytest.mark.parametrize("estimator", ["reference", "corrected"])
@pytest.mark.parametrize("ab", ABS, ids=[f"{x}_{y}" for x, y in ABS])
def test_photometric(engines, maxima, photometric_pair, ab, estimator):
    a = photometric_pair
    for lvl in (0, 2):
        for T in _poses(a).values():
            _check(engines, maxima, "photometric", estimator, a["gref"], a["gcur"], lvl, T, a["K"], ab=ab)
    _check(engines, maxima, "photometric", estimator, a["gref"], a["gcur"], 0, _rot_z(20.0), a["K"], ab=ab)
