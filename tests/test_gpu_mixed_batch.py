"""Fused batches whose pairs differ in everything a batch allows to differ, against single alignments and the oracle.

A batch shares one launch plan and one level geometry, taken from its first reference; everything else is per pair: the
current camera's intrinsics (they go into each pair's K T and Jacobian constants), the reference and current pyramids'
level counts, the context and stream a pyramid was built on, and pyramids shared between pairs.  "Batch == single, bit
for bit" is the guard against state that leaks from one pair to another, so it is asserted here on batches where no two
neighbouring pairs have the same intrinsics.  Also: an engine on a caller-supplied stream, and a batch of mixed sizes.
"""
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

from helpers import nan_equal, pose_delta
from test_gpu_generic_tiles import _rot_z, _shift_z
from tile_geometry import TILE_H, TILE_W

pytestmark = pytest.mark.gpu

COARSE_TILES = 110          # make_launch_plan (csrc/launch_plan.h): a level of at most this many tiles runs one CTA per pair
CTAS_PER_SM = 2             # the level kernel's occupancy on an H100 (DESIGN.md)
PP = np.array([[2000.0, -30.0], [-30.0, 9000.0]], dtype=np.float32)


def _grid():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count * CTAS_PER_SM


def _tiles(w, h):
    return -(-w // TILE_W) * -(-h // TILE_H)


def _same(a, b):
    return (np.array_equal(a.transformation, b.transformation) and np.array_equal(a.information, b.information)
            and (a.log_likelihood == b.log_likelihood or (np.isnan(a.log_likelihood) and np.isnan(b.log_likelihood)))
            and repr(a.levels) == repr(b.levels))


def _flow(levels):
    return [l["termination"] for l in levels], [l["num_iterations"] for l in levels]


# ---- 1. mixed intrinsics, 160 x 120, one walking group ----
W, H = 160, 120
NPAIRS = 96
BASE_K = (129.325, 129.125, 79.65, 63.825)            # fr1 / 4
# 8 intrinsics sets: focal lengths from -9 % to +12 %, principal points moved by up to 4 px
K_SETS = [(BASE_K[0] * s, BASE_K[1] * s * q, BASE_K[2] + dx, BASE_K[3] + dy)
          for s, q, dx, dy in ((1.0, 1.0, 0.0, 0.0), (0.91, 1.004, 2.5, -1.5), (1.12, 0.997, -3.0, 2.0), (1.05, 1.01, 1.2, 3.7),
                               (0.95, 0.99, -4.0, -2.2), (1.08, 1.0, 3.3, 0.4), (0.97, 1.006, -1.1, -3.9), (1.02, 0.994, 0.7, 1.9))]


def _perturbed(K):
    """the current camera's intrinsics off by a few percent from the reference's"""
    fx, fy, ox, oy = K
    return (fx * 1.03, fy * 0.975, ox + 1.5, oy - 1.25)


def _pair_spec(i):
    """(intrinsics set, current K differs from reference K, reference levels, current levels, built on the second engine)"""
    return i % 8, i % 4 == 3, 4 if i % 3 == 0 else 3, 3 if i % 2 == 0 else 4, i % 5 == 1


@pytest.fixture(scope="module")
def second_engine():
    from dvo_slam_b200.engine import Engine
    eng = Engine(device=0)
    yield eng
    eng.close()


@pytest.fixture(scope="module")
def small_batch(engine, second_engine):
    from dvo_slam_b200 import synth
    imgs, specs = [], []
    for i in range(NPAIRS):
        ks, pert, lr, lc, other = _pair_spec(i)
        p = synth.make_pair(3000 + i, synth.SceneConfig(width=W, height=H, intrinsics=K_SETS[ks]))
        imgs.append({k: p[k].numpy() for k in ("I_ref", "Z_ref", "I_cur", "Z_cur")})
        specs.append(dict(Kr=K_SETS[ks], Kc=_perturbed(K_SETS[ks]) if pert else K_SETS[ks], lr=lr, lc=lc, other=other, ks=ks,
                          pert=pert))
    # one pyramid_batch call per (engine, intrinsics, level count, side): 2 x 8 x ... calls of a few images each
    refs, curs = [None] * NPAIRS, [None] * NPAIRS
    for side, out in (("ref", refs), ("cur", curs)):
        groups = {}
        for i, s in enumerate(specs):
            key = (s["other"], s["Kr"] if side == "ref" else s["Kc"], s["lr"] if side == "ref" else s["lc"])
            groups.setdefault(key, []).append(i)
        for (other, K, lv), idx in groups.items():
            eng = second_engine if other else engine
            I = np.stack([imgs[i]["I_" + side] for i in idx]); Z = np.stack([imgs[i]["Z_" + side] for i in idx])
            for i, p in zip(idx, eng.pyramid_batch(I, Z, K, lv)):
                out[i] = p
    pairs = [(refs[i], curs[i], i) for i in range(NPAIRS)]
    # a pyramid shared between pairs: reference 0 is the reference of two more pairs and the current of another
    pairs += [(refs[0], curs[0], 0), (curs[0], refs[0], -1), (refs[0], curs[0], 0)]
    return dict(imgs=imgs, specs=specs, refs=refs, curs=curs, pairs=pairs)


def _cfg(first, last):
    from dvo_slam_b200.engine import Config
    return Config(first_level=first, last_level=last, max_iterations_per_level=50, precision=1e-4)


def test_small_batch_is_one_walking_group(small_batch):
    """every level of 160 x 120 is coarse and the batch holds more than grid / 4 pairs: the whole match is one launch in
    which each CTA walks its pair through all levels"""
    assert len(small_batch["pairs"]) >= _grid() // 4
    assert all(_tiles(W >> l, H >> l) <= COARSE_TILES for l in range(3))
    s = small_batch["specs"]
    assert {x["ks"] for x in s} == set(range(8)) and sum(x["pert"] for x in s) == NPAIRS // 4
    assert {x["lr"] for x in s} == {3, 4} and {x["lc"] for x in s} == {3, 4} and any(x["other"] for x in s)


def test_small_batch_equals_single_and_the_oracle(engine, oracle, small_batch):
    cfg = _cfg(2, 0)
    pairs = small_batch["pairs"]
    refs, curs = [p[0] for p in pairs], [p[1] for p in pairs]
    res = engine.match_batch(refs, curs, cfg)
    again = engine.match_batch(refs, curs, cfg)
    for k, (r, c, _) in enumerate(pairs):
        assert _same(res[k], again[k]), k
        assert _same(res[k], engine.match(r, c, cfg)), k
        assert not res[k].is_nan(), k
    assert _same(res[0], res[NPAIRS]) and _same(res[0], res[NPAIRS + 2])

    # the oracle: every pair whose current K differs, and the first two pairs of every intrinsics set
    specs, imgs = small_batch["specs"], small_batch["imgs"]
    check = sorted({i for i, s in enumerate(specs) if s["pert"]} |
                   {i for ks in range(8) for i in [j for j, s in enumerate(specs) if s["ks"] == ks and not s["pert"]][:2]})
    assert len(check) >= 12
    ocfg = oracle.config(first_level=2, last_level=0, max_iterations_per_level=50, precision=1e-4)

    def cpu(i):
        s, a = specs[i], imgs[i]
        oref = oracle.Pyramid(a["I_ref"], a["Z_ref"], s["Kr"], s["lr"])
        ocur = oracle.Pyramid(a["I_cur"], a["Z_cur"], s["Kc"], s["lc"])
        return oracle.match(oref, ocur, ocfg, oracle.mode("mirror"))

    with ThreadPoolExecutor(os.cpu_count() or 8) as ex:
        orc = dict(zip(check, ex.map(cpu, check)))
    same = 0
    for i in check:
        o, r = orc[i], res[i]
        assert [l["valid_pixels"] for l in r.levels] == [l["valid_pixels"] for l in o["levels"]], i
        if _flow(r.levels) == _flow(o["levels"]):
            same += 1
            dt, dr = pose_delta(o["T"], r.transformation)
            assert dt < 1e-4 and dr < 1e-4, (i, dt, dr)
    assert same >= len(check) // 2, (same, len(check))
    print(f"\n{len(check)} pairs against MIRROR, {same} with MIRROR's control flow")


def test_current_intrinsics_at_a_fixed_pose(engine, oracle, small_batch):
    """the current camera's K, not the reference's, projects the points: residual records and the error image bit-exact,
    P / LL / A / b to 2e-6, where the two differ"""
    specs, imgs = small_batch["specs"], small_batch["imgs"]
    mir = oracle.mode("mirror")
    T = _rot_z(0.7) @ _shift_z(0.008)
    T[0, 3] = -0.005
    idx = [i for i, s in enumerate(specs) if s["pert"]][:3]
    for i in idx:
        s, a = specs[i], imgs[i]
        gref, gcur = small_batch["refs"][i], small_batch["curs"][i]
        assert gref.level_info(0)[2] != gcur.level_info(0)[2]
        oref = oracle.Pyramid(a["I_ref"], a["Z_ref"], s["Kr"], s["lr"])
        ocur = oracle.Pyramid(a["I_cur"], a["Z_cur"], s["Kc"], s["lc"])
        for lvl in range(3):
            n_g, img_g = engine.residual_image(gref, gcur, lvl, T)
            n_o, img_o = oracle.residual_image(oref, ocur, lvl, T, mir)
            assert n_g == n_o > 0 and nan_equal(img_g, img_o), (i, lvl)
            # and the reference's K would have given other records
            ocur_k = oracle.Pyramid(a["I_cur"], a["Z_cur"], s["Kr"], s["lc"])
            assert not nan_equal(oracle.residual_image(oref, ocur_k, lvl, T, mir)[1], img_o)
            ne_g, err_g = engine.intensity_error_image(gref, gcur, lvl, T)
            ne_o, err_o = oracle.intensity_error_image(oref, ocur, lvl, T, mir)
            assert ne_g == ne_o and np.array_equal(err_g, err_o), (i, lvl)
            for uw in (False, True):
                lg = engine.linearize(gref, gcur, lvl, T, uw, PP)
                lo = oracle.linearize(oref, ocur, lvl, T, mir, uw, PP)
                assert lg["n"] == lo["n"] == n_o
                assert np.allclose(lg["precision"], lo["precision"], rtol=0, atol=2e-6 * np.abs(lo["precision"]).max())
                assert abs(lg["ll"] - lo["ll"]) <= 2e-6 * abs(lo["ll"]) + 0.5
                assert np.allclose(lg["A"], lo["A"], rtol=0, atol=2e-6 * np.abs(lo["A"]).max())
                assert np.allclose(lg["b"], lo["b"], rtol=0, atol=2e-6 * np.abs(lo["b"]).max())


# ---- 2. mixed intrinsics, 640 x 480: level 0 in squads of several CTAs ----
FULL_PAIRS = 72
FR1 = (517.3, 516.5, 318.6, 255.3)
FULL_K_SETS = [(FR1[0] * s, FR1[1] * s * q, FR1[2] + dx, FR1[3] + dy)
               for s, q, dx, dy in ((1.0, 1.0, 0.0, 0.0), (0.92, 1.003, 6.0, -4.0), (1.1, 0.996, -8.0, 5.0),
                                    (1.04, 1.008, 3.0, 9.0), (0.96, 0.992, -10.0, -6.0), (1.07, 1.0, 8.5, 1.0))]


@pytest.fixture(scope="module")
def full_batch(engine):
    import torch
    from dvo_slam_b200 import synth
    dev = torch.device("cuda", 0)
    refs, curs = [None] * FULL_PAIRS, [None] * FULL_PAIRS
    for ks, K in enumerate(FULL_K_SETS):
        idx = [i for i in range(FULL_PAIRS) if i % len(FULL_K_SETS) == ks]
        ps = [synth.make_pair(4000 + i, synth.SceneConfig(intrinsics=K), device=dev) for i in idx]
        for side, out in (("ref", refs), ("cur", curs)):
            I = np.stack([p["I_" + side].cpu().numpy() for p in ps]); Z = np.stack([p["Z_" + side].cpu().numpy() for p in ps])
            for i, p in zip(idx, engine.pyramid_batch(I, Z, K, 5)):
                out[i] = p
    return refs, curs


@pytest.mark.parametrize("estimator", ["reference", "corrected"])
def test_full_size_mixed_intrinsics_equal_single(engine, full_batch, estimator):
    from dvo_slam_b200.engine import Engine
    refs, curs = full_batch
    assert FULL_PAIRS >= _grid() // 4 and _tiles(640, 480) > COARSE_TILES      # level 0 is a fine level: squads, walked
    assert len({r.level_info(0)[2] for r in refs[:len(FULL_K_SETS)]}) == len(FULL_K_SETS)
    eng = engine if estimator == "reference" else Engine(device=0, estimator="corrected")
    try:
        cfg = _cfg(4, 0)
        res = eng.match_batch(refs, curs, cfg)
        for i in range(FULL_PAIRS):
            assert _same(res[i], eng.match(refs[i], curs[i], cfg)), i
            assert not res[i].is_nan(), i
    finally:
        if eng is not engine:
            eng.close()


# ---- 3. a caller-supplied stream ----
def test_caller_supplied_stream(engine, small_batch):
    import torch
    from dvo_slam_b200.engine import Engine
    specs, imgs = small_batch["specs"], small_batch["imgs"]
    n = 6
    K = specs[0]["Kr"]
    Ir = np.stack([imgs[i]["I_ref"] for i in range(n)]); Zr = np.stack([imgs[i]["Z_ref"] for i in range(n)])
    Ic = np.stack([imgs[i]["I_cur"] for i in range(n)]); Zc = np.stack([imgs[i]["Z_cur"] for i in range(n)])
    stream = torch.cuda.Stream(device=0)
    eng = Engine(device=0, stream=stream.cuda_stream)
    try:
        assert eng.stream == stream.cuda_stream
        outs = []
        for e in (engine, eng):
            refs, curs = e.pyramid_batch(Ir, Zr, K, 3), e.pyramid_batch(Ic, Zc, K, 3)
            o = [bytes(e.match_batch(refs, curs, _cfg(2, 0), raw=True))]
            T = _rot_z(1.0) @ _shift_z(0.01)
            for i in range(n):
                for lvl in range(3):
                    o += [refs[i].download(lvl), curs[i].download(lvl), refs[i].select(lvl)[1]]
                    o += list(e.residual_image(refs[i], curs[i], lvl, T)) + list(e.intensity_error_image(refs[i], curs[i], lvl, T))
                    for uw in (False, True):
                        o += list(e.linearize(refs[i], curs[i], lvl, T, uw, PP).values())
            outs.append(o)
            for p in refs + curs:
                p.release()
        for k, (a, b) in enumerate(zip(*outs)):
            if isinstance(a, np.ndarray):
                assert np.array_equal(a.view(np.uint8), b.view(np.uint8)), k
            else:
                assert a == b or (a != a and b != b), k
    finally:
        eng.close()
    # the stream is the caller's: closing the engine leaves it usable
    with torch.cuda.stream(stream):
        x = torch.arange(1000, device="cuda", dtype=torch.float64) * 2.0
        s = x.sum()
    stream.synchronize()
    assert float(s) == 999000.0


# ---- 4. a batch of mixed sizes ----
def test_shape_mismatch_is_a_status(engine, small_batch):
    from dvo_slam_b200 import synth
    cfg = _cfg(2, 0)
    r0, c0 = small_batch["refs"][2], small_batch["curs"][2]
    before = engine.match(r0, c0, cfg)
    p = synth.make_pair(5, synth.SceneConfig(width=W + 2, height=H, intrinsics=K_SETS[0]))
    other = engine.pyramid(p["I_ref"].numpy(), p["Z_ref"].numpy(), K_SETS[0], 3)
    for refs, curs in (([r0, other], [c0, other]), ([r0, r0], [c0, other]), ([other], [c0])):
        with pytest.raises(RuntimeError, match="status -4"):          # DVO_B200_ERR_SHAPE_MISMATCH
            engine.match_batch(refs, curs, cfg)
    # the context keeps working, on both sizes
    assert _same(engine.match(r0, c0, cfg), before)
    r = engine.match(other, other, cfg)
    assert not r.is_nan() and _same(r, engine.match_batch([other, other], [other, other], cfg)[1])
