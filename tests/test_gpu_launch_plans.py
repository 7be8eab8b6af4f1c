"""Every launch plan of the level kernel returns, for every pair of a batch, the bits of the pair's single alignment.

The plan is chosen on the host (csrc/launch_plan.h: make_launch_plan) from the batch size, the grid (SMs x resident CTAs
per SM) and the level geometry: one launch per level with squads of up to 69 CTAs for small batches; for batches of at
least grid/4 pairs a coarse segment with one CTA per pair, fused with up to three slices of the fine levels with squads of
g, 2g and 4g CTAs; and the developer overrides DVO_B200_* on top.  The strict oracle comparisons run on the single-pair
path, so they speak for a batch only if every plan returns the same bits.

The plan is restated in plain Python in launch_plan_model.py.  It picks the batch sizes -- the first and last size of
every plan shape -- and each case asserts the shape it exists for; on the device the number of persistent launches the
profiler counts must equal the restatement's.  Batches mix ordinary seeded pairs with pairs that finish at very different
times (a current frame without depth: TooFewConstraints on every level; identical frames; masked references; keyframe
pairs that share one reference pyramid), placed at both ends of the batch and of every slice.  Expected results are single
alignments, one per (pair, configuration, estimator), computed once with no override set.
"""
import contextlib
import ctypes as C
import os

import numpy as np
import pytest

from launch_plan_model import KNOBS, OVERRIDES, boundary_sizes, level_geometry, plan, shape, size_of_shape


def special_positions(n, p):
    """both ends of the batch and of every fine slice"""
    pos = {0, n - 1}
    for _, b, c in p["slices"]:
        pos |= {b, b + c - 1}
    return sorted(pos)


GEOM_640 = level_geometry(640, 480, 5)
GEOM_1280 = level_geometry(1280, 960, 6)
SIZES_264 = [1, 2, 65, 66, 67, 88, 89, 132, 133, 264, 265, 294, 295, 370, 371, 382, 383, 441, 442, 512]


def test_restated_plan_at_264_ctas():
    """The plan on an H100 SXM (132 SMs x 2 CTAs) at 640x480, levels 4..0, for every batch size up to 1077, as DESIGN 4.1
    and the sizes of this file rely on; and the other geometries' shapes."""
    grid = 264
    g0 = []
    for n in range(1, 1078):
        p = plan(GEOM_640, 4, 0, grid, n)
        if n <= 65:
            assert not p["walk"] and p["launches"] == 5 and [G["nlev"] for G in p["groups"]] == [1] * 5, n
            g0.append(p["groups"][-1]["g"])
            continue
        assert p["walk"] and p["fused"] and p["launches"] == 1, n
        assert [(G["first_li"], G["nlev"], G["g"]) for G in p["groups"]][0] == (0, 4, 1), n   # levels 4..1, one CTA per pair
        # from 371 pairs on, the fine level takes squads of 2: one slice until the first keeps two pairs per squad beside
        # the second (383), two until it does so beside the third as well (442)
        want = ((4,) if n == 66 else (3,) if n <= 88 else (2,) if n <= 132 else (1,) if n <= 264 else (3, 6) if n <= 294
                else (3, 6, 12) if n <= 370 else (2,) if n <= 382 else (2, 4) if n <= 441 else (2, 4, 8) if n <= 879
                else (1, 2) if n <= 884 else (1, 2, 4))
        assert tuple(s[0] for s in p["slices"]) == want, (n, p["slices"])
        if n in (265, 294):
            assert [s[2] for s in p["slices"]] == [n - 79, 79]
    assert g0[0] == 69 and sorted(set(g0), reverse=True)[:3] == [69, 35, 23] and g0[-1] == 4
    assert all(a >= b for a, b in zip(g0, g0[1:]))
    assert plan(GEOM_640, 4, 0, grid, 265)["slices"] == [(3, 0, 186), (6, 186, 79)]
    assert plan(GEOM_640, 4, 0, grid, 512)["slices"] == [(2, 0, 334), (4, 334, 119), (8, 453, 59)]   # DESIGN 4.1
    assert plan(GEOM_640, 4, 0, grid, 371)["slices"] == [(2, 0, 371)]
    assert plan(GEOM_640, 4, 0, grid, 383)["slices"] == [(2, 0, 264), (4, 264, 119)]
    assert plan(GEOM_640, 4, 0, grid, 442)["slices"] == [(2, 0, 264), (4, 264, 119), (8, 383, 59)]
    assert boundary_sizes(GEOM_640, 4, 0, grid) == SIZES_264
    # 1280x960, levels 5..0: a fine group of two levels (1 and 0) behind the coarse walk; three slices of 6 / 12 / 24 at 148..167
    for n in range(148, 168):
        p = plan(GEOM_1280, 5, 0, grid, n)
        assert p["fused"] and p["groups"][1]["nlev"] == 2 and [s[0] for s in p["slices"]] == [6, 12, 24], n
    assert [s[0] for s in plan(GEOM_1280, 5, 0, grid, 168)["slices"]] == [1]
    assert size_of_shape(GEOM_1280, 5, 0, grid, ("fused", 6, 12, 24), pick="first") == 148
    assert size_of_shape(GEOM_1280, 5, 0, grid, ("fused", 6, 12, 24), pick="last") == 167
    # levels 3..1: a coarse-only walk (one launch instead of three); level 0 alone: a walk without fusion
    for n in (66, 100, 512):
        p = plan(GEOM_640, 3, 1, grid, n)
        assert not p["fused"] and [(G["nlev"], G["g"]) for G in p["groups"]] == [(3, 1)] and p["launches"] == 1
        q = plan(GEOM_640, 0, 0, grid, n)
        assert q["walk"] and not q["fused"] and len(q["groups"]) == 1 and q["launches"] == 1
    assert plan(GEOM_640, 3, 1, grid, 65)["launches"] == 3
    # the overrides at 512
    env = lambda **kw: {f"DVO_B200_{k}": v for k, v in kw.items()}
    assert plan(GEOM_640, 4, 0, grid, 512, env(NO_WALK="1"))["launches"] == 5
    assert plan(GEOM_640, 4, 0, grid, 512, env(NO_FUSE="1"))["launches"] == 2
    assert [G["nlev"] for G in plan(GEOM_640, 4, 0, grid, 512, env(COARSE_TILES="0"))["groups"]] == [5]
    p = plan(GEOM_640, 4, 0, grid, 512, env(COARSE_TILES="40"))
    assert p["fused"] and [G["nlev"] for G in p["groups"]] == [3, 2]
    p = plan(GEOM_640, 4, 0, grid, 512, env(COARSE_TILES="400"))
    assert [(G["nlev"], G["g"]) for G in p["groups"]] == [(5, 1)] and p["launches"] == 1
    assert plan(GEOM_640, 4, 0, grid, 512, env(TAIL="0,0"))["slices"] == [(2, 0, 512)]
    assert plan(GEOM_640, 4, 0, grid, 512, env(TAIL="60,30"))["slices"] == [(2, 0, 422), (4, 422, 60), (8, 482, 30)]
    assert plan(GEOM_640, 4, 0, grid, 512, env(TAIL="180,90"))["slices"] == [(2, 0, 332), (4, 332, 180)]
    assert plan(GEOM_640, 4, 0, grid, 512, env(STRIPS_PER_CTA="1"))["slices"] == [(69, 0, 512)]
    assert plan(GEOM_640, 4, 0, grid, 512, env(STRIPS_PER_CTA="3"))["slices"] == [(23, 0, 503), (46, 503, 9)]
    assert plan(GEOM_640, 4, 0, grid, 512, env(STRIPS_PER_CTA="69"))["slices"] == [(1, 0, 512)]
    assert plan(GEOM_640, 4, 0, grid, 512, env(FINE_G="1"))["slices"] == [(1, 0, 512)]
    assert plan(GEOM_640, 4, 0, grid, 512, env(FINE_G="4"))["slices"] == [(4, 0, 424), (8, 424, 59), (16, 483, 29)]
    assert plan(GEOM_640, 4, 0, grid, 512, env(FINE_G="8"))["slices"] == [(8, 0, 469), (16, 469, 29), (32, 498, 14)]


# ---- the device side ----
CFGS = {
    "4..0": dict(first_level=4, last_level=0, max_iterations_per_level=50, precision=1e-4),
    "3..1": dict(first_level=3, last_level=1, max_iterations_per_level=50, precision=1e-4),
    "0..0": dict(first_level=0, last_level=0, max_iterations_per_level=50, precision=1e-4),
    "5..0": dict(first_level=5, last_level=0, max_iterations_per_level=50, precision=1e-4),
    # iteration logs, a prior and per-pair initial estimates
    "4..0 init": dict(first_level=4, last_level=0, max_iterations_per_level=50, precision=1e-4, mu=0.05, use_initial_estimate=1),
}


@contextlib.contextmanager
def _no_overrides():
    saved = {k: os.environ.pop(k) for k in KNOBS if k in os.environ}
    try:
        yield
    finally:
        os.environ.update(saved)


def _raw(eng, refs, curs, cfg, T=None, log=False):
    """dvo_b200_match_batch -> per pair: the result record's bytes, followed by its iteration-log slots' bytes with log"""
    from dvo_slam_b200.engine import CResult, IterationStats
    n = len(refs)
    rh = (C.c_void_p * n)(*[p.handle for p in refs])
    ch = (C.c_void_p * n)(*[p.handle for p in curs])
    max_log = (cfg.first_level - cfg.last_level + 1) * (cfg.max_iterations_per_level + 1) if log else 0
    res = (CResult * n)()
    lg = (IterationStats * (n * max_log))() if log else None
    Tp = None if T is None else np.ascontiguousarray(np.asarray(T, np.float64).reshape(n, 16))
    eng._check(eng.lib.dvo_b200_match_batch(eng.ctx, C.byref(cfg), n, rh, ch,
                                            None if Tp is None else Tp.ctypes.data_as(C.POINTER(C.c_double)), res, lg, max_log))
    rb, lb = bytes(res), bytes(lg) if log else b""
    r, s = C.sizeof(CResult), C.sizeof(IterationStats) * max_log
    return [rb[i * r:(i + 1) * r] + lb[i * s:(i + 1) * s] for i in range(n)]


def _diff(got, want):
    """the first field in which two records differ"""
    from dvo_slam_b200.engine import CResult, IterationStats
    r = C.sizeof(CResult)
    a, b = CResult.from_buffer_copy(got[:r]), CResult.from_buffer_copy(want[:r])
    for f, _ in CResult._fields_:
        va, vb = getattr(a, f), getattr(b, f)
        if hasattr(va, "_length_") or isinstance(va, C.Structure):
            if bytes(va) != bytes(vb):
                return f
        elif not (va == vb or (va != va and vb != vb)):
            return f"{f} {va} != {vb}"
    s = C.sizeof(IterationStats)
    for k in range((len(got) - r) // s):
        if got[r + k * s:r + (k + 1) * s] != want[r + k * s:r + (k + 1) * s]:
            return f"iteration log entry {k}"
    return "bytes"


class Pool:
    """Distinct pairs of one image size, as pyramids on one context.  Kinds: ordinary seeded pairs; keyframe pairs that
    share one reference pyramid; a current frame without depth (TooFewConstraints on every level); identical frames (the
    reference pyramid passed as the current one); masked references."""

    def __init__(self, eng, scfg, levels, n_ord, seed0):
        import torch
        from dvo_slam_b200 import synth
        dev = torch.device("cuda", 0)
        self.w, self.h, self.levels, self.K = scfg.width, scfg.height, levels, scfg.intrinsics
        self.kinds, self.handles = [], []
        I = np.empty((2 * n_ord, scfg.height, scfg.width), np.float32)
        Z = np.empty_like(I)
        xi = []
        for i in range(n_ord):
            p = synth.make_pair(seed0 + i, scfg, device=dev)
            I[i], Z[i] = p["I_ref"].cpu().numpy(), p["Z_ref"].cpu().numpy()
            I[n_ord + i], Z[n_ord + i] = p["I_cur"].cpu().numpy(), p["Z_cur"].cpu().numpy()
            xi.append(p["xi"])
        pyr = self._keep(eng.pyramid_batch(I, Z, self.K, levels))
        self.ordinary = [self._kind(f"seed{seed0 + i}", pyr[i], pyr[n_ord + i], synth.se3_exp(0.8 * xi[i])) for i in range(n_ord)]
        frames, _ = synth.make_sequence(seed0 + 500, 5, scfg, device=dev)
        fI = np.stack([f[0].cpu().numpy() for f in frames])
        fZ = np.stack([f[1].cpu().numpy() for f in frames])
        key = self._keep(eng.pyramid_batch(fI, fZ, self.K, levels))
        rng = np.random.default_rng(seed0)
        self.keyframe = [self._kind(f"keyframe{k}", key[0], key[k], synth.se3_exp(rng.uniform(-0.01, 0.01, 6))) for k in range(1, 5)]
        nan_cur = self._keep(eng.pyramid_batch(I[n_ord:n_ord + 2], np.full_like(Z[:2], np.nan), self.K, levels))
        self.nan = [self._kind(f"nan-depth{i}", pyr[i], nan_cur[i], np.eye(4)) for i in range(2)]
        self.identical = [self._kind("identical0", pyr[2], pyr[2], np.eye(4)),
                          self._kind("identical1", key[0], key[0], synth.se3_exp(rng.uniform(-0.01, 0.01, 6)))]
        self.masked = []
        for j in range(2):
            m = synth.make_moving_object_pair(seed0 + 900 + j, scfg)
            ref = self._keep([eng.pyramid(m["I_ref"], m["Z_ref"], self.K, levels, mask=m["mask"])])[0]
            cur = self._keep([eng.pyramid(m["I_cur"], m["Z_cur"], self.K, levels)])[0]
            self.masked.append(self._kind(f"masked{j}", ref, cur, synth.se3_exp(0.5 * m["xi"])))
        self.special = [self.nan[0], self.identical[0], self.masked[0], self.keyframe[0],
                        self.nan[1], self.identical[1], self.masked[1], self.keyframe[1]]
        self.geom = level_geometry(self.w, self.h, levels)

    def _keep(self, pyrs):
        self.handles += pyrs
        return pyrs

    def _kind(self, name, ref, cur, T):
        k = len(self.kinds)
        self.kinds.append({"name": name, "ref": ref, "cur": cur, "T": np.asarray(T, np.float64)})
        return k

    def compose(self, n, special):
        """a batch of n kinds: the special kinds at the given positions, keyframe pairs every 41 slots, ordinary pairs
        (neighbours always different) elsewhere"""
        no = len(self.ordinary)
        slots = [self.ordinary[(5 * i + n) % no] for i in range(n)]
        for p in range(17, n - 1, 41):
            slots[p] = self.keyframe[(p // 41) % len(self.keyframe)]
        for j, p in enumerate(special):
            slots[p] = self.special[j % len(self.special)]
        return slots

    def release(self):
        for p in self.handles:
            p.release()


class Ctx:
    """the two estimator engines (profiled), the pools and the single-alignment results"""

    def __init__(self):
        import torch
        from dvo_slam_b200 import synth
        from dvo_slam_b200.engine import Engine
        self.eng = {"reference": Engine(device=0), "corrected": Engine(device=0, estimator="corrected")}
        for e in self.eng.values():
            e.profile_enable(True)
        self.grid = torch.cuda.get_device_properties(0).multi_processor_count * 2
        self.p640 = Pool(self.eng["reference"], synth.SceneConfig(), 5, 48, 3000)
        self.p1280 = Pool(self.eng["reference"], synth.SceneConfig().scaled(2), 6, 32, 4000)
        self._single = {}

    def cfg(self, name):
        from dvo_slam_b200.engine import Config
        return Config(**CFGS[name])

    def expected(self, est, name, pool, slots):
        """the single alignment of every slot's kind, computed once per (kind, configuration, estimator)"""
        init = "init" in name
        with _no_overrides():
            for k in sorted(set(slots)):
                key = (est, name, id(pool), k)
                if key not in self._single:
                    kd = pool.kinds[k]
                    self._single[key] = _raw(self.eng[est], [kd["ref"]], [kd["cur"]], self.cfg(name),
                                             [kd["T"]] if init else None, init)[0]
        return [self._single[(est, name, id(pool), k)] for k in slots]

    def batch(self, est, name, pool, slots):
        """one batch call -> (records, persistent launches the profiler counted)"""
        init = "init" in name
        kd = [pool.kinds[k] for k in slots]
        eng = self.eng[est]
        eng.profile_read(reset=True)
        got = _raw(eng, [d["ref"] for d in kd], [d["cur"] for d in kd], self.cfg(name),
                   [d["T"] for d in kd] if init else None, init)
        return got, eng.profile_read(reset=True)["residual"]["launches"]

    def check(self, est, name, pool, slots, got, what):
        want = self.expected(est, name, pool, slots)
        bad = [(i, pool.kinds[k]["name"], _diff(g, w)) for i, (k, g, w) in enumerate(zip(slots, got, want)) if g != w]
        assert not bad, f"{what}: {len(bad)} of {len(slots)} pairs differ from their single alignments, first: {bad[:6]}"

    def run(self, est, name, pool, n, first, last, env=None, what=""):
        """plan -> batch with the special kinds at the plan's boundaries -> launches and bits checked"""
        p = plan(pool.geom, first, last, self.grid, n, env)
        slots = pool.compose(n, special_positions(n, p))
        got, launches = self.batch(est, name, pool, slots)
        assert launches == p["launches"], (f"{what}: {launches} persistent launches, the restated plan has {p['launches']} "
                                           f"({p}) at grid {self.grid}")
        self.check(est, name, pool, slots, got, f"{what} n={n} plan {shape(p)} {est}")
        return p

    def close(self):
        self.p640.release()
        self.p1280.release()
        for e in self.eng.values():
            e.close()


@pytest.fixture(scope="module")
def ctx(engine):
    c = Ctx()
    yield c
    c.close()


@pytest.mark.gpu
def test_grid_is_two_ctas_per_sm(ctx):
    """The sizes of this file come from the grid: batches of grid/4 - 1 pairs run one launch per level, grid/4 pairs one
    fused launch."""
    n = ctx.grid // 4
    for m, want in ((n - 1, 5), (n, 1)):
        p = plan(ctx.p640.geom, 4, 0, ctx.grid, m)
        assert p["launches"] == want
        slots = ctx.p640.compose(m, [0, m - 1])
        got, launches = ctx.batch("reference", "4..0", ctx.p640, slots)
        assert launches == want, (f"{m} pairs ran {launches} persistent launches, {want} expected at {ctx.grid // 2} SMs x 2 "
                                  "CTAs: the persistent kernel's occupancy is no longer two CTAs per SM")
        ctx.check("reference", "4..0", ctx.p640, slots, got, f"n={m}")


@pytest.mark.gpu
@pytest.mark.parametrize("est", ["reference", "corrected"])
@pytest.mark.parametrize("k", range(len(SIZES_264)), ids=[f"n{n}" for n in SIZES_264])
def test_every_plan_shape_equals_single_alignments(ctx, k, est):
    """640x480, levels 4..0: the first and last batch size of every plan shape (the sizes in the id are those of 132 SMs)"""
    sizes = boundary_sizes(ctx.p640.geom, 4, 0, ctx.grid)
    assert len(sizes) == len(SIZES_264), f"grid {ctx.grid}: plan shapes give the sizes {sizes}, this file expects {len(SIZES_264)}"
    if ctx.grid == 264:
        assert sizes == SIZES_264
    ctx.run(est, "4..0", ctx.p640, sizes[k], 4, 0, what="640x480 4..0")


@pytest.mark.gpu
@pytest.mark.parametrize("est", ["reference", "corrected"])
def test_two_fine_levels_at_1280x960(ctx, est):
    """1280x960, levels 5..0: levels 1 and 0 form the fine group, in three slices of 6 / 12 / 24 CTAs on 132 SMs"""
    pool = ctx.p1280
    n = size_of_shape(pool.geom, 5, 0, ctx.grid, shape(plan(pool.geom, 5, 0, ctx.grid, 160)), pick="first")
    p = ctx.run(est, "5..0", pool, n, 5, 0, what="1280x960 5..0")
    assert p["fused"] and p["groups"][1]["nlev"] == 2 and len(p["slices"]) == 3, p
    if ctx.grid == 264:
        assert n == 148 and [s[0] for s in p["slices"]] == [6, 12, 24]


@pytest.mark.gpu
@pytest.mark.parametrize("est", ["reference", "corrected"])
@pytest.mark.parametrize("levels", ["3..1", "0..0"])
def test_coarse_only_and_fine_only_walks(ctx, levels, est):
    first, last = (3, 1) if levels == "3..1" else (0, 0)
    n = ctx.grid // 4 + 34
    p = ctx.run(est, levels, ctx.p640, n, first, last, what=f"640x480 {levels}")
    assert p["walk"] and not p["fused"] and len(p["groups"]) == 1
    assert p["groups"][0]["g"] == (1 if levels == "3..1" else p["g_level"][0])


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["g1", "two-slices", "2-4-8"])
def test_iteration_logs_and_initial_estimates(ctx, which):
    """with_iterations, use_initial_estimate with per-pair T_init and mu = 0.05: every log entry equals the single
    alignment's.  The shapes are those of 3/4 grid, grid + 15 and 512 pairs: one slice of g = 1, two slices of 3 and 6, and
    the benchmark's 2 / 4 / 8 on 132 SMs."""
    geom = ctx.p640.geom
    probe = {"g1": ctx.grid * 3 // 4, "two-slices": ctx.grid + 15, "2-4-8": 512}[which]
    want = shape(plan(geom, 4, 0, ctx.grid, probe))
    if ctx.grid == 264:
        assert want == {"g1": ("fused", 1), "two-slices": ("fused", 3, 6), "2-4-8": ("fused", 2, 4, 8)}[which]
    n = size_of_shape(geom, 4, 0, ctx.grid, want, pick="last" if which == "2-4-8" else "middle")
    ctx.run("reference", "4..0 init", ctx.p640, n, 4, 0, what="logs and T_init")


@pytest.mark.gpu
def test_one_context_across_plans(ctx):
    """One fresh context through 512 -> 1 -> 300 -> 66 -> 512 pairs: its workspace, squad states and ready ring are reused
    by every plan, and the results do not change."""
    from dvo_slam_b200.engine import Engine
    pool = ctx.p640
    eng = Engine(device=0)
    try:
        eng.profile_enable(True)
        for n in (512, 1, 300, 66, 512):
            p = plan(pool.geom, 4, 0, ctx.grid, n)
            slots = pool.compose(n, special_positions(n, p))
            eng.profile_read(reset=True)
            got = _raw(eng, [pool.kinds[k]["ref"] for k in slots], [pool.kinds[k]["cur"] for k in slots], ctx.cfg("4..0"))
            assert eng.profile_read(reset=True)["residual"]["launches"] == p["launches"], n
            ctx.check("reference", "4..0", pool, slots, got, f"fresh context, n={n} plan {shape(p)}")
    finally:
        eng.close()


@pytest.mark.gpu
def test_match_batch_device_three_slices(ctx):
    """dvo_b200_match_batch_device on a three-slice batch: the records in a torch buffer equal single alignments"""
    import torch
    from dvo_slam_b200.engine import CResult
    pool = ctx.p640
    want_shape = shape(plan(pool.geom, 4, 0, ctx.grid, 512))
    assert len(want_shape) == 4, f"no three-slice plan at 512 pairs on grid {ctx.grid}: {want_shape}"
    n = size_of_shape(pool.geom, 4, 0, ctx.grid, want_shape)
    p = plan(pool.geom, 4, 0, ctx.grid, n)
    slots = pool.compose(n, special_positions(n, p))
    eng = ctx.eng["reference"]
    buf = torch.full((n * C.sizeof(CResult),), 0x5A, dtype=torch.uint8, device="cuda:0")
    eng.profile_read(reset=True)
    eng.match_batch_device([pool.kinds[k]["ref"] for k in slots], [pool.kinds[k]["cur"] for k in slots], ctx.cfg("4..0"),
                           buf.data_ptr())
    eng.synchronize()
    assert eng.profile_read(reset=True)["residual"]["launches"] == 1
    raw = buf.cpu().numpy().tobytes()
    r = C.sizeof(CResult)
    ctx.check("reference", "4..0", pool, slots, [raw[i * r:(i + 1) * r] for i in range(n)], f"match_batch_device n={n}")


@pytest.mark.gpu
def test_two_shards_on_one_device(ctx):
    """ShardedEngine([0, 0]) at 512 pairs: each shard aligns 256 pairs, a plan of its own (one slice of g = 1 on 132 SMs)"""
    from dvo_slam_b200.engine import CResult, ShardedEngine
    pool = ctx.p640
    n = 512
    p = plan(pool.geom, 4, 0, ctx.grid, n)
    slots = pool.compose(n, special_positions(n, p) + [255, 256])
    shard_plan = plan(pool.geom, 4, 0, ctx.grid, n // 2)
    assert shape(shard_plan) != shape(p)
    sh = ShardedEngine([0, 0])
    try:
        res = sh.match_batch([C.c_void_p(pool.kinds[k]["ref"].handle) for k in slots],
                             [C.c_void_p(pool.kinds[k]["cur"].handle) for k in slots], ctx.cfg("4..0"))
    finally:
        sh.close()
    raw, r = bytes(res), C.sizeof(CResult)
    ctx.check("reference", "4..0", pool, slots, [raw[i * r:(i + 1) * r] for i in range(n)], f"two shards, plan {shape(shard_plan)}")


@pytest.mark.gpu
@pytest.mark.parametrize("n", [512, 24])
@pytest.mark.parametrize("knob,value", OVERRIDES, ids=[f"{k}={v}" for k, v in OVERRIDES])
def test_developer_overrides(ctx, monkeypatch, knob, value, n):
    """Every DVO_B200_* override gives every pair its single alignment's bits (the knobs are read on every call)."""
    env = {f"DVO_B200_{knob}": value}
    monkeypatch.setenv(f"DVO_B200_{knob}", value)
    p = ctx.run("reference", "4..0", ctx.p640, n, 4, 0, env=env, what=f"DVO_B200_{knob}={value}")
    if n == 512 and knob not in ("CONTIGUOUS",):
        assert p != plan(ctx.p640.geom, 4, 0, ctx.grid, n), f"DVO_B200_{knob}={value} does not change the plan at {n} pairs"
