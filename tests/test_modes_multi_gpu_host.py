"""Every alignment mode with device outputs and over several GPUs, without a GPU: the shard slicing and the up-front checks of
dvo_b200_match_batch_modes_device / _modes_sharded (csrc/modes_args.h) built for the host with fakes for the pointer and
pyramid queries; the marshalling of Engine.match_batch_modes_device and ShardedEngine.match_batch_modes against a recording
fake of the C library; and a world-size-2 gloo all-gather of every per-pair output of a device call, shards of unequal size."""
import ctypes as C
import gc
import multiprocessing as mp
import os
import shutil
import subprocess
import tempfile

import numpy as np
import pytest
import torch
import torch.distributed as dist

import test_engine_calls_host as tec
from dvo_slam_b200 import engine as E

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RES, LOG = C.sizeof(E.CResult), C.sizeof(E.IterationStats)
DEV, REGION = 0x10000000, 0x10000000          # the fake's device memory
INVALID, SHAPE = -1, -4


@pytest.fixture(scope="module")
def lib():
    tmp = tempfile.mkdtemp(prefix="dvo_modes_args_")
    try:
        out = os.path.join(tmp, "libmodes_args.so")
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-Wall", "-fPIC", "-shared", "-I", os.path.join(ROOT, "dvo_slam_b200", "csrc"),
                               "-o", out, os.path.join(ROOT, "tests", "native", "modes_args.cpp")])
        L = C.CDLL(out)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    i64p, dp, ip = C.POINTER(C.c_longlong), C.POINTER(C.c_double), C.POINTER(C.c_int)
    L.ms_slice.argtypes = [C.c_int, C.c_int, C.c_int, C.c_longlong, C.c_longlong, C.c_longlong, C.c_longlong, i64p]
    L.ms_check.argtypes = [C.c_int, C.c_int, ip, C.c_int, C.c_int, C.c_double, C.c_int, C.c_int, ip, C.c_int, dp, C.c_int, dp, dp, i64p,
                           C.c_int, C.POINTER(E.WeightMaps), C.c_longlong, C.c_longlong, C.c_char_p, C.c_int]
    return L


@pytest.mark.parametrize("k", [0, 1, 3])
@pytest.mark.parametrize("b,e", [(0, 4), (4, 7), (7, 7)])
def test_shard_slice_moves_every_per_pair_pointer(lib, k, b, e):
    n, max_log, wb, mb = 7, 5, 4 * 80 * 60 + 64, 320 * 240
    off = (C.c_longlong * 16)()
    assert lib.ms_slice(n, k, max_log, b, e, wb, mb, off) == e - b
    per = max(k, 1)
    want = [8 * b, 8 * b, 8 * 16 * per * b, 8 * 36 * per * b, 8 * 2 * per * b, 16 * b, 16 * k * b, RES * b, 4 * b, 8 * k * b, RES * k * b,
            LOG * max_log * b, wb * b, mb * b, 128 * b, 16 * b]
    assert list(off) == want


def _maps(memory="device", base=DEV, mask=True):
    m = E.WeightMaps()
    m.memory = E.MAPS_MEMORY[memory]
    m.weight = E.MapPlane(base, 4 * 320, 4 * 320 * 240)
    if mask:
        m.mask = E.MapPlane(base + 0x1000000, 320, 320 * 240)
        m.mask_weight = 0.3
    return m


def _spd(seed):
    M = np.random.default_rng(seed).normal(size=(6, 6))
    return M @ M.T


@pytest.fixture(scope="module")
def check(lib):
    def run(form="device", n=3, k=0, devices=(0,), views=None, H=None, s=2, prior=None, ab0=None, outputs=None, max_log=0, maps=None,
            first=2, last=0, mu=0.0, use_init=1):
        views = views if views is not None else [[3, devices[0], 320, 240]] * (2 * n)
        dev = (C.c_int * len(devices))(*devices)
        vw = (C.c_int * (4 * len(views)))(*[int(x) for v in views for x in v])
        arr = lambda a: None if a is None else np.ascontiguousarray(a, dtype=np.float64)
        H = arr(np.tile(np.eye(4), (n, max(k, 1), 1, 1)) if H is None else H)
        prior, ab0 = arr(prior), arr(ab0)
        ptr = lambda a: None if a is None else a.ctypes.data_as(C.POINTER(C.c_double))
        o = {"photometric": 0, "screen_photometric": 0, "results": DEV, "best": 0, "scores": 0, "screen_results": 0, "iterations": 0}
        o.update(outputs or {})
        outs = (C.c_longlong * 7)(*o.values())
        buf = C.create_string_buffer(512)
        rc = lib.ms_check(1 if form == "sharded" else 0, len(devices), dev, first, last, mu, use_init, n, vw, k, ptr(H), s, ptr(prior), ptr(ab0),
                          outs, max_log, C.byref(maps) if maps is not None else None, DEV, DEV + REGION, buf, 512)
        return rc, buf.value.decode()
    return run


def test_accepted(check):
    assert check() == (0, "")
    assert check(k=3, outputs={"best": DEV + 0x100000, "scores": DEV + 0x200000}, maps=_maps()) == (0, "")
    assert check(form="sharded", devices=(0, 0), outputs={"results": 0x1000}, maps=_maps("host", base=0x4000000000)) == (0, "")


def test_device_output_refusals(check):
    FN = "match_batch_modes_device: "
    cases = [
        (dict(outputs={"results": 0x1000}), "results is not device or managed memory of device 0"),
        (dict(outputs={"results": DEV + REGION - 8}), "results is not device or managed memory of device 0"),   # its last byte
        (dict(outputs={"results": DEV + 4}), "results is misaligned"),
        (dict(outputs={"photometric": DEV + 0x100000 + 4}), "photometric is misaligned"),
        (dict(outputs={"iterations": 0x1000}, max_log=4), "iteration_stats is not device or managed memory"),
        (dict(outputs={"best": DEV + 0x100000}), "best is only written with k >= 1"),
        (dict(outputs={"scores": DEV + 0x100000}), "scores is only written with k >= 1"),
        (dict(outputs={"screen_results": DEV + 0x100000}), "screen_results is only written with k >= 1"),
        (dict(outputs={"screen_photometric": DEV + 0x100000, "photometric": DEV + 0x200000}), "screen_photometric is only written"),
        (dict(ab0=np.tile([1.0, 0.0], (3, 1))), "photometric_init without photometric"),
        (dict(maps=_maps("host", base=0x4000000000)), "maps must be DVO_B200_MAPS_DEVICE"),
        (dict(k=2, outputs={"best": DEV + 0x100000, "scores": 0x1000}), "scores is not device or managed memory"),
    ]
    for kw, want in cases:
        rc, msg = check(**kw)
        assert rc == INVALID and msg.startswith(FN) and want in msg, (kw, msg)
    # an iteration log is only placed when it has entries
    assert check(outputs={"iterations": 0x1000}, max_log=0) == (0, "")


def test_the_order_of_the_checks(check):
    # E's argument checks first, with E's messages: a NULL results before a host-memory best
    assert check(outputs={"results": 0, "best": 0x1000}) == (INVALID, "match_batch: null argument")
    # E's batch checks next: too few levels and a batch of mixed sizes before any check of the form
    few = [[2, 0, 320, 240]] * 6
    assert check(views=few, outputs={"best": 0x1000})[1] == "match: pyramid has fewer levels than FirstLevel+1"
    mixed = [[3, 0, 320, 240]] * 5 + [[3, 0, 160, 120]]
    assert check(views=mixed, outputs={"results": 0x1000}) == (SHAPE, "match: all pyramids of a batch must share width/height")
    # E of the arguments: a prior makes it match_batch_prior, maps make it match_batch_maps
    bad = np.stack([_spd(0), _spd(1), _spd(2)])
    bad[2, 0, 1] += 1.0
    assert check(prior=bad, outputs={"results": 0x1000})[1] == "match_batch_prior: prior_information of pair 2 is not symmetric"
    assert check(prior=bad, maps=_maps(mask=False), mu=0.1)[1] == "match_batch_prior: cfg->mu must be 0: the prior replaces mu I"
    nan_ab = np.tile([1.0, 0.0], (3, 1))
    nan_ab[1, 0] = np.nan
    assert check(ab0=nan_ab, outputs={"photometric": DEV + 0x100000})[1] == "match_batch_photometric: photometric_init is not finite"
    assert check(maps=_maps(base=0x4000000000))[1].startswith("match_batch_maps: weight is not device or managed memory")
    # k >= 1: the multi-hypothesis call's checks, naming the hypothesis, before the form's
    kbad = np.stack([np.stack([_spd(3 * p + j) for j in range(3)]) for p in range(3)])
    kbad[1, 2, 3, 4] += 1.0
    rc, msg = check(k=3, prior=kbad, outputs={"best": 0x1000})
    assert msg == "match_batch_hypotheses: prior_information of hypothesis 2 of pair 1 is not symmetric"
    assert check(k=3, s=5, outputs={"best": 0x1000})[1].startswith("match_batch_hypotheses: screen_level = 5 outside")
    # then the form's own: k-only outputs, maps memory, then each output
    assert "best is only written" in check(outputs={"best": DEV + 0x100000, "results": 0x1000}, maps=_maps("host", base=0x4000000000))[1]
    assert "maps must be DVO_B200_MAPS_DEVICE" in check(outputs={"results": 0x1000}, maps=_maps("host", base=0x4000000000))[1]


def test_sharded_refusals(check):
    FN = "match_batch_modes_sharded: "
    host = {"results": 0x1000}
    # n = 3 over two shards: pairs 0, 1 on shard 0 and pair 2 on shard 1, whose current pyramid is on device 0
    views = [[3, 0, 320, 240]] * 2 + [[3, 1, 320, 240]] + [[3, 0, 320, 240]] * 3   # refs 0..2, then curs 0..2
    rc, msg = check(form="sharded", devices=(0, 1), outputs=host, views=views)
    assert rc == INVALID and msg == FN + "pair 2 belongs to shard 1 (device 1) but its pyramids live on devices 1 / 0", msg
    rc, msg = check(form="sharded", devices=(0, 0), outputs=host, maps=_maps("device"))
    assert msg == FN + "maps must be DVO_B200_MAPS_HOST"
    # a bad Lambda on the last shard's pair refuses the whole batch, first
    lam = np.stack([np.stack([_spd(3 * p + j) for j in range(2)]) for p in range(5)])
    lam[4, 1, 0, 0] = np.inf
    rc, msg = check(form="sharded", devices=(0, 0), n=5, k=2, prior=lam, outputs=dict(host, best=0x2000), maps=_maps("device"))
    assert msg == "match_batch_hypotheses: prior_information of hypothesis 1 of pair 4 is not finite"
    # the placement refusal comes after E's checks
    rc, msg = check(form="sharded", devices=(0, 1), outputs={"results": 0}, views=views)
    assert msg == "match_batch: null argument"


# ---- marshalling against the recording fake of the C library ----

def _kinds(fake, name, a):
    if name in ("match_batch_modes_device", "match_batch_modes_sharded"):
        n, k = a[2], a[5]
        rows = n * max(k, 1)
        outputs = [tec.S] * 7 if name.endswith("device") else [tec.OUT] * 7
        return [tec.CTX, tec.CFG, tec.S, 8 * n, 8 * n, tec.S, 128 * rows, tec.S, tec.S, 288 * rows, 16 * rows] + outputs + [tec.S, tec.OUT]
    return KINDS(fake, name, a)


KINDS = tec._kinds


@pytest.fixture
def fake(monkeypatch):
    monkeypatch.setattr(tec, "_kinds", _kinds)
    f = tec.FakeLib()
    monkeypatch.setattr(E, "_lib", f)
    yield f
    gc.collect()
    for o in gc.get_objects():   # nothing made here may reach the real library once the fake is gone
        if type(o) is E.Pyramid and o.handle in f.handles:
            o.handle = None


def test_engine_match_batch_modes_device(fake, monkeypatch):
    eng = E.Engine()
    ordered = []
    monkeypatch.setattr(E.Engine, "_ordered_with_torch", lambda self, ts, call: (ordered.append([t.data_ptr() for t in ts]), call())[1])
    fake.calls.clear()
    pyr = eng.pyramid_batch(np.zeros((2, 8, 8), np.float32), np.zeros((2, 8, 8), np.float32), tec.K, 3)
    fake.calls.clear()
    n, k, cfg = 1, 2, E.Config(first_level=2, last_level=0, max_iterations_per_level=3, use_initial_estimate=1)
    H = np.random.default_rng(1).normal(size=(n, k, 4, 4))
    H[..., 3, :] = [0, 0, 0, 1]
    lam = np.stack([np.stack([_spd(j) for j in range(k)])])
    ab0 = np.full((n, k, 2), 0.5)
    out = {name: torch.zeros(shape, dtype=getattr(torch, dt)) for name, (shape, dt) in
           E._modes_outputs(n, k, 12, True, True).items()}
    eng.match_batch_modes_device(pyr[:1], pyr[1:], cfg, out, hypotheses=H, screen_level=1, min_constraint_ratio=0.25,
                                 prior_information=lam, photometric_init=ab0)
    addr = {name: t.data_ptr() for name, t in out.items()}
    assert ordered == [list(addr.values())]   # every output is ordered with torch's stream
    (call,) = fake.calls
    b = lambda a: np.ascontiguousarray(a, dtype=np.float64).tobytes()
    handles = lambda ps: np.array([p.handle for p in ps], dtype=np.uint64).tobytes()
    assert call == ("match_batch_modes_device", tec.CTX, bytes(cfg), n, handles(pyr[:1]), handles(pyr[1:]), k, b(H), 1, 0.25, b(lam), b(ab0),
                    addr["photometric"], addr["screen_photometric"], addr["results"], addr["best"], addr["scores"],
                    addr["screen_results"], addr["iterations"], 12, None)
    # k = 0: T_init per pair, and no k-only output
    fake.calls.clear()
    out = {name: torch.zeros(shape, dtype=getattr(torch, dt)) for name, (shape, dt) in E._modes_outputs(2, 0, 0, False, False).items()}
    eng.match_batch_modes_device(pyr, pyr[::-1], cfg, out, T_init=np.tile(np.eye(4), (2, 1, 1)))
    assert fake.calls[0][7:] == (b(np.tile(np.eye(4), (2, 1, 1))), 0, 0.0, None, None, None, None, out["results"].data_ptr(), None, None,
                                 None, None, 0, None)
    with pytest.raises(ValueError, match="out\\['best'\\]"):
        eng.match_batch_modes_device(pyr, pyr, cfg, dict(out, best=torch.zeros(2, dtype=torch.int32)))
    with pytest.raises(ValueError, match="without screen_level"):
        eng.match_batch_modes_device(pyr[:1], pyr[1:], cfg, out, hypotheses=H)


def test_sharded_match_batch_modes(fake):
    s = E.ShardedEngine([0, 0])
    pyr = s.pyramid_batch(np.zeros((3, 8, 8), np.float32), np.zeros((3, 8, 8), np.float32), tec.K, 3)
    fake.calls.clear()
    cfg = E.Config(first_level=2, last_level=0, max_iterations_per_level=3)
    lam = np.stack([_spd(p) for p in range(3)])
    res, maps, ab = s.match_batch_modes(pyr, pyr[::-1], cfg, T_init=np.tile(np.eye(4), (3, 1, 1)), prior_information=lam, photometric=True,
                                        mask_weight=0.4, with_iterations=True)
    assert [c[0] for c in fake.calls] == ["pyramid_level_info"] * 6 + ["match_batch_modes_sharded"]
    call = fake.calls[-1]
    b = lambda a: np.ascontiguousarray(a, dtype=np.float64).tobytes()
    assert call[1:12] == (tec.CTX, bytes(cfg), 3, np.array([p.value for p in pyr], np.uint64).tobytes(),
                          np.array([p.value for p in pyr[::-1]], np.uint64).tobytes(), 0, b(np.tile(np.eye(4), (3, 1, 1))), 0, 0.0, b(lam), None)
    assert call[12:] == (tec.OUT, None, tec.OUT, None, None, None, tec.OUT, 12, tec.OUT)
    assert len(res) == 3 and ab.shape == (3, 2)
    assert {key: v.shape for key, v in maps.items()} == {"weight": (3, 8, 8), "residual_i": (3, 8, 8), "residual_z": (3, 8, 8),
                                                         "estimate": (3, 4, 4), "precision": (3, 2, 2), "mask": (3, 8, 8)}
    # k >= 1 returns what Engine.match_batch_hypotheses returns
    fake.calls.clear()
    H = np.tile(np.eye(4), (3, 2, 1, 1))
    out = s.match_batch_modes(pyr, pyr, hypotheses=H, screen_level=1, screen_results=True, photometric=True)
    assert len(out) == 6 and out[1].shape == (3,) and out[2].shape == (3, 2) and len(out[3]) == 3 and out[5].shape == (3, 2, 2)
    (call,) = fake.calls
    assert call[6:9] == (2, b(H), 1) and call[12:] == (tec.OUT, tec.OUT, tec.OUT, tec.OUT, tec.OUT, tec.OUT, None, 0, None)
    s.close()


# ---- the all-gather of a device call's outputs ----

def _gather_worker(rank, world, port, total, k, q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from dvo_slam_b200.distributed import all_gather_results, shard_range, tensor_to_results
        b, e = shard_range(total, world, rank)
        rows = np.arange(b, e)
        res = torch.zeros((e - b, RES), dtype=torch.uint8)
        res[:, :8] = torch.from_numpy(rows.astype(np.float64)).view(torch.uint8).reshape(-1, 8)   # transformation[0] = pair
        ab = torch.from_numpy(np.stack([1.0 + rows, -0.5 * rows], 1))
        best = torch.from_numpy((rows % k).astype(np.int32)).reshape(-1, 1)
        scores = torch.from_numpy(rows[:, None] + np.arange(k)[None] / 10.0)
        g = [all_gather_results(t, total) for t in (res, ab, best, scores)]
        allrows = np.arange(total)
        ok = ([r.transformation[0] for r in tensor_to_results(g[0])] == list(allrows.astype(float)) and
              np.array_equal(g[1].numpy(), np.stack([1.0 + allrows, -0.5 * allrows], 1)) and
              np.array_equal(g[2].numpy()[:, 0], allrows % k) and g[2].dtype == torch.int32 and
              np.array_equal(g[3].numpy(), allrows[:, None] + np.arange(k)[None] / 10.0))
        q.put((rank, bool(ok)))
    finally:
        dist.destroy_process_group()


def test_all_gather_of_device_outputs_world_size_2_gloo():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    total, k = 7, 3
    port = 31500 + (os.getpid() % 2000)
    procs = [ctx.Process(target=_gather_worker, args=(r, 2, port, total, k, q)) for r in range(2)]
    for p in procs:
        p.start()
    got = [q.get(timeout=120) for _ in range(2)]
    for p in procs:
        p.join(timeout=60)
    assert sorted(got) == [(0, True), (1, True)]
