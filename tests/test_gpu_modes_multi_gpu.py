"""Every alignment mode with its outputs in device memory and over several GPUs, on the GPU: dvo_b200_match_batch_modes_device
writes, byte for byte, what the host-output entry point of its mode returns (plain, photometric, prior, maps, multi-hypothesis),
under both estimators, with masks, mixed intrinsics and a three-slice launch plan, moves no device-to-host byte and stages and
launches what that call does; dvo_b200_match_batch_device is it with every mode NULL; its output refusals move no counter.
dvo_b200_match_batch_modes_sharded over two shards and one equals the one-context call, with an empty shard too, and refuses
a bad batch before any shard launches."""
import ctypes as C

import numpy as np
import pytest
import torch

from dvo_slam_b200 import synth
from dvo_slam_b200.engine import CResult, IterationStats, ShardedEngine, _weight_maps
from test_gpu_hypotheses import FIRST, LAST, SCENE, _cfg, _hypotheses, _mask, _same
from test_gpu_hypotheses_modes import MASK_WEIGHT, _ab0, _lam

pytestmark = pytest.mark.gpu
DP = C.POINTER(C.c_double)
P = lambda a: None if a is None else np.ascontiguousarray(a, dtype=np.float64).ctypes.data_as(DP)
MODES = {"plain": {}, "photometric": dict(photometric=True), "prior": dict(prior=True),
         "photometric+prior": dict(photometric=True, prior=True), "maps": dict(maps=True),
         "photometric+prior+maps": dict(photometric=True, prior=True, maps=True)}


def _pairs(engine, n, seed=200, kws=None, scenes=None):
    out = []
    for i in range(n):
        scene = scenes[i] if scenes else SCENE
        kw = kws[i] if kws else {}
        p = synth.make_pair(seed + i % 5, scene)
        out.append({"ref": engine.pyramid(p["I_ref"].numpy(), p["Z_ref"].numpy(), scene.intrinsics, 3, **kw),
                    "cur": engine.pyramid(synth.exposure(p["I_cur"].numpy(), 1.0 + 0.03 * (i % 3), -2.0 * (i % 4)), p["Z_cur"].numpy(),
                                          scene.intrinsics, 3, **kw), "pair": p})
    return out


def _inputs(batch, k, mode, seed=1):
    """(T_init or hypotheses, Lambda, (alpha, beta)_0) of a call: k = 0 per pair, else per hypothesis"""
    rng = np.random.default_rng(seed)
    kk = max(k, 2)
    H = np.stack([_hypotheses(q["pair"], kk, i) for i, q in enumerate(batch)])
    lam = np.stack([_lam(rng, kk) for _ in batch]) if mode.get("prior") else None
    ab0 = np.stack([_ab0(rng, kk) for _ in batch]) if mode.get("photometric") else None
    if k:
        return H[:, :k], None if lam is None else lam[:, :k], None if ab0 is None else ab0[:, :k]
    return H[:, 1], None if lam is None else lam[:, 1], None if ab0 is None else ab0[:, 1]


def _host(engine, refs, curs, cfg, k, H, s, lam, ab0, photometric, screen, logs, maps):
    """the host-output entry point E of the arguments, through the C ABI: {output name: bytes or a numpy array}"""
    n = len(refs)
    L = engine.lib
    rh, ch = (C.c_void_p * n)(*[r.handle for r in refs]), (C.c_void_p * n)(*[c.handle for c in curs])
    res = (CResult * n)()
    max_log = (cfg.first_level - cfg.last_level + 1) * (cfg.max_iterations_per_level + 1) if logs else 0
    log = (IterationStats * (n * max_log))() if logs else None
    ab = np.zeros((n, 2)) if photometric else None
    dmaps, wm = engine._device_maps(refs, cfg, MASK_WEIGHT) if maps else (None, None)
    out = {}
    if k:
        best, scores = np.zeros(n, np.int32), np.zeros((n, k))
        scr = (CResult * (n * k))() if screen else None
        scr_ab = np.zeros((n, k, 2)) if photometric and screen else None
        rc = L.dvo_b200_match_batch_hypotheses_modes(engine.ctx, C.byref(cfg), n, rh, ch, k, P(H), s, 0.3, P(lam), P(ab0),
                                                     None if ab is None else ab.ctypes.data_as(DP),
                                                     None if scr_ab is None else scr_ab.ctypes.data_as(DP), res,
                                                     best.ctypes.data_as(C.POINTER(C.c_int32)), scores.ctypes.data_as(DP), scr, log,
                                                     max_log, C.byref(wm) if wm is not None else None)
        out.update(best=best, scores=scores)
        if screen:
            out["screen_results"] = bytes(scr)
            if photometric:
                out["screen_photometric"] = scr_ab
    else:
        abp = None if ab is None else ab.ctypes.data_as(DP)
        head = (engine.ctx, C.byref(cfg), n, rh, ch, P(H))
        if maps:
            rc = L.dvo_b200_match_batch_maps(*head, P(lam), P(ab0), abp, res, log, max_log, C.byref(wm))
        elif lam is not None:
            rc = L.dvo_b200_match_batch_prior(*head, P(lam), P(ab0), abp, res, log, max_log)
        elif photometric:
            rc = L.dvo_b200_match_batch_photometric(*head, P(ab0), res, abp, log, max_log)
        else:
            rc = L.dvo_b200_match_batch(*head, res, log, max_log)
    assert rc == 0, L.dvo_b200_last_error(engine.ctx).decode()
    out["results"] = bytes(res)
    if photometric:
        out["photometric"] = ab
    if logs:
        out["iterations"] = bytes(log)
    if maps:
        out["maps"] = {key: v.cpu().numpy() for key, v in dmaps.items()}
    return out


def _device(engine, refs, curs, cfg, k, H, s, lam, ab0, photometric, screen, logs, maps):
    """match_batch_modes_device, read back from its torch tensors after the engine's stream: the dict of _host"""
    out = engine.device_outputs(refs, cfg, k, screen_results=screen, photometric=photometric, with_iterations=logs,
                                mask_weight=MASK_WEIGHT if maps else None)
    engine.match_batch_modes_device(refs, curs, cfg, out, T_init=None if k else H, hypotheses=H if k else None, screen_level=s,
                                    min_constraint_ratio=0.3 if k else 0.0, prior_information=lam, photometric_init=ab0)
    engine.synchronize()
    got = {}
    for key, v in out.items():
        if key == "maps":
            got[key] = {m: t.cpu().numpy() for m, t in v.items()}
        elif key == "mask_weight":
            continue
        elif key in ("results", "screen_results", "iterations"):
            got[key] = v.cpu().numpy().tobytes()
        else:
            got[key] = v.cpu().numpy()
    return got


def _same_outputs(a, b):
    assert a.keys() == b.keys(), (sorted(a), sorted(b))
    for key in a:
        if key == "maps":
            _same_outputs(a[key], b[key])
        elif isinstance(a[key], bytes):
            assert a[key] == b[key], key
        else:
            x, y = np.asarray(a[key]), np.asarray(b[key])
            assert x.dtype == y.dtype and x.tobytes() == y.tobytes(), key


def _compare(engine, batch, cfg, k, s, mode, screen=True, logs=True, seed=1):
    """the device call against E, byte for byte, and its counters against E's"""
    refs, curs = [q["ref"] for q in batch], [q["cur"] for q in batch]
    H, lam, ab0 = _inputs(batch, k, mode, seed)
    args = (engine, refs, curs, cfg, k, H, s, lam, ab0, mode.get("photometric", False), screen and k > 0, logs, mode.get("maps", False))
    engine.synchronize()
    h0, l0 = engine.h2d_bytes(), engine.kernel_launches()
    want = _host(*args)
    h1, l1, d1 = engine.h2d_bytes(), engine.kernel_launches(), engine.d2h_bytes()
    got = _device(*args)
    assert engine.d2h_bytes() == d1
    assert engine.h2d_bytes() - h1 == h1 - h0 and engine.kernel_launches() - l1 == l1 - l0
    _same_outputs(want, got)


@pytest.fixture(scope="module")
def batch(engine):
    return _pairs(engine, 4)


@pytest.mark.parametrize("estimator", ["reference", "corrected"])
@pytest.mark.parametrize("mode", list(MODES), ids=str)
def test_device_k0_is_the_entry_point_of_its_mode(engine, batch, estimator, mode):
    engine.set_estimator(estimator)
    try:
        _compare(engine, batch, _cfg(), 0, 0, MODES[mode])
    finally:
        engine.set_estimator("reference")


@pytest.mark.parametrize("estimator", ["reference", "corrected"])
@pytest.mark.parametrize("mode", ["plain", "photometric+prior+maps"], ids=str)
def test_device_hypotheses_are_the_modes_call(engine, batch, estimator, mode):
    engine.set_estimator(estimator)
    try:
        for s in (FIRST, FIRST - 1, LAST):
            _compare(engine, batch, _cfg(), 4, s, MODES[mode], seed=10 + s)
    finally:
        engine.set_estimator("reference")


def test_device_masks_mixed_intrinsics_and_a_big_batch(engine):
    other = synth.SceneConfig(width=320, height=240, intrinsics=(287.0, 291.5, 161.0, 118.5))
    kws = [{}, {"mask": _mask(1), "mask_roles": "reference"}, {"mask": _mask(2), "mask_roles": "both"}, {}]
    mixed = _pairs(engine, 4, 300, kws=kws, scenes=[SCENE, SCENE, other, other])
    full = MODES["photometric+prior+maps"]
    for k, s in ((0, 0), (4, FIRST - 1)):
        _compare(engine, mixed, _cfg(), k, s, full)
    big = _pairs(engine, 8, 400)
    idx = [i % 8 for i in range(512)]
    big = [big[i] for i in idx]   # 512 pairs: a launch plan of three slices
    _compare(engine, big, _cfg(), 0, 0, MODES["photometric+prior"], logs=False)
    _compare(engine, big, _cfg(), 2, FIRST - 1, MODES["plain"], logs=False, screen=False)


def test_match_batch_device_is_the_modes_call_without_modes(engine, batch):
    refs, curs = [q["ref"] for q in batch], [q["cur"] for q in batch]
    H, _, _ = _inputs(batch, 0, {})
    old = torch.zeros((len(refs), C.sizeof(CResult)), dtype=torch.uint8, device="cuda:0")
    torch.cuda.synchronize()
    engine.match_batch_device(refs, curs, _cfg(), old.data_ptr(), T_init=H)
    engine.synchronize()
    out = engine.device_outputs(refs, _cfg())
    engine.match_batch_modes_device(refs, curs, _cfg(), out, T_init=H)
    engine.synchronize()
    assert torch.equal(old.cpu(), out["results"].cpu())


def _raw_device(engine, refs, curs, cfg, results, best=None, maps=None, k=0, H=None):
    n = len(refs)
    rh, ch = (C.c_void_p * n)(*[r.handle for r in refs]), (C.c_void_p * n)(*[c.handle for c in curs])
    return engine.lib.dvo_b200_match_batch_modes_device(engine.ctx, C.byref(cfg), n, rh, ch, k, P(H), 1, 0.0, None, None, None, None,
                                                        C.c_void_p(results), None if best is None else C.c_void_p(best), None, None,
                                                        None, 0, None if maps is None else C.byref(maps))


def test_device_refusals_move_no_counters(engine, batch):
    refs, curs = [batch[0]["ref"]], [batch[0]["cur"]]
    dev = torch.zeros(2 * C.sizeof(CResult), dtype=torch.uint8, device="cuda:0")
    host = np.zeros(C.sizeof(CResult), np.uint8)
    best = torch.zeros(4, dtype=torch.int32, device="cuda:0")
    dmaps, wm = engine._device_maps(refs, _cfg(), MASK_WEIGHT)
    bufs = {key: np.zeros(v.shape, dtype=str(v.dtype).split(".")[1]) for key, v in dmaps.items()}
    hm = _weight_maps(bufs, "host", MASK_WEIGHT)
    engine.synchronize()
    counters = lambda: (engine.h2d_bytes(), engine.kernel_launches(), engine.d2h_bytes())
    c0 = counters()
    cases = [(dict(results=host.ctypes.data), "results is not device or managed memory of device 0"),
             (dict(results=dev.data_ptr() + 4), "results is misaligned"),
             (dict(results=dev.data_ptr(), best=best.data_ptr()), "best is only written with k >= 1"),
             (dict(results=dev.data_ptr(), maps=hm), "maps must be DVO_B200_MAPS_DEVICE")]
    for kw, want in cases:
        rc = _raw_device(engine, refs, curs, _cfg(), **kw)
        msg = engine.lib.dvo_b200_last_error(engine.ctx).decode()
        assert rc == -1 and msg.startswith("match_batch_modes_device: ") and want in msg, (want, msg)
        assert counters() == c0, want
    # E's refusals come first: a NULL results before a host-memory best
    rc = _raw_device(engine, refs, curs, _cfg(), None, best=host.ctypes.data)
    assert rc == -1 and engine.lib.dvo_b200_last_error(engine.ctx).decode() == "match_batch: null argument"
    assert counters() == c0
    assert _raw_device(engine, refs, curs, _cfg(), dev.data_ptr(), maps=wm) == 0
    engine.synchronize()
    assert counters()[2] == c0[2] and counters()[1] > c0[1]


def _engine_call(engine, refs, curs, cfg, **kw):
    """the one-context call of ShardedEngine.match_batch_modes' arguments, through Engine"""
    if kw.get("hypotheses") is not None:
        kw.pop("T_init", None)
        return engine.match_batch_hypotheses(refs, curs, kw.pop("hypotheses"), kw.pop("screen_level"), kw.pop("min_constraint_ratio"), cfg,
                                             **kw)
    kw = {key: v for key, v in kw.items() if key not in ("hypotheses", "screen_level", "min_constraint_ratio", "screen_results")}
    kw.pop("maps", None)
    if kw.get("mask_weight") is not None:
        return engine.match_batch_maps(refs, curs, cfg, **kw)
    kw.pop("mask_weight", None)
    photometric = kw.pop("photometric", False)
    if photometric:
        return engine.match_batch_photometric(refs, curs, cfg, kw.pop("T_init"), kw.pop("photometric_init"), **kw)
    kw.pop("photometric_init", None)
    return engine.match_batch(refs, curs, cfg, kw.pop("T_init"), **kw)


def _same_returns(a, b):
    if isinstance(a, tuple):
        assert isinstance(b, tuple) and len(a) == len(b)
        for x, y in zip(a, b):
            _same_returns(x, y)
    elif isinstance(a, list):
        assert len(a) == len(b)
        for x, y in zip(a, b):
            _same_returns(x, y)
    elif isinstance(a, dict):
        assert a.keys() == b.keys()
        host = lambda v: v.cpu().numpy() if hasattr(v, "cpu") else np.asarray(v)
        for key in a:
            x, y = host(a[key]), host(b[key])
            assert x.dtype == y.dtype and x.tobytes() == y.tobytes(), key
    elif isinstance(a, np.ndarray):
        assert a.dtype == b.dtype and a.tobytes() == np.asarray(b).tobytes()
    else:
        assert _same(a, b, iterations=True)


@pytest.fixture(scope="module")
def sharded():
    two, one = ShardedEngine([0, 0]), ShardedEngine([0])
    yield two, one
    two.close()
    one.close()


@pytest.mark.parametrize("estimator", ["reference", "corrected"])
@pytest.mark.parametrize("n", [7, 1])
def test_sharded_equals_one_context(engine, sharded, estimator, n):
    pairs = _pairs(engine, n, 500)
    refs, curs = [q["ref"] for q in pairs], [q["cur"] for q in pairs]
    engine.set_estimator(estimator)
    for s in sharded:
        s.set_estimator(estimator)
    try:
        for name, mode in MODES.items():
            for k in (0, 4):
                H, lam, ab0 = _inputs(pairs, k, mode, seed=len(name) + k)
                kw = dict(T_init=None if k else H, hypotheses=H if k else None, screen_level=FIRST - 1 if k else None,
                          min_constraint_ratio=0.3 if k else 0.0, with_iterations=True, screen_results=k > 0,
                          prior_information=lam, photometric_init=ab0, photometric=mode.get("photometric", False),
                          maps=mode.get("maps", False), mask_weight=MASK_WEIGHT if mode.get("maps") else None)
                want = _engine_call(engine, refs, curs, _cfg(), **dict(kw))
                for s in sharded:
                    _same_returns(want, s.match_batch_modes(refs, curs, _cfg(), **kw))
    finally:
        engine.set_estimator("reference")
        for s in sharded:
            s.set_estimator("reference")


def test_sharded_refusals_leave_every_shard_untouched(engine, sharded):
    two, _ = sharded
    pairs = _pairs(engine, 5, 600)
    refs, curs = [q["ref"] for q in pairs], [q["cur"] for q in pairs]
    ctxs = [two.lib.dvo_b200_sharded_ctx(two.h, i) for i in range(2)]
    counters = lambda: [(two.lib.dvo_b200_kernel_launches(c), two.lib.dvo_b200_h2d_bytes(c)) for c in ctxs]
    c0 = counters()
    H, lam, _ = _inputs(pairs, 3, {"prior": True}, seed=3)
    bad = lam.copy()
    bad[4, 2, 0, 1] = 1.0          # pair 4 belongs to the last shard
    with pytest.raises(RuntimeError, match="prior_information of hypothesis 2 of pair 4 is not symmetric"):
        two.match_batch_modes(refs, curs, _cfg(), hypotheses=H, screen_level=FIRST, prior_information=bad)
    assert counters() == c0
    n = len(refs)
    wm = engine._device_maps(refs, _cfg(), MASK_WEIGHT)[1]
    rh, ch = (C.c_void_p * n)(*[r.handle for r in refs]), (C.c_void_p * n)(*[c.handle for c in curs])
    res = (CResult * n)()
    rc = two.lib.dvo_b200_match_batch_modes_sharded(two.h, C.byref(_cfg()), n, rh, ch, 0, None, 0, 0.0, None, None, None, None, res, None,
                                                     None, None, None, 0, C.byref(wm))
    assert rc == -1 and "maps must be DVO_B200_MAPS_HOST" in two.lib.dvo_b200_sharded_last_error(two.h).decode()
    assert counters() == c0
    if torch.cuda.device_count() >= 2:
        other = ShardedEngine([0, 1])
        try:
            with pytest.raises(RuntimeError, match="pair 3 belongs to shard 1"):
                other.match_batch_modes(refs, curs, _cfg())
        finally:
            other.close()
    assert two.match_batch_modes(refs, curs, _cfg(), hypotheses=H, screen_level=FIRST, prior_information=lam)[1].shape == (n,)
    assert all(c[0] > c0[i][0] for i, c in enumerate(counters()))
