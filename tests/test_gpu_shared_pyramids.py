"""Pyramids shared between contexts, streams and host threads (INTEGRATION.md §E).

A pyramid may be used by any context while its build is still queued on the building context's stream, may be released
as soon as the calls that used it have returned (on any context, dvo_b200_match_batch_device included), and may outlive
the context that built it.  The rest of the suite builds every pyramid synchronously and reads results through blocking
calls, so none of that is exercised there.  Here the building context's stream is held by a device-side spin
(torch.cuda._sleep) while the build is queued behind it, and every case asserts that the build (or, in the release case,
the foreign alignment) has not completed when the call under test is issued: a hold that is too short fails loudly
instead of passing vacuously.

Every output is compared bit for bit with the oracle (pyramid planes, selections, residual records, error images) or
with the same call on a single context whose builds were all synchronised (linearisations, alignments).

HOLD_CYCLES is a count of SM clock cycles, so the hold's length follows the clock.  On an H100 80GB HBM3 at a 400 W power
limit (maximum SM clock 1980 MHz) it lasted 151 ms, and the call under test was issued at most 0.36 ms after the hold
started: a margin of over 400 times.
"""
import ctypes as C
import threading
import time

import numpy as np
import pytest

from helpers import nan_equal
from test_gpu_geometry import _identical

pytestmark = pytest.mark.gpu

HOLD_CYCLES = 300_000_000
DEPTH_SCALE = 1.0 / 5000.0
SMALL = (160, 120, 3)           # (width, height, levels): sizes where the oracle is the reference
FULL = (640, 480, 5)            # sizes where a single-context run is the reference
SELECTIONS = [(0.0, 0.0), (4.0, 0.02), (8.0, 0.05)]       # the defaults and two (intensity, depth) threshold pairs
PP = np.array([[2000.0, -30.0], [-30.0, 9000.0]], dtype=np.float32)


def _T():
    from dvo_slam_b200 import synth
    return synth.se3_exp(np.array([0.004, -0.003, 0.008, 0.004, -0.003, 0.006]))


def _cfg(first, last, sel=(0.0, 0.0)):
    from dvo_slam_b200.engine import Config
    return Config(first_level=first, last_level=last, max_iterations_per_level=50, precision=1e-4,
                  intensity_derivative_threshold=sel[0], depth_derivative_threshold=sel[1])


# ---- holding a stream ----
def _torch_stream(eng):
    import torch
    return torch.cuda.ExternalStream(eng.stream, device=torch.device("cuda", 0))


def _hold(eng):
    """queue a device-side spin of HOLD_CYCLES on the engine's stream: work the engine enqueues next waits behind it"""
    import torch
    s = _torch_stream(eng)
    with torch.cuda.stream(s):
        torch.cuda._sleep(HOLD_CYCLES)
    return time.perf_counter()


def _mark(eng):
    """an event recorded on the engine's stream after everything enqueued so far"""
    import torch
    ev = torch.cuda.Event()
    ev.record(_torch_stream(eng))
    return ev


def _assert_pending(ev, t_hold=None):
    assert not ev.query(), "the held work finished before the call under test was issued: the hold is too short"
    if t_hold is not None:
        print(f"call issued {1e3 * (time.perf_counter() - t_hold):.2f} ms after the hold started")


# ---- calls with an explicit context (the Pyramid methods use the building engine's) ----
def _download(ctx, p, lvl):
    from dvo_slam_b200.engine import load_library
    w, h, _ = p.level_info(lvl)
    out = np.empty((6, h, w), dtype=np.float32)
    rc = load_library().dvo_b200_pyramid_download(ctx, p.handle, lvl, out.ctypes.data_as(C.POINTER(C.c_float)))
    assert rc == 0, rc
    return out


def _select(eng, p, lvl, sel):
    from dvo_slam_b200.engine import load_library
    w, h, _ = p.level_info(lvl)
    mask = np.zeros((h, w), dtype=np.uint8)
    cnt = C.c_int64()
    eng._check(load_library().dvo_b200_pyramid_select(eng.ctx, p.handle, lvl, sel[0], sel[1], C.byref(cnt),
                                                      mask.ctypes.data_as(C.POINTER(C.c_uint8))))
    return cnt.value, mask


def _result(r):
    return [r.transformation, r.information, r.log_likelihood, repr(r.levels)]


def _device_results(eng, refs, curs, cfg):
    """dvo_b200_match_batch_device into a torch buffer; returns (buffer, decode) where decode() reads it after a sync"""
    import torch
    from dvo_slam_b200.engine import CResult, Result
    n = len(refs)
    buf = torch.zeros(n * C.sizeof(CResult), dtype=torch.uint8, device="cuda:0")
    eng.match_batch_device(refs, curs, cfg, buf.data_ptr())

    def decode():
        res = (CResult * n).from_buffer_copy(buf.cpu().numpy().tobytes())
        return [_result(Result(res[i])) for i in range(n)]
    return buf, decode


# ---- inputs ----
class Inputs:
    """n frames of one scene in the three host formats, in pinned memory, and the float images the oracle sees"""

    def __init__(self, frames, K, levels, seed):
        import torch
        rng = np.random.default_rng(seed)
        self.K, self.levels = K, levels
        self.n = len(frames)
        self.h, self.w = frames[0][0].shape
        grey = np.stack([I for I, _ in frames]).astype(np.uint8)
        assert np.array_equal(grey.astype(np.float32), np.stack([I for I, _ in frames]))
        raw = np.stack([np.where(np.isnan(Z), 0, np.round(np.nan_to_num(Z) / DEPTH_SCALE)).astype(np.uint16) for _, Z in frames])
        bgr = np.clip(grey[..., None].astype(np.int32) + rng.integers(-20, 21, size=grey.shape + (3,)), 0, 255).astype(np.uint8)
        from oracle import oracle_py as orc
        self.depth = np.stack([orc.convert_raw_depth(r, DEPTH_SCALE) for r in raw])
        self.grey_f = grey.astype(np.float32)
        self.bgr_grey = np.stack([orc.bgr_to_grey(b) for b in bgr])
        pin = lambda a: torch.from_numpy(np.ascontiguousarray(a)).pin_memory()
        self.p_grey, self.p_raw, self.p_bgr = pin(grey), pin(raw), pin(bgr)
        self.p_I, self.p_Z = pin(self.grey_f), pin(self.depth)

    def build(self, eng, path):
        """enqueue the build of all n frames through one input path; nothing synchronises"""
        dims = (self.n, self.h, self.w)
        if path == "raw":
            return eng.pyramid_raw_batch((self.p_grey.data_ptr(), self.p_raw.data_ptr()) + dims, DEPTH_SCALE, self.K, self.levels)
        if path == "bgr":
            return eng.pyramid_bgr_batch((self.p_bgr.data_ptr(), self.p_raw.data_ptr()) + dims, DEPTH_SCALE, self.K, self.levels)
        assert path == "float"
        return eng.pyramid_batch(None, None, self.K, self.levels, host_ptrs=(self.p_I.data_ptr(), self.p_Z.data_ptr()) + dims)

    def intensity(self, path, i):
        return self.bgr_grey[i] if path == "bgr" else self.grey_f[i]


def _scene(seed, w, h):
    from dvo_slam_b200 import synth
    K = tuple(v * w / 640 for v in synth.FR1_INTRINSICS)
    p = synth.make_pair(seed, synth.SceneConfig(width=w, height=h, intrinsics=K))
    return [(p["I_ref"].numpy(), p["Z_ref"].numpy()), (p["I_cur"].numpy(), p["Z_cur"].numpy())], K


_cache = {}


def _small(which="pair"):
    """160 x 120, 3 levels: the (reference, current) pair under test, or a decoy of another scene"""
    if which not in _cache:
        w, h, levels = SMALL
        frames, K = _scene(41 if which == "pair" else 97, w, h)
        _cache[which] = Inputs(frames, K, levels, seed=3 if which == "pair" else 4)
    return _cache[which]


def _oracle_pyramid(inp, path, i):
    from oracle import oracle_py as orc
    key = ("oracle", id(inp), path, i)
    if key not in _cache:
        _cache[key] = orc.Pyramid(inp.intensity(path, i), inp.depth[i], inp.K, inp.levels)
    return _cache[key]


def _release(pyrs):
    for p in pyrs:
        p.release()


def _held_build(eng, inp, decoy, path):
    """Build the decoy (another scene) synchronously and release it, so that the pool holds a slab of the right size with
    other contents and the staging buffer is allocated; then hold the stream and queue the real build behind the hold."""
    _release(decoy.build(eng, path))
    eng.synchronize()
    t = _hold(eng)
    pyrs = inp.build(eng, path)
    return pyrs, _mark(eng), t


# ---- the calls of case 1: each returns its outputs as a list ----
def _call_select(sel):
    def f(eng, ref, cur, levels):
        return [v for p in (ref, cur) for l in range(levels) for v in _select(eng, p, l, sel)]
    return f


def _call_download(null_ctx):
    def f(eng, ref, cur, levels):
        return [_download(None if null_ctx else eng.ctx, p, l) for p in (ref, cur) for l in range(levels)]
    return f


def _call_residual(eng, ref, cur, levels):
    return [v for l in range(levels) for v in eng.residual_image(ref, cur, l, _T(), _cfg(l, l))]


def _call_error_image(eng, ref, cur, levels):
    return [v for l in range(levels) for v in eng.intensity_error_image(ref, cur, l, _T(), _cfg(l, l))]


def _call_linearize(eng, ref, cur, levels):
    return [v for l in range(levels) for uw in (False, True) for v in eng.linearize(ref, cur, l, _T(), uw, PP, _cfg(l, l)).values()]


def _call_match(eng, ref, cur, levels):
    return _result(eng.match(ref, cur, _cfg(levels - 1, 0)))


def _call_match_device(eng, ref, cur, levels):
    _, decode = _device_results(eng, [ref], [cur], _cfg(levels - 1, 0))
    eng.synchronize()
    return decode()[0]


CALLS = {
    "select_default": _call_select(SELECTIONS[0]),
    "select_thresholds": _call_select(SELECTIONS[1]),
    "download": _call_download(False),
    "download_null_ctx": _call_download(True),
    "residual_image": _call_residual,
    "intensity_error_image": _call_error_image,
    "linearize": _call_linearize,
    "match": _call_match,
    "match_batch_device": _call_match_device,
}
PATHS = ["raw", "bgr", "float"]


def _check_against_oracle(call, got, inp, path):
    from oracle import oracle_py as orc
    levels = inp.levels
    oref, ocur = _oracle_pyramid(inp, path, 0), _oracle_pyramid(inp, path, 1)
    if call.startswith("select"):
        sel = SELECTIONS[0] if call == "select_default" else SELECTIONS[1]
        want = [v for op in (oref, ocur) for l in range(levels) for v in orc.select(op, l, *sel)]
        for k in range(0, len(want), 2):
            assert got[k] == want[k] and np.array_equal(got[k + 1], want[k + 1]), k // 2
    elif call.startswith("download"):
        k = 0
        for op in (oref, ocur):
            for l in range(levels):
                want = op.planes(l)
                want[1][np.isnan(want).any(axis=0)] = np.nan        # device depth is masked where any channel is NaN
                assert all(nan_equal(got[k][c], want[c]) for c in range(6)), (k, l)
                k += 1
    elif call in ("residual_image", "intensity_error_image"):
        fn = orc.residual_image if call == "residual_image" else orc.intensity_error_image
        for l in range(levels):
            n_o, img_o = fn(oref, ocur, l, _T(), orc.mode("mirror"))
            assert got[2 * l] == n_o and nan_equal(got[2 * l + 1], img_o), l


@pytest.fixture(scope="module")
def single_context():
    """outputs of every call on one context whose builds were synchronised, per (input path, call)"""
    from dvo_slam_b200.engine import Engine
    out = {}
    inp = _small()
    for path in PATHS:
        for call, fn in CALLS.items():
            eng = Engine(device=0)
            try:
                ref, cur = inp.build(eng, path)
                eng.synchronize()
                out[(path, call)] = fn(eng, ref, cur, inp.levels)
                _release([ref, cur])
            finally:
                eng.close()
    return out


def test_the_hold_lasts_long_enough():
    """the hold, timed by CUDA events on the stream it holds: long against the few milliseconds the calls under test take
    to be issued, short enough to keep the file fast"""
    import torch
    A = _engines(1)[0]
    try:
        s = _torch_stream(A)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(s)
        _hold(A)
        b.record(s)
        b.synchronize()
        ms = a.elapsed_time(b)
        print(f"hold of {HOLD_CYCLES} cycles: {ms:.1f} ms")
        assert 50.0 < ms < 1000.0, ms
    finally:
        A.close()


def _engines(n):
    from dvo_slam_b200.engine import Engine
    return [Engine(device=0) for _ in range(n)]


# ---- 1. consumed before built ----
@pytest.mark.parametrize("call", list(CALLS))
@pytest.mark.parametrize("path", PATHS)
def test_consumed_before_built(oracle, single_context, path, call):
    """Context A queues the build of a (reference, current) pair behind a hold; context B makes one call on the pyramids
    before the build has run, with no host synchronisation in between.  The outputs must be the oracle's and the
    single-context ones."""
    A, B = _engines(2)
    inp = _small()
    pyrs = []
    try:
        pyrs, built, t = _held_build(A, inp, _small("decoy"), path)
        _assert_pending(built, t)
        got = CALLS[call](B, pyrs[0], pyrs[1], inp.levels)
        _check_against_oracle(call, got, inp, path)
        _identical(got, single_context[(path, call)])
    finally:
        _release(pyrs)
        A.close()
        B.close()


# ---- 2. the selection state after a foreign select on an unfinished pyramid ----
@pytest.fixture(scope="module")
def single_context_matches():
    """per (input path, selection): the single-context alignment of the small pair (the BGR path has its own grey image)"""
    from dvo_slam_b200.engine import Engine
    inp = _small()
    out = {}
    for path in PATHS:
        eng = Engine(device=0)
        try:
            ref, cur = inp.build(eng, path)
            eng.synchronize()
            for sel in SELECTIONS:
                out[(path, sel)] = _result(eng.match(ref, cur, _cfg(inp.levels - 1, 0, sel)))
            _release([ref, cur])
        finally:
            eng.close()
    return out


@pytest.mark.parametrize("path", PATHS)
def test_selection_state_after_a_foreign_select_on_an_unfinished_pyramid(oracle, single_context_matches, path):
    """B selects with non-default thresholds while A's build of the pyramid is still queued.  Then B's alignment at those
    thresholds, A's alignment and selection at the defaults, and rounds that alternate the thresholds between the two
    contexts must all equal the single-context alignments and the oracle's selections: the per-pyramid selection cache
    (thresholds on the host, masks on the device) has to agree every time."""
    A, B = _engines(2)
    inp = _small()
    levels = inp.levels
    oref = _oracle_pyramid(inp, path, 0)
    pyrs = []

    def check_select(eng, ref, sel):
        for l in range(levels):
            S, mask = _select(eng, ref, l, sel)
            So, masko = oracle.select(oref, l, *sel)
            assert S == So and np.array_equal(mask, masko), (l, sel, S, So)

    def check_match(eng, ref, cur, sel):
        _identical(_result(eng.match(ref, cur, _cfg(levels - 1, 0, sel))), single_context_matches[(path, sel)])

    try:
        pyrs, built, t = _held_build(A, inp, _small("decoy"), path)
        ref, cur = pyrs
        _assert_pending(built, t)
        check_select(B, ref, SELECTIONS[1])
        check_match(B, ref, cur, SELECTIONS[1])
        check_match(A, ref, cur, SELECTIONS[0])
        check_select(A, ref, SELECTIONS[0])
        rounds = [(B, SELECTIONS[2]), (A, SELECTIONS[1]), (B, SELECTIONS[0]), (A, SELECTIONS[2]), (B, SELECTIONS[1]),
                  (A, SELECTIONS[0])]
        for eng, sel in rounds:
            check_match(eng, ref, cur, sel)
            check_select(eng, ref, sel)
    finally:
        _release(pyrs)
        A.close()
        B.close()


# ---- 3. release after an asynchronous foreign match ----
NPAIRS_ASYNC = 256
NCUR = 8


@pytest.fixture(scope="module")
def full_scenes(oracle):
    """640 x 480, 5 levels: a sequence (frame 0 is the reference P, frames 1.. the currents) and another scene Q"""
    from dvo_slam_b200 import synth
    w, h, levels = FULL
    frames, _ = synth.make_sequence(77, NCUR + 1)
    seq = Inputs([(I.numpy(), Z.numpy()) for I, Z in frames], synth.FR1_INTRINSICS, levels, seed=5)
    qframes, K = _scene(78, w, h)
    q = Inputs(qframes[:1], K, levels, seed=6)
    return seq, q


def _one(eng, inp, i):
    """frame i of inp alone (n = 1, from the pinned float images): a pyramid whose slab has a size of its own"""
    dims = (1, inp.h, inp.w)
    I, Z = inp.p_I[i], inp.p_Z[i]
    return eng.pyramid_batch(None, None, inp.K, inp.levels, host_ptrs=(I.data_ptr(), Z.data_ptr()) + dims)[0]


def _async_pairs(P, curs):
    return [P] * NPAIRS_ASYNC, [curs[i % NCUR] for i in range(NPAIRS_ASYNC)]


@pytest.fixture(scope="module")
def undisturbed(full_scenes):
    """the batch of case 3 on one context, nothing released early; and Q's level planes"""
    from dvo_slam_b200.engine import Engine
    seq, q = full_scenes
    eng = Engine(device=0)
    try:
        P = _one(eng, seq, 0)
        curs = seq.build(eng, "float")[1:]
        eng.synchronize()
        refs, cs = _async_pairs(P, curs)
        res = [_result(r) for r in eng.match_batch(refs, cs, _cfg(FULL[2] - 1, 0))]
        Q = _one(eng, q, 0)
        eng.synchronize()
        planes = [_download(eng.ctx, Q, l) for l in range(FULL[2])]
        _release([P, Q] + curs)
    finally:
        eng.close()
    return res, planes


@pytest.mark.parametrize("contexts", ["two", "one"])
def test_release_after_an_asynchronous_foreign_match(full_scenes, undisturbed, contexts):
    """A builds P alone.  B queues dvo_b200_match_batch_device on 256 pairs that all use P as reference (its currents are
    B's own), releases its handles, the last reference to P is dropped at once, and A immediately builds a pyramid of the
    same geometry from another scene, which takes P's memory.  The foreign alignment must still read P: its results equal
    an undisturbed run bit for bit, and so does the new pyramid.  "one": the same sequence on a single context, where the
    stream orders it."""
    seq, q = full_scenes
    want, q_planes = undisturbed
    A = _engines(1)[0]
    B = _engines(1)[0] if contexts == "two" else A
    new = None
    try:
        P = _one(A, seq, 0)
        A.synchronize()
        curs = seq.build(B, "float")[1:]
        B.synchronize()
        refs, cs = _async_pairs(P, curs)
        buf, decode = _device_results(B, refs, cs, _cfg(FULL[2] - 1, 0))
        done = _mark(B)
        del refs, cs
        _release(curs)
        P.release()
        new = _one(A, q, 0)
        _assert_pending(done)                     # the alignment was still running when P's memory was rebuilt
        B.synchronize()
        A.synchronize()
        got = decode()
        for i in range(NPAIRS_ASYNC):
            _identical(got[i], want[i])
        _identical([_download(A.ctx, new, l) for l in range(FULL[2])], q_planes)
    finally:
        if new is not None:
            new.release()
        A.close()
        if B is not A:
            B.close()


# ---- 4. pyramids outliving their context ----
def _current_device():
    import torch
    return torch.cuda.current_device()


def test_pyramids_outlive_their_context(oracle, single_context):
    """A queues the build of the pair behind a hold and is destroyed at once.  B aligns the pair, and download with a NULL
    context reads it: all of it as the oracle and the single-context run.  B is destroyed too, and the last release
    happens on another host thread, which frees the memory of the closed pool.  Releasing and download with a NULL context
    leave the calling thread's current device as it was (checked on a device other than the pyramids' where there is
    one)."""
    import torch
    A, B = _engines(2)
    inp = _small()
    path = "raw"
    pyrs = []
    try:
        pyrs, built, t = _held_build(A, inp, _small("decoy"), path)
        _assert_pending(built, t)
        A.close()
        ref, cur = pyrs
        for call in ("match", "residual_image", "select_default", "download_null_ctx"):
            got = CALLS[call](B, ref, cur, inp.levels)
            _check_against_oracle(call, got, inp, path)
            _identical(got, single_context[(path, call)])
    finally:
        A.close()
        B.close()
    other = 1 if torch.cuda.device_count() > 1 else 0
    errors = []

    def last_release():
        try:
            from dvo_slam_b200.engine import load_library
            torch.cuda.set_device(other)
            got = [_download(None, p, l) for p in pyrs for l in range(inp.levels)]
            assert _current_device() == other
            _identical(got, single_context[(path, "download_null_ctx")])
            for p in pyrs:
                assert load_library().dvo_b200_pyramid_release(p.handle) == 0
                p.handle = None
            assert _current_device() == other
        except BaseException as e:          # noqa: BLE001 -- re-raised on the test's thread
            errors.append(e)
    th = threading.Thread(target=last_release)
    th.start()
    th.join()
    if errors:
        raise errors[0]


# ---- 5. concurrent host threads, each with its own context ----
NTHREADS, NROUNDS = 4, 3


@pytest.fixture(scope="module")
def thread_scenes(oracle):
    """640 x 480, 4 levels: 4 shared references and 4 currents per thread (one sequence: reference k, current k + 1)"""
    from dvo_slam_b200 import synth
    w, h, _ = FULL
    levels = 4
    frames, _ = synth.make_sequence(91, 5 * NTHREADS)
    fr = [(I.numpy(), Z.numpy()) for I, Z in frames]
    refs = Inputs([fr[k] for k in range(4)], synth.FR1_INTRINSICS, levels, seed=7)
    curs = [Inputs([fr[(k + 1 + 4 * t) % len(fr)] for k in range(4)], synth.FR1_INTRINSICS, levels, seed=8 + t)
            for t in range(NTHREADS)]
    return refs, curs


def test_concurrent_threads_align_against_shared_references(thread_scenes):
    """A fifth context queues the build of 4 reference pyramids behind a hold.  Four host threads, each with its own
    context and its own currents, align all of them against the shared references for several rounds at the default
    thresholds, concurrently.  Every result equals the serial single-context result bit for bit."""
    from dvo_slam_b200.engine import Engine
    refs_in, curs_in = thread_scenes
    cfg = _cfg(3, 0)
    solo = Engine(device=0)
    try:
        srefs = refs_in.build(solo, "float")
        want = []
        for t in range(NTHREADS):
            scurs = curs_in[t].build(solo, "float")
            solo.synchronize()
            want.append([_result(r) for r in solo.match_batch(srefs, scurs, cfg)])
            _release(scurs)
        _release(srefs)
    finally:
        solo.close()

    E = Engine(device=0)
    engines = _engines(NTHREADS)
    curs = []
    for t in range(NTHREADS):
        curs.append(curs_in[t].build(engines[t], "float"))
        engines[t].synchronize()
    shared = []
    results = [[] for _ in range(NTHREADS)]
    errors = []
    start = threading.Barrier(NTHREADS)

    def worker(t):
        try:
            start.wait()
            for _ in range(NROUNDS):
                results[t].append([_result(r) for r in engines[t].match_batch(shared, curs[t], cfg)])
        except BaseException as e:          # noqa: BLE001 -- re-raised on the test's thread
            errors.append(e)

    try:
        shared, built, t0 = _held_build(E, refs_in, curs_in[0], "float")
        _assert_pending(built, t0)
        threads = [threading.Thread(target=worker, args=(t,)) for t in range(NTHREADS)]
        for th in threads:
            th.start()
        for th in threads:
            th.join()
        if errors:
            raise errors[0]
        for t in range(NTHREADS):
            assert len(results[t]) == NROUNDS
            for r in results[t]:
                for i in range(len(shared)):
                    _identical(r[i], want[t][i])
    finally:
        for t in range(NTHREADS):
            _release(curs[t])
        _release(shared)
        E.close()
        for eng in engines:
            eng.close()
