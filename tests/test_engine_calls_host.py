"""The marshalling of Engine and ShardedEngine, pinned on the CPU.  A recording fake of the C library stands in for
libdvo_b200.so: its creates hand out handles and its level_info answers sizes.  Each case checks the sequence of C calls
with their scalar arguments, the bytes behind each pointer (read when the call is made, through the sizes the call
implies), where the engine synchronises, and which inputs raise.  Paths that need torch CUDA tensors (the device creates,
the weight maps) are left to the GPU tests."""
import ctypes as C
import gc
import itertools

import numpy as np
import pytest

from dvo_slam_b200 import engine as E

CTX, OUT = "ctx", "out"
S = None          # a scalar argument, recorded as its value
CFG = C.sizeof(E.Config)
PIXEL_BYTES = {0: (4, 4), 1: (1, 2), 2: (3, 2)}   # image and depth bytes per pixel of each dvo_b200_input_format


def _kinds(fake, name, a):
    """what each argument of a call is: S, CTX, OUT (an output: only whether it is passed), or the bytes behind a pointer"""
    n = a[1] if len(a) > 1 and isinstance(a[1], int) else None
    if name == "create":
        return [S, S, OUT]
    if name in ("synchronize", "set_estimator", "get_estimator", "last_error", "stream"):
        return [CTX] + [S] * (len(a) - 1)
    if name == "pyramid_level_info":
        return [S, S, OUT, OUT, OUT]
    if name == "pyramid_create":
        px = a[3] * a[4]
        return [CTX, 4 * px, 4 * px] + [S] * 7 + [OUT]
    if name == "pyramid_create_raw":
        px = a[4] * a[5]
        return [CTX, px, 2 * px] + [S] * 8 + [OUT]
    if name in ("pyramid_create_batch", "sharded_pyramid_create_batch"):
        px = n * a[4] * a[5]
        return [CTX, S, 4 * px, 4 * px] + [S] * 7 + [OUT]
    if name in ("pyramid_create_raw_batch", "pyramid_create_bgr_batch"):
        px = n * a[5] * a[6]
        return [CTX, S, (3 if "bgr" in name else 1) * px, 2 * px] + [S] * 8 + [OUT]
    if name == "pyramid_create_masked_batch_roles":
        px = n * a[8] * a[9]
        bi, bz = PIXEL_BYTES[a[2]]
        return [CTX, S, S, bi * px, bz * px, S, px] + [S] * 8 + [OUT]
    if name == "pyramid_create_rectified_batch":
        n, px = a[2], a[2] * a[9] * a[10]
        bi, bz = PIXEL_BYTES[a[3]]
        return [CTX, S, S, S, bi * px, bz * px, S, px, S, S, S, S, OUT]
    if name == "pyramid_create_registered_batch":
        n, px = a[3], a[3] * a[10] * a[11]
        bi, bz = PIXEL_BYTES[a[4]]
        dw, dh = fake.registrations[a[1]]
        return [CTX, S, S, S, S, bi * px, bz * n * dw * dh, S, px, S, S, S, S, OUT]
    if name == "rectifier_create":
        return [CTX, S, S, S, S, 4 * a[3] * a[4], 4 * a[3] * a[4], 16, OUT]
    if name == "depth_registration_create":
        dw, dh = a[1], a[2]
        return [CTX, S, S, 4 * dw * dh, 4 * dw * dh, 4 * (dw + 1) * (dh + 1), 4 * (dw + 1) * (dh + 1), 128, S, S, 16, OUT]
    if name == "sharded_create":
        return [S, 4 * a[0], OUT]
    n = a[2]
    pairs = [CTX, CFG, S, 8 * n, 8 * n]
    if name in ("match_batch", "match_batch_sharded"):
        return pairs + [128 * n, OUT, OUT, S]
    if name == "match_batch_photometric":
        return pairs + [128 * n, 16 * n, OUT, OUT, OUT, S]
    if name == "match_batch_prior":
        return pairs + [128 * n, 288 * n, 16 * n, OUT, OUT, OUT, S]
    if name == "match_batch_device":
        return pairs + [128 * n, S]
    if name == "match_batch_hypotheses_modes":
        nk = n * a[5]
        return pairs + [S, 128 * nk, S, S, 288 * nk, 16 * nk] + [OUT] * 7 + [S, OUT]
    hook = [CTX, CFG, S, S, S, 128]
    if name in ("residual_image", "intensity_error_image"):
        return hook + [OUT, OUT]
    if name == "residual_image_photometric":
        return hook + [16, OUT, OUT]
    if name == "linearize":
        return hook + [S, 16] + [OUT] * 5
    if name == "linearize_photometric":
        return hook + [16, S, 16] + [OUT] * 5
    raise AssertionError(f"no argument kinds for dvo_b200_{name}")


def _addr(a):
    if isinstance(a, int):
        return a
    if isinstance(a, C.c_void_p):
        return a.value
    if type(a).__name__ == "CArgObject":
        return C.addressof(a._obj)
    if isinstance(a, C.Array):
        return C.addressof(a)
    if isinstance(a, C._Pointer):
        return C.cast(a, C.c_void_p).value
    raise TypeError(f"not a pointer: {type(a)}")


def _scalar(a):
    if isinstance(a, C.c_void_p):
        return a.value
    assert isinstance(a, (int, float)), type(a)
    return a


class FakeLib:
    """Records every dvo_b200_* call but the releases; creates hand out handles, level_info answers level 0 >> level."""

    def __init__(self):
        self.calls, self.handles, self.sizes, self.registrations = [], set(), {}, {}
        self.ctx, self.sharded = 0xC7000, 0x5A000
        self._next = itertools.count(0x100000, 0x100)

    def __getattr__(self, attr):
        if not attr.startswith("dvo_b200_"):
            raise AttributeError(attr)
        name = attr[len("dvo_b200_"):]

        def call(*a):
            if name.endswith("release") or name.endswith("destroy"):
                return 0
            rec = []
            for kind, v in zip(_kinds(self, name, a), a, strict=True):
                if v is None:
                    rec.append(None)
                elif kind is S:
                    rec.append(_scalar(v))
                elif kind == CTX:
                    rec.append(CTX if _addr(v) in (self.ctx, self.sharded) else _addr(v))
                elif kind == OUT:
                    rec.append(OUT)
                else:
                    rec.append(C.string_at(_addr(v), kind))
            self.calls.append((name, *rec))
            return self._act(name, a)
        return call

    def _handle(self, w, h):
        p = next(self._next)
        self.handles.add(p)
        self.sizes[p] = (w, h)
        return p

    def _act(self, name, a):
        if name == "create":
            a[2]._obj.value = self.ctx
        elif name == "sharded_create":
            a[2]._obj.value = self.sharded
        elif name == "last_error":
            return b"fake"
        elif name == "pyramid_level_info":
            w, h = self.sizes[a[0]]
            a[2]._obj.value, a[3]._obj.value = w >> a[1], h >> a[1]
        elif name.startswith("pyramid_create") or name == "sharded_pyramid_create_batch":
            if name in ("pyramid_create_rectified_batch", "pyramid_create_registered_batch"):
                w, h = self.sizes[a[1]]
            else:
                w, h = {"pyramid_create": (a[3], a[4]), "pyramid_create_masked_batch_roles": (a[8], a[9])}.get(name, (a[-8], a[-7]))
            out = a[-1]
            if isinstance(out, C.Array):
                for i in range(len(out)):
                    out[i] = self._handle(w, h)
            else:                               # one handle by reference
                out._obj.value = self._handle(w, h)
        elif name == "rectifier_create":
            a[-1]._obj.value = self._handle(a[3], a[4])
        elif name == "depth_registration_create":
            a[-1]._obj.value = p = self._handle(a[8], a[9])
            self.registrations[p] = (a[1], a[2])
        return 0


@pytest.fixture
def fake(monkeypatch):
    f = FakeLib()
    monkeypatch.setattr(E, "_lib", f)
    yield f
    gc.collect()
    for o in gc.get_objects():   # nothing made here may reach the real library once the fake is gone
        if type(o) in (E.Pyramid, E.Rectifier, E.DepthRegistration) and o.handle in f.handles:
            o.handle = None


@pytest.fixture
def eng(fake):
    e = E.Engine()
    assert fake.calls == [("create", 0, None, OUT), ("set_estimator", CTX, 0)]
    fake.calls.clear()
    return e


K = (525.0, 520.5, 160.25, 119.75)
N, H, W, LV = 3, 6, 8, 3
SYNC = ("synchronize", CTX)
rng = np.random.default_rng(7)


def b(a, dtype):
    return np.ascontiguousarray(a, dtype=dtype).tobytes()


def handles(ps):
    return np.array([p.handle for p in ps], np.uint64).tobytes()


def frames(n, fmt, h=H, w=W):
    if fmt == 0:
        return rng.random((n, h, w), dtype=np.float32), rng.random((n, h, w), dtype=np.float32) + 0.5
    img = rng.integers(0, 256, (n, h, w, 3) if fmt == 2 else (n, h, w), dtype=np.uint8)
    return img, rng.integers(0, 5000, (n, h, w), dtype=np.uint16)


def masks_of(kind, n, h=H, w=W):
    """(masks argument, bytes the create receives, whether the binding converts them)"""
    base = (rng.random((n, h, w)) < 0.7).astype(np.uint8)
    if kind == "hw":
        return base[0], np.broadcast_to(base[0], (n, h, w)).tobytes(), n > 1
    if kind == "nhw":
        return base, base.tobytes(), False
    if kind == "bool":
        return base.astype(bool), base.tobytes(), True
    if kind == "strided":
        big = np.ascontiguousarray(np.repeat(base, 2, axis=2) * 3)   # uint8 values pass as they are
        return big[:, :, ::2], (base * 3).tobytes(), True
    if kind == "ptr":
        return base.ctypes.data, base.tobytes(), False, base
    raise AssertionError(kind)


MASK_KINDS = [None, "hw", "nhw", "bool", "strided", "ptr"]


def call_masks(kind, n):
    if kind is None:
        return None, None, False, None
    m = masks_of(kind, n)
    return m if len(m) == 4 else m + (None,)


def masked(n, fmt, I, Z, scale, M, roles, w=W, h=H, levels=LV):
    return ("pyramid_create_masked_batch_roles", CTX, n, fmt, I, Z, scale, M, roles, w, h, *K, levels, OUT)


# ---- host creates ----
@pytest.mark.parametrize("kind", MASK_KINDS)
@pytest.mark.parametrize("roles", ["reference", "both"])
@pytest.mark.parametrize("ptrs", [False, True])
def test_pyramid_batch(eng, fake, kind, roles, ptrs):
    I, Z = frames(N, 0)
    m, mb, converted, _keep = call_masks(kind, N)
    if ptrs:
        ps = eng.pyramid_batch(None, None, K, LV, host_ptrs=(I.ctypes.data, Z.ctypes.data, N, H, W), masks=m, mask_roles=roles)
    else:
        ps = eng.pyramid_batch(I, Z, K, LV, masks=m, mask_roles=roles)
    if kind is None:
        want = [("pyramid_create_batch", CTX, N, I.tobytes(), Z.tobytes(), W, H, *K, LV, OUT)]
    else:
        want = [masked(N, 0, I.tobytes(), Z.tobytes(), 0.0, mb, E.MASK_ROLES[roles])] + [SYNC] * converted
    assert fake.calls == want + [SYNC] * (not ptrs)
    assert len(ps) == N and len({p.handle for p in ps} & fake.handles) == N


def test_pyramid_batch_from_other_dtypes(eng, fake):
    I, Z = frames(N, 0)
    eng.pyramid_batch(I.astype(np.float64), Z.tolist(), K, LV)
    assert fake.calls == [("pyramid_create_batch", CTX, N, I.tobytes(), Z.tobytes(), W, H, *K, LV, OUT), SYNC]


@pytest.mark.parametrize("kind", MASK_KINDS)
@pytest.mark.parametrize("roles", ["reference", "both"])
@pytest.mark.parametrize("raw", [False, True])
def test_pyramid_single(eng, fake, kind, roles, raw):
    I, Z = frames(1, 1 if raw else 0)
    m, mb, converted, _keep = call_masks(kind, 1)
    if raw:
        p = eng.pyramid_raw(I[0], Z[0], 0.001, K, LV, mask=m, mask_roles=roles)
    else:
        p = eng.pyramid(I[0], Z[0], K, LV, mask=m, mask_roles=roles)
    fmt = int(raw)
    if kind is None:
        want = [("pyramid_create_raw", CTX, I.tobytes(), Z.tobytes(), 0.001, W, H, *K, LV, OUT) if raw else
                ("pyramid_create", CTX, I.tobytes(), Z.tobytes(), W, H, *K, LV, OUT)]
    else:
        want = [masked(1, fmt, I.tobytes(), Z.tobytes(), 0.001 if raw else 0.0, mb, E.MASK_ROLES[roles])] + [SYNC] * converted
    assert fake.calls == want + [SYNC]
    assert p.handle in fake.handles


def test_pyramid_single_converts(eng, fake):
    I, Z = frames(1, 1)
    eng.pyramid_raw(I[0].astype(np.int32), Z[0].astype(np.float64), 0.002, K, LV)
    eng.pyramid(I[0], Z[0], K, LV)
    assert fake.calls == [("pyramid_create_raw", CTX, I.tobytes(), Z.tobytes(), 0.002, W, H, *K, LV, OUT), SYNC,
                          ("pyramid_create", CTX, b(I, np.float32), b(Z, np.float32), W, H, *K, LV, OUT), SYNC]


@pytest.mark.parametrize("kind", MASK_KINDS)
@pytest.mark.parametrize("roles", ["reference", "both"])
@pytest.mark.parametrize("bgr", [False, True])
def test_pyramid_raw_and_bgr_batch(eng, fake, kind, roles, bgr):
    I, Z = frames(N, 2 if bgr else 1)
    m, mb, converted, _keep = call_masks(kind, N)
    f = eng.pyramid_bgr_batch if bgr else eng.pyramid_raw_batch
    ps = f((I.ctypes.data, Z.ctypes.data, N, H, W), 0.001, K, LV, masks=m, mask_roles=roles)
    if kind is None:
        want = [("pyramid_create_bgr_batch" if bgr else "pyramid_create_raw_batch", CTX, N, I.tobytes(), Z.tobytes(), 0.001, W, H, *K,
                 LV, OUT)]
    else:
        want = [masked(N, 2 if bgr else 1, I.tobytes(), Z.tobytes(), 0.001, mb, E.MASK_ROLES[roles])] + [SYNC] * converted
    assert fake.calls == want
    assert len(ps) == N


@pytest.mark.parametrize("kind", [None, "hw", "nhw", "bool", "ptr"])
@pytest.mark.parametrize("fmt", [0, 1, 2])
@pytest.mark.parametrize("roles", ["reference", "both"])
def test_pyramid_rectified_batch(eng, fake, kind, fmt, roles):
    mx, my = rng.random((4, 5), dtype=np.float32), rng.random((4, 5), dtype=np.float32)
    rect = eng.rectifier((W, H), mx.astype(np.float64), my, (100.0, 101.0, 2.5, 1.5))
    assert fake.calls == [("rectifier_create", CTX, W, H, 5, 4, mx.tobytes(), my.tobytes(), b([100.0, 101.0, 2.5, 1.5], np.float32),
                           OUT)]
    fake.calls.clear()
    I, Z = frames(N, fmt)
    m, mb, _converted, _keep = call_masks(kind, N)
    scale = None if fmt == 0 else 0.001
    ps = eng.pyramid_rectified_batch(rect, I, Z, LV, depth_scale=scale, masks=m, mask_roles=roles)
    assert fake.calls == [("pyramid_create_rectified_batch", CTX, rect.handle, N, fmt, I.tobytes(), Z.tobytes(), scale or 0.0, mb,
                           E.MASK_ROLES[roles], W, H, LV, OUT), SYNC]
    assert len(ps) == N and all(fake.sizes[p.handle] == (5, 4) for p in ps)


@pytest.mark.parametrize("kind", [None, "hw", "ptr"])
@pytest.mark.parametrize("fmt", [0, 1, 2])
@pytest.mark.parametrize("with_rect", [False, True])
def test_pyramid_registered_batch(eng, fake, kind, fmt, with_rect):
    dw, dh = 5, 4
    rays = [rng.random(s, dtype=np.float32) for s in [(dh, dw), (dh, dw), (dh + 1, dw + 1), (dh + 1, dw + 1)]]
    T = np.eye(4)
    T[0, 3] = 0.025
    reg = eng.depth_registration((dw, dh), [r.astype(np.float64) for r in rays], T, (W, H), K)
    rect = eng.rectifier((W, H), np.zeros((H, W), np.float32), np.zeros((H, W), np.float32), K) if with_rect else None
    assert fake.calls[0] == ("depth_registration_create", CTX, dw, dh, *(r.tobytes() for r in rays), T.tobytes(), W, H, b(K, np.float32),
                             OUT)
    fake.calls.clear()
    I, _ = frames(N, fmt)
    Z = rng.random((N, dh, dw), dtype=np.float32) if fmt == 0 else rng.integers(0, 5000, (N, dh, dw), dtype=np.uint16)
    m, mb, _converted, _keep = call_masks(kind, N)
    ps = eng.pyramid_registered_batch(reg, I, Z, LV, depth_scale=None if fmt == 0 else 0.001, masks=m, mask_roles="both",
                                      rectifier=rect)
    assert fake.calls == [("pyramid_create_registered_batch", CTX, reg.handle, rect.handle if rect else None, N, fmt, I.tobytes(),
                           Z.tobytes(), 0.0 if fmt == 0 else 0.001, mb, 3, W, H, LV, OUT), SYNC]
    assert len(ps) == N


def test_create_refusals(eng, fake):
    I, Z = frames(N, 0)
    G, D = frames(N, 1)
    ptrs = (I.ctypes.data, Z.ctypes.data, N, H, W)
    rect = eng.rectifier((W, H), np.zeros((H, W), np.float32), np.zeros((H, W), np.float32), K)
    fake.calls.clear()
    refused = [
        (ValueError, lambda: eng.pyramid_batch(I, Z, K, LV, masks=np.ones((H, W + 1)))),
        (ValueError, lambda: eng.pyramid_batch(None, None, K, LV, host_ptrs=ptrs, masks=np.ones(7))),
        (ValueError, lambda: eng.pyramid_batch(I, Z, K, LV, masks=np.ones((N, H, W)), mask_roles="current")),
        (ValueError, lambda: eng.pyramid_raw_batch(ptrs, 0.001, K, LV, masks=np.ones((N + 1, H, W)))),
        (ValueError, lambda: eng.pyramid_bgr_batch(ptrs, 0.001, K, LV, masks=np.ones((N, H, W)), mask_roles="none")),
        (ValueError, lambda: eng.pyramid(I[0], Z[0], K, LV, mask=np.ones((H + 1, W)))),
        (ValueError, lambda: eng.pyramid_raw(G[0], D[0], 0.001, K, LV, mask=np.ones((H, W)), mask_roles="x")),
        (AssertionError, lambda: eng.pyramid(I[0], Z[0, :-1], K, LV)),
        (AssertionError, lambda: eng.pyramid(I, Z, K, LV)),
        (AssertionError, lambda: eng.pyramid_raw(G[0], D[0, :, :-1], 0.001, K, LV, mask=np.ones((H, W)))),
        (AssertionError, lambda: eng.pyramid_batch(I, Z[:, :-1], K, LV)),
        (AssertionError, lambda: eng.pyramid_batch(I[0], Z[0], K, LV, masks=np.ones((H, W)))),
        (ValueError, lambda: eng.pyramid(I[0], Z[0], K + (1.0,), LV)),
        (ValueError, lambda: eng.pyramid_raw(G[0], D[0], 0.001, K[:3], LV, mask=np.ones((H, W)))),
        (ValueError, lambda: eng.pyramid_batch(I, Z, K[:3], LV)),
        (ValueError, lambda: eng.pyramid_raw_batch(ptrs, 0.001, K + (1.0,), LV)),
        (ValueError, lambda: eng.pyramid_bgr_batch(ptrs, 0.001, K[:3], LV, masks=np.ones((N, H, W), np.uint8))),
        (ValueError, lambda: eng.pyramid_rectified_batch(rect, G, D, LV)),                      # raw depth without depth_scale
        (ValueError, lambda: eng.pyramid_rectified_batch(rect, I, D, LV, depth_scale=0.001)),   # float32 image, uint16 depth
        (ValueError, lambda: eng.pyramid_rectified_batch(rect, I, Z[:, :-1], LV)),
        (ValueError, lambda: eng.pyramid_rectified_batch(rect, I, Z, LV, masks=np.ones((2, H, W)))),
        (ValueError, lambda: eng.pyramid_rectified_batch(rect, I, Z, LV, masks=np.ones((N, H, W)), mask_roles="x")),
    ]
    for i, (exc, f) in enumerate(refused):
        with pytest.raises(exc):
            f()
        assert fake.calls == [], i


# ---- alignment ----
def pair_set(eng, n):
    I, Z = frames(2 * n, 0)
    ps = eng.pyramid_batch(I, Z, K, LV)
    return ps[:n], ps[n:]


def cfg_of(**kw):
    return E.Config(first_level=2, last_level=0, max_iterations_per_level=7, precision=1e-4, **kw)


def spd(*shape):
    a = rng.standard_normal(shape + (6, 6))
    return a @ np.swapaxes(a, -1, -2) + 6 * np.eye(6)


@pytest.mark.parametrize("t_init", [False, True])
@pytest.mark.parametrize("with_iterations", [False, True])
@pytest.mark.parametrize("prior", [False, True])
@pytest.mark.parametrize("raw", [False, True])
def test_match_batch(eng, fake, t_init, with_iterations, prior, raw):
    refs, curs = pair_set(eng, N)
    fake.calls.clear()
    cfg = cfg_of(use_initial_estimate=int(t_init))
    T = np.tile(np.eye(4, dtype=np.float32), (N, 1, 1)) + 0.01 * rng.random((N, 4, 4), dtype=np.float32) if t_init else None
    lam = spd(N) if prior else None
    out = eng.match_batch(refs, curs, cfg, T, with_iterations, raw=raw, prior_information=lam)
    max_log = 3 * 8 if with_iterations else 0
    Tb = b(T, np.float64) if t_init else None
    rest = (OUT, OUT if with_iterations else None, max_log)
    if prior:
        want = ("match_batch_prior", CTX, bytes(cfg), N, handles(refs), handles(curs), Tb, lam.tobytes(), None, None) + rest
    else:
        want = ("match_batch", CTX, bytes(cfg), N, handles(refs), handles(curs), Tb) + rest
    assert fake.calls == [want]
    assert len(out) == N and isinstance(out[0], E.CResult if raw else E.Result)


@pytest.mark.parametrize("t_init", [False, True])
@pytest.mark.parametrize("ab0", [False, True])
@pytest.mark.parametrize("with_iterations", [False, True])
@pytest.mark.parametrize("prior", [False, True])
def test_match_batch_photometric(eng, fake, t_init, ab0, with_iterations, prior):
    refs, curs = pair_set(eng, N)
    fake.calls.clear()
    cfg = cfg_of(use_initial_estimate=int(t_init))
    T = [np.eye(4).ravel().tolist()] * N if t_init else None
    A0 = [(1.0 + 0.1 * i, 0.01 * i) for i in range(N)] if ab0 else None
    lam = spd(N).astype(np.float32) if prior else None
    res, ab = eng.match_batch_photometric(refs, curs, cfg, T, A0, with_iterations, prior_information=lam)
    Tb = b(T, np.float64) if t_init else None
    A0b = b(A0, np.float64) if ab0 else None
    log = (OUT if with_iterations else None, 24 if with_iterations else 0)
    if prior:
        want = ("match_batch_prior", CTX, bytes(cfg), N, handles(refs), handles(curs), Tb, b(lam, np.float64), A0b, OUT, OUT) + log
    else:
        want = ("match_batch_photometric", CTX, bytes(cfg), N, handles(refs), handles(curs), Tb, A0b, OUT, OUT) + log
    assert fake.calls == [want]
    assert len(res) == N and ab.shape == (N, 2) and ab.dtype == np.float64


def test_match_single(eng, fake):
    (ref,), (cur,) = pair_set(eng, 1)
    fake.calls.clear()
    cfg = cfg_of(use_initial_estimate=1)
    T = np.eye(4)
    T[2, 3] = 0.125
    r = eng.match(ref, cur, cfg, T, with_iterations=True)
    eng.match(ref, cur, cfg)
    hs = (handles([ref]), handles([cur]))
    assert fake.calls == [("match_batch", CTX, bytes(cfg), 1, *hs, T.tobytes(), OUT, OUT, 24),
                          ("match_batch", CTX, bytes(cfg), 1, *hs, None, OUT, None, 0)]
    assert isinstance(r, E.Result)


@pytest.mark.parametrize("t_init", [False, True])
def test_match_batch_device(eng, fake, t_init):
    refs, curs = pair_set(eng, N)
    fake.calls.clear()
    cfg = cfg_of()
    T = np.tile(np.eye(4), (N, 1)) if t_init else None     # [4n, 4]: any shape of n * 16 values
    assert eng.match_batch_device(refs, curs, cfg, 0xDE00, T) is None
    assert fake.calls == [("match_batch_device", CTX, bytes(cfg), N, handles(refs), handles(curs), b(T, np.float64) if t_init else None,
                           0xDE00)]


@pytest.mark.parametrize("k", [1, 3])
@pytest.mark.parametrize("prior", [False, True])
@pytest.mark.parametrize("photometric", [False, "default", "init"])
@pytest.mark.parametrize("screen", [False, True])
@pytest.mark.parametrize("with_iterations", [False, True])
def test_match_batch_hypotheses(eng, fake, k, prior, photometric, screen, with_iterations):
    refs, curs = pair_set(eng, N)
    fake.calls.clear()
    Hy = np.tile(np.eye(4), (N, k, 1, 1)) + 0.01 * rng.random((N, k, 4, 4))
    lam = spd(N, k) if prior else None
    A0 = rng.random((N, k, 2)) if photometric == "init" else None
    cfg = None if k == 1 else cfg_of(use_initial_estimate=1)
    out = eng.match_batch_hypotheses(refs, curs, Hy, 1, 0.25, cfg, with_iterations, screen, prior_information=lam, photometric_init=A0,
                                     photometric=bool(photometric))
    c = E.Config(use_initial_estimate=1) if cfg is None else cfg
    max_log = (c.first_level - c.last_level + 1) * (c.max_iterations_per_level + 1) if with_iterations else 0
    p = bool(photometric)
    assert fake.calls == [("match_batch_hypotheses_modes", CTX, bytes(c), N, handles(refs), handles(curs), k, Hy.tobytes(), 1, 0.25,
                           lam.tobytes() if prior else None, A0.tobytes() if A0 is not None else None, OUT if p else None,
                           OUT if p and screen else None, OUT, OUT, OUT, OUT if screen else None, OUT if with_iterations else None,
                           max_log, None)]
    res, best, scores = out[:3]
    assert len(res) == N and best.shape == (N,) and best.dtype == np.int32 and scores.shape == (N, k)
    assert len(out) == 3 + screen + p * (1 + screen)
    if screen:
        assert [len(s) for s in out[3]] == [k] * N
    if p:
        assert out[3 + screen].shape == (N, 2) and (not screen or out[4 + screen].shape == (N, k, 2))


def test_match_refusals(eng, fake):
    refs, curs = pair_set(eng, N)
    fake.calls.clear()
    cfg = cfg_of()
    Hy = np.tile(np.eye(4), (N, 2, 1, 1))
    refused = [
        (AssertionError, lambda: eng.match_batch(refs, curs[:-1], cfg)),
        (AssertionError, lambda: eng.match_batch([], [], cfg)),
        (ValueError, lambda: eng.match_batch(refs, curs, cfg, np.eye(4))),
        (ValueError, lambda: eng.match_batch(refs, curs, cfg, prior_information=spd(N - 1))),
        (ValueError, lambda: eng.match_batch(refs, curs, cfg, prior_information=np.eye(6))),
        (ValueError, lambda: eng.match_batch_photometric(refs, curs, cfg, photometric_init=np.ones((N, 3)))),
        (ValueError, lambda: eng.match_batch_photometric(refs, curs, cfg, np.ones((N, 15)))),
        (ValueError, lambda: eng.match_batch_photometric(refs, curs, cfg, prior_information=spd(N, 2))),
        (ValueError, lambda: eng.match_batch_device(refs, curs, cfg, 0xDE00, np.eye(4))),
        (ValueError, lambda: eng.match_batch_hypotheses(refs, curs, Hy[:, 0], 1)),
        (ValueError, lambda: eng.match_batch_hypotheses(refs, curs, Hy[:-1], 1)),
        (ValueError, lambda: eng.match_batch_hypotheses(refs, curs, Hy[..., :3], 1)),
        (ValueError, lambda: eng.match_batch_hypotheses(refs, curs, Hy, 1, prior_information=spd(N))),
        (ValueError, lambda: eng.match_batch_hypotheses(refs, curs, Hy, 1, photometric=True, photometric_init=np.ones((N, 2)))),
        (ValueError, lambda: eng.match_batch_hypotheses(refs, curs, Hy, 1, photometric_init=np.ones((N, 2, 2)))),
        (AssertionError, lambda: eng.match_batch_hypotheses(refs, curs[:1], Hy, 1)),
        (ValueError, lambda: eng.residual_image(refs[0], curs[0], 0, np.eye(3))),
        (ValueError, lambda: eng.linearize(refs[0], curs[0], 0, np.eye(4), ab=(1.0, 0.0, 0.0))),
        (ValueError, lambda: eng.linearize(refs[0], curs[0], 0, np.eye(4), prev_precision=np.eye(3))),
        (ValueError, lambda: eng.intensity_error_image(refs[0], curs[0], 0, np.ones(15))),
    ]
    for i, (exc, f) in enumerate(refused):
        fake.calls.clear()
        with pytest.raises(exc):
            f()
        assert [c for c in fake.calls if c[0] != "pyramid_level_info"] == [], i


# ---- test hooks ----
@pytest.mark.parametrize("ab", [None, (1.25, -0.5)])
@pytest.mark.parametrize("level", [0, 2])
def test_hooks(eng, fake, ab, level):
    (ref,), (cur,) = pair_set(eng, 1)
    fake.calls.clear()
    T = np.eye(4, dtype=np.float32)
    T[0, 3] = 0.5
    Tb, abb = b(T, np.float64), None if ab is None else b(ab, np.float64)
    cfg = cfg_of()
    hs = (ref.handle, cur.handle, level)
    info = ("pyramid_level_info", ref.handle, level, OUT, OUT, OUT)
    n, img = eng.residual_image(ref, cur, level, T.ravel(), cfg, ab=ab)
    assert img.shape == (7, H >> level, W >> level)
    if ab is None:
        want = [info, ("residual_image", CTX, bytes(cfg), *hs, Tb, OUT, OUT)]
    else:
        want = [info, ("residual_image_photometric", CTX, bytes(cfg), *hs, Tb, abb, OUT, OUT)]
    n, img = eng.intensity_error_image(ref, cur, level, T)
    assert img.shape == (H >> level, W >> level)
    want += [info, ("intensity_error_image", CTX, bytes(E.Config()), *hs, Tb, OUT, OUT)]
    for weights, pp in ((False, None), (True, [[2.0, 0.5], [0.5, 3.0]])):
        out = eng.linearize(ref, cur, level, T, weights, pp, cfg, ab=ab)
        ppb = b(pp if pp is not None else np.zeros(4), np.float32)
        if ab is None:
            want.append(("linearize", CTX, bytes(cfg), *hs, Tb, int(weights), ppb, OUT, OUT, OUT, OUT, OUT))
        else:
            want.append(("linearize_photometric", CTX, bytes(cfg), *hs, Tb, abb, int(weights), ppb, OUT, OUT, OUT, OUT, OUT))
        k = 6 if ab is None else 8
        assert out["A"].shape == (k, k) and out["b"].shape == (k,) and out["precision"].shape == (2, 2)
    assert fake.calls == want


# ---- several devices ----
@pytest.mark.parametrize("t_init", [False, True])
def test_sharded(fake, t_init):
    s = E.ShardedEngine([0, 1])
    I, Z = frames(2 * N, 0)
    hs = s.pyramid_batch(I.astype(np.float64), Z, [int(v) if v == int(v) else v for v in K], LV)
    refs, curs = hs[:N], hs[N:]
    cfg = cfg_of(use_initial_estimate=int(t_init))
    T = np.tile(np.eye(4), (N, 1, 1)) if t_init else None
    res = s.match_batch(refs, curs, cfg, T)
    assert len(res) == N and isinstance(res[0], E.CResult)
    hb = lambda ps: np.array([p.value for p in ps], np.uint64).tobytes()
    assert fake.calls == [("sharded_create", 2, b([0, 1], np.int32), OUT),
                          ("sharded_pyramid_create_batch", CTX, 2 * N, I.tobytes(), Z.tobytes(), W, H, *K, LV, OUT),
                          ("match_batch_sharded", CTX, bytes(cfg), N, hb(refs), hb(curs), T.tobytes() if t_init else None, OUT, None, 0)]
    s.close()
