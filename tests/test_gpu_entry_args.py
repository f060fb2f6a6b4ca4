"""GPU: the argument rules every one-shot audio entry point (device and host form) and every stream create share.

Each one-shot entry rejects B = 0, B = 65536 (on a real [65536, 1] batch) and S = 0 (flac accepts S = 0: an empty row is
a valid stream); each host entry rejects n_in = [-1] and [S + 1]; each create rejects 0 and 65536 slots, chunk 0 and
the chunk limit + 1.  After every rejection the context still gives the same bits as before it.  Every buffer is large
enough for the arguments it goes with, so a missing check fails an assertion, never reads out of bounds."""
import ctypes as C

import numpy as np
import pytest
import torch

from viettts_b200 import _lib

pytestmark = pytest.mark.gpu

SR = 16000
S0 = 4096
BIG = 65536          # one row past the batch limit
BANK = SR            # samples of the bed bank's one entry
IR = 64              # reverb taps
NB = 513             # denoiser bias bins


@pytest.fixture(scope="module")
def eng():
    from viettts_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


def P(a):
    if a is None:
        return None
    return a.data_ptr() if isinstance(a, torch.Tensor) else a.ctypes.data


class Bufs:
    """Every buffer a call of B rows of S samples may touch, on the host (host form) or the device (device form)."""

    def __init__(self, host, B, S, x=None):
        rows = max(B, 1)
        Y = 4 * max(S, 1) + 16
        dev = (lambda a: a) if host else (lambda a: torch.from_numpy(a).cuda())
        self.x = dev(np.zeros(rows * max(S, 1), np.float32) if x is None else x)
        self.codes = dev(np.zeros(rows * max(S, 1), np.int16))
        self.y = dev(np.zeros(rows * Y, np.float32))
        self.r = dev(np.zeros(rows * 4, np.float32))
        self.nb = dev(np.zeros(rows, np.int32))
        self.gain = dev(np.zeros(rows, np.float32))
        self.ir = dev(np.r_[np.float32(1.0), np.full(IR - 1, 0.01, np.float32)])
        self.bias = dev(np.full(NB, 1e-3, np.float32))
        self.keys = dev(np.array([7], np.int64))
        self.yb = dev(np.zeros(rows * _lib.load().vtts_flac_bound(max(S, 0), 4096), np.uint8))
        # host in both forms
        self.semis = np.full(rows, 3.0, np.float32)
        self.formants = np.zeros(rows, np.float32)
        self.tempo = np.full(rows, 1.25, np.float32)
        self.bed = np.zeros(rows, np.int32)
        self.sos = np.zeros(6, np.float64)
        K = C.c_int()
        assert _lib.load().vtts_eq_design(1, SR, 3000.0, 0.707, 6.0, 2, self.sos.ctypes.data, C.byref(K)) == 0
        self.K = K.value

    def outputs(self):
        return [(a.cpu().numpy() if isinstance(a, torch.Tensor) else a).copy() for a in (self.y, self.r, self.nb, self.yb)]


def one_shot(eng, bank):
    """name -> call(host, B, S, b, n): the entry point on b's buffers and the host or device row lengths n (or None)"""
    L, h = eng.lib, eng.h
    offs = np.array([0], np.int64)
    lens = np.array([BANK], np.int32)

    def sfx(host):
        return "_host" if host else ""

    def f(name, *args):
        def call(host, B, S, b, n):
            fn = getattr(L, "vtts_" + name + sfx(host))
            a = [P(v) if isinstance(v, (np.ndarray, torch.Tensor)) else v for v in args[0](b)]
            return fn(h, P(b.x) if name != "decode" else P(b.codes), P(n), *[v(B, S) if callable(v) else v for v in a],
                      *([] if host else [None]))
        return call

    return {
        "compress": f("compress", lambda b: [lambda B, S: B, lambda B, S: S, SR, -30.0, 4.0, 6.0, 5.0, 50.0, 0.0, b.y, b.r]),
        "deess": f("deess", lambda b: [lambda B, S: B, lambda B, S: S, SR, 5000.0, -30.0, 4.0, 6.0, 1.0, 50.0, 12.0, b.y, b.r]),
        "eq": f("eq", lambda b: [lambda B, S: B, lambda B, S: S, b.sos, b.K, b.y]),
        "loudness": f("loudness", lambda b: [lambda B, S: B, lambda B, S: S, SR, b.y]),
        "loudness_normalize": f("loudness_normalize", lambda b: [lambda B, S: B, lambda B, S: S, SR, -23.0, -1.0, b.y, b.r]),
        "loudness_normalize_limited": f("loudness_normalize_limited",
                                        lambda b: [lambda B, S: B, lambda B, S: S, SR, -23.0, -1.0, 5.0, 50.0, b.y, b.r]),
        "bed_mix": f("bed_mix", lambda b: [lambda B, S: B, lambda B, S: S, SR, bank, offs, lens, 1, b.bed, 12.0, -40.0, 10.0, 200.0,
                                           0, 0, 0, 0, b.y, b.r]),
        "reverb": f("reverb", lambda b: [lambda B, S: B, lambda B, S: S, SR, b.ir, IR, 0.3, b.y]),
        "watermark": f("watermark", lambda b: [lambda B, S: B, lambda B, S: S, 7, 0.05, b.y]),
        "watermark_detect": f("watermark_detect", lambda b: [lambda B, S: B, lambda B, S: S, SR, b.keys, 1, 0, b.y, b.nb]),
        "denoise": f("denoise", lambda b: [lambda B, S: B, lambda B, S: S, 0.5, b.bias, b.y]),
        "pitch_shift": f("pitch_shift", lambda b: [lambda B, S: B, lambda B, S: S, b.semis, b.y]),
        "voice_shift": f("voice_shift", lambda b: [lambda B, S: B, lambda B, S: S, b.semis, b.formants, b.y]),
        "time_stretch": f("time_stretch", lambda b: [lambda B, S: B, lambda B, S: S, b.tempo, b.y, lambda B, S: 2 * max(S, 1)]),
        "resample": f("resample", lambda b: [lambda B, S: B, lambda B, S: S, SR, 3 * SR, b.y]),
        "encode": f("encode", lambda b: [lambda B, S: B, lambda B, S: S, 0, b.y]),
        "decode": f("decode", lambda b: [lambda B, S: B, lambda B, S: S, 0, b.y]),
        "flac_encode": f("flac_encode", lambda b: [lambda B, S: B, lambda B, S: S, SR, 4096, b.yb,
                                                   lambda B, S: _lib.load().vtts_flac_bound(max(S, 0), 4096), b.nb]),
    }


def limit_call(eng):
    L, h = eng.lib, eng.h

    def call(host, B, S, b, n):
        fn = L.vtts_limit_host if host else L.vtts_limit
        return fn(h, P(b.x), P(n), P(b.gain), B, S, SR, -1.0, 5.0, 50.0, P(b.y), P(b.r), *([] if host else [None]))
    return call


@pytest.fixture(scope="module")
def entries(eng):
    bank = torch.from_numpy(np.random.default_rng(1).standard_normal(BANK).astype(np.float32) * 0.1).cuda()
    e = one_shot(eng, bank)
    e["limit"] = limit_call(eng)
    e["_bank"] = bank
    return e


NAMES = ["compress", "deess", "eq", "limit", "loudness", "loudness_normalize", "loudness_normalize_limited", "bed_mix", "reverb",
         "watermark", "watermark_detect", "denoise", "pitch_shift", "voice_shift", "time_stretch", "resample", "encode", "decode",
         "flac_encode"]


def rows(host, lengths):
    a = np.array(lengths, np.int32)
    return a if host else torch.from_numpy(a).cuda()


def baseline(call, host):
    x = (np.random.default_rng(3).standard_normal(2 * S0) * 0.2).astype(np.float32)
    b = Bufs(host, 2, S0, x)
    if not host:
        b.codes.copy_(torch.from_numpy((x * 8000).astype(np.int16)).cuda())
    else:
        b.codes[:] = (x * 8000).astype(np.int16)
    n = rows(host, [S0, S0 - 100])
    return b, n


def run_ok(eng, call, host, B, S, b, n):
    _lib.check(eng.h, call(host, B, S, b, n))
    torch.cuda.synchronize()


@pytest.mark.parametrize("host", [False, True], ids=["device", "host"])
@pytest.mark.parametrize("name", NAMES)
def test_one_shot_shape_rules(eng, entries, name, host):
    call = entries[name]
    b, n = baseline(call, host)
    run_ok(eng, call, host, 2, S0, b, n)
    want = b.outputs()

    def still_same():
        b2, n2 = baseline(call, host)
        run_ok(eng, call, host, 2, S0, b2, n2)
        for u, v in zip(want, b2.outputs()):
            assert u.tobytes() == v.tobytes()

    z = Bufs(host, 1, 1)
    with pytest.raises(_lib.VttsError):
        _lib.check(eng.h, call(host, 0, 1, z, None))
    still_same()
    big = Bufs(host, BIG, 1)
    with pytest.raises(_lib.VttsError):
        _lib.check(eng.h, call(host, BIG, 1, big, None))
    del big
    still_same()
    e = Bufs(host, 1, 0)
    if name == "flac_encode":
        run_ok(eng, call, host, 1, 0, e, None)
    else:
        with pytest.raises(_lib.VttsError):
            _lib.check(eng.h, call(host, 1, 0, e, None))
    still_same()
    if host:
        for bad in (-1, S0 + 1):
            with pytest.raises(_lib.VttsError, match="outside"):
                _lib.check(eng.h, call(host, 1, S0, Bufs(host, 1, S0), np.array([bad], np.int32)))
            still_same()


def creates(eng, bank):
    """name -> (create(max_streams, chunk) -> (rc, handle), destroy, chunk limit, needs loaded weights)"""
    L, h = eng.lib, eng.h
    bias = np.full(NB, 1e-3, np.float32)
    ir = np.r_[np.float32(1.0), np.full(IR - 1, 0.01, np.float32)]
    sos = np.zeros(6, np.float64)
    K = C.c_int()
    L.vtts_eq_design(1, SR, 3000.0, 0.707, 6.0, 2, sos.ctypes.data, C.byref(K))
    offs = np.array([0], np.int64)
    lens = np.array([BANK], np.int32)
    p = C.c_int()
    p64 = C.c_int64()
    keep = (bias, ir, sos, offs, lens)   # host arrays the creates read, alive as long as the closures

    def mk(name, *args, pitch=True, wide=False):
        def create(S, F, keep=keep):
            out = C.c_void_p()
            extra = [C.byref(p64 if wide else p)] if pitch else []
            rc = getattr(L, f"vtts_{name}_stream_create")(h, S, F, *args, C.byref(out), *extra)
            return rc, out
        return create, getattr(L, f"vtts_{name}_stream_destroy")

    return {
        "resample": (*mk("resample", SR, 3 * SR), 1 << 22),
        "denoise": (*mk("denoise", 0.5, P(bias)), 1 << 22),
        "pitch_shift": (*mk("pitch_shift"), 1 << 22),
        "time_stretch": (*mk("time_stretch"), 1 << 22),
        "loudness": (*mk("loudness", SR, 60, pitch=False), 1 << 22),
        "limiter": (*mk("limiter", SR, -1.0, 5.0, 50.0), 1 << 22),
        "eq": (*mk("eq", P(sos), K.value, pitch=False), 1 << 22),
        "compressor": (*mk("compressor", SR, -30.0, 4.0, 6.0, 5.0, 50.0, 0.0, pitch=False), 1 << 22),
        "deesser": (*mk("deesser", SR, 5000.0, -30.0, 4.0, 6.0, 1.0, 50.0, 12.0, pitch=False), 1 << 22),
        "reverb": (*mk("reverb", SR, P(ir), IR, 0.3), 1 << 22),
        "bed": (*mk("bed", SR, P(bank), P(offs), P(lens), 1, 12.0, -40.0, 10.0, 200.0, 0, 0, 0, 0), 1 << 22),
        "watermark": (*mk("watermark", 7, 0.05), 1 << 22),
        "flac": (*mk("flac", SR, 4096, wide=True), 1 << 22),
        "vocoder": (*mk("vocoder", pitch=False), 4096),
        "acoustic": (*mk("acoustic", 64, 16, 0, 0, pitch=False), 4096),
    }


CREATES = ["resample", "denoise", "pitch_shift", "time_stretch", "loudness", "limiter", "eq", "compressor", "deesser", "reverb", "bed",
           "watermark", "flac", "vocoder", "acoustic"]


@pytest.mark.parametrize("name", CREATES)
def test_stream_create_dimension_rules(eng, entries, name):
    create, destroy, chunk_max = creates(eng, entries["_bank"])[name]
    call = entries["eq"]
    b, n = baseline(call, False)
    run_ok(eng, call, False, 2, S0, b, n)
    want = b.outputs()
    for S, F in ((0, 256), (BIG, 256), (4, 0), (4, chunk_max + 1)):
        rc, out = create(S, F)
        assert rc != 0 and not out.value
        assert "max_streams=" in _lib.load().vtts_last_error(eng.h).decode()
        b2, n2 = baseline(call, False)
        run_ok(eng, call, False, 2, S0, b2, n2)
        for u, v in zip(want, b2.outputs()):
            assert u.tobytes() == v.tobytes()
    if name not in ("vocoder", "acoustic"):   # the model streams need loaded weights
        rc, out = create(4, 256)
        _lib.check(eng.h, rc)
        _lib.check(eng.h, destroy(eng.h, out))
