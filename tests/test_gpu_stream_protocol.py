"""GPU: the slot protocol every per-slot stream shares (resample, denoise, pitch shift, time stretch, loudness, limiter,
equalizer, vocoder), called through the C ABI on device buffers, and the error paths of the host-buffer entry points.

A rejected push names the entry point and the first bad slot, launches nothing and leaves the stream as it was: the
valid pushes around it produce the bits of a stream that never saw it."""
import ctypes as C

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
S = 2


@pytest.fixture(scope="module")
def eng(hifigan_params):
    from viettts_b200.engine import Engine
    e = Engine(0)
    e.load_hifigan(hifigan_params)
    yield e
    e.close()


def _p(t):
    return None if t is None else C.c_void_p(t.data_ptr())


# each opener returns the stream, its device push entry point, the input shape [S, F(, 80)] and the output shape
def _resample(eng):
    st = eng.open_resample_stream(S, 64, 48000)
    return st, "resample_stream_push", (S, 64), (S, st.out_pitch)


def _denoise(eng):
    st = eng.open_denoise_stream(S, 512, 1.0)
    return st, "denoise_stream_push", (S, 512), (S, st.out_pitch)


def _pitch(eng):
    st = eng.open_pitch_shift_stream(S, 512)
    return st, "pitch_shift_stream_push", (S, 512), (S, st.out_pitch)


def _time_stretch(eng):
    st = eng.open_time_stretch_stream(S, 512)
    return st, "time_stretch_stream_push", (S, 512), (S, st.out_pitch)


def _loudness(eng):
    st = eng.open_loudness_meter(S, 1600)
    return st, "loudness_stream_push", (S, 1600), (S, 4)


def _limiter(eng):
    st = eng.open_limiter_stream(S, 64)
    return st, "limiter_stream_push", (S, 64), (S, st.out_pitch)


def _eq(eng):
    st = eng.open_eq_stream(S, 64, "hp:100,pk:1000:1:3")
    return st, "eq_stream_push", (S, 64), (S, st.out_pitch)


def _vocoder(eng):
    st = eng.open_vocoder_stream(S, 8)
    return st, "vocoder_stream_push", (S, 8, 80), (S, st.wav_ld)


STREAMS = {"resample": _resample, "denoise": _denoise, "pitch": _pitch, "time_stretch": _time_stretch, "loudness": _loudness,
           "limiter": _limiter, "eq": _eq, "vocoder": _vocoder}


def _push(eng, name, st, ctx, x, n_new, flags, y, n_out):
    """the raw device push; returns (rc, the context's last error)"""
    lib, s = eng.lib, torch.cuda.current_stream().cuda_stream
    n = None if n_new is None else np.ascontiguousarray(n_new, np.int32)
    f = None if flags is None else np.ascontiguousarray(flags, np.uint8)
    ptr = lambda a: None if a is None else a.ctypes.data
    no = None if n_out is None else n_out.ctypes.data
    if name in ("pitch_shift_stream_push", "time_stretch_stream_push"):
        par = np.full(S, 3.0 if name == "pitch_shift_stream_push" else 1.5, np.float32)   # semitones / tempo
        rc = getattr(lib, "vtts_" + name)(ctx, st.h, _p(x), ptr(n), ptr(f), par.ctypes.data, _p(y), no, s)
    elif name == "limiter_stream_push":
        gain, red = np.full(S, 6.0, np.float32), torch.zeros(S, device="cuda")
        rc = lib.vtts_limiter_stream_push(ctx, st.h, _p(x), ptr(n), ptr(f), gain.ctypes.data, _p(y), no, _p(red), s)
    elif name == "loudness_stream_push":
        rc = lib.vtts_loudness_stream_push(ctx, st.h, _p(x), ptr(n), ptr(f), _p(y), s)
    else:
        rc = getattr(lib, "vtts_" + name)(ctx, st.h, _p(x), ptr(n), ptr(f), _p(y), no, s)
    msg = lib.vtts_last_error(ctx)
    return rc, msg.decode() if msg else ""


def _valid_run(eng, name, st, x_shape, y_shape, rejects=()):
    """two valid pushes (BEGIN on both slots, then END), each preceded by the rejected pushes `rejects`"""
    F = x_shape[1]
    rng = np.random.default_rng(7)
    outs = []
    for flags in ([1, 1], [2, 2]):
        for bad in rejects:
            bad()
        x = torch.from_numpy((rng.standard_normal(x_shape) * 0.1).astype(np.float32)).cuda()
        y = torch.zeros(y_shape, device="cuda")
        n_out = np.zeros(S, np.int32)
        rc, msg = _push(eng, name, st, eng.h, x, [F, F // 2], flags, y, n_out)
        assert rc == 0, msg
        torch.cuda.synchronize()
        outs.append((y.cpu().numpy(), n_out.copy()))
    return outs


@pytest.mark.parametrize("kind", list(STREAMS))
def test_rejections(eng, kind):
    from viettts_b200.engine import Engine
    st, name, x_shape, y_shape = STREAMS[kind](eng)
    ref_st, *_ = STREAMS[kind](eng)
    F = x_shape[1]
    x = torch.zeros(x_shape, device="cuda")
    y = torch.zeros(y_shape, device="cuda")
    n_out = np.zeros(S, np.int32)
    other = Engine(0)
    cases = [
        (eng.h, x, [0, F + 1], [1, 1], f"{name}: n_new[1]={F + 1} outside [0, {F}]"),
        (eng.h, x, [-1, 0], [1, 1], f"{name}: n_new[0]=-1 outside [0, {F}]"),
        (eng.h, x, [1, 1], [1, 4], f"{name}: flags[1]=4 (bit0 BEGIN, bit1 END)"),
        (eng.h, x, [0, 3], [0, 0], f"{name}: slot 1 is not open (push BEGIN first, also after END)"),
        (eng.h, None, [1, 1], [1, 1], f"{name}: null pointer"),
        (eng.h, x, None, [1, 1], f"{name}: null pointer"),
        (other.h, x, [1, 1], [1, 1], f"{name}: the stream belongs to another context"),
    ]

    def reject(case):
        ctx, xx, n, f, want = case
        before = eng.launch_count()
        rc, msg = _push(eng, name, st, ctx, xx, n, f, y, n_out)
        assert rc == -1 and msg == want
        assert eng.launch_count() == before

    try:
        for case in cases:
            reject(case)
        got = _valid_run(eng, name, st, x_shape, y_shape, rejects=[lambda c=c: reject(c) for c in cases[:3]])
        want = _valid_run(eng, name, ref_st, x_shape, y_shape)
        for (yg, ng), (yw, nw) in zip(got, want):
            assert np.array_equal(ng, nw)
            assert np.array_equal(yg, yw)
        # after END the slots are closed again
        rc, msg = _push(eng, name, st, eng.h, x, [1, 0], [0, 0], y, n_out)
        assert rc == -1 and msg == f"{name}: slot 0 is not open (push BEGIN first, also after END)"
    finally:
        st.close()
        ref_st.close()
        other.close()


def test_host_calls_before_load(eng, hifigan_params):
    """a host call that fails in its device stage leaves the context ready for the next call"""
    from viettts_b200.engine import Engine
    mel = (np.random.default_rng(3).standard_normal((2, 24, 80)) * 0.5 - 4.0).astype(np.float32)
    B, T, _ = mel.shape
    wav = np.empty((B, T * 256), np.float32)
    e = Engine(0)
    try:
        assert e.lib.vtts_mel2wave_host(e.h, mel.ctypes.data, None, B, T, wav.ctypes.data) != 0
        assert b"not loaded" in e.lib.vtts_last_error(e.h)
        e.load_hifigan(hifigan_params)
        assert np.array_equal(e.mel2wave(mel), eng.mel2wave(mel))

        x = (np.random.default_rng(4).standard_normal((2, 4096)) * 0.1).astype(np.float32)
        mel_out = np.empty((2, 16, 80), np.float32)
        assert e.lib.vtts_melspec_host(e.h, x.ctypes.data, 2, 4096, mel_out.ctypes.data) != 0
        assert b"not loaded" in e.lib.vtts_last_error(e.h)
        assert np.array_equal(e.melspec(x), eng.melspec(x))
    finally:
        e.close()


def test_stream_checks_keep_their_place(eng):
    """a stream's own checks run in the slot loop: a bad slot 0 is reported before a bad n_new of slot 1"""
    x = torch.zeros((S, 512), device="cuda")
    y = torch.zeros((S, 4096), device="cuda")
    n, f, n_out = np.array([1, 513], np.int32), np.array([1, 1], np.uint8), np.zeros(S, np.int32)
    st = torch.cuda.current_stream().cuda_stream
    with eng.open_pitch_shift_stream(S, 512) as ps:
        sem = np.array([20.0, 0.0], np.float32)
        rc = eng.lib.vtts_pitch_shift_stream_push(eng.h, ps.h, _p(x), n.ctypes.data, f.ctypes.data, sem.ctypes.data, _p(y),
                                                  n_out.ctypes.data, st)
        assert rc == -1 and eng.lib.vtts_last_error(eng.h).decode() == \
            "pitch_shift_stream_push: semitones[0] = 20 (finite, in [-12, 12])"
    with eng.open_loudness_meter(S, 17600, max_seconds=1) as lm:
        xl = torch.zeros((S, 17600), device="cuda")
        nl = np.array([17600, 17601], np.int32)
        rc = eng.lib.vtts_loudness_stream_push(eng.h, lm.h, _p(xl), nl.ctypes.data, f.ctypes.data, _p(y[:, :4].contiguous()), st)
        assert rc == -1 and eng.lib.vtts_last_error(eng.h).decode() == \
            "loudness_stream_push: slot 0 would hold 17600 samples, more than max_seconds (10 sub-blocks)"
    with eng.open_vocoder_stream(S, 8) as vs:
        eng.set_precision("fp32")
        try:
            xm, yv = torch.zeros((S, 8, 80), device="cuda"), torch.zeros((S, vs.wav_ld), device="cuda")
            nv = np.array([1, 9], np.int32)
            rc = eng.lib.vtts_vocoder_stream_push(eng.h, vs.h, _p(xm), nv.ctypes.data, f.ctypes.data, _p(yv), n_out.ctypes.data, st)
            assert rc == -1 and eng.lib.vtts_last_error(eng.h).decode() == \
                "vocoder_stream_push: the strict fp32 mode has no streaming path; use bf16x3 or fp16"
        finally:
            eng.set_precision("bf16x3")
