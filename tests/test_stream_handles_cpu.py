"""CPU: what the Python stream handles hand to the library.  A recording fake `lib` stands in for libviettts_b200: every
pointer argument is resolved to the array or tensor it came from and copied at the call, so the tests see the bytes,
dtype and layout of each argument, and the fake writes outputs the handles must slice by n_out."""
import ctypes as C

import numpy as np
import pytest
import torch

from viettts_b200 import engine as E

S, F, PITCH, LOOK = 3, 20, 40, 3
# argument positions of the output and n_out of the host pushes that differ from (-2, -1)
HOST_OUT = {"vtts_loudness_stream_push_host": (-1, None), "vtts_limiter_stream_push_host": (-3, -2)}
# the BEGIN parameter of a push: keyword, value, what the slots [BEGIN, idle, BEGIN] of a fresh stream get
PARAMS = {"pitch": ("semitones", 2.0, [2.0, 0.0, 2.0]), "time_stretch": ("tempo", 1.5, [1.5, 1.0, 1.5]),
          "limiter": ("gain_db", 2.0, [2.0, 0.0, 2.0])}
KINDS = ["resample", "denoise", "pitch", "time_stretch", "loudness", "limiter", "eq", "vocoder"]


class FakeLib:
    def __init__(self):
        self.calls = []        # (name, [argument records])
        self.arrays = {}       # address -> array / tensor passed through engine._ptr

    def record(self, a):
        if a is not None:
            self.arrays[a.ctypes.data if isinstance(a, np.ndarray) else a.data_ptr()] = a
        return a

    def _arg(self, v):
        if isinstance(v, int) and v in self.arrays:
            a = self.arrays[v]
            if isinstance(a, np.ndarray):
                return {"dtype": a.dtype, "contig": a.flags.c_contiguous, "data": a.copy(), "obj": a}
            return {"dtype": a.dtype, "contig": a.is_contiguous(), "data": a.clone(), "obj": a}
        return v

    def __getattr__(self, name):
        def fn(*args):
            rec = [self._arg(a) for a in args]
            self.calls.append((name, rec))
            if name.endswith("_lookahead"):
                return LOOK
            if name.endswith("_create"):
                for a in args:
                    if type(a).__name__ == "CArgObject":
                        o = a._obj
                        o.value = 0x1234 if isinstance(o, C.c_void_p) else PITCH
            if name.endswith("_push_host"):
                # inputs n_new at args[3]; the output and n_out at HOST_OUT's positions
                n = rec[3]["data"]
                o, no = HOST_OUT.get(name, (-2, -1))
                out = rec[o]["obj"]
                out[...] = np.arange(out.size, dtype=np.float32).reshape(out.shape)
                if no is not None:
                    rec[no]["obj"][...] = np.minimum(n, 2)
                if name == "vtts_limiter_stream_push_host":
                    rec[-1]["obj"][...] = -np.arange(S, dtype=np.float32)
            return 0
        return fn

    def named(self, name):
        return [r for n, r in self.calls if n == name]


@pytest.fixture
def eng(monkeypatch):
    lib = FakeLib()
    monkeypatch.setattr(E, "_ptr", lambda a: None if lib.record(a) is None else (a.ctypes.data if isinstance(a, np.ndarray)
                                                                                  else a.data_ptr()))
    e = E.Engine.__new__(E.Engine)
    e.lib, e.h, e.device = lib, C.c_void_p(99), 0
    return e


def _streams(eng):
    bias = np.ones(E.DENOISE_BINS, np.float32)
    return {
        "resample": (E.ResampleStream(eng, S, F, 48000), "vtts_resample_stream_push", PITCH),
        "denoise": (E.DenoiseStream(eng, S, F, 1.0, bias=bias), "vtts_denoise_stream_push", PITCH),
        "pitch": (E.PitchShiftStream(eng, S, F), "vtts_pitch_shift_stream_push", PITCH),
        "time_stretch": (E.TimeStretchStream(eng, S, F), "vtts_time_stretch_stream_push", PITCH),
        "loudness": (E.LoudnessMeter(eng, S, F), "vtts_loudness_stream_push", 4),
        "limiter": (E.LimiterStream(eng, S, F), "vtts_limiter_stream_push", PITCH),
        "eq": (E.EqStream(eng, S, F, [[1.0, 0.5, 0.0, 1.0, -0.25, 0.0]]), "vtts_eq_stream_push", F),
        "vocoder": (E.VocoderStream(eng, S, F), "vtts_vocoder_stream_push", 256 * (F + LOOK)),
    }


@pytest.mark.parametrize("kind", KINDS)
def test_host_push_marshalling(eng, kind):
    st, name, width = _streams(eng)[kind]
    row = (80,) if kind == "vocoder" else ()
    x = np.arange(S * 7 * int(np.prod(row)), dtype=np.float64).reshape((S, 7) + row)   # short chunk, wrong dtype
    extra = {PARAMS[kind][0]: PARAMS[kind][1]} if kind in PARAMS else {}
    res = st.push(x, [7, 0, 5], begin=[True, False, True], end=[False, False, True], **extra)
    (rec,) = eng.lib.named(name + "_host")
    xr, nr, fr = rec[2], rec[3], rec[4]
    assert xr["dtype"] == np.float32 and xr["contig"] and xr["data"].shape == (S, F) + row
    assert np.array_equal(xr["data"][:, :7], x.astype(np.float32)) and not xr["data"][:, 7:].any()
    assert nr["dtype"] == np.int32 and nr["contig"] and list(nr["data"]) == [7, 0, 5]
    assert fr["dtype"] == np.uint8 and fr["contig"] and list(fr["data"]) == [1, 0, 3]
    if kind in PARAMS:
        assert rec[5]["dtype"] == np.float32 and rec[5]["contig"] and list(rec[5]["data"]) == PARAMS[kind][2]
    if kind == "loudness":
        assert res.shape == (S, 4) and res.dtype == np.float32
        return
    if kind == "limiter":
        assert rec[-1]["dtype"] == np.float32 and rec[-1]["data"].shape == (S,)
        assert np.array_equal(st.reduction_db, -np.arange(S, dtype=np.float32))
    out = rec[HOST_OUT.get(name + "_host", (-2, -1))[0]]["obj"]
    assert out.dtype == np.float32 and out.shape == (S, width)
    scale = 256 if kind == "vocoder" else 1
    for s, n in enumerate([2, 0, 2]):
        assert np.array_equal(res[s], out[s, : n * scale])


def test_pitch_shift_carry(eng):
    st = E.PitchShiftStream(eng, S, F)
    x = np.zeros((S, F), np.float32)
    st.push(x, [1, 1, 0], begin=[True, True, False], semitones=[3.0, -2.0, 5.0])
    st.push(x, [1, 1, 1], begin=[False, False, True], semitones=7.0)
    st.push(x, [1, 0, 0], begin=[True, False, False], semitones=[-1.0, 9.0, 9.0])
    sems = [list(r[5]["data"]) for r in eng.lib.named("vtts_pitch_shift_stream_push_host")]
    assert sems == [[3.0, -2.0, 0.0], [3.0, -2.0, 7.0], [-1.0, -2.0, 7.0]]
    assert list(st.shift) == [-1.0, -2.0, 7.0]
    with pytest.raises(ValueError):
        st.push(x, [1, 0, 0], begin=[True, False, False])


def test_time_stretch_carry(eng):
    st = E.TimeStretchStream(eng, S, F)
    x = np.zeros((S, F), np.float32)
    st.push(x, [1, 1, 0], begin=[True, True, False], tempo=[1.5, 0.75, 2.0])
    st.push(x, [1, 1, 1], begin=[False, False, True], tempo=0.5)
    st.push(x, [1, 0, 0], begin=[True, False, False], tempo=[1.25, 9.0, 9.0])
    tps = [list(r[5]["data"]) for r in eng.lib.named("vtts_time_stretch_stream_push_host")]
    assert tps == [[1.5, 0.75, 1.0], [1.5, 0.75, 0.5], [1.25, 0.75, 0.5]]
    assert list(st.tempo) == [1.25, 0.75, 0.5]
    with pytest.raises(ValueError):
        st.push(x, [1, 0, 0], begin=[True, False, False])


def test_limiter_gain_carry(eng):
    st = E.LimiterStream(eng, S, F)
    x = np.zeros((S, F), np.float32)
    st.push(x, [1, 1, 0], begin=[True, True, False], gain_db=[3.0, -2.0, 5.0])
    st.push(x, [1, 1, 1], begin=[False, False, True])                             # 0 dB when left out
    st.push(x, [1, 0, 0], begin=[True, False, False], gain_db=[6.0, 99.0, 99.0])    # values of other slots are not read
    gains = [list(r[5]["data"]) for r in eng.lib.named("vtts_limiter_stream_push_host")]
    assert gains == [[3.0, -2.0, 0.0], [3.0, -2.0, 0.0], [6.0, -2.0, 0.0]]
    assert list(st.gain_db) == [6.0, -2.0, 0.0]
    n = len(eng.lib.calls)
    with pytest.raises(ValueError, match=r"got 71\.0$"):                 # the value given, not the carried array
        st.push(x, [1, 0, 0], begin=[True, False, False], gain_db=71.0)
    assert len(eng.lib.calls) == n and list(st.gain_db) == [6.0, -2.0, 0.0]


@pytest.mark.parametrize("kind", KINDS)
def test_device_push_marshalling(eng, kind):
    st, name, width = _streams(eng)[kind]
    row = (80,) if kind == "vocoder" else ()
    x_t = torch.zeros((S, F) + row)
    out_t = torch.zeros((S, width))
    extra = {PARAMS[kind][0]: PARAMS[kind][1]} if kind in PARAMS else {}
    red_t = torch.zeros(S)
    if kind == "limiter":
        extra["reduction_t"] = red_t
    st.push_device(x_t, [1, 2, 3], np.array([1, 0, 2]), out_t, stream=77, **extra)
    (rec,) = eng.lib.named(name)
    assert rec[2]["obj"] is x_t and rec[{"loudness": -2, "limiter": -4}.get(kind, -3)]["obj"] is out_t
    if kind in PARAMS:
        assert rec[5]["dtype"] == np.float32 and list(rec[5]["data"]) == [PARAMS[kind][1]] + 2 * [PARAMS[kind][2][1]]
    if kind == "limiter":
        assert rec[-2]["obj"] is red_t
        with pytest.raises(ValueError):
            st.push_device(x_t, [1, 2, 3], [0, 0, 0], out_t, reduction_t=torch.zeros(S + 1), stream=77)
        with pytest.raises(ValueError):                                 # a host buffer would be written on the device
            st.push_device(x_t, [1, 2, 3], [0, 0, 0], out_t, None, stream=77)
        with pytest.raises(TypeError):
            st.push_device(x_t, [1, 2, 3], [0, 0, 0], out_t, stream=77)
        assert len(eng.lib.named(name)) == 1
    assert rec[3]["dtype"] == np.int32 and list(rec[3]["data"]) == [1, 2, 3]
    assert rec[4]["dtype"] == np.uint8 and list(rec[4]["data"]) == [1, 0, 2]
    assert rec[-1] == 77
    with pytest.raises(ValueError):
        st.push_device(torch.zeros((S, F + 1) + row), [1, 2, 3], [0, 0, 0], out_t, stream=77, **extra)
    with pytest.raises(ValueError):
        st.push_device(x_t, [1, 2, 3], [0, 0, 0], torch.zeros((S, width), dtype=torch.float64), stream=77, **extra)
    with pytest.raises(ValueError):
        st.push(np.zeros((S, F + 1) + row, np.float32), [1, 2, 3])


@pytest.mark.parametrize("kind", KINDS + ["acoustic"])
def test_close_twice(eng, kind):
    if kind == "acoustic":
        st, name = E.AcousticStream(eng, S, F, 100, 50), "vtts_acoustic_stream_destroy"
    else:
        st, push, _ = _streams(eng)[kind]
        name = push.replace("_push", "_destroy")
    with st:
        pass
    st.close()
    assert len(eng.lib.named(name)) == 1


# ---- the audio chain after the vocoder -----------------------------------------------------------------------------

class RecordingEngine:
    """stands in for Engine in the one-shot chain: records each call and hands the audio through"""
    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        def call(w, *args, **kw):
            self.calls.append(name)
            return (w, 0.0) if name in ("limit", "normalize_loudness") else w
        return call


ONE_SHOT = {E.DenoiseStream: "denoise", E.PitchShiftStream: "pitch_shift", E.TimeStretchStream: "time_stretch",
            E.ResampleStream: "resample", E.EqStream: "equalize", E.LimiterStream: "limit"}


def test_chain_order_is_shared(eng, monkeypatch):
    """the one-shot chain (the CLI's) calls the stages the stream chain (TtsStream's) opens, in the same order"""
    monkeypatch.setattr(eng, "_bias_arg", lambda bias: np.ones(E.DENOISE_BINS, np.float32))
    sos = [[1.0, 0.5, 0.0, 1.0, -0.25, 0.0]]
    chain = E.AudioChain(denoise=0.5, semitones=2.0, tempo=1.25, output_rate=48000, eq=sos, limit=-2.0, gain_db=3.0, meter=True)
    rec = RecordingEngine()
    chain.run(rec, np.zeros(100, np.float32))
    opened = list(chain.streams(eng, S, 256 * F, 100))
    assert [name for name, _ in opened] == ["dn", "ps", "ts", "rs", "eq", "lm", "mt"]
    assert [ONE_SHOT[type(st)] for _, st in opened if type(st) in ONE_SHOT] == rec.calls
    assert rec.calls == ["denoise", "pitch_shift", "time_stretch", "resample", "equalize", "limit"]
    assert [st.max_chunk_samples for _, st in opened] == [256 * F] + [PITCH] * 6   # each takes the previous width
    assert opened[5][1].rate == opened[6][1].rate == 48000 and opened[5][1].ceiling == -2.0

    loud = E.AudioChain(output_rate=48000, loudness=-16.0, true_peak=-1.5)
    rec = RecordingEngine()
    loud.run(rec, np.zeros(100, np.float32))
    assert rec.calls == ["resample", "normalize_loudness"]
    with pytest.raises(ValueError, match="no streaming form"):
        list(loud.streams(eng, S, 256 * F, 100))


@pytest.mark.parametrize("argv, calls", [
    (["--denoise", "0.5", "--pitch", "2", "--tempo", "1.25", "--output-rate", "48000", "--eq", "hp:100", "--limiter"],
     ["denoise", "pitch_shift", "time_stretch", "resample", "equalize", "limit"]),
    (["--eq", "hp:100", "--loudness", "-16", "--limiter"], ["equalize", "normalize_loudness"]),
    ([], []),
])
def test_cli_runs_the_chain(monkeypatch, tmp_path, argv, calls):
    from viettts_b200 import synthesizer
    from viettts_b200.hifigan import mel2wave
    from viettts_b200.nat import text2mel
    rec = RecordingEngine()
    monkeypatch.setattr(E, "get_engine", lambda device=None: rec)
    monkeypatch.setattr(text2mel, "text2mel", lambda *a, **k: np.zeros((1, 4, 80), np.float32))
    monkeypatch.setattr(mel2wave, "mel2wave", lambda mel: np.zeros((1, 1024), np.float32))
    assert synthesizer.main(["--text", "xin chào", "--output", str(tmp_path / "o.wav"), *argv]) == 0
    assert rec.calls == calls


def test_push_signatures():
    """the handles keep their push arguments: names, order and the BEGIN parameter's place"""
    import inspect
    base_h, base_d = ["x", "n_new", "begin", "end"], ["x_t", "n_new", "flags", "out_t"]
    want = {E.VocoderStream: (["mel", "n_new", "begin", "end"], ["mel_t", "n_new", "flags", "out_t", "stream"]),
            E.PitchShiftStream: (base_h + ["semitones"], base_d + ["semitones", "stream"]),
            E.TimeStretchStream: (base_h + ["tempo"], base_d + ["tempo", "stream"]),
            E.LimiterStream: (base_h + ["gain_db"], base_d + ["reduction_t", "gain_db", "stream"])}
    for cls in (E.ResampleStream, E.DenoiseStream, E.LoudnessMeter, E.EqStream):
        want[cls] = (base_h, base_d + ["stream"])
    for cls, (h, d) in want.items():
        assert list(inspect.signature(cls.push).parameters)[1:] == h, cls
        assert list(inspect.signature(cls.push_device).parameters)[1:] == d, cls


@pytest.mark.parametrize("argv, flag", [(["--pitch", "13"], "--pitch"), (["--tempo", "3"], "--tempo"), (["--denoise", "-1"], "--denoise"),
                                        (["--output-rate", "16001"], "--output-rate"), (["--eq", "wobble"], "--eq"),
                                        (["--limiter", "--true-peak", "-30"], "--limiter"), (["--loudness", "-80"], "--loudness")])
def test_cli_errors_name_the_flag(capsys, argv, flag):
    from viettts_b200 import synthesizer
    with pytest.raises(SystemExit):
        synthesizer.main(["--text", "xin chào", *argv])
    assert f"error: {flag}: " in capsys.readouterr().err
