"""CPU: what the Python stream handles hand to the library.  A recording fake `lib` stands in for libviettts_b200: every
pointer argument is resolved to the array or tensor it came from and copied at the call, so the tests see the bytes,
dtype and layout of each argument, and the fake writes outputs the handles must slice by n_out."""
import ctypes as C

import numpy as np
import pytest
import torch

from viettts_b200 import engine as E

S, F, PITCH, LOOK = 3, 20, 40, 3


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
                # inputs n_new at args[3]; n_out is the last argument, the output before it
                n = rec[3]["data"]
                out = rec[-2]["obj"] if name != "vtts_loudness_stream_push_host" else rec[-1]["obj"]
                out[...] = np.arange(out.size, dtype=np.float32).reshape(out.shape)
                if name != "vtts_loudness_stream_push_host":
                    rec[-1]["obj"][...] = np.minimum(n, 2)
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
        "loudness": (E.LoudnessMeter(eng, S, F), "vtts_loudness_stream_push", 4),
        "vocoder": (E.VocoderStream(eng, S, F), "vtts_vocoder_stream_push", 256 * (F + LOOK)),
    }


@pytest.mark.parametrize("kind", ["resample", "denoise", "pitch", "loudness", "vocoder"])
def test_host_push_marshalling(eng, kind):
    st, name, width = _streams(eng)[kind]
    row = (80,) if kind == "vocoder" else ()
    x = np.arange(S * 7 * int(np.prod(row)), dtype=np.float64).reshape((S, 7) + row)   # short chunk, wrong dtype
    extra = {"semitones": 2.0} if kind == "pitch" else {}
    res = st.push(x, [7, 0, 5], begin=[True, False, True], end=[False, False, True], **extra)
    (rec,) = eng.lib.named(name + "_host")
    xr, nr, fr = rec[2], rec[3], rec[4]
    assert xr["dtype"] == np.float32 and xr["contig"] and xr["data"].shape == (S, F) + row
    assert np.array_equal(xr["data"][:, :7], x.astype(np.float32)) and not xr["data"][:, 7:].any()
    assert nr["dtype"] == np.int32 and nr["contig"] and list(nr["data"]) == [7, 0, 5]
    assert fr["dtype"] == np.uint8 and fr["contig"] and list(fr["data"]) == [1, 0, 3]
    if kind == "pitch":
        assert rec[5]["dtype"] == np.float32 and list(rec[5]["data"]) == [2.0, 0.0, 2.0]
    if kind == "loudness":
        assert res.shape == (S, 4) and res.dtype == np.float32
        return
    out = rec[-2]["obj"]
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


@pytest.mark.parametrize("kind", ["resample", "denoise", "pitch", "loudness", "vocoder"])
def test_device_push_marshalling(eng, kind):
    st, name, width = _streams(eng)[kind]
    row = (80,) if kind == "vocoder" else ()
    x_t = torch.zeros((S, F) + row)
    out_t = torch.zeros((S, width))
    extra = {"semitones": 1.0} if kind == "pitch" else {}
    st.push_device(x_t, [1, 2, 3], np.array([1, 0, 2]), out_t, stream=77, **extra)
    (rec,) = eng.lib.named(name)
    assert rec[2]["obj"] is x_t and rec[-2 if kind == "loudness" else -3]["obj"] is out_t
    assert rec[3]["dtype"] == np.int32 and list(rec[3]["data"]) == [1, 2, 3]
    assert rec[4]["dtype"] == np.uint8 and list(rec[4]["data"]) == [1, 0, 2]
    assert rec[-1] == 77
    with pytest.raises(ValueError):
        st.push_device(torch.zeros((S, F + 1) + row), [1, 2, 3], [0, 0, 0], out_t, stream=77, **extra)
    with pytest.raises(ValueError):
        st.push_device(x_t, [1, 2, 3], [0, 0, 0], torch.zeros((S, width), dtype=torch.float64), stream=77, **extra)
    with pytest.raises(ValueError):
        st.push(np.zeros((S, F + 1) + row, np.float32), [1, 2, 3])


@pytest.mark.parametrize("kind", ["resample", "denoise", "pitch", "loudness", "vocoder", "acoustic"])
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
