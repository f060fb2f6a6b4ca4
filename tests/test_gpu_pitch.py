"""GPU: the pitch shifter (Engine.pitch_shift / pitch_shift_forward, vtts_pitch_shift*), its stream
(Engine.open_pitch_shift_stream) and the `semitones=` stage of the text-to-speech stream and the CLI's --pitch.

One-shot outputs are held to the float64 definition under the device's own discrete decisions (vtts_debug_pitch_decisions)
per element, |y - y64| <= TOL * error_scale (TOL from tests/test_pitch_cpu.py, over 4x an fp32 emulation of the kernels),
and the device's decisions may differ from float64's only where float64's margin is below DEC_MARGIN of the frame's norm.
Everything that streams, and every precision mode, batch position and repeat, is compared bit for bit with the one-shot
call."""
import json
import pickle

import numpy as np
import pytest
import torch

from oracle import denoise_oracle as do
from oracle import pitch_oracle as po
from test_denoise_cpu import signal_of
from test_pitch_cpu import DEC_MARGIN, TOL, decision_margins, voiced_of
from viettts_b200 import config, synthetic
from viettts_b200.engine import STREAM_BEGIN, STREAM_END

pytestmark = pytest.mark.gpu
KEY = np.array([7, 1234567], np.uint32)
RAGGED = [0, 1, 512, 513, 1023, 1025, 80128]
SHIFTS = [3.0, -5.0, 7.0, 12.0, -12.0, 2.5, -7.25]


@pytest.fixture(scope="module")
def eng():
    from viettts_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


def decisions(eng, x, sem, lens=None):
    dev = torch.device("cuda", 0)
    lt = None if lens is None else torch.from_numpy(np.asarray(lens, np.int32)).to(dev)
    return eng.debug_pitch_decisions(torch.from_numpy(np.ascontiguousarray(x, np.float32)).to(dev), sem, lt)


def check_decisions(dec, x, s, what):
    """the device's decisions differ from float64's only at comparisons whose float64 margin is below DEC_MARGIN"""
    dec64 = po.decisions_of(x, s)
    flag_m, branch_m = decision_margins(x, dec64)
    f_dev, f64 = (dec & 1) == 1, (dec64 & 1) == 1
    flips = f_dev != f64
    assert np.all(flag_m[flips] < DEC_MARGIN), (what, float(flag_m[flips].max()))
    both = f_dev & f64
    side = both & ((dec >> 1 & 1) != (dec64 >> 1 & 1))
    assert np.all(branch_m[side] < DEC_MARGIN), (what, float(branch_m[side].max()))


def check_row(y, x, n, s, dec, what=""):
    """y: the full output row of an input row x of which n samples are valid; dec: the device's decisions of the row"""
    if n <= do.PAD or s == 0:
        assert np.array_equal(y[:n].view(np.uint32), x[:n].view(np.uint32)), what     # a bit copy
        assert not dec.any(), what
    else:
        F = do.n_frames(n)
        assert not dec[F:].any(), what
        check_decisions(dec[:F], x[:n], s, what)
        y64 = po.pitch_shift(x[:n], s, decisions=dec[:F])
        ratio = np.abs(y[:n].astype(np.float64) - y64) / po.error_scale(x[:n], s)
        assert np.all(ratio <= TOL), (what, float(ratio.max()), int(ratio.argmax()))
    assert np.all(y[n:] == 0), what


def ragged_batch():
    S = max(RAGGED)
    lens = np.array(RAGGED, np.int32)
    x = np.stack([(voiced_of if b % 2 else signal_of)(S, 40 + b) for b in range(lens.size)])
    for b, n in enumerate(lens):
        x[b, n:] = np.nan                             # past a row's length: never read
    return x, lens


def test_one_shot_ragged_batch_against_float64(eng):
    x, lens = ragged_batch()
    sem = np.array(SHIFTS, np.float32)
    y = eng.pitch_shift(x, sem, lengths=lens)
    assert y.shape == x.shape
    dec = decisions(eng, x, sem, lens)
    assert dec.shape == (len(lens), do.n_frames(x.shape[1]), do.N_BINS)
    for b, n in enumerate(lens):
        check_row(y[b], x[b], int(n), float(sem[b]), dec[b], (b, n, sem[b]))
    # the device entry point computes the same bits
    dev = torch.device("cuda", 0)
    yt = eng.pitch_shift_forward(torch.from_numpy(x).to(dev), sem, lengths_t=torch.from_numpy(lens).to(dev))
    assert np.array_equal(yt.cpu().numpy(), y)


def test_three_minute_row(eng):
    n = 3 * 60 * 16000 + 77
    x = voiced_of(n, 11)
    y = eng.pitch_shift(x, -4.0)
    check_row(y, x, n, -4.0, decisions(eng, x[None], -4.0)[0], "3 min")


def test_same_bits_in_every_mode_alone_in_a_batch_and_repeated(eng):
    S = 20000
    lens = np.array([S, 7000, 513, 300], np.int32)
    sem = np.array([5.0, -3.0, 12.0, 4.0], np.float32)
    x = np.stack([voiced_of(S, 60 + b) for b in range(lens.size)])
    ys = []
    for mode in ("fp32", "bf16x3", "fp16"):
        eng.set_precision(mode)
        ys.append(eng.pitch_shift(x, sem, lengths=lens))
        ys.append(eng.pitch_shift(x, sem, lengths=lens))
    eng.set_precision("bf16x3")
    for y in ys[1:]:
        assert np.array_equal(y, ys[0])
    for b, n in enumerate(lens):
        alone = eng.pitch_shift(x[b, :n], float(sem[b]))
        assert np.array_equal(alone, ys[0][b, :n]), b


def test_zero_shift_is_the_input(eng):
    x = voiced_of(9000, 3)
    assert np.array_equal(eng.pitch_shift(x, 0.0), x)
    y = eng.pitch_shift(np.stack([x, x]), [0.0, 2.0])
    assert np.array_equal(y[0], x) and not np.array_equal(y[1], x)


# ---- stream ------------------------------------------------------------------------------------------------------

def push_plans(kind, F, rng):
    """utterances of one slot, each a list of push sizes (END with the last one)"""
    if kind == "ones":
        return [[1] * int(rng.integers(1100, 1500))]
    if kind in (255, 256, 1000):
        return [[min(kind, F)] * int(rng.integers(4, 12))]
    if kind == "max":
        return [[F] * int(rng.integers(2, 5)) + [int(rng.integers(1, F))]]
    if kind == "end_empty":
        return [[int(v) for v in rng.integers(1, F + 1, size=4)] + [0]]
    if kind == "short":
        return [[int(rng.integers(1, 200)), int(rng.integers(0, 200))], [512], [513]]
    if kind == "reuse":
        return [[int(v) for v in rng.integers(1, F + 1, size=3)], [int(v) for v in rng.integers(1, F + 1, size=5)]]
    if kind == "late":
        return [[0] * int(rng.integers(2, 6))] + [[int(v) for v in rng.integers(1, F + 1, size=6)]]
    return []    # idle


KINDS = ["ones", 255, 256, 1000, "max", "end_empty", "short", "reuse", "late", "idle"]
STREAM_SHIFTS = [3.0, -5.0, 0.0, 12.0, -12.0, 7.5, -1.0]


def run_stream(eng, S, F, kinds, seed):
    """each slot runs its plan (a slot's "late" plan starts it some pushes after the others), every utterance with its
    own shift; the concatenated outputs must equal the one-shot call and each push must issue five launches"""
    rng = np.random.default_rng(seed)
    dev = torch.device("cuda", 0)
    plans = []
    for k in kinds:
        flat = []
        for u, sizes in enumerate(push_plans(k, F, rng)):
            if k == "late" and u == 0:
                flat += [(0, 0, None)] * len(sizes)                     # idle pushes before the slot begins
                continue
            for q, n in enumerate(sizes):
                flat.append((n, (STREAM_BEGIN if q == 0 else 0) | (STREAM_END if q == len(sizes) - 1 else 0), u))
        plans.append(flat)
    data = [dict() for _ in range(S)]
    got = [dict() for _ in range(S)]
    shift = [dict() for _ in range(S)]
    P = np.zeros(S, np.int64)
    E = np.zeros(S, np.int64)
    with eng.open_pitch_shift_stream(S, F) as ps:
        assert ps.lookahead == do.LOOKAHEAD
        xt = torch.zeros((S, F), device=dev)
        yt = torch.empty((S, ps.out_pitch), device=dev)
        for c in range(max(len(p) for p in plans)):
            n_new = np.zeros(S, np.int32)
            flags = np.zeros(S, np.uint8)
            sem = np.full(S, np.nan, np.float32)                       # read only for the slots that begin
            x = np.full((S, F), np.nan, np.float32)                    # past n_new: never read
            for s in range(S):
                if c >= len(plans[s]) or plans[s][c][2] is None:
                    continue
                n, f, u = plans[s][c]
                n_new[s], flags[s] = n, f
                chunk = voiced_of(max(n, 1), 1000 * s + 10 * c + u)[:n]
                x[s, :n] = chunk
                if f & STREAM_BEGIN:
                    data[s][u], got[s][u] = [], []
                    shift[s][u] = sem[s] = STREAM_SHIFTS[int(rng.integers(len(STREAM_SHIFTS)))]
                    P[s] = E[s] = 0
                data[s][u].append(chunk)
            xt.copy_(torch.from_numpy(x))
            yt.fill_(12345.0)
            before = eng.launch_count()
            n_out = ps.push_device(xt, n_new, flags, yt, semitones=sem)
            assert eng.launch_count() - before == 5
            y = yt.cpu().numpy()
            for s in range(S):
                if n_new[s] == 0 and flags[s] == 0:
                    assert n_out[s] == 0 and np.all(y[s] == 12345.0), (s, c)     # idle: untouched
                    continue
                P[s] += n_new[s]
                e = int(P[s]) if flags[s] & STREAM_END else po.emitted_closed_form(int(P[s]))
                assert n_out[s] == e - E[s], (kinds[s], s, c, int(P[s]), int(n_out[s]), e - E[s])
                E[s] = e
                got[s][plans[s][c][2]].append(y[s, : n_out[s]].copy())
    for s in range(S):
        for u, chunks in data[s].items():
            xs = np.concatenate(chunks)
            out = np.concatenate(got[s][u])
            ref = eng.pitch_shift(xs, shift[s][u])
            assert out.shape == ref.shape and np.array_equal(out, ref), (kinds[s], s, u, xs.size, shift[s][u])
            if shift[s][u] == 0:
                assert np.array_equal(out, xs)


@pytest.mark.parametrize("S", [1, 3, 32])
def test_stream_equals_one_shot(eng, S):
    F = 1000
    kinds = ["max"] if S == 1 else [KINDS[(s + S) % len(KINDS)] for s in range(S)]
    run_stream(eng, S, F, kinds, seed=S)


def test_stream_one_sample_pushes_and_edges(eng):
    run_stream(eng, 4, 1024, ["ones", 255, 256, "short"], seed=99)


def test_stream_large_chunks(eng):
    run_stream(eng, 2, 48000, ["max", "reuse"], seed=7)


def test_stream_host_push_equals_device_push(eng):
    F = 700
    x = voiced_of(5000, 4)
    with eng.open_pitch_shift_stream(2, F) as ps:
        out = [[], []]
        for p0 in range(0, 5000, F):
            n = min(F, 5000 - p0)
            ys = ps.push(np.stack([x[p0: p0 + n], -x[p0: p0 + n]]), [n, n], begin=[p0 == 0] * 2, end=[p0 + n == 5000] * 2,
                         semitones=[4.0, -6.0])
            for s in range(2):
                out[s].append(ys[s])
    ref = eng.pitch_shift(np.stack([x, -x]), [4.0, -6.0])
    for s in range(2):
        assert np.array_equal(np.concatenate(out[s]), ref[s])


def test_launches_are_fixed(eng):
    with eng.open_pitch_shift_stream(4, 512) as ps:
        counts = []
        for n_new, flags in (([0, 0, 0, 0], [0, 0, 0, 0]), ([512, 1, 0, 7], [1, 1, 0, 3]), ([512, 0, 0, 0], [0, 2, 0, 0]),
                             ([0, 0, 0, 0], [0, 0, 0, 0])):
            before = eng.launch_count()
            ps.push(np.zeros((4, 512), np.float32), n_new, begin=np.array(flags) & 1, end=np.array(flags) & 2, semitones=3.0)
            counts.append(eng.launch_count() - before)
    assert counts == [5, 5, 5, 5]
    before = eng.launch_count()
    eng.pitch_shift(np.zeros((3, 1000), np.float32), 2.0)
    assert eng.launch_count() - before == 4


def test_argument_errors(eng):
    from viettts_b200._lib import VttsError
    x = voiced_of(2000, 1)
    y = np.zeros_like(x)
    for bad in (float("nan"), float("inf"), 13.0, -13.0, 12.001):
        with pytest.raises(ValueError):
            eng.pitch_shift(x, bad)
        # the library checks too, before anything is launched
        c0 = eng.launch_count()
        sem = np.array([bad], np.float32)
        assert eng.lib.vtts_pitch_shift_host(eng.h, x.ctypes.data, None, 1, x.size, sem.ctypes.data, y.ctypes.data) == -1
        assert eng.launch_count() == c0
    with pytest.raises(VttsError, match="outside"):
        eng.pitch_shift(np.stack([x, x]), 2.0, lengths=[2000, 2001])
    with pytest.raises(ValueError):
        eng.pitch_shift(np.stack([x, x]), [1.0, 2.0, 3.0])
    xt = torch.from_numpy(x[None]).cuda()
    sem = np.array([2.0], np.float32)
    assert eng.lib.vtts_pitch_shift(eng.h, xt.data_ptr(), None, 1, x.size, sem.ctypes.data, xt.data_ptr(), None) == -1   # y aliases x
    assert eng.lib.vtts_pitch_shift(eng.h, xt.data_ptr(), None, 1, x.size, None, xt.data_ptr() + 4, None) == -1          # no shifts
    for S, F in ((0, 16), (65536, 16), (1, 0), (1, (1 << 22) + 1)):
        with pytest.raises(VttsError, match="pitch_shift_stream_create"):
            eng.open_pitch_shift_stream(S, F)
    with eng.open_pitch_shift_stream(2, 16) as ps:
        z = np.zeros((2, 16), np.float32)
        c0 = eng.launch_count()
        with pytest.raises(VttsError, match="not open"):
            ps.push(z, [4, 0])
        with pytest.raises(VttsError, match="outside"):
            ps.push(z, [17, 0], begin=[True, False], semitones=1.0)
        for bad in (float("nan"), 13.0, -13.0):
            with pytest.raises(VttsError, match="semitones"):
                ps.push(z, [4, 0], begin=[True, False], semitones=[bad, 0.0])
        with pytest.raises(ValueError, match="semitones"):
            ps.push(z, [4, 0], begin=[True, False])
        assert eng.launch_count() == c0                                 # nothing was launched
        ps.push(z, [4, 0], begin=[True, False], semitones=[3.0, 0.0])
        c0 = eng.launch_count()
        n = np.array([4, 0], np.int32)
        f = np.zeros(2, np.uint8)
        for changed in (np.array([5.0, 0.0], np.float32), np.array([np.nan, 0.0], np.float32)):
            with pytest.raises(VttsError, match="until END"):
                eng._ck(eng.lib.vtts_pitch_shift_stream_push_host(eng.h, ps.h, z.ctypes.data, n.ctypes.data, f.ctypes.data,
                                                                  changed.ctypes.data, np.zeros((2, ps.out_pitch), np.float32).ctypes.data,
                                                                  np.zeros(2, np.int32).ctypes.data))
        assert eng.launch_count() == c0
        ps.push(z, [4, 0], end=[True, False])
        with pytest.raises(VttsError, match="not open"):
            ps.push(z, [4, 0])                        # ended: BEGIN first
        y = ps.push(np.stack([x[:16], x[:16]]), [16, 0], begin=[True, False], end=[True, False], semitones=5.0)[0]
        assert np.array_equal(y, x[:16])              # a short row is a copy, and the failed calls left the stream usable


# ---- text-to-speech stream and CLI -------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def tts_eng(acoustic_ckpt, hifigan_params):
    from viettts_b200.engine import Engine
    e = Engine(0)
    e.load_acoustic(acoustic_ckpt)
    e.load_hifigan(hifigan_params)
    e.load_duration(synthetic.duration_ckpt(1234))
    yield e
    e.close()


def tts_tokens(seed, L):
    rng = np.random.default_rng(seed)
    t = rng.integers(4, 90, size=L).astype(np.int32)
    t[4::5] = 3
    t[0] = t[-1] = 0
    return t


@pytest.mark.parametrize("kind", ["off", "reference"])
@pytest.mark.parametrize("denoise,rate", [(None, None), (0.5, 48000)])
def test_tts_stream_pitch_equals_shifted_tts(tts_eng, denoise, rate, kind):
    eng = tts_eng
    eng.set_precision("bf16x3")
    eng.set_fused_pairs(False)
    try:
        lens = [30, 7, 55, 20]
        shifts = [None, -4.0, None, 6.5]                              # None: the stream's default
        default = 3.0
        kw = {"off": {}, "reference": {"rng": KEY}}[kind]
        toks = [tts_tokens(90 + b, n) for b, n in enumerate(lens)]
        expect = []
        for t, sh in zip(toks, shifts):
            w = eng.tts(t[None], silence_duration=0.1, **kw)[0][0]
            if denoise is not None:
                w = eng.denoise(w, denoise)
            w = eng.pitch_shift(w, default if sh is None else sh)
            expect.append(w if rate is None else eng.resample(w, rate))
        pieces = {b: [] for b in range(len(toks))}
        with eng.open_tts_stream(2, 16, 2000, 100, output_rate=rate, denoise=denoise, semitones=default, **kw) as ts:
            queue, owner = list(range(len(toks))), {}
            while queue or ts.busy().any():
                for s in np.flatnonzero(~ts.busy()):
                    if queue:
                        b = queue.pop(0)
                        owner[int(s)] = b
                        ts.begin(int(s), toks[b], silence_duration=0.1, semitones=shifts[b])
                for s, w in ts.step().items():
                    pieces[owner[s]].append(w)
        for b in range(len(toks)):
            audio = np.concatenate(pieces[b])
            assert audio.shape == expect[b].shape and np.array_equal(audio, expect[b]), (denoise, rate, kind, b)
    finally:
        eng.set_fused_pairs(True)


def test_tts_stream_pitch_with_meter(tts_eng):
    eng = tts_eng
    eng.set_precision("bf16x3")
    eng.set_fused_pairs(False)
    try:
        toks = [tts_tokens(120 + b, n) for b, n in enumerate([25, 40])]
        audio = {0: [], 1: []}
        last = {}
        with eng.open_tts_stream(2, 16, 2000, 100, semitones=-2.0, meter=True) as ts:
            ts.begin(0, toks[0], silence_duration=0.1)
            ts.begin(1, toks[1], silence_duration=0.1, semitones=5.0)
            while ts.busy().any():
                for s, w in ts.step().items():
                    audio[s].append(w)
                last.update(ts.meter())
        for s, sh in ((0, -2.0), (1, 5.0)):
            a = np.concatenate(audio[s])
            assert np.array_equal(a, eng.pitch_shift(eng.tts(toks[s][None], silence_duration=0.1)[0][0], sh)), s
            ref = eng.loudness(a)
            assert np.array_equal(np.array(last[s], np.float32), np.array(ref, np.float32)), s
        with pytest.raises(ValueError):
            eng.open_tts_stream(1, 16, 2000, 100, semitones=13.0)
        with eng.open_tts_stream(1, 16, 2000, 100) as ts:
            with pytest.raises(ValueError, match="semitones"):
                ts.begin(0, toks[0], semitones=2.0)
    finally:
        eng.set_fused_pairs(True)


def test_cli_pitch(tts_eng, acoustic_ckpt, hifigan_params, golden_dir, tmp_path, monkeypatch):
    from viettts_b200 import synthesizer
    from viettts_b200.engine import get_engine
    from viettts_b200.hifigan.mel2wave import mel2wave
    from viettts_b200.nat.text2mel import text2mel
    (tmp_path / "assets/hifigan").mkdir(parents=True)
    (tmp_path / "assets/infore/hifigan").mkdir(parents=True)
    (tmp_path / "assets/infore/nat").mkdir(parents=True)
    (tmp_path / "assets/hifigan/config.json").write_text(json.dumps(config.HIFIGAN))
    for path, obj in (("assets/infore/hifigan/hk_hifi.pickle", hifigan_params), ("assets/infore/nat/acoustic_latest_ckpt.pickle", acoustic_ckpt),
                      ("assets/infore/nat/duration_latest_ckpt.pickle", synthetic.duration_ckpt(1234))):
        with open(tmp_path / path, "wb") as f:
            pickle.dump(obj, f)
    monkeypatch.chdir(tmp_path)
    lex = str(golden_dir / "lexicon_small.txt")
    ge = get_engine(0)
    text = "Xin chào, tôi là trợ lý ảo."
    assert synthesizer.main(["--text", text, "--output", "one.wav", "--lexicon-file", lex, "--silence-duration", "0.1",
                             "--pitch", "3"]) == 0
    wave = np.ravel(mel2wave(text2mel(synthesizer.nat_normalize_text(text), lex, 0.1)))
    pcm, sr = synthesizer.read_wav(tmp_path / "one.wav")
    assert sr == 16000
    expect = synthesizer.float_to_pcm16(ge.pitch_shift(wave, 3.0)).astype(np.int32)
    raw = np.frombuffer((tmp_path / "one.wav").read_bytes()[44:], "<i2").astype(np.int32)
    assert raw.shape == expect.shape and np.abs(raw - expect).max() <= 1

    lines = ["Xin chào, tôi là trợ lý ảo.", "hôm nay trời đẹp quá! bạn có khỏe không?"]
    (tmp_path / "lines.txt").write_text("\n".join(lines) + "\n")
    assert synthesizer.main(["--text-file", "lines.txt", "--output", "out.wav", "--lexicon-file", lex, "--silence-duration", "0.1",
                             "--seed", "5", "--denoise", "0.3", "--pitch", "-2.5", "--output-rate", "48000"]) == 0
    waves = synthesizer.synthesize_lines(lines, lex, 0.1, seed=5)
    for i, w in enumerate(waves):
        raw = (tmp_path / f"out_{i:04d}.wav").read_bytes()
        assert raw[44:] == synthesizer.float_to_pcm16(ge.resample(ge.pitch_shift(ge.denoise(w, 0.3), -2.5), 48000)).tobytes()

    for bad in ("13", "nan", "-12.5"):
        with pytest.raises(SystemExit):
            synthesizer.main(["--text", text, "--pitch", bad, "--lexicon-file", lex])
