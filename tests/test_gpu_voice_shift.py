"""GPU: the voice shifter (Engine.pitch_shift(..., formant=), vtts_voice_shift*), its stream (Engine.open_voice_shift_stream)
and the `formant=` option of the audio chain, the text-to-speech stream and the CLI's --formant.

One-shot outputs are held to oracle/voice_shift_oracle.py per element, |y - y64| <= TOL_F * error_scale (TOL_F from
tests/test_voice_shift_cpu.py, over 4x an fp32 emulation of the kernels), under the device's own decisions where the
pitch moves; rows with s = 0 and a formant shift have no decisions and are compared as they are.  Without a formant the
calls are the pitch shifter bit for bit.  Everything that streams, every precision mode, batch position and repeat is
compared bit for bit with the one-shot call."""
import numpy as np
import pytest
import torch

from helpers import slot_streams as ss
from oracle import denoise_oracle as do
from oracle import pitch_oracle as po
from oracle import voice_shift_oracle as vo
from test_denoise_cpu import signal_of
from test_gpu_pitch import check_decisions, decisions, tts_tokens
from test_pitch_cpu import voiced_of
from test_voice_shift_cpu import KEEP_MOVE, LEGACY, SIGNALS, SR, TOL_F, expected_steps, f0_of, warp_steps
from viettts_b200 import synthetic
from viettts_b200.engine import AudioChain

pytestmark = pytest.mark.gpu
RAGGED = [0, 1, 512, 513, 1023, 1025, 80128, 30000, 24000]
CASES = [(3.0, 0.0), (-5.0, 4.0), (7.0, -5.0), (12.0, 0.0), (-12.0, 4.0), (0.0, 3.0), (5.0, -2.0), (0.0, 0.0), (0.0, -5.0)]


@pytest.fixture(scope="module")
def eng():
    from viettts_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


def check_row(y, x, n, s, phi, dec, what=""):
    """y: the output row of input x with n valid samples at (s, phi); dec: the device's pitch decisions of the row"""
    if n <= do.PAD or (s == 0 and phi == 0):
        assert np.array_equal(y[:n].view(np.uint32), x[:n].view(np.uint32)), what     # a bit copy
    elif s == 0:
        y64 = vo.voice_shift(x[:n], s, phi)
        ratio = np.abs(y[:n].astype(np.float64) - y64) / vo.error_scale(x[:n], s, phi)
        assert np.all(ratio <= TOL_F), (what, float(ratio.max()))
        return float(ratio.max())
    else:
        F = do.n_frames(n)
        check_decisions(dec[:F], x[:n], s, what)
        y64 = vo.voice_shift(x[:n], s, phi, decisions=dec[:F])
        ratio = np.abs(y[:n].astype(np.float64) - y64) / vo.error_scale(x[:n], s, phi)
        assert np.all(ratio <= TOL_F), (what, float(ratio.max()), int(ratio.argmax()))
        assert np.all(y[n:] == 0), what
        return float(ratio.max())
    assert np.all(y[n:] == 0), what
    return 0.0


def test_no_formant_is_the_pitch_shift_bit_for_bit(eng):
    """formant=None and vtts_voice_shift with formants = NULL are vtts_pitch_shift, through every entry point"""
    S = max(RAGGED)
    lens = np.array(RAGGED, np.int32)
    x = np.stack([(voiced_of if b % 2 else signal_of)(S, 40 + b) for b in range(lens.size)])
    sem = np.array([3.0, -5.0, 7.0, 12.0, -12.0, 2.5, -7.25, 0.0, 4.0], np.float32)
    ref = eng.pitch_shift(x, sem, lengths=lens)
    y = np.empty_like(x)
    assert eng.lib.vtts_voice_shift_host(eng.h, x.ctypes.data, lens.ctypes.data, len(lens), S, sem.ctypes.data, None, y.ctypes.data) == 0
    assert np.array_equal(y, ref)
    dev = torch.device("cuda", 0)
    xt, lt = torch.from_numpy(x).to(dev), torch.from_numpy(lens).to(dev)
    yt = torch.empty_like(xt)
    assert eng.lib.vtts_voice_shift(eng.h, xt.data_ptr(), lt.data_ptr(), len(lens), S, sem.ctypes.data, None, yt.data_ptr(), None) == 0
    torch.cuda.synchronize()
    assert np.array_equal(yt.cpu().numpy(), ref)
    assert np.array_equal(eng.pitch_shift_forward(xt, sem, lengths_t=lt, formant=None).cpu().numpy(), ref)


def test_one_shot_ragged_batch_against_float64(eng):
    S = max(RAGGED)
    lens = np.array(RAGGED, np.int32)
    x = np.stack([(voiced_of if b % 2 else signal_of)(S, 70 + b) for b in range(lens.size)])
    for b, n in enumerate(lens):
        x[b, n:] = np.nan                             # past a row's length: never read
    sem = np.array([c[0] for c in CASES], np.float32)
    fmt = np.array([c[1] for c in CASES], np.float32)
    y = eng.pitch_shift(x, sem, lengths=lens, formant=fmt)
    dec = decisions(eng, x, sem, lens)
    worst = max(check_row(y[b], x[b], int(n), float(sem[b]), float(fmt[b]), dec[b], (b, n, sem[b], fmt[b])) for b, n in enumerate(lens))
    print(f"worst |y - y64| / error_scale {worst:.2e} (TOL_F {TOL_F:.0e})")
    dev = torch.device("cuda", 0)
    yt = eng.pitch_shift_forward(torch.from_numpy(x).to(dev), sem, lengths_t=torch.from_numpy(lens).to(dev), formant=fmt)
    assert np.array_equal(yt.cpu().numpy(), y)


def test_three_minute_row(eng):
    n = 3 * 60 * 16000 + 77
    x = voiced_of(n, 11)
    y = eng.pitch_shift(x, 5.0, formant=-2.0)
    print(f"3 min: {check_row(y, x, n, 5.0, -2.0, decisions(eng, x[None], 5.0)[0], '3 min'):.2e}")


def test_same_bits_in_every_mode_alone_in_a_batch_and_repeated(eng):
    S = 20000
    lens = np.array([S, 7000, 513, 300, 15000], np.int32)
    sem = np.array([5.0, -3.0, 12.0, 4.0, 0.0], np.float32)
    fmt = np.array([0.0, 4.0, -5.0, 1.0, -3.0], np.float32)
    x = np.stack([voiced_of(S, 60 + b) for b in range(lens.size)])
    ys = []
    for mode in ("fp32", "bf16x3", "fp16"):
        eng.set_precision(mode)
        ys.append(eng.pitch_shift(x, sem, lengths=lens, formant=fmt))
        ys.append(eng.pitch_shift(x, sem, lengths=lens, formant=fmt))
    eng.set_precision("bf16x3")
    for y in ys[1:]:
        assert np.array_equal(y, ys[0])
    for b, n in enumerate(lens):
        alone = eng.pitch_shift(x[b, :n], float(sem[b]), formant=float(fmt[b]))
        assert np.array_equal(alone, ys[0][b, :n]), b


def test_envelope_warp_and_pitch_on_the_device(eng):
    """the LPC envelope warp of the device's output is f with a formant shift (within 4 steps of 1/48 octave) and r
    without one (within 1), and the steady vowels' F0 is r F0 within 2 %"""
    report = []
    for name, sig in SIGNALS.items():
        x = sig()
        for s, phi in KEEP_MOVE + LEGACY:
            y = eng.pitch_shift(x, float(s), formant=phi)
            j, want = warp_steps(x, y), expected_steps(s, phi)
            report.append(f"{name} ({s}, {phi}): {j} steps, expected {want:.1f}")
            assert abs(j - want) <= (1 if phi is None else 4), (name, s, phi, j, want)
            if name != "speech":
                f0y, f0x = f0_of(y[SR // 4: 3 * SR // 4]), f0_of(x[SR // 4: 3 * SR // 4])
                assert abs(f0y / (float(po.ratio(s)) * f0x) - 1) <= 0.02, (name, s, phi, f0y, f0x)
    print("\n".join(report))


# ---- stream ------------------------------------------------------------------------------------------------------

STREAM_CASES = [(3.0, 0.0), (-5.0, 4.0), (0.0, -3.0), (12.0, None), (-12.0, 2.0), (7.5, -1.0), (0.0, 0.0), (-1.0, None)]


def run_stream(eng, S, F, kinds, seed, host=False):
    """slot s runs plan kinds[s] with its own (s, phi) per utterance (phi None: the formants follow the pitch), held to
    the stream's contract and the pitch stream's five launches on every push (tests/helpers/slot_streams.py); without a
    formant the stream is the pitch shifter"""
    rng = np.random.default_rng(seed)
    plans = [ss.push_plan(k, F, rng) for k in kinds]
    cases = [[STREAM_CASES[int(rng.integers(len(STREAM_CASES)))] for _ in p] for p in plans]
    for row in ss.run(ss.stage(eng, "voice_shift", S, F), plans, lambda s, u, n: voiced_of(n, 1000 * s + u), cases, host=host):
        for x, (sh, phi), y, _ in filter(None, row):
            if phi is None:
                assert np.array_equal(y, eng.pitch_shift(x, sh))


@pytest.mark.parametrize("S", [1, 3, 16])
def test_stream_equals_one_shot(eng, S):
    kinds = ["max"] if S == 1 else [ss.KINDS[(s + S) % len(ss.KINDS)] for s in range(S)]
    run_stream(eng, S, 1000, kinds, seed=S)


def test_stream_one_sample_pushes_large_chunks_and_host_push(eng):
    run_stream(eng, 4, 1024, ["ones", 255, 256, "short"], seed=99)
    run_stream(eng, 2, 48000, ["max", "reuse"], seed=7)
    run_stream(eng, 3, 700, ["reuse", 1000, "max"], seed=5, host=True)


def test_stream_reads_formant_with_begin_only(eng):
    from viettts_b200._lib import VttsError
    x = voiced_of(4000, 9)
    with eng.open_voice_shift_stream(2, 2000) as ps:
        z = np.zeros((2, 2000), np.float32)
        c0 = eng.launch_count()
        for bad in (np.nan, np.inf, 12.5, -13.0):
            with pytest.raises(VttsError, match="formants"):
                ps.push(z, [4, 0], begin=[True, False], semitones=2.0, formant=[bad, 0.0])
        assert eng.launch_count() == c0
        a = ps.push(np.stack([x[:2000], x[:2000]]), [2000, 2000], begin=[True, True], semitones=[2.0, 2.0], formant=[1.0, 1.0])
        n, f, sem = np.array([10, 0], np.int32), np.zeros(2, np.uint8), np.array([2.0, 2.0], np.float32)
        for changed in ([3.0, 1.0], [np.nan, 1.0]):                               # a change without BEGIN
            fmt = np.array(changed, np.float32)
            with pytest.raises(VttsError, match="until END"):
                eng._ck(eng.lib.vtts_voice_shift_stream_push_host(eng.h, ps.h, z.ctypes.data, n.ctypes.data, f.ctypes.data, sem.ctypes.data,
                                                                  fmt.ctypes.data, np.zeros((2, ps.out_pitch), np.float32).ctypes.data,
                                                                  np.zeros(2, np.int32).ctypes.data))
        assert eng.launch_count() == c0 + 5
        b = ps.push(np.stack([x[2000:], x[2000:]]), [2000, 2000], end=[True, True], semitones=[2.0, 2.0], formant=[1.0, 1.0])
    ref = eng.pitch_shift(x, 2.0, formant=1.0)
    for s in range(2):
        assert np.array_equal(np.concatenate([a[s], b[s]]), ref)


def test_argument_errors(eng):
    x = np.stack([voiced_of(2000, 1)] * 2)
    y = np.zeros_like(x)
    sem = np.zeros(2, np.float32)
    for bad in (np.nan, np.inf, 13.0, -12.001):
        with pytest.raises(ValueError):
            eng.pitch_shift(x, 0.0, formant=bad)
        c0 = eng.launch_count()
        fmt = np.array([0.0, bad], np.float32)
        assert eng.lib.vtts_voice_shift_host(eng.h, x.ctypes.data, None, 2, 2000, sem.ctypes.data, fmt.ctypes.data, y.ctypes.data) == -1
        assert eng.launch_count() == c0
    with pytest.raises(ValueError):
        eng.pitch_shift(x, 0.0, formant=[1.0, 2.0, 3.0])


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


@pytest.mark.parametrize("semitones,formant,rate,meter", [(3.0, 0.0, None, False), (None, -3.0, 48000, True)])
def test_tts_stream_equals_the_chain(tts_eng, semitones, formant, rate, meter):
    eng = tts_eng
    eng.set_precision("bf16x3")
    eng.set_fused_pairs(False)
    try:
        lens = [30, 7, 55, 20]
        over = [None, {"formant": 2.0}, {"semitones": -4.0, "formant": 0.0}, {"formant": -1.5}]
        toks = [tts_tokens(150 + b, n) for b, n in enumerate(lens)]
        expect = []
        for t, o in zip(toks, over):
            o = o or {}
            ch = AudioChain(semitones=o.get("semitones", semitones), formant=o.get("formant", formant), output_rate=rate, meter=meter)
            expect.append(ch.run(eng, eng.tts(t[None], silence_duration=0.1)[0][0]))
        pieces = {b: [] for b in range(len(toks))}
        last = {}
        with eng.open_tts_stream(2, 16, 2000, 100, semitones=semitones, formant=formant, output_rate=rate, meter=meter) as ts:
            queue, owner = list(range(len(toks))), {}
            while queue or ts.busy().any():
                for s in np.flatnonzero(~ts.busy()):
                    if queue:
                        b = queue.pop(0)
                        owner[int(s)] = b
                        ts.begin(int(s), toks[b], silence_duration=0.1, **(over[b] or {}))
                for s, w in ts.step().items():
                    pieces[owner[s]].append(w)
                if meter:
                    for s, m in ts.meter().items():
                        last[owner[s]] = m
        for b in range(len(toks)):
            audio = np.concatenate(pieces[b])
            assert audio.shape == expect[b].shape and np.array_equal(audio, expect[b]), (semitones, formant, b)
            if meter:
                assert np.array_equal(np.array(last[b], np.float32), np.array(eng.loudness(audio, rate), np.float32)), b
        with eng.open_tts_stream(1, 16, 2000, 100, semitones=2.0) as ts:
            with pytest.raises(ValueError, match="formant"):
                ts.begin(0, toks[0], formant=1.0)
        with pytest.raises(ValueError):
            eng.open_tts_stream(1, 16, 2000, 100, formant=13.0)
    finally:
        eng.set_fused_pairs(True)


def test_cli_formant(tts_eng, acoustic_ckpt, hifigan_params, golden_dir, tmp_path, monkeypatch):
    import json
    import pickle
    from viettts_b200 import config, synthesizer
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
                             "--pitch", "4", "--formant", "0"]) == 0
    wave = np.ravel(mel2wave(text2mel(synthesizer.nat_normalize_text(text), lex, 0.1)))
    expect = synthesizer.float_to_pcm16(AudioChain(semitones=4.0, formant=0.0).run(ge, wave)).astype(np.int32)
    raw = np.frombuffer((tmp_path / "one.wav").read_bytes()[44:], "<i2").astype(np.int32)
    assert raw.shape == expect.shape and np.abs(raw - expect).max() <= 1
    for bad in ("13", "nan"):
        with pytest.raises(SystemExit):
            synthesizer.main(["--text", text, "--formant", bad, "--lexicon-file", lex])
