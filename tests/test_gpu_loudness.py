"""GPU: the loudness meter and normalizer (Engine.loudness / normalize_loudness / *_forward, vtts_loudness*), the meter
stream (Engine.open_loudness_meter), the TTS stream's `meter=True` and the CLI's --loudness / --true-peak.

One-shot readings are held to the float64 definition within L_TOL LU (tests/test_loudness_cpu.py, over 4x an fp32
emulation of the kernels); the true peak to the fp32 4x resampler's own outputs; everything that streams, and every
precision mode, batch position and repeat, is compared bit for bit with the one-shot call."""
import json
import pickle

import numpy as np
import pytest
import torch

from oracle import loudness_oracle as lo
from test_loudness_cpu import L_TOL, RATES, bursts, noise, sine
from viettts_b200 import config, synthetic
from viettts_b200.engine import STREAM_BEGIN, STREAM_END

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    from viettts_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


def row_signal(kind, n, rate, seed):
    if n == 0:
        return np.zeros(0, np.float32)
    secs = n / rate + 0.01
    x = {"noise": noise(secs, rate, seed), "bursts": bursts(secs, rate, seed), "sine": sine(997, secs, rate, 0.5)}[kind]
    return x[:n].astype(np.float32)


def expected_peak(eng, x, rate):
    """max(max |x|, max |Engine.resample(x, 4 rate, rate)|): the device's own oversampled outputs"""
    if x.size == 0:
        return 0.0
    u = eng.resample(x, 4 * rate, rate)
    return float(max(np.abs(x).max(), np.abs(u).max()))


def check_reading(got, x, rate, eng, what):
    ref = lo.gate(lo.energies(x, rate), rate // 10)
    for g, r, name in zip(got[:3], ref, ("integrated", "momentary", "short-term")):
        if np.isinf(r):
            assert g == r, (what, name, g, r)
        else:
            assert abs(float(g) - r) <= L_TOL, (what, name, float(g) - r)
    P = expected_peak(eng, x, rate)
    if P == 0:
        assert got[3] == -np.inf, what
    else:
        # the same peak up to the rounding of 20 log10f: a few ulp of the reading (one fp32 ulp of P moves it by 5e-7 dB)
        ref = 20 * np.log10(P)
        assert abs(float(got[3]) - ref) <= 4 * float(np.spacing(np.float32(abs(ref)))) + 1e-6, (what, float(got[3]), ref)


@pytest.mark.parametrize("rate", RATES)
def test_one_shot_ragged_batch_against_float64(eng, rate):
    m = rate // 10
    lens = [0, 1, 4 * m - 1, 4 * m, 4 * m + 1, 5 * rate + 17, 8 * rate]
    kinds = ["noise", "noise", "sine", "bursts", "noise", "noise", "bursts"]
    S = max(lens)
    x = np.full((len(lens), S), np.nan, np.float32)           # past a row's length: never read
    rows = []
    for b, (n, k) in enumerate(zip(lens, kinds)):
        rows.append(row_signal(k, n, rate, 10 * b + rate))
        x[b, :n] = rows[-1]
    got = eng.loudness(x, rate, lengths=lens)
    for b, n in enumerate(lens):
        check_reading([got.integrated[b], got.momentary[b], got.short_term[b], got.true_peak[b]], rows[b], rate, eng, (rate, b, n))
    # the device entry point computes the same bits
    dev = torch.device("cuda", 0)
    out = eng.loudness_forward(torch.from_numpy(x).to(dev), rate, lengths_t=torch.from_numpy(np.array(lens, np.int32)).to(dev)).cpu().numpy()
    assert np.array_equal(out, np.stack(got, axis=1))


def test_three_minute_row_and_generator_output(eng, hifigan_params):
    x = bursts(180, 16000, 5).astype(np.float32)
    r = eng.loudness(x, 16000)
    check_reading(list(r), x, 16000, eng, "3 min")
    eng.load_hifigan(hifigan_params)
    wav = eng.mel2wave(synthetic.mel_input(4, 2, 400))
    for b in range(2):
        r = eng.loudness(wav[b], 16000)
        check_reading(list(r), wav[b], 16000, eng, ("generator", b))
        w48 = eng.resample(wav[b], 48000)
        check_reading(list(eng.loudness(w48, 48000)), w48, 48000, eng, ("generator 48k", b))


def test_same_bits_in_every_mode_alone_in_a_batch_and_repeated(eng):
    rate = 16000
    lens = np.array([6 * rate, 3 * rate + 5, 7000, 0], np.int32)
    x = np.stack([row_signal("bursts", int(lens.max()), rate, 70 + b) for b in range(lens.size)])
    outs = []
    for mode in ("fp32", "bf16x3", "fp16"):
        eng.set_precision(mode)
        for _ in range(2):
            outs.append(np.stack(eng.loudness(x, rate, lengths=lens), axis=1))
            outs.append(eng.normalize_loudness(x, -20.0, rate, true_peak=-2.0, lengths=lens))
    eng.set_precision("bf16x3")
    for o in outs[2::2]:
        assert np.array_equal(o, outs[0])
    for y, g in outs[3::2]:
        assert np.array_equal(y, outs[1][0]) and np.array_equal(g, outs[1][1])
    for b, n in enumerate(lens):
        alone = np.array(eng.loudness(x[b, :n], rate), np.float32) if n else np.full(4, -np.inf, np.float32)
        assert np.array_equal(alone, outs[0][b]), b


# ---- normalization -------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("rate", [16000, 48000])
@pytest.mark.parametrize("ceiling", [None, -1.0, -6.0])
def test_normalize(eng, rate, ceiling):
    target = -16.0
    lens = [0, 3 * rate // 10, 5 * rate, 4 * rate + 3, 6 * rate]
    S = max(lens)
    x = np.full((len(lens), S), np.nan, np.float32)
    rows = []
    for b, n in enumerate(lens):
        rows.append(row_signal(["noise", "noise", "bursts", "sine", "noise"][b], n, rate, 5 * b) * np.float32(0.05 * (b + 1)))
        x[b, :n] = rows[-1]
    x[4, :lens[4]] = 0                                        # a silent row: L = -inf
    rows[4] = x[4, :lens[4]].copy()
    y, g = eng.normalize_loudness(x, target, rate, true_peak=ceiling, lengths=lens)
    for b, n in enumerate(lens):
        xb = rows[b]
        assert np.all(y[b, n:] == 0), b
        L = lo.measure(xb, rate)[0] if n else -np.inf
        if not np.isfinite(L):
            assert g[b] == 0 and np.array_equal(y[b, :n].view(np.uint32), xb.view(np.uint32)), b
            continue
        g_ref = lo.gain(xb, rate, target, ceiling)
        assert abs(float(g[b]) - g_ref) <= L_TOL + 1e-4, (b, float(g[b]), g_ref)   # + the fp32 resampler's peak
        f = np.float32(10.0 ** (np.float64(g[b]) / 20.0))
        assert np.array_equal(y[b, :n], xb * f), b
        if ceiling is None:
            assert abs(lo.measure(y[b, :n], rate)[0] - target) <= 1e-3, b
        else:
            assert lo.true_peak(y[b, :n]) <= ceiling + 1e-3, b
            assert lo.measure(y[b, :n], rate)[0] <= target + 1e-3, b
    # the device entry point, out of place and in place, computes the same bits
    dev = torch.device("cuda", 0)
    xt = torch.from_numpy(x).to(dev)
    lt = torch.from_numpy(np.array(lens, np.int32)).to(dev)
    yt, gt = eng.normalize_loudness_forward(xt, target, rate, true_peak=ceiling, lengths_t=lt)
    assert np.array_equal(yt.cpu().numpy(), y) and np.array_equal(gt.cpu().numpy(), g)
    y2, _ = eng.normalize_loudness_forward(xt, target, rate, true_peak=ceiling, lengths_t=lt, out=xt)
    assert y2.data_ptr() == xt.data_ptr() and np.array_equal(xt.cpu().numpy(), y)


def test_argument_errors(eng):
    from viettts_b200._lib import VttsError
    x = noise(1, 16000).astype(np.float32)
    for rate in (11025, 7990, 192010, 16005):
        with pytest.raises(ValueError):
            eng.loudness(x, rate)
        with pytest.raises(VttsError, match="rate"):
            eng._ck(eng.lib.vtts_loudness_host(eng.h, x.ctypes.data, None, 1, x.size, rate, np.zeros(4, np.float32).ctypes.data))
    for t, c in ((-71.0, None), (0.5, None), (float("nan"), None), (-16.0, 0.5), (-16.0, -21.0), (-16.0, float("nan"))):
        with pytest.raises(ValueError):
            eng.normalize_loudness(x, t, true_peak=c)
    y = np.zeros_like(x)
    for t, c in ((-71.0, float("inf")), (-16.0, 0.5), (-16.0, -float("inf")), (float("nan"), float("inf"))):
        with pytest.raises(VttsError, match="loudness_normalize_host"):
            eng._ck(eng.lib.vtts_loudness_normalize_host(eng.h, x.ctypes.data, None, 1, x.size, 16000, t, c, y.ctypes.data, None))
    with pytest.raises(VttsError, match="null"):
        eng._ck(eng.lib.vtts_loudness_host(eng.h, None, None, 1, x.size, 16000, y.ctypes.data))
    with pytest.raises(VttsError, match="null"):
        eng._ck(eng.lib.vtts_loudness(eng.h, None, None, 1, x.size, 16000, None, None))
    with pytest.raises(VttsError, match="outside"):
        eng.loudness(np.stack([x, x]), 16000, lengths=[-1, 5])
    with pytest.raises(VttsError, match="outside"):
        eng.normalize_loudness(np.stack([x, x]), -16.0, lengths=[5, x.size + 1])


# ---- meter stream --------------------------------------------------------------------------------------------------

def push_plan(kind, F, m, rng):
    """push sizes of one utterance (END with the last)"""
    if kind == "ones":
        return [1] * 900 + [int(v) for v in rng.integers(1, F + 1, size=8)]
    if kind == 255:
        return [255] * int(rng.integers(20, 40))
    if kind == "m":
        return [min(m, F)] * int(rng.integers(5, 40))
    if kind == "random":
        return [int(v) for v in rng.integers(0, F + 1, size=int(rng.integers(5, 30)))]
    return []


def run_meter(eng, S, F, rate, kinds, seed, long_slot=None):
    """drives a meter: slot s runs plan kinds[s] (several utterances for 'reuse' slots begin mid-run); after every push
    the readings of each active slot equal the one-shot readings of its prefix (integrated, momentary, short-term bit
    for bit; the true peak at END)"""
    rng = np.random.default_rng(seed)
    m = rate // 10
    plans = {s: [push_plan(k, F, m, rng) for _ in range(2 if s % 3 == 1 else 1)] for s, k in enumerate(kinds)}
    if long_slot is not None:
        plans[long_slot] = [[F] * (200 * rate // F)]
    start = {s: int(rng.integers(0, 4)) for s in range(S)}    # BEGIN in mid-run
    sigs = {s: [] for s in range(S)}
    heard = {s: np.zeros(0, np.float32) for s in range(S)}
    state = {s: (0, 0) for s in range(S)}                     # (utterance, push)
    last = np.full((S, 4), -np.inf, np.float32)
    with eng.open_loudness_meter(S, F, rate, max_seconds=240) as mt:
        assert mt.lookahead == lo.LOOKAHEAD
        step = 0
        while any(state[s][0] < len(plans[s]) for s in range(S)):
            x = np.zeros((S, F), np.float32)
            n = np.zeros(S, np.int32)
            begin = np.zeros(S, bool)
            end = np.zeros(S, bool)
            for s in range(S):
                u, p = state[s]
                if step < start[s] or u >= len(plans[s]):
                    continue
                plan = plans[s][u]
                if not plan:
                    state[s] = (u + 1, 0)
                    continue
                if p == 0:
                    begin[s] = True
                    sigs[s] = row_signal(["noise", "bursts"][(s + u) % 2], sum(plan) + 1, rate, 100 * s + u)[: sum(plan)]
                    heard[s] = np.zeros(0, np.float32)
                k = plan[p]
                pos = heard[s].size
                x[s, :k] = sigs[s][pos: pos + k]
                n[s] = k
                heard[s] = sigs[s][: pos + k]
                end[s] = p == len(plan) - 1
                state[s] = (u + 1, 0) if end[s] else (u, p + 1)
            c0 = eng.launch_count()
            out = mt.push(x, n, begin, end)
            assert eng.launch_count() - c0 == 7
            act = begin | end | (n > 0)
            for s in np.flatnonzero(~act):
                assert np.array_equal(out[s], last[s]), s  # idle slots keep their readings
            idx = [int(s) for s in np.flatnonzero(act)]
            if idx:
                lens = np.array([heard[s].size for s in idx], np.int32)
                X = np.zeros((len(idx), max(1, int(lens.max()))), np.float32)
                for i, s in enumerate(idx):
                    X[i, : lens[i]] = heard[s]
                ref = np.stack(eng.loudness(X, rate, lengths=lens), axis=1)
                for i, s in enumerate(idx):
                    assert np.array_equal(out[s, :3], ref[i, :3]), (step, s, out[s], ref[i])
                    if end[s]:
                        assert out[s, 3] == ref[i, 3], (step, s)
                    else:
                        assert out[s, 3] <= ref[i, 3] or np.isnan(ref[i, 3]), (step, s)
            last = out
            step += 1


@pytest.mark.parametrize("rate", [16000, 48000])
def test_meter_one_slot(eng, rate):
    run_meter(eng, 1, 4096, rate, ["ones"], 1)
    run_meter(eng, 1, rate // 10, rate, ["m"], 2)


@pytest.mark.parametrize("rate", [8000, 16000, 44100])
def test_meter_eight_slots(eng, rate):
    run_meter(eng, 8, 2048, rate, [255, "m", "random", "random", "idle", 255, "random", "m"], 3 + rate)


def test_meter_long_slot(eng):
    run_meter(eng, 3, 32000, 16000, ["random", "idle", "m"], 9, long_slot=1)


def test_meter_history_overflow_launches_nothing(eng):
    from viettts_b200._lib import VttsError
    rate, F = 16000, 8000
    x = noise(2, rate, 1).astype(np.float32)
    with eng.open_loudness_meter(2, F, rate, max_seconds=1) as mt:
        mt.push(np.stack([x[:F], x[:F]]), [F, 0], [True, False])
        r1 = mt.push(np.stack([x[F:2 * F], x[:F]]), [F, 0])        # 16000 samples: exactly the 10 sub-blocks it holds
        c0 = eng.launch_count()
        with pytest.raises(VttsError, match="max_seconds"):
            mt.push(np.stack([x[:F], x[:F]]), [F, 0])                # would complete sub-block 15 of 10
        assert eng.launch_count() == c0
        r2 = mt.push(np.zeros((2, F), np.float32), [0, 0], [False, False], [True, False])
        assert np.array_equal(r2[0, :3], r1[0, :3])
        assert np.array_equal(r2[0], np.array(eng.loudness(x[:2 * F], rate), np.float32))


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


@pytest.mark.parametrize("rate,denoise", [(None, None), (48000, None), (None, 0.1), (48000, 0.1)])
def test_tts_stream_meter_equals_one_shot(tts_eng, rate, denoise):
    eng = tts_eng
    eng.set_precision("bf16x3")
    lens = [30, 7, 55]
    toks = [tts_tokens(90 + b, n) for b, n in enumerate(lens)]

    def stream(meter):
        pieces, readings = {b: [] for b in range(len(toks))}, {}
        with eng.open_tts_stream(2, 16, 2000, 100, output_rate=rate, denoise=denoise, meter=meter) as ts:
            queue, owner = list(range(len(toks))), {}
            while queue or ts.busy().any():
                for s in np.flatnonzero(~ts.busy()):
                    if queue:
                        b = queue.pop(0)
                        owner[int(s)] = b
                        ts.begin(int(s), toks[b], silence_duration=0.1)
                busy = ts.busy()
                out = ts.step()
                for s, w in out.items():
                    pieces[owner[s]].append(w)
                if meter:
                    got = ts.meter()
                    assert sorted(got) == sorted(out)
                    for s in out:
                        if not ts.busy()[s] and busy[s]:
                            readings[owner[s]] = got[s]
        return {b: np.concatenate(p) for b, p in pieces.items()}, readings

    plain, _ = stream(False)
    audio, readings = stream(True)
    for b in range(len(toks)):
        assert np.array_equal(audio[b], plain[b]), b                      # the meter does not touch the audio
        ref = eng.loudness(audio[b], rate or config.SAMPLE_RATE)
        assert np.array_equal(np.array(readings[b], np.float32), np.array(ref, np.float32)), (b, readings[b], ref)
    with pytest.raises(ValueError):
        eng.open_tts_stream(2, 16, 2000, 100, output_rate=11025, meter=True)
    eng.open_tts_stream(1, 16, 2000, 100, output_rate=11025).close()     # without the meter 11025 Hz stays available


def test_cli_loudness(tts_eng, acoustic_ckpt, hifigan_params, golden_dir, tmp_path, monkeypatch):
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
    text = "Xin chào, tôi là trợ lý ảo. hôm nay trời đẹp quá! bạn có khỏe không?"
    assert synthesizer.main(["--text", text, "--output", "one.wav", "--lexicon-file", lex, "--silence-duration", "0.1",
                             "--loudness", "-16"]) == 0
    wave = np.ravel(mel2wave(text2mel(synthesizer.nat_normalize_text(text), lex, 0.1)))
    y, g = ge.normalize_loudness(wave, -16.0, 16000, true_peak=-1.0)
    raw = (tmp_path / "one.wav").read_bytes()
    assert raw[44:] == synthesizer.float_to_pcm16(y).tobytes()
    pcm, sr = synthesizer.read_wav(tmp_path / "one.wav")
    assert sr == 16000
    L, _, _, tp = lo.measure(pcm, sr)
    assert 10 ** (tp / 20) <= 10 ** ((-1.0 + 1e-3) / 20) + 0.5 / 32767, tp    # PCM rounding moves samples by half a step
    if abs(g - (-16.0 - lo.measure(wave, 16000)[0])) <= 1e-3:
        assert abs(L + 16.0) <= 0.01, L                                    # the target is reachable under the ceiling
    else:
        assert L < -16.0 and abs(lo.true_peak(y) + 1.0) <= 1e-3            # the ceiling holds the gain back

    lines = ["Xin chào, tôi là trợ lý ảo.", "hôm nay trời đẹp quá! bạn có khỏe không?"]
    (tmp_path / "lines.txt").write_text("\n".join(lines) + "\n")
    assert synthesizer.main(["--text-file", "lines.txt", "--output", "out.wav", "--lexicon-file", lex, "--silence-duration", "0.1",
                             "--seed", "5", "--denoise", "0.3", "--output-rate", "48000", "--loudness", "-23", "--true-peak", "-2"]) == 0
    waves = synthesizer.synthesize_lines(lines, lex, 0.1, seed=5)
    for i, w in enumerate(waves):
        raw = (tmp_path / f"out_{i:04d}.wav").read_bytes()
        expect = ge.normalize_loudness(ge.resample(ge.denoise(w, 0.3), 48000), -23.0, 48000, true_peak=-2.0)[0]
        assert raw[44:] == synthesizer.float_to_pcm16(expect).tobytes()

    for bad in (["--true-peak", "-1"], ["--output-rate", "11025", "--loudness", "-16"], ["--loudness", "-80"],
                ["--loudness", "-16", "--true-peak", "1"]):
        with pytest.raises(SystemExit):
            synthesizer.main(["--text", text, "--lexicon-file", lex, *bad])
