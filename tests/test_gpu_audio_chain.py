"""GPU: the audio chain on its own speech.

A. Stage by stage against float64 (one-shot): `AudioChain.run` by hand, one stage at a time, on a ragged batch of the
   vocoder's output for a few seeded utterances.  Each device stage is held to its float64 oracle fed the device's own
   input to that stage, within the bound and TOL of the stage's own GPU test (imported from its test_<stage>_cpu.py);
   the pitch shifter and the time stretcher under the device's own decisions, with the DEC_MARGIN rule.  The meter's
   reading of the final audio is held to loudness_oracle within L_TOL, the true peak under the limiter's ceiling, the
   codes to g711_oracle bit for bit, and each batch row to `AudioChain.run` of it alone bit for bit.  The worst error
   of every stage is printed in that stage's own units.
B. The all-stages TTS stream under continuous batching (staggered BEGINs, per-utterance overrides, a slot reused the
   step after its END, an utterance that plans no frames) equals the one-shot chain bit for bit: codes, float audio
   and the meter's readings; then with each stream stage left out in turn, and at the meter's capacity edge."""
import numpy as np
import pytest
import torch

from oracle import bed_oracle as bo
from oracle import compressor_oracle as co
from oracle import denoise_oracle as dno
from oracle import eq_oracle as eo
from oracle import g711_oracle as go
from oracle import limiter_oracle as lm
from oracle import loudness_oracle as lo
from oracle import pitch_oracle as po
from oracle import resample_oracle as ro
from oracle import reverb_oracle as rvo
from oracle import time_stretch_oracle as tso
from oracle import watermark_oracle as wo
import test_bed_cpu
import test_compressor_cpu
import test_deesser_cpu
import test_denoise_cpu
import test_eq_cpu
import test_limiter_cpu
import test_loudness_cpu
import test_pitch_cpu
import test_resample_cpu
import test_reverb_cpu
import test_time_stretch_cpu
import test_watermark_cpu
from test_audio_chain_cpu import ALL_ON, out_pitch_rule
from viettts_b200 import config, synthetic

pytestmark = pytest.mark.gpu
KEY = np.array([7, 1234567], np.uint32)
SD = 0.1                                               # silence_duration of every utterance
BANK = ["pink,seed=5", "pink,seed=6,level=-22"]
EMPTY = np.array([3, 3, 3, 0], np.int32)               # only word ends before a trailing silence: nothing left to vocode


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


# ---- A. stage by stage against float64 -------------------------------------------------------------------------------

def dev_rows(x):
    return torch.from_numpy(np.ascontiguousarray(x, np.float32)).cuda()


def dec_margin_ok(dec, dec64, flag_m, branch_m, margin):
    """the device's decisions differ from float64's only where float64's margin is below `margin` (the stage's
    DEC_MARGIN)"""
    f_dev, f64 = (dec & 1) == 1, (dec64 & 1) == 1
    side = f_dev & f64 & ((dec >> 1 & 1) != (dec64 >> 1 & 1))
    return bool(np.all(flag_m[f_dev != f64] < margin) and np.all(branch_m[side] < margin))


def reduction_ok(red, rref):
    """a device reduction against float64's, as the stage's own GPU test holds it"""
    return abs(float(red) - rref) <= 1e-3 * max(1.0, abs(rref)), (red, rref)


def stage_error(eng, name, chain, x, y, n, m, row, extra):
    """(worst error of one row in the stage's own units, its TOL): x the device's input row (n valid samples), y the
    device's output row (m valid samples); every output past m must be 0.  Stages that report a gain reduction leave
    float64's in extra["rref"][row]."""
    assert not y[m:].any(), name
    x, y = x[:n], y[:m]
    r = chain.rate
    if name == "dn":
        if n <= dno.PAD:
            assert np.array_equal(y.view(np.uint32), x.view(np.uint32))
            return 0.0, test_denoise_cpu.TOL
        bias = extra["bias"]
        e = np.abs(y - dno.denoise(x, chain.denoise, bias)) / dno.error_scale(x, chain.denoise, bias)
        return float(e.max()), test_denoise_cpu.TOL
    if name == "ps":
        s = extra["semitones"][row]
        dec = extra["dec"][row]
        if n <= dno.PAD or s == 0:
            assert np.array_equal(y.view(np.uint32), x.view(np.uint32))
            assert not dec.any()
            return 0.0, test_pitch_cpu.TOL
        F = dno.n_frames(n)
        assert not dec[F:].any()
        dec = dec[:F]
        dec64 = po.decisions_of(x, s)
        assert dec_margin_ok(dec, dec64, *test_pitch_cpu.decision_margins(x, dec64), test_pitch_cpu.DEC_MARGIN), "pitch decisions"
        e = np.abs(y - po.pitch_shift(x, s, decisions=dec)) / po.error_scale(x, s)
        return float(e.max()), test_pitch_cpu.TOL
    if name == "ts":
        a = extra["tempo"][row]
        dec = extra["dec"][row]
        if n <= dno.PAD or float(np.float32(a)) == 1.0:
            k = min(n, m)
            assert np.array_equal(y[:k].view(np.uint32), x[:k].view(np.uint32))
            assert not dec.any()
            return 0.0, test_time_stretch_cpu.TOL
        T = dno.n_frames(m)
        assert not dec[T:].any()
        dec = dec[:T]
        dec64 = tso.stretch_decisions_of(x, a)
        assert dec_margin_ok(dec, dec64, *test_time_stretch_cpu.decision_margins(x, a), test_time_stretch_cpu.DEC_MARGIN), \
            "time-stretch decisions"
        e = np.abs(y - tso.time_stretch(x, a, decisions=dec)) / tso.stretch_error_scale(x, a)
        return float(e.max()), test_time_stretch_cpu.TOL
    if name == "wm":
        eps = chain.watermark["strength"]
        if n <= dno.PAD:
            assert np.array_equal(y, x)
            return 0.0, test_watermark_cpu.TOL_EMBED
        e = np.abs(y - wo.embed(x, chain.watermark["key"], np.float32(eps))) / test_watermark_cpu.embed_scale(x, eps)
        return float(e.max()), test_watermark_cpu.TOL_EMBED
    if name == "rs":
        rates = (config.SAMPLE_RATE, chain.output_rate)
        e = np.abs(y - ro.resample(x, *rates)) / np.maximum(ro.abs_sum(x, *rates), 1e-30)
        return float(e.max()), test_resample_cpu.TOL
    if name == "eq":
        return test_eq_cpu.error_units(y, eo.sosfilt(chain.eq, x), x, chain.eq), test_eq_cpu.TOL
    if name == "cp":
        ref, rref, P = co.compress(x, r, parts=True, **chain.compress)
        assert reduction_ok(extra["red"][row], rref)[0], ("compressor reduction", extra["red"][row], rref)
        extra["rref"][row] = rref
        return test_compressor_cpu.error_units(y, ref, P), test_compressor_cpu.TOL
    if name == "ds":
        ref, rref, P = test_deesser_cpu.parts(x, r, **chain.deess)
        assert reduction_ok(extra["red"][row], rref)[0], ("de-esser reduction", extra["red"][row], rref)
        extra["rref"][row] = rref
        return test_deesser_cpu.error_units(y, ref, x, P), test_deesser_cpu.TOL
    if name == "rv":
        p = extra["params"]
        return test_reverb_cpu.error_units(y, rvo.reverb(x, p["ir"], p["mix"]), x, p["ir"], p["mix"]), test_reverb_cpu.TOL
    if name == "bd":
        bank, idx = extra["bank"], extra["index"][row]
        if idx < 0:
            assert np.array_equal(y, x)
            return 0.0, test_bed_cpu.TOL
        p = bank.params[0]
        b = bank.audio.cpu().numpy()[bank.offsets[idx]: bank.offsets[idx] + bank.lengths[idx]]
        ref, rref, P = bo.mix(x, b, r, p["Fi"], p["Tt"], p["C"], p["o"], parts=True,
                              **{k: p[k] for k in ("duck", "threshold", "attack", "release")})
        assert ref.size == m
        assert reduction_ok(extra["red"][row], rref)[0], ("bed reduction", extra["red"][row], rref)
        extra["rref"][row] = rref
        return test_bed_cpu.error_units(y, ref, P), test_bed_cpu.TOL
    if name == "lm":
        ref, rref, P = lm.limit(x, r, chain.limit, extra["gain_db"][row], 5.0, 100.0, parts=True)
        red = extra["red"][row]
        assert abs(float(red) - rref) <= 1e-3 or (np.isinf(rref) and np.isinf(red)), ("limiter reduction", red, rref)
        extra["rref"][row] = rref
        c = np.float32(10 ** (chain.limit / 20))
        assert np.abs(y).max() <= c * (1 + 2 ** -22), "sample peak over the ceiling"
        assert lo.true_peak(y) <= chain.limit + test_limiter_cpu.TP_MARGIN, ("true peak", lo.true_peak(y))
        return test_limiter_cpu.error_units(y, ref, P), test_limiter_cpu.Y_TOL
    raise ValueError(name)


def run_by_hand(eng, chain, wavs, rows):
    """AudioChain.run's stages on a ragged batch, one at a time; `rows` the per-row BEGIN values (semitones, tempo, bed)
    and `over_db`: None for the limiter's pre-gain of the chain, else a pre-gain that puts the row's sample peak that
    many dB over the ceiling.  Checks each stage's every row against its oracle, and that every stage with a gain
    reduction (compressor, de-esser, bed, limiter) acted on at least one row; returns (final float rows, lengths, worst
    error per stage in its units, TOL per stage, float64's deepest reduction per such stage)."""
    lens = np.array([w.size for w in wavs], np.int32)
    x = np.zeros((len(wavs), int(lens.max())), np.float32)
    for b, w in enumerate(wavs):
        x[b, : w.size] = w
    r = chain.rate
    worst, tols, deepest = {}, {}, {}
    for name, _, _ in chain._stages():
        if name == "mt":
            continue
        extra = {"rref": {}}
        if name == "dn":
            extra["bias"] = eng.denoiser_bias()
            y = eng.denoise(x, chain.denoise, lengths=lens)
            out = lens
        elif name == "ps":
            sem = np.array(rows["semitones"], np.float32)
            extra["semitones"] = [float(s) for s in sem]
            extra["dec"] = eng.debug_pitch_decisions(dev_rows(x), sem, torch.from_numpy(lens).cuda())
            y = eng.pitch_shift(x, sem, lengths=lens)
            out = lens
        elif name == "ts":
            tp = np.array(rows["tempo"], np.float32)
            extra["tempo"] = [float(a) for a in tp]
            extra["dec"] = eng.debug_time_stretch_decisions(dev_rows(x), tp, torch.from_numpy(lens).cuda())
            y = eng.time_stretch(x, tp, lengths=lens)
            out = np.array([tso.stretch_length(int(n), float(a)) for n, a in zip(lens, tp)], np.int32)
        elif name == "wm":
            y = eng.watermark(x, chain.watermark, lengths=lens)
            out = lens
        elif name == "rs":
            y = eng.resample(x, chain.output_rate, lengths=lens)
            out = np.array([ro.out_len(int(n), config.SAMPLE_RATE, chain.output_rate) for n in lens], np.int32)
        elif name == "eq":
            y = eng.equalize(x, chain.eq, r, lengths=lens)
            out = lens
        elif name == "cp":
            y, extra["red"] = eng.compress(x, chain.compress, r, lengths=lens)
            out = lens
        elif name == "ds":
            y, extra["red"] = eng.deess(x, chain.deess, r, lengths=lens)
            out = lens
        elif name == "rv":
            from viettts_b200.engine import reverb_params
            extra["params"] = reverb_params(chain.reverb, r)
            y = eng.reverb(x, chain.reverb, r, lengths=lens)
            out = lens
        elif name == "bd":
            bank = chain._bank(eng)
            idx = np.array(rows["bed"], np.int32)
            extra.update(bank=bank, index=idx)
            y, extra["red"] = eng.mix_bed(x, bank, r, lengths=lens, index=idx)
            out = lens + np.where(idx >= 0, bank.params[0]["Tt"], 0).astype(np.int32)
        elif name == "lm":
            peak_db = [20 * np.log10(max(float(np.abs(x[b, :n]).max()), 1e-30)) for b, n in enumerate(lens)]
            g = np.array([chain.gain_db if o is None else np.clip(o + chain.limit - p, -70.0, 70.0)
                          for o, p in zip(rows["over_db"], peak_db)], np.float32)
            extra["gain_db"] = [float(v) for v in g]
            y, extra["red"] = eng.limit(x, chain.limit, r, gain_db=g, lengths=lens)
            out = lens
        errs = [stage_error(eng, name, chain, x[b], y[b], int(lens[b]), int(out[b]), b, extra) for b in range(len(wavs))]
        worst[name] = max(e for e, _ in errs)
        tols[name] = errs[0][1]
        assert worst[name] <= tols[name], (name, worst[name], tols[name])
        if extra["rref"]:
            deepest[name] = min(extra["rref"].values())
            assert deepest[name] < 0, (name, "never acted on this speech", extra["rref"])
        x, lens = y, out
    return x, lens, worst, tols, deepest


def check_meter(eng, y, lens, rate, worst):
    """the meter's reading of the final audio against loudness_oracle within L_TOL; its true peak against the fp32
    oversampler's own outputs, as tests/test_gpu_loudness.py holds it"""
    got = eng.loudness(y, rate, lengths=lens)
    err = 0.0
    for b, n in enumerate(lens):
        ref = lo.gate(lo.energies(y[b, :n], rate), rate // 10)
        for g, v in zip((got.integrated[b], got.momentary[b], got.short_term[b]), ref):
            if np.isinf(v):
                assert g == v, (b, g, v)
            else:
                err = max(err, abs(float(g) - v))
        u = eng.resample(y[b, :n], 4 * rate, rate)
        P = float(max(np.abs(y[b, :n]).max(), np.abs(u).max()))
        ref_tp = 20 * np.log10(P)
        assert abs(float(got.true_peak[b]) - ref_tp) <= 4 * float(np.spacing(np.float32(abs(ref_tp)))) + 1e-6, (b, got.true_peak[b], ref_tp)
    worst["mt"] = err
    assert err <= test_loudness_cpu.L_TOL, err
    return got


# (AudioChain options, tokens per row, bank entry per row, the limiter's pre-gain per row as dB over the ceiling)
CONFIGS = {
    "all48k": (dict(ALL_ON, output_rate=48000), [25, 40, 32], [0, 0, 0], [None, 6.0, 12.0]),
    "phone8k": (dict(output_rate=8000, eq="telephone", compress="voice", limit=-3.0, meter=True, encoding="ulaw"), [30, 52], [0, 0],
                [None, 9.0]),
    "room44k": (dict(output_rate=44100, reverb="room", bed=BANK, compress="voice", limit=-1.0, meter=True), [28, 45, 36], [0, 1, -1],
                [None, 6.0, 12.0]),
}


@pytest.mark.parametrize("config_name", list(CONFIGS))
def test_stages_against_float64_on_the_chains_own_speech(tts_eng, config_name):
    from viettts_b200.engine import AudioChain
    eng = tts_eng
    eng.set_precision("bf16x3")
    opts, lengths, beds, over_db = CONFIGS[config_name]
    chain = AudioChain(**opts)
    toks = [tts_tokens(300 + 7 * b + len(config_name), L) for b, L in enumerate(lengths)]
    wavs = [eng.tts(t[None], silence_duration=SD)[0][0] for t in toks]
    B = len(wavs)
    rows = {"semitones": [chain.semitones] * B, "tempo": [chain.tempo] * B, "over_db": over_db, "bed": beds}
    y, lens, worst, tols, deepest = run_by_hand(eng, chain, wavs, rows)
    if chain.meter:
        check_meter(eng, y, lens, chain.rate, worst)
        tols["mt"] = test_loudness_cpu.L_TOL
    if chain.encoding is not None:
        codes = eng.encode(y, chain.encoding, lengths=lens)
        assert np.array_equal(codes, go.encode(y, chain.encoding, lengths=lens))
    # each row alone through AudioChain.run: the same bits (rows on a bank entry other than the chain's default 0, or
    # with a pre-gain of their own, differ)
    for b in range(B):
        if (beds[b] != 0 and chain.bed is not None) or (over_db[b] is not None and chain.limit is not None):
            continue
        one = chain.run(eng, wavs[b])
        want = y[b, : lens[b]] if chain.encoding is None else codes[b, : lens[b]]
        assert one.shape == want.shape and np.array_equal(one, want), b
    print(f"\n{config_name}: worst |err| / scale per stage (TOL): "
          + ", ".join(f"{k} {worst[k]:.3g} ({tols[k]:g})" for k in worst)
          + "; deepest float64 reduction (dB): " + ", ".join(f"{k} {v:.2f}" for k, v in deepest.items()))


# ---- B. the all-stages TTS stream under continuous batching --------------------------------------------------------------

STREAM_OPTS = dict(output_rate=48000, denoise=0.5, semitones=3.0, tempo=0.8, watermark="key=1", eq="hs:6000:3", compress="voice",
                   deess="voice", reverb="hall", bed=BANK, limit=-1.0, meter=True)
OVERRIDES = ("semitones", "tempo", "gain_db", "bed")
OPENED_WITH = {"semitones": "semitones", "tempo": "tempo", "gain_db": "limit", "bed": "bed"}   # the option each override needs
STAGE_OPTION = {"dn": "denoise", "ps": "semitones", "ts": "tempo", "wm": "watermark", "rs": "output_rate", "eq": "eq", "cp": "compress",
                "ds": "deess", "rv": "reverb", "bd": "bed", "lm": "limit"}


def schedule():
    """(first step it may begin in, slot, tokens, overrides) per utterance; a slot's utterances run in this order, each
    begun as soon as the slot is free from that step on.  Slot 0 runs two utterances back to back; slot 3 begins an
    utterance with nothing to vocode mid-run, then another."""
    from viettts_b200.engine import MIN_TEMPO
    return [
        (0, 0, tts_tokens(500, 25), {}),
        (1, 1, tts_tokens(501, 40), dict(semitones=-5.0, tempo=MIN_TEMPO, gain_db=4.0, bed=1)),
        (3, 2, tts_tokens(502, 30), dict(semitones=7.0, tempo=1.6, gain_db=-6.0, bed=-1)),
        (2, 4, tts_tokens(503, 50), dict(tempo=0.9, gain_db=10.0)),
        (5, 3, EMPTY, dict(semitones=1.0, bed=1)),
        (0, 0, tts_tokens(504, 35), dict(semitones=-2.5, tempo=1.25, bed=0)),
        (6, 5, tts_tokens(505, 28), dict(semitones=12.0, tempo=MIN_TEMPO, bed=1, gain_db=-2.0)),
        (7, 3, tts_tokens(506, 26), dict(tempo=2.0, gain_db=1.5, bed=-1)),
    ]


def run_tts_stream(eng, sched, S, max_frames, opts, kw):
    """runs `sched` through open_tts_stream(S, 16, max_frames, 100, **opts, **kw); returns per utterance (its steps'
    outputs concatenated, the meter's reading after its last step or None, the frames begin planned)"""
    pending = [list() for _ in range(S)]
    for u, (start, slot, _, _) in enumerate(sched):
        pending[slot].append(u)
    pieces = {u: [] for u in range(len(sched))}
    meter, frames, ended, begun = {}, {}, {}, {}
    owner = [None] * S
    with eng.open_tts_stream(S, 16, max_frames, 100, **opts, **kw) as ts:
        step = 0
        while any(pending) or ts.busy().any():
            busy = ts.busy()
            for s in range(S):
                if not busy[s] and pending[s] and sched[pending[s][0]][0] <= step:
                    u = pending[s].pop(0)
                    ov = {k: v for k, v in sched[u][3].items() if opts.get(OPENED_WITH[k]) is not None}
                    frames[u] = ts.begin(s, sched[u][2], silence_duration=SD, **ov)
                    owner[s], begun[u] = u, step
            out = ts.step()
            m = ts.meter() if ts.mt is not None else {}
            busy = ts.busy()
            for s, w in out.items():
                u = owner[s]
                pieces[u].append(w)
                if s in m:
                    meter[u] = m[s]
                if not busy[s]:
                    ended[u] = step
            step += 1
            assert step < 2000
    for s in range(S):                                     # a slot's next utterance began in the step after its END
        us = [u for u in range(len(sched)) if sched[u][1] == s]
        for a, b in zip(us, us[1:]):
            if sched[b][0] <= ended[a] + 1:
                assert begun[b] == ended[a] + 1, (s, a, b)
    return {u: (np.concatenate(pieces[u]) if pieces[u] else None, meter.get(u), frames[u]) for u in range(len(sched))}


def one_shot(eng, opts, tokens, ov, kw, encoding):
    """AudioChain.run of the utterance's tts audio with its overrides, as a stream slot runs it"""
    from viettts_b200.engine import AudioChain
    o = dict(opts)
    for k, v in ov.items():
        if opts.get(OPENED_WITH[k]) is not None and k != "bed":
            o[k] = v
    if o.get("bed") is not None:                           # the slot's bank entry, alone
        bank = o["bed"] if isinstance(o["bed"], list) else [o["bed"]]
        v = ov.get("bed", 0)
        o["bed"] = None if v == -1 else bank[v]
    wav = eng.tts(tokens[None], silence_duration=SD, **kw)[0][0]
    return AudioChain(**o, encoding=encoding).run(eng, wav)


def check_stream_against_one_shot(eng, sched, S, max_frames, opts, kw, float_run=True):
    coded = run_tts_stream(eng, sched, S, max_frames, dict(opts, encoding="pcm16"), kw)
    flt = run_tts_stream(eng, sched, S, max_frames, opts, kw) if float_run else None
    for u, (_, _, tokens, ov) in enumerate(sched):
        codes, reading, frames = coded[u]
        if frames == 0:                                    # planned no frames: one empty output, no reading
            assert codes is not None and codes.size == 0 and codes.dtype == np.int16 and reading is None, u
            if flt is not None:
                assert flt[u][0].size == 0 and flt[u][0].dtype == np.float32, u
            continue
        want = one_shot(eng, opts, tokens, ov, kw, "pcm16")
        assert codes.shape == want.shape and np.array_equal(codes, want), ("codes", u)
        audio = one_shot(eng, opts, tokens, ov, kw, None)
        if flt is not None:
            assert np.array_equal(flt[u][0], audio), ("float audio", u)
            assert np.array_equal(eng.encode(flt[u][0], "pcm16"), codes), ("encoded float audio", u)
        if opts.get("meter"):
            ref = np.array(eng.loudness(audio, opts.get("output_rate") or config.SAMPLE_RATE), np.float32)
            assert np.array_equal(np.array(reading, np.float32), ref), ("meter", u, reading, ref)
            if flt is not None:
                assert np.array_equal(np.array(flt[u][1], np.float32), ref), ("meter, float run", u)


@pytest.mark.parametrize("kind", ["off", "reference"])
@pytest.mark.parametrize("mode", ["bf16x3", "fp16"])
def test_all_stages_tts_stream_equals_one_shot_chain(tts_eng, mode, kind):
    eng = tts_eng
    eng.set_precision(mode)
    eng.set_fused_pairs(False)
    try:
        sched = schedule()
        kw = {"off": {}, "reference": {"rng": KEY}}[kind]
        assert eng.tts_plan(EMPTY[None], silence_duration=SD)[3][0] == 0
        check_stream_against_one_shot(eng, sched, 6, 2000, STREAM_OPTS, kw)
    finally:
        eng.set_fused_pairs(True)
        eng.set_precision("bf16x3")


@pytest.mark.parametrize("left_out", list(STAGE_OPTION))
def test_tts_stream_with_one_stage_left_out(tts_eng, left_out):
    """every stream stage but the meter off in turn: each pair of stages two apart in the order meets once"""
    eng = tts_eng
    eng.set_precision("bf16x3")
    eng.set_fused_pairs(False)
    try:
        opts = dict(STREAM_OPTS)
        opts[STAGE_OPTION[left_out]] = None
        sched = [(0, 0, tts_tokens(600 + len(left_out), 27), dict(semitones=-3.0, tempo=0.6, gain_db=3.0, bed=1)),
                 (2, 1, tts_tokens(610 + len(left_out), 33), dict(tempo=1.4, bed=-1))]
        check_stream_against_one_shot(eng, sched, 2, 2000, opts, {}, float_run=False)
    finally:
        eng.set_fused_pairs(True)


def test_tts_stream_at_capacity(tts_eng):
    """one utterance of exactly max_frames frames at MIN_TEMPO under a bed with the longest tail (10 s): every stage's
    width follows the stated rule and the stream equals the one-shot chain at max_frames.  The meter's history is not
    at its edge here: its `seconds` keeps a second of margin over any utterance the stream accepts, so no utterance can
    fill it; the sizing rule is held at every max_frames by test_audio_chain_cpu.py
    (test_the_meter_holds_an_utterance_of_max_frames)."""
    from viettts_b200.engine import MIN_TEMPO, AudioChain
    eng = tts_eng
    eng.set_precision("bf16x3")
    eng.set_fused_pairs(False)
    try:
        for seed in range(700, 740):                       # an utterance the trim leaves whole: n_emit = n_frames
            tok = tts_tokens(seed, 60)
            tok[-1] = 40
            _, _, nf, ne = eng.tts_plan(tok[None], silence_duration=SD)
            if ne[0] == nf[0]:
                break
        assert ne[0] == nf[0]
        max_frames = int(nf[0])
        opts = dict(STREAM_OPTS, tempo=MIN_TEMPO, bed="pink,tail=10000")
        chain = AudioChain(**{k: v for k, v in opts.items()})
        assert chain.bed[0]["Tt"] == 10 * 48000
        sched = [(0, 1, tok, {})]
        with eng.open_tts_stream(2, 16, max_frames, 100, **opts) as ts:
            p = ts.voc.wav_ld
            for st in ts._built[2:]:
                name = next(k for k in STAGE_OPTION if getattr(ts, k) is st) if st is not ts.mt else "mt"
                if name != "mt":
                    assert st.out_pitch == out_pitch_rule(name, p, chain), name
                    p = st.out_pitch
        got = run_tts_stream(eng, sched, 2, max_frames, dict(opts, encoding="pcm16"), {})
        codes, reading, frames = got[0]
        assert frames == max_frames
        want = one_shot(eng, opts, tok, {}, {}, "pcm16")
        assert codes.shape == want.shape and np.array_equal(codes, want)
        audio = one_shot(eng, opts, tok, {}, {}, None)
        n = tso.stretch_length(max_frames * config.HOP, MIN_TEMPO)
        assert audio.size == ro.out_len(n, config.SAMPLE_RATE, 48000) + 10 * 48000
        assert np.array_equal(np.array(reading, np.float32), np.array(eng.loudness(audio, 48000), np.float32))
    finally:
        eng.set_fused_pairs(True)
