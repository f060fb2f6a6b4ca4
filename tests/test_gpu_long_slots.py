"""GPU: every per-slot sample stream deep into a long-lived slot, past 2^24 and 2^31 samples (and 2^32).

A stream slot now lives as long as text keeps arriving (TtsStream.append), so every stage's carried state and absolute
sample positions run on for hours.  Each stream here opens two slots with 2^22-sample pushes, pushes digital silence
from BEGIN (one device buffer, no host copies) until the slot's input position reaches a mark, then a few seconds of
speech in ragged chunks (1-sample pushes included) with END on the last one.  Every push's emission count is held to the
stage's counting formula, evaluated in Python ints.  The probe's outputs are then held to

  * the same stream given a short silence prefix of the same length modulo the stage's period, bit for bit.  Digital
    silence leaves every carried state where it was after a few frames of silence, so only the position modulo the
    stage's grid can matter: 256 for the STFT hop (denoise, pitch shift) and the compressor's scan block, 512 for the
    reverb's partition, 1024 for the equalizer's block (and the de-esser's sidechain, which runs it), 1024 for the
    limiter (its 256-sample release blocks and 1024-sample tiles), 65536 for the watermark's chip period, `down`
    inputs for a resampler at up / down, rate / 10 for the loudness meter's sub-blocks, the bed's loop period (with the
    ducker's 256-sample block) for the bed, and for the time stretcher the period of its frame centres
    rint(256 t alpha) in double, which rounds halves to even: with 256 alpha = p / q in lowest terms, frame t + q sits at
    a_t + p when q = 1, and frame t + 2q at a_t + 2p otherwise (p is then odd, and a shift by odd p moves an exact half
    to the other even neighbour);
  * for the stages keyed to absolute position or carrying phase (resample, pitch shift, time stretch, watermark, bed)
    and for the meter, also the stage's float64 oracle on the probe plus a silent context, evaluated at the absolute
    offset, within the bound the stage's ragged-rows test uses.
"""
import time
from fractions import Fraction
from math import gcd

import numpy as np
import pytest
import torch

from helpers import slot_streams as ss
from oracle import bed_oracle as bo
from oracle import loudness_oracle as lo
from oracle import pitch_oracle as po
from oracle import resample_oracle as ro
from oracle import time_stretch_oracle as tso
from oracle import watermark_oracle as wo
from test_bed_cpu import TOL as BED_TOL, error_units
from test_loudness_cpu import L_TOL
from test_pitch_cpu import TOL as PITCH_TOL
from test_resample_cpu import TOL as RS_TOL
from test_time_stretch_cpu import TOL as TS_TOL
from test_watermark_cpu import KEY, TOL_EMBED, embed_scale, speech
from viettts_b200 import config
from viettts_b200.engine import STREAM_BEGIN, STREAM_END

pytestmark = pytest.mark.gpu
SR = config.SAMPLE_RATE
F = 1 << 22
MARKS = [(1 << 24) + 12345, (1 << 31) - 20000, (1 << 31) + 6789, (1 << 32) + 4321]
SESSIONS = [(MARKS[0], MARKS[1]), (MARKS[2], MARKS[3])]      # the two slots of one stream
PROBE = speech(3.0, 2.0).astype(np.float32)
CHUNKS = [1, 1, 1, 255, 256, 257, 1, 1023, 1025, 1, 4096, 8191, 1]
OUT_RATE = 44100                                        # up / down = 441 / 160 from 16 kHz
BANK = ["pink,seed=1,length=0.6,fade_in=250,tail=300,xfade=50,offset=0.1"]


@pytest.fixture(scope="module")
def eng():
    from viettts_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


def probe_chunks():
    out, left = [], PROBE.size - sum(CHUNKS)
    while left > 0:
        out.append(min(left, 20000))
        left -= out[-1]
    return CHUNKS + out


def ts_period(tempo):
    """input samples and frames after which the time stretcher's frame centres rint(256 t alpha) repeat exactly"""
    r = Fraction(float(np.float32(tempo))) * 256
    k = 1 if r.denominator == 1 else 2
    return k * r.numerator, k * r.denominator


def bed_period(eng):
    bank = eng.prepare_beds(BANK, SR)
    p = bank.params[0]
    P = int(bank.lengths[0]) - p["C"]
    return P * 256 // gcd(P, 256)


def long_stage(eng, name):
    """(stage, BEGIN value, period) of stream `name` as the probe runs it: two slots of chunk F from the table"""
    if name.startswith("time_stretch_"):
        tempo = float(name.rsplit("_", 1)[1])
        return ss.stage(eng, "time_stretch", 2, F), tempo, ts_period(tempo)[0]
    spec, value, period = {
        "resample": (dict(out_rate=OUT_RATE), None, ro.ratio(SR, OUT_RATE)[1]),
        "denoise": (dict(strength=0.5, bias=np.full(513, 1e-3, np.float32)), None, 256),
        "pitch": ({}, 3.0, 256),
        "limiter": (dict(ceiling=-1.0), 12.0, 1024),
        "eq": (dict(eq="telephone"), None, 1024),
        "compressor": (dict(spec="voice"), None, 256),
        "deesser": (dict(spec="voice"), None, 1024),
        "reverb": (dict(spec="room"), None, 512),
        "watermark": (dict(spec=KEY), None, wo.PERIOD),
        "bed": (dict(bed=BANK), 0, None),
        "loudness": (dict(max_seconds=1 << 20), None, SR // 10),
    }[name]
    return ss.stage(eng, name, 2, F, **spec), value, bed_period(eng) if name == "bed" else period


def plan(mark):
    """[(n_new, probe offset or None, end)] of one slot: silence up to `mark`, then the probe"""
    p = [(F, None, False)] * (mark // F) + ([(mark % F, None, False)] if mark % F else [])
    off = 0
    chunks = probe_chunks()
    for i, k in enumerate(chunks):
        p.append((k, off, i == len(chunks) - 1))
        off += k
    return p


def run(eng, stage, value, marks):
    """runs both slots of one stream, BEGIN value `value`, to their marks and through the probe; per slot: the probe
    pushes' outputs (a list of arrays), the last reduction (or meter reading) and the wall time"""
    dev = torch.device("cuda", 0)
    t0 = time.perf_counter()
    st = stage.open()
    kw = stage.begin([value] * 2)[0]
    S = 2
    width = 4 if stage.meter else st.out_pitch
    x_t = torch.zeros((S, F), dtype=torch.float32, device=dev)
    y_t = torch.zeros((S, width), dtype=torch.float32, device=dev)
    red_t = torch.zeros(S, dtype=torch.float32, device=dev)
    probe_t = torch.from_numpy(PROBE).to(dev)
    plans = [plan(m) for m in marks]
    outs, last = [[] for _ in range(S)], [None] * S
    P = [0] * S
    try:
        for i in range(max(map(len, plans))):
            n_new = np.zeros(S, np.int32)
            flags = np.zeros(S, np.uint8)
            for s in range(S):
                if i >= len(plans[s]):
                    continue
                n, off, end = plans[s][i]
                if off is not None:
                    x_t[s, :n].copy_(probe_t[off:off + n])
                n_new[s] = n
                flags[s] = (STREAM_BEGIN if i == 0 else 0) | (STREAM_END if end else 0)
            n_out = stage.push_device(st, x_t, n_new, flags, y_t, red_t, kw)
            for s in range(S):
                if i >= len(plans[s]):
                    continue
                n, off, end = plans[s][i]
                P0, P[s] = P[s], P[s] + n
                if n_out is not None:
                    want = stage.emitted(P[s], end, value) - (0 if i == 0 else stage.emitted(P0, False, value))
                    assert int(n_out[s]) == want, (stage.name, marks[s], i, P[s], int(n_out[s]), want)
                if off is not None:
                    if n_out is not None:
                        outs[s].append(y_t[s, :int(n_out[s])].cpu().numpy().copy())
                    if end:
                        last[s] = (y_t[s].cpu().numpy().copy() if stage.meter else float(red_t[s]))
        torch.cuda.synchronize()
    finally:
        st.close()
    return outs, last, time.perf_counter() - t0


def short(mark, period, floor=1 << 15):
    """a short prefix of the same length as `mark` modulo `period`"""
    L = mark % period
    while L < floor:
        L += period
    return L


# ---- float64 oracles at the absolute offset ----
def window(c):
    """the probe after c samples of silent context: a slot's input from absolute sample mark - c on, for a probe pushed
    at `mark`"""
    return np.concatenate([np.zeros(c, np.float32), PROBE])


def rel(y, ref, scale):
    """max |y - ref| / scale, where a zero scale (silence) admits no error at all"""
    d = np.abs(y.astype(np.float64) - ref)
    z = scale <= 0
    return float(np.max(np.where(z, np.where(d == 0, 0.0, np.inf), d / np.where(z, 1.0, scale))))


def oracle_resample(eng, stage, mark, y):
    up, down, _ = ro.ratio(SR, OUT_RATE)
    c = mark % down + 40 * down                      # s0 = mark - c is a multiple of down: output s0 up / down is sample 0
    s0 = mark - c
    E0 = stage.emitted(mark, False)
    m0 = E0 - s0 * up // down
    w = window(c)
    y64 = ro.resample(w, SR, OUT_RATE, m_range=(m0, m0 + y.size))
    scale = ro.abs_sum(w, SR, OUT_RATE, m_range=(m0, m0 + y.size))
    assert m0 + y.size == ro.out_len(w.size, SR, OUT_RATE)
    err = np.abs(y.astype(np.float64) - y64) / np.maximum(scale, 1e-30)
    return float(err.max()), RS_TOL


def oracle_watermark(eng, stage, mark, y):
    c = mark % 256 + 2048
    s0 = mark - c
    w = window(c)
    ref = wo.embed(w, KEY, np.float32(0.1), frame0=s0 // 256)
    u0 = stage.emitted(mark, False) - s0
    assert u0 + y.size == w.size
    return rel(y, ref[u0:], embed_scale(w, 0.1)[u0:]), TOL_EMBED


def oracle_pitch(eng, stage, mark, y):
    c = mark % 256 + 2048                              # frames at 256 t: the window's grid is the slot's
    s0 = mark - c
    w = window(c)
    dec = eng.debug_pitch_decisions(torch.from_numpy(w[None]).cuda(), 3.0)[0]
    ref = po.pitch_shift(w, 3.0, decisions=dec)
    u0 = stage.emitted(mark, False) - s0
    assert u0 + y.size == w.size
    return rel(y, ref[u0:], po.error_scale(w, 3.0)[u0:]), PITCH_TOL


def oracle_stretch(eng, stage, mark, y):
    tempo = 1.25
    p, q = ts_period(tempo)                          # 320 inputs per frame: frame centres a_t = 320 t exactly
    c = mark % p + 8 * p
    s0 = mark - c
    w = window(c)
    M = tso.stretch_length(w.size, tempo)
    dec = eng.debug_time_stretch_decisions(torch.from_numpy(w[None]).cuda(), tempo)[0, :M // 256 + 1]
    ref = tso.time_stretch(w, tempo, decisions=dec)
    u0 = stage.emitted(mark, False, tempo) - s0 * q * 256 // p
    assert u0 + y.size == M, (u0, y.size, M)
    return rel(y, ref[u0:], tso.stretch_error_scale(w, tempo)[u0:]), TS_TOL


def oracle_bed(eng, stage, mark, y, red):
    bank = eng.prepare_beds(BANK, SR)
    p = bank.params[0]
    b = bank.audio.cpu().numpy()[bank.offsets[0]:bank.offsets[0] + bank.lengths[0]]
    c = 4096
    w = window(c)
    ref, rr, parts = bo.mix(w, b, SR, 0, p["Tt"], p["C"], p["o"] + mark - c, parts=True,
                            **{k: p[k] for k in ("duck", "threshold", "attack", "release")})
    assert c + y.size == ref.size
    full = np.concatenate([ref[:c], y])             # the context's outputs are not under test: they add no error
    assert abs(red - rr) <= 1e-3 * max(1.0, abs(rr)), (red, rr)
    return error_units(full, ref, parts), BED_TOL


def oracle_meter(eng, mark, got):
    m = SR // 10
    w = window(mark % m + 10 * m)              # whole sub-blocks of silence before: the slot's grid
    ref = lo.gate(lo.energies(w, SR), m)
    err = 0.0
    for g, r in zip(got[:3], ref):
        if np.isinf(r):
            assert g == r, (g, r)
        else:
            err = max(err, abs(float(g) - r))
    u = eng.resample(PROBE, 4 * SR, SR)
    peak = 20 * np.log10(max(np.abs(PROBE).max(), np.abs(u).max()))
    assert abs(float(got[3]) - peak) <= 4 * float(np.spacing(np.float32(abs(peak)))) + 1e-6, (float(got[3]), peak)
    return err, L_TOL


ORACLES = {"resample": oracle_resample, "watermark": oracle_watermark, "pitch": oracle_pitch,
           "time_stretch_1.25": oracle_stretch}


STAGE_NAMES = ["resample", "denoise", "pitch", "time_stretch_1.25", "time_stretch_0.9", "limiter", "eq", "compressor",
               "deesser", "reverb", "watermark", "bed", "loudness"]


@pytest.mark.parametrize("session", [0, 1], ids=["2^24,2^31-", "2^31+,2^32+"])
@pytest.mark.parametrize("name", STAGE_NAMES)
def test_probe_deep_in_a_slot(eng, name, session):
    stage, value, period = long_stage(eng, name)
    marks = SESSIONS[session]
    outs, last, secs = run(eng, stage, value, marks)
    ref_marks = [short(m, period) for m in marks]
    routs, rlast, _ = run(eng, stage, value, ref_marks)
    for s, mark in enumerate(marks):
        what = (name, mark, ref_marks[s])
        if stage.meter:
            assert np.array_equal(last[s], rlast[s]), (what, last[s], rlast[s])
            err, tol = oracle_meter(eng, mark, last[s])
        else:
            assert [o.size for o in outs[s]] == [o.size for o in routs[s]], what
            y = np.concatenate(outs[s])
            assert np.array_equal(y.view(np.uint32), np.concatenate(routs[s]).view(np.uint32)), what
            if stage.reduction:
                assert last[s] == rlast[s], (what, last[s], rlast[s])
            err, tol = None, None
            if name == "bed":
                err, tol = oracle_bed(eng, stage, mark, y, last[s])
            elif name in ORACLES:
                err, tol = ORACLES[name](eng, stage, mark, y)
        if err is not None:
            print(f"{name} mark {mark}: worst error {err:.3g} (bound {tol:g}), bit-identical to a {ref_marks[s]}-sample prefix")
            assert err <= tol, (what, err, tol)
        else:
            print(f"{name} mark {mark}: bit-identical to a {ref_marks[s]}-sample prefix")
    print(f"{name} marks {marks}: {secs:.1f} s")


def test_meter_to_its_history_cap(eng):
    """One meter slot at 8 kHz and the largest max_seconds the API accepts (2^20 s, 10 * 2^20 sub-blocks of 800
    samples) filled to its last sample: silence, then the probe ending at (hcap + 1) 800 - 1 samples, 8.4e9.  Its
    readings there against float64; the next sample is refused before anything is launched, and the slot keeps its
    readings and still takes END."""
    from viettts_b200._lib import VttsError
    rate, max_seconds = 8000, 1 << 20
    m, hcap = rate // 10, 10 * max_seconds
    cap = (hcap + 1) * m - 1                        # the most samples a slot holds: hcap complete sub-blocks
    mark = cap - PROBE.size
    dev = torch.device("cuda", 0)
    t0 = time.perf_counter()
    with eng.open_loudness_meter(1, F, rate, max_seconds=max_seconds) as mt:
        with pytest.raises(VttsError, match="max_seconds"):
            eng.open_loudness_meter(1, F, rate, max_seconds=max_seconds + 1)
        x_t = torch.zeros((1, F), dtype=torch.float32, device=dev)
        y_t = torch.zeros((1, 4), dtype=torch.float32, device=dev)
        probe_t = torch.from_numpy(PROBE).to(dev)
        pushes = [(n, None) for n, _, _ in plan(mark)[:-len(probe_chunks())]]
        off = 0
        for k in probe_chunks():
            pushes.append((k, off))
            off += k
        P = 0
        for i, (n, o) in enumerate(pushes):
            if o is not None:
                x_t[0, :n].copy_(probe_t[o:o + n])
            mt.push_device(x_t, np.array([n], np.int32), np.array([STREAM_BEGIN if i == 0 else 0], np.uint8), y_t)
            P += n
        assert P == cap
        r1 = y_t.cpu().numpy()[0].copy()
        c0 = eng.launch_count()
        with pytest.raises(VttsError, match="max_seconds"):
            mt.push_device(x_t, np.array([1], np.int32), np.zeros(1, np.uint8), y_t)
        assert eng.launch_count() == c0
        assert np.array_equal(y_t.cpu().numpy()[0], r1)
        mt.push_device(x_t, np.zeros(1, np.int32), np.array([STREAM_END], np.uint8), y_t)
        r2 = y_t.cpu().numpy()[0].copy()
    secs = time.perf_counter() - t0
    assert np.array_equal(r2[:3], r1[:3])
    w = window(mark % m + 10 * m)                  # whole sub-blocks of silence before: the slot's grid
    ref = lo.gate(lo.energies(w, rate), m)
    err = 0.0
    for g, v in zip(r2[:3], ref):
        assert np.isfinite(v), ref
        err = max(err, abs(float(g) - v))
    assert err <= L_TOL, (err, r2, ref)
    u = eng.resample(PROBE, 4 * rate, rate)
    peak = 20 * np.log10(max(np.abs(PROBE).max(), np.abs(u).max()))
    assert abs(float(r2[3]) - peak) <= 4 * float(np.spacing(np.float32(abs(peak)))) + 1e-6, (float(r2[3]), peak)
    print(f"meter at its cap of {cap} samples: worst error {err:.3g} LU (bound {L_TOL:g}); {secs:.1f} s")


# ---- a long-lived TTS slot ------------------------------------------------------------------------------------------------

LONG_FRAMES = (1 << 24) // config.HOP + 64        # the joined utterance passes 2^24 samples at the native rate


@pytest.fixture(scope="module")
def tts_long(acoustic_ckpt, hifigan_params):
    """an engine with the synthetic models, and sentences whose joined utterance passes LONG_FRAMES frames"""
    from test_gpu_audio_chain import SD, tts_tokens
    from viettts_b200 import synthetic
    from viettts_b200.engine import Engine
    e = Engine(0)
    e.load_acoustic(acoustic_ckpt)
    e.load_hifigan(hifigan_params)
    e.load_duration(synthetic.duration_ckpt(1234))
    e.set_precision("bf16x3")
    cand = [tts_tokens(5000 + i, 40 + i % 51) for i in range(1500)]
    tok = np.zeros((len(cand), 100), np.int32)
    for b, t in enumerate(cand):
        tok[b, :t.size] = t
    _, _, nf, ne = e.tts_plan(tok, [t.size for t in cand], silence_duration=SD)
    k = int(np.searchsorted(np.cumsum(ne), LONG_FRAMES)) + 1
    assert k <= len(cand)
    yield e, cand[:k], int(ne[:k].sum()), int(nf[:k].max())
    e.close()


def last_window_stages(eng, chain, wav):
    """The chain's frame-local and finite-memory stages over the last 10 s of the long utterance against float64: each
    stage's input is the device's previous stage over the whole utterance (one-shot calls, which the stream equals bit
    for bit), and float64 runs on a window that starts on the stage's grid, far enough back to cover its memory:
    the denoiser on 256-sample frames, the watermark on frames keyed from the window's absolute first frame
    (watermark_oracle.embed's frame0), the resampler from an input that is a multiple of `down`.  Returns
    {stage: (worst error, bound)}."""
    from test_denoise_cpu import TOL as DN_TOL
    from oracle import denoise_oracle as dno
    r0 = config.SAMPLE_RATE
    tail = 10 * r0
    worst = {}
    x = wav
    bias = eng.denoiser_bias()
    y = eng.denoise(x, chain.denoise)
    s0 = (x.size - tail - 4096) // 256 * 256
    ref = dno.denoise(x[s0:], chain.denoise, bias)
    sc = dno.error_scale(x[s0:], chain.denoise, bias)
    worst["dn"] = (rel(y[s0 + 2048:], ref[2048:], sc[2048:]), DN_TOL)
    x = eng.time_stretch(eng.pitch_shift(y, chain.semitones), chain.tempo)
    wm = chain.watermark
    y = eng.watermark(x, wm)
    s0 = (x.size - tail - 4096) // 256 * 256
    ref = wo.embed(x[s0:], wm["key"], np.float32(wm["strength"]), frame0=s0 // 256)
    worst["wm"] = (rel(y[s0 + 2048:], ref[2048:], embed_scale(x[s0:], wm["strength"])[2048:]), TOL_EMBED)
    if chain.output_rate is not None and chain.output_rate != r0:
        x = y
        rates = (r0, chain.output_rate)
        up, down, _ = ro.ratio(*rates)
        y = eng.resample(x, chain.output_rate)
        s0 = (x.size - tail - 4096) // down * down
        m0 = s0 * up // down + 4096 * up // down
        ref = ro.resample(x[s0:], *rates, m_range=(m0 - s0 * up // down, y.size - s0 * up // down))
        sc = ro.abs_sum(x[s0:], *rates, m_range=(m0 - s0 * up // down, y.size - s0 * up // down))
        worst["rs"] = (rel(y[m0:], ref, sc), RS_TOL)
    for k, (e, tol) in worst.items():
        assert e <= tol, (k, e, tol)
    return worst


@pytest.mark.parametrize("output_rate", [None, 48000], ids=["native", "48k"])
def test_long_tts_slot_equals_one_shot_chain(tts_long, output_rate):
    """One TTS stream slot, every audio stage on and the meter (test_gpu_audio_chain's `all48k` configuration, at the
    native rate and at 48 kHz), fed sentence after sentence through `append` past 2^24 samples: its audio equals
    AudioChain.run of tts_joined of the same sentences bit for bit, and its meter reading equals Engine.loudness of it"""
    from test_gpu_audio_chain import CONFIGS, SD
    from viettts_b200.engine import AudioChain
    eng, sents, frames, max_nf = tts_long
    opts = dict(CONFIGS["all48k"][0], output_rate=output_rate)
    t0 = time.perf_counter()
    pieces, reading = [], None
    with eng.open_tts_stream(1, 64, max_nf, 100, max_joined_frames=frames, **opts) as ts:
        got = ts.begin(0, sents[0], silence_duration=SD, more=True)
        for i, t in enumerate(sents[1:]):
            got += ts.append(0, t, more=i + 2 < len(sents))
        assert got == frames
        steps = 0
        while ts.busy().any():
            out = ts.step()
            pieces.append(out[0])
            m = ts.meter()
            if 0 in m:
                reading = m[0]
            steps += 1
    y = np.concatenate(pieces)
    t_stream = time.perf_counter() - t0
    t0 = time.perf_counter()
    wav = eng.tts_joined([sents], silence_duration=SD)[0][0]
    assert wav.size == frames * config.HOP
    want = AudioChain(**opts).run(eng, wav)
    t_one = time.perf_counter() - t0
    rate = output_rate or config.SAMPLE_RATE
    assert wav.size > 1 << 24
    assert y.shape == want.shape and np.array_equal(y.view(np.uint32), want.view(np.uint32)), (y.shape, want.shape)
    ref = np.array(eng.loudness(want, rate), np.float32)
    assert np.array_equal(np.array(reading, np.float32), ref), (reading, ref)
    worst = last_window_stages(eng, AudioChain(**opts), wav)
    print(f"long TTS slot ({output_rate or 'native'}): last 10 s against float64: "
          + ", ".join(f"{k} {v[0]:.3g} ({v[1]:g})" for k, v in worst.items()))
    print(f"long TTS slot ({output_rate or 'native'}): {len(sents)} sentences, {frames} frames, {y.size} output samples; "
          f"stream {t_stream:.1f} s in {steps} steps, one-shot chain {t_one:.1f} s")
