"""The audio chain's stage order and stream sizing, without a device.

`AudioChain.streams` opens the stream stages in order and hands each the previous one's output width (`out_pitch`) as
its input width.  That is right only if no stage ever emits more in one push than its `out_pitch`, for any input of
at most its own input width.  The largest push of a stage is the one with END (it releases what the stage held back);
it is derived here from the oracles' emission schedules (`emitted` / `released` counted from each output's last input)
for the worst position of the push, and compared with the width each stage states in include/viettts_b200.h.  The
meter of a chain must also hold a whole utterance: `max_frames` vocoder frames, slowed down by the time stretcher at
MIN_TEMPO, resampled and lengthened by the bed's tail.

The stream classes are replaced by stand-ins that record what `AudioChain.streams` gives them, so the hand-off code
itself runs here; tests/test_gpu_audio_chain.py checks the library's widths against `out_pitch_rule` and runs the
chain at its capacity edge on the device."""
import numpy as np
import pytest

from oracle import denoise_oracle as dno
from oracle import limiter_oracle as lm
from oracle import resample_oracle as ro
from oracle import time_stretch_oracle as tso
from viettts_b200 import config

ALL_ON = dict(denoise=0.5, semitones=3.0, tempo=0.8, watermark="key=1", eq="hs:6000:3", compress="voice", deess="voice",
              reverb="hall", bed="pink", limit=-1.0, meter=True)
ORDER = ["dn", "ps", "ts", "wm", "rs", "eq", "cp", "ds", "rv", "bd", "lm", "mt"]
STREAM_CLASSES = {"dn": "DenoiseStream", "ps": "PitchShiftStream", "ts": "TimeStretchStream", "wm": "WatermarkStream",
                  "rs": "ResampleStream", "eq": "EqStream", "cp": "CompressorStream", "ds": "DeesserStream",
                  "rv": "ReverbStream", "bd": "BedStream", "lm": "LimiterStream", "mt": "LoudnessMeter"}

# (AudioChain options, its stages in order): every stage on, then the tables of the per-stage modules, one row each
STAGE_ORDERS = [
    (dict(ALL_ON, output_rate=48000), ORDER),
    (dict(ALL_ON, output_rate=48000, limit=None, meter=False, loudness=-16.0), ORDER[:-1]),
    (dict(ALL_ON), ORDER[:4] + ORDER[5:]),
    (dict(output_rate=48000, compress="voice", reverb="room", bed="pink", limit=-1.0, meter=True), ["rs", "cp", "rv", "bd", "lm", "mt"]),
    (dict(bed="pink,duck=6", loudness=-16.0, encoding="ulaw"), ["bd", "lm"]),
    (dict(output_rate=48000, eq="hs:6000:3", compress="voice", deess="voice", reverb="hall", limit=-1.0, meter=True),
     ["rs", "eq", "cp", "ds", "rv", "lm", "mt"]),
    (dict(reverb="room", denoise=0.5, compress="voice"), ["dn", "cp", "rv"]),
    (dict(output_rate=48000, eq="hs:6000:3", compress="voice", deess="voice", limit=-1.0, meter=True), ["rs", "eq", "cp", "ds", "lm", "mt"]),
    (dict(deess="voice", denoise=0.5, compress="voice"), ["dn", "cp", "ds"]),
    (dict(output_rate=48000, eq="telephone", compress="voice", limit=-1.0, meter=True), ["rs", "eq", "cp", "lm", "mt"]),
    (dict(compress="voice", denoise=0.5), ["dn", "cp"]),
    (dict(output_rate=8000, eq="telephone", encoding="ulaw", meter=True), ["rs", "eq", "mt"]),
    (dict(denoise=0.5, watermark="key=1", output_rate=44100), ["dn", "wm", "rs"]),
    (dict(semitones=-2.0, tempo=1.5, watermark=7), ["ps", "ts", "wm"]),
    (dict(), []),
]


@pytest.mark.parametrize("opts,order", STAGE_ORDERS)
def test_stage_order(opts, order):
    from viettts_b200.engine import AudioChain
    assert [s[0] for s in AudioChain(**opts)._stages()] == order


def limiter_lookahead(rate: int) -> int:
    """the limiter stream's lookahead at the chain's 5 ms: W + 19 (limiter_oracle.stream_lookahead)"""
    return lm.stream_lookahead(lm.params(rate, 5.0, 100.0)[0])


def out_pitch_rule(name: str, width: int, chain) -> int:
    """the outputs per slot of a push's output buffer that include/viettts_b200.h states for a stage of `chain` opened
    with input width `width` (the meter has none)"""
    if name in ("dn", "ps", "wm"):
        return width + 1023
    if name == "ts":
        return 2 * width + 2048
    if name == "rs":
        up, down, half = ro.ratio(config.SAMPLE_RATE, chain.output_rate)
        return -(-(width * up + half + 1) // down)
    if name in ("eq", "cp", "ds"):
        return width
    if name == "rv":
        return width + 511
    if name == "bd":
        return width + chain.bed[0]["Tt"]
    if name == "lm":
        return width + limiter_lookahead(chain.rate)
    raise ValueError(name)


def largest_end_push(name: str, width: int, chain) -> int:
    """the most a stage emits in one push with END that brings at most `width` samples, over every number P of samples
    the slot received before it: total(P + width) - emitted(P), total the stage's whole output.  For the denoiser's STFT
    schedule, the resampler, the reverb and the limiter, P - emitted(P) repeats with a period of one hop, `down`
    inputs or one block, or stops growing once P passes the lookahead, and the sweeps cover that, so they find the
    worst P.  The time stretcher's schedule repeats only after many frames at some tempos (25 frames at 1.37), so its
    bound is derived instead (see below) and the sweep only checks it at a few positions."""
    from viettts_b200.engine import reverb_stream_emitted
    if name in ("dn", "ps", "wm"):          # the pitch shifter and the watermark share the denoiser's STFT schedule
        return max(P + width - dno.emitted(P) for P in range(0, 5 * dno.HOP))
    if name == "ts":
        # Before END every frame q with 256 q a + 0.5 <= P - 512 is scanned (rint adds at most 0.5), so Q > (P - 512.5) /
        # (256 a) frames and E(P) = 256 Q - 511 > (P - 512.5) / a - 511 (E = 0 and P <= 512 give less still).  END brings
        # the total to floor((P + w) / a + 0.5), so it emits less than (w + 512.5) / a + 511.5 <= 2 w + 1536.5 at a >= 1/2.
        bound = 2 * width + 1536
        swept = max(tso.stretch_length(P + width, a) - tso.stretch_emitted(P, a)
                    for a in (tso.MIN_TEMPO, 0.8, 1.0, 1.37, tso.MAX_TEMPO) for P in range(0, 8 * dno.HOP))
        assert swept <= bound, (width, swept, bound)
        return bound
    if name == "rs":
        rates = (config.SAMPLE_RATE, chain.output_rate)
        up, down, half = ro.ratio(*rates)
        return max(ro.emitted(P + width, *rates, end=True) - ro.emitted(P, *rates) for P in range(0, 2 * down + half // max(up, 1) + 2))
    if name in ("eq", "cp", "ds"):          # n_out = n_new
        return width
    if name == "rv":
        return max(reverb_stream_emitted(P + width, end=True) - reverb_stream_emitted(P) for P in range(0, 1024))
    if name == "bd":                        # every sample it brings, and the tail at END
        return width + chain.bed[0]["Tt"]
    if name == "lm":
        W = lm.params(chain.rate, 5.0, 100.0)[0]
        L = limiter_lookahead(chain.rate)
        return max(lm.released(P + width, W, end=True) - lm.released(P, W) for P in range(0, 2 * L + 2))
    raise ValueError(name)


def longest_output(chain, n: int) -> int:
    """the most samples the meter of `chain` receives for n vocoder samples: the time stretcher at MIN_TEMPO, the
    resampler's ceil(n up / down) and the bed's tail"""
    if chain.tempo is not None:
        n = tso.stretch_length(n, tso.MIN_TEMPO)
    if chain.output_rate is not None:
        n = ro.out_len(n, config.SAMPLE_RATE, chain.output_rate)
    if chain.bed is not None:
        n += chain.bed[0]["Tt"]
    return n


def opened(monkeypatch, chain, width: int, max_frames: int, S: int = 3):
    """[(name, input width, out_pitch or None, args)] of the stages `chain.streams` opens, through stand-ins that take
    the rule's out_pitch"""
    from viettts_b200 import engine
    log = []

    class FakeEngine:
        def prepare_beds(self, bed, rate):
            return ("bank", rate)

    for name, cls in STREAM_CLASSES.items():
        def make(e, max_streams, p, *args, _name=name):
            assert max_streams == S
            st = type("Stand-in", (), {})()
            if _name != "mt":
                st.out_pitch = out_pitch_rule(_name, p, chain)
            log.append((_name, p, getattr(st, "out_pitch", None), args))
            return st
        monkeypatch.setattr(engine, cls, make)
    for name, st in chain.streams(FakeEngine(), S, width, max_frames):
        assert log[-1][0] == name
    return log


CHAINS = [
    dict(ALL_ON, output_rate=48000),
    dict(ALL_ON, output_rate=44100, reverb="room", bed=["pink,seed=1,tail=10000", "pink,seed=2,level=-24,tail=10000"]),
    dict(ALL_ON, tempo=None),
    dict(output_rate=8000, eq="telephone", compress="voice", limit=-3.0, meter=True, encoding="ulaw"),
    dict(denoise=0.5, semitones=-4.0, tempo=0.5, watermark="key=9", meter=True),
    dict(ALL_ON, output_rate=48000, bed="pink,tail=10000", tempo=0.5),
]


@pytest.mark.parametrize("F", [1, 16, 64])
@pytest.mark.parametrize("opts", CHAINS)
def test_every_stage_holds_the_largest_push_of_the_one_before(monkeypatch, opts, F):
    """The first stage takes the vocoder stream's width 256 (F + 10); every next stage's input width is the previous
    stage's out_pitch, which holds the largest push that stage can emit at END."""
    from viettts_b200.engine import AudioChain
    chain = AudioChain(**opts)
    width = config.HOP * (F + 10)
    log = opened(monkeypatch, chain, width, 2000)
    assert [e[0] for e in log] == [s[0] for s in chain._stages()]
    p = width
    for name, p_in, pitch, _ in log:
        assert p_in == p, (name, p_in, p)                                   # the previous stage's width
        if name == "mt":
            break
        need = largest_end_push(name, p_in, chain)
        assert need <= pitch, (name, p_in, need, pitch)
        p = pitch


@pytest.mark.parametrize("max_frames", [1, 16, 937, 1000, 2000, 6250])
@pytest.mark.parametrize("opts", CHAINS)
def test_the_meter_holds_an_utterance_of_max_frames(monkeypatch, opts, max_frames):
    """The meter keeps 10 max_seconds + 1 sub-blocks of rate / 10 samples per slot (vtts_loudness_stream_push refuses a
    push past them); the chain's `seconds` must cover the longest utterance it can receive."""
    from viettts_b200.engine import AudioChain
    chain = AudioChain(**opts)
    if not chain.meter:
        pytest.skip("no meter")
    log = opened(monkeypatch, chain, config.HOP * 26, max_frames)
    name, _, _, args = log[-1]
    assert name == "mt"
    rate, seconds = args
    assert rate == chain.rate
    n = longest_output(chain, max_frames * config.HOP)
    assert n // (rate // 10) <= 10 * seconds, (n, rate, seconds)
