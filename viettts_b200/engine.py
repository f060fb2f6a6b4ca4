"""Engine: one libviettts_b200 context per GPU + the host-side plumbing around it.

Host buffers are numpy arrays (the reference's seams take/return numpy / jax
arrays on the host); device buffers are torch tensors used purely as memory
containers (`tensor.data_ptr()` is what crosses the C ABI)."""
from __future__ import annotations

import ctypes as C
import threading
from typing import NamedTuple

import numpy as np

from . import _lib, config, weights

DROPOUT_OFF, DROPOUT_MASK, DROPOUT_SEED, DROPOUT_REFERENCE = 0, 1, 2, 3


def _chunk_seed(seed: int, chunk: int) -> int:
    """Key of the on-device dropout stream for the chunk-th slice of an over-long batch (a distinct 64-bit key per
    chunk: `seed + offset` would alias the next seed's first chunk)."""
    return (int(seed) ^ (chunk * 0x9E3779B97F4A7C15)) & 0xFFFFFFFFFFFFFFFF


def _rng_seed(rng, *others) -> int:
    """The `seed` argument of VTTS_DROPOUT_REFERENCE for a checkpoint `rng` (uint32[2]): (rng[0] << 32) | rng[1].
    `others` are the mask / seed arguments of the same call, which must be None alongside `rng`."""
    if any(o is not None for o in others):
        raise ValueError("rng= selects the reference's own mask stream; it cannot be combined with masks= or seed=")
    w = np.asarray(rng).ravel()
    if w.size != 2 or not np.issubdtype(w.dtype, np.integer):
        raise ValueError(f"rng must hold exactly two integer words (the checkpoint's uint32[2] rng), got {np.asarray(rng).shape}")
    return ((int(w[0]) & 0xFFFFFFFF) << 32) | (int(w[1]) & 0xFFFFFFFF)
PRECISION_FP32, PRECISION_BF16X3, PRECISION_FP16 = 0, 1, 2
PRECISIONS = {"fp32": PRECISION_FP32, "bf16x3": PRECISION_BF16X3, "fp16": PRECISION_FP16}
MAX_ACOUSTIC_ROWS = 128   # rows per vtts_acoustic_forward call (csrc/nat.cu MAX_ROWS)


def resample_ratio(in_rate: int, out_rate: int):
    """(up, down): out_rate / in_rate in lowest terms, as vtts_resample takes it (each must be <= 1024)"""
    from math import gcd
    in_rate, out_rate = int(in_rate), int(out_rate)
    if in_rate <= 0 or out_rate <= 0:
        raise ValueError(f"sample rates must be positive, got {in_rate} -> {out_rate}")
    g = gcd(in_rate, out_rate)
    return out_rate // g, in_rate // g


def resample_length(n: int, in_rate: int, out_rate: int) -> int:
    """ceil(n * up / down): the samples `Engine.resample` makes of n input samples"""
    up, down = resample_ratio(in_rate, out_rate)
    return -(-int(n) * up // down)


DENOISE_BINS = config.N_FFT // 2 + 1   # 513
DENOISE_BIAS_FRAMES = 88                # the all-zero mel [1, 88, 80] the default denoiser bias is taken from


def _strength(s) -> float:
    s = float(s)
    if not (np.isfinite(s) and s >= 0):
        raise ValueError(f"denoise strength must be finite and >= 0, got {s}")
    return s


def _per_row(v, n: int, name: str, lo: float, hi: float, shown=None) -> np.ndarray:
    """float32 [n]: a scalar for every row, or one value per row, each finite and in [lo, hi] (errors show `shown`, by
    default v)"""
    a = np.asarray(v, np.float32)
    a = np.full(n, a, np.float32) if a.ndim == 0 else np.ascontiguousarray(a.reshape(-1), np.float32)
    if a.shape != (n,):
        raise ValueError(f"{name}: one value or one per row ({n}), got {np.shape(v)}")
    if not (np.all(np.isfinite(a)) and np.all((a >= lo) & (a <= hi))):
        raise ValueError(f"{name} must be finite and lie in [{lo:g}, {hi:g}], got {v if shown is None else shown}")
    return a


class _BeginParam(NamedTuple):
    """A per-row effect parameter that a stream slot takes with BEGIN and keeps until END."""
    name: str                       # keyword of the calls and of `TtsStream.begin`
    neutral: float                  # a slot's value before its first BEGIN
    lo: float
    hi: float
    default: float | None = None    # a push's value when the keyword is left out (None: required with BEGIN)
    host_check: bool = False        # a push checks the range here (else the library rejects a bad BEGIN value)
    optional: bool = False          # may be left out with BEGIN: the library gets NULL and the slots take `neutral`

    def rows(self, v, n: int) -> np.ndarray:
        return _per_row(v, n, self.name, self.lo, self.hi)


MAX_SEMITONES = 12.0
MIN_TEMPO, MAX_TEMPO = 0.5, 2.0
LIMIT_MAX_GAIN_DB = 70.0
SEMITONES = _BeginParam("semitones", 0.0, -MAX_SEMITONES, MAX_SEMITONES)
# the formant shift of the voice shifter; NaN (a slot's value without one): the formants follow the pitch
FORMANT = _BeginParam("formant", float("nan"), -MAX_SEMITONES, MAX_SEMITONES, optional=True)
TEMPO = _BeginParam("tempo", 1.0, MIN_TEMPO, MAX_TEMPO)
GAIN_DB = _BeginParam("gain_db", 0.0, -LIMIT_MAX_GAIN_DB, LIMIT_MAX_GAIN_DB, default=0.0, host_check=True)
BED = _BeginParam("bed", -1.0, -1.0, 7.0, default=0, host_check=True)     # a bank entry; the bank's size bounds it


EQ_MAX_SECTIONS = 8
EQ_PRESETS = {"telephone": "hp:300:4,lp:3400:4"}   # the ITU-T G.712 telephone band
# band name -> (vtts_eq_kind, its value names, how many of them may be left out)
_EQ_BANDS = {"hp": (0, ("F", "ORDER"), 1), "lp": (1, ("F", "ORDER"), 1), "ls": (2, ("F", "GAIN", "S"), 1),
             "hs": (3, ("F", "GAIN", "S"), 1), "pk": (4, ("F", "Q", "GAIN"), 0), "notch": (5, ("F", "Q"), 0)}


def _eq_stable(row) -> bool:
    """a section b0 b1 b2 a0 a1 a2 is finite, a0 != 0 and strictly stable with every pole radius <= 1 - 1e-6"""
    if not np.all(np.isfinite(row)) or row[3] == 0:
        return False
    a1, a2 = row[4] / row[3], row[5] / row[3]
    if not (abs(a2) < 1 and abs(a1) < 1 + a2):
        return False
    disc = a1 * a1 - 4 * a2      # the poles of z^2 + a1 z + a2
    return (np.sqrt(a2) if disc < 0 else (abs(a1) + np.sqrt(disc)) / 2) <= 1 - 1e-6


def eq_sections(spec, rate: int) -> np.ndarray:
    """float64 [K,6] (rows b0 b1 b2 a0 a1 a2, 1 <= K <= 8) of an equalizer `spec` at `rate` Hz, designed by the library
    (vtts_eq_design; needs no device).  `spec` is an sos array, or comma-separated bands: hp:F[:ORDER] and lp:F[:ORDER]
    (Butterworth, order 1..8, default 2), ls:F:GAIN[:S] and hs:F:GAIN[:S] (RBJ shelves, slope S in (0, 1], default 1),
    pk:F:Q:GAIN (RBJ peaking), notch:F:Q, or the preset `telephone` (hp:300:4,lp:3400:4).  F in [10, 0.45 rate] Hz, Q in
    [0.1, 30], GAIN in [-24, 24] dB, rate in [8000, 192000].  Raises ValueError for anything else, for more than 8
    sections, and for a section that is not finite and strictly stable."""
    try:
        r = float(rate)
    except (TypeError, ValueError):
        r = None
    if r is None or not (8000 <= r <= 192000 and r == int(r)):
        raise ValueError(f"eq: rate {rate} must be an integer in [8000, 192000]")
    r = int(r)
    if not isinstance(spec, str):
        sos = np.array(spec, np.float64, order="C")   # a copy in the [K][6] row-major layout the library reads
        if sos.ndim != 2 or sos.shape[1] != 6 or not 1 <= sos.shape[0] <= EQ_MAX_SECTIONS:
            raise ValueError(f"eq: an sos array must be [K,6] with 1 <= K <= {EQ_MAX_SECTIONS}, got {np.shape(spec)}")
        for j, row in enumerate(sos):
            if not _eq_stable(row):
                raise ValueError(f"eq: section {j} {row.tolist()} must be finite with a0 != 0 and strictly stable")
        return sos
    lib = _lib.load()
    rows = []
    for band in spec.split(","):
        band = band.strip().lower()
        if band in EQ_PRESETS:
            rows.append(eq_sections(EQ_PRESETS[band], r))
            continue
        name, *vals = band.split(":")
        if name not in _EQ_BANDS:
            raise ValueError(f"eq: unknown band {band!r} (hp, lp, ls, hs, pk, notch or {', '.join(EQ_PRESETS)})")
        kind, names, optional = _EQ_BANDS[name]
        if not len(names) - optional <= len(vals) <= len(names):
            raise ValueError(f"eq: band {band!r} takes {name}:{':'.join(names[:len(names) - optional])}"
                             + "".join(f"[:{n}]" for n in names[len(names) - optional:]))
        try:
            v = dict(zip(names, (float(s) for s in vals)))
        except ValueError:
            raise ValueError(f"eq: band {band!r} has a value that is not a number") from None
        order = v.get("ORDER", 2.0)
        if not (np.isfinite(order) and order == int(order)):
            raise ValueError(f"eq: band {band!r}: the order must be an integer in [1, 8]")
        buf = np.zeros((EQ_MAX_SECTIONS, 6), np.float64)
        k = C.c_int()
        rc = lib.vtts_eq_design(kind, r, v["F"], v.get("Q", v.get("S", 1.0)), v.get("GAIN", 0.0), int(order), _ptr(buf), C.byref(k))
        if rc != 0:
            raise ValueError(f"eq: band {band!r} at {r} Hz is out of range (F in [10, {0.45 * r:g}] Hz, ORDER in [1, 8], "
                             "Q in [0.1, 30], S in (0, 1], GAIN in [-24, 24] dB)")
        rows.append(buf[:k.value])
    sos = np.concatenate(rows) if rows else np.zeros((0, 6))
    if not 1 <= sos.shape[0] <= EQ_MAX_SECTIONS:
        raise ValueError(f"eq: {spec!r} makes {sos.shape[0]} sections (1 to {EQ_MAX_SECTIONS})")
    return sos


# the compressor's parameters in vtts_compress's order, with their ranges and the `voice` preset
COMPRESSOR_RANGES = {"threshold": (-60.0, 0.0), "ratio": (1.0, 20.0), "knee": (0.0, 24.0), "attack": (0.5, 200.0),
                     "release": (5.0, 5000.0), "makeup": (-24.0, 24.0)}
COMPRESSOR_PRESETS = {"voice": {"threshold": -24.0, "ratio": 3.0, "knee": 6.0, "attack": 5.0, "release": 80.0, "makeup": 0.0}}


def compressor_params(spec, rate: int) -> dict:
    """{threshold, ratio, knee, attack, release, makeup} (float32 values, in vtts_compress's order) of a compressor
    `spec` at `rate` Hz (an integer in [8000, 192000]).  `spec` is the preset `voice` (-24 dBFS threshold, 3:1 ratio,
    6 dB knee, 5 ms attack, 80 ms release, 0 dB makeup), comma-separated key=value pairs over those six keys, or a dict
    of them; keys left out take the voice preset.  threshold dBFS in [-60, 0], ratio in [1, 20], knee dB in [0, 24],
    attack ms in [0.5, 200], release ms in [5, 5000], makeup dB in [-24, 24].  Raises ValueError naming the key."""
    _check_rate("compress", rate)
    return _keyed_params("compress", spec, COMPRESSOR_RANGES, COMPRESSOR_PRESETS)


# the de-esser's parameters in vtts_deess's order, with their ranges and the `voice` preset; freq's upper end is a
# fraction of the rate (deesser_params puts in 0.45 rate), and the detector's ranges are the compressor's
DEESSER_RANGES = {"freq": (1000.0, 0.45), "threshold": (-60.0, 0.0), "ratio": (1.0, 20.0), "knee": (0.0, 24.0), "attack": (0.5, 200.0),
                  "release": (5.0, 5000.0), "range": (0.0, 24.0)}
DEESSER_PRESETS = {"voice": {"freq": 5000.0, "threshold": -30.0, "ratio": 4.0, "knee": 6.0, "attack": 1.0, "release": 60.0,
                             "range": 12.0}}


def deesser_params(spec, rate: int) -> dict:
    """{freq, threshold, ratio, knee, attack, release, range} (float32 values, in vtts_deess's order) of a de-esser
    `spec` at `rate` Hz (an integer in [8000, 192000]).  `spec` is the preset `voice` (5000 Hz crossover, -30 dBFS
    threshold, 4:1 ratio, 6 dB knee, 1 ms attack, 60 ms release, 12 dB range), comma-separated key=value pairs over
    those seven keys, or a dict of them; keys left out take the voice preset.  freq Hz in [1000, 0.45 rate] (so the voice
    preset needs rate >= 11112 Hz), range dB in [0, 24], the others in the compressor's ranges.  Raises ValueError
    naming the key."""
    _check_rate("deess", rate)
    ranges = dict(DEESSER_RANGES, freq=(1000.0, 0.45 * float(rate)))
    return _keyed_params("deess", spec, ranges, DEESSER_PRESETS)


# the synthetic room's parameters with their ranges (seed: an integer) and the presets; an IR may be at most 5 s long
REVERB_RANGES = {"rt60": (0.1, 4.0), "predelay": (0.0, 200.0), "mix": (0.0, 1.0), "seed": (0.0, float(2 ** 24))}
REVERB_PRESETS = {"room": {"rt60": 0.35, "predelay": 8.0, "mix": 0.15, "seed": 0.0},
                  "hall": {"rt60": 1.8, "predelay": 25.0, "mix": 0.22, "seed": 0.0}}
REVERB_MAX_IR_SECONDS = 5


def reverb_ir(rt60: float, predelay_ms: float, seed: int, rate: int) -> np.ndarray:
    """The synthetic room's impulse response (float32 [d + N]): d = round(predelay_ms rate / 1000) zeros, then Gaussian
    noise e = default_rng(seed).standard_normal(N), N = ceil(rt60 rate), under the envelope 10^(-3 i / (rt60 rate)) (60 dB
    down after rt60 seconds), scaled to unit energy in float64 and cast once."""
    d = int(np.round(float(predelay_ms) * rate / 1000.0))
    n = int(np.ceil(float(rt60) * rate))
    e = np.random.default_rng(int(seed)).standard_normal(n)
    h = np.zeros(d + n)
    h[d:] = e * 10.0 ** (-3.0 * np.arange(n) / (float(rt60) * rate))
    return (h / np.sqrt(np.sum(h * h))).astype(np.float32)


def reverb_params(spec, rate: int) -> dict:
    """{ir: float32 [L], mix: float32 value} of a reverb `spec` at `rate` Hz (an integer in [8000, 192000]).  `spec` is
    a preset (`room`: rt60 0.35 s, predelay 8 ms, mix 0.15; `hall`: rt60 1.8 s, predelay 25 ms, mix 0.22; seed 0),
    comma-separated key=value pairs over rt60, predelay, mix and seed (keys left out keep the room values), or a dict of
    them; these give the synthetic room of `reverb_ir`, and the dict also carries rt60, predelay and seed.  rt60 s in
    [0.1, 4], predelay ms in [0, 200], mix in [0, 1], seed an integer >= 0.  A dict may instead give `ir` (a float
    array of 1 to 5 rate finite taps, used as given, not normalized) and `mix` (default the room's).  Raises ValueError
    naming the key."""
    _check_rate("reverb", rate)
    rate = int(rate)
    if isinstance(spec, dict) and "ir" in spec:
        extra = set(spec) - {"ir", "mix"}
        if extra:
            raise ValueError(f"reverb: with ir= the only other key is mix, got {', '.join(sorted(extra))}")
        try:
            ir = np.ascontiguousarray(np.asarray(spec["ir"], np.float64).astype(np.float32)).ravel()
        except (TypeError, ValueError):
            raise ValueError("reverb: ir= must be an array of numbers") from None
        if not 1 <= ir.size <= REVERB_MAX_IR_SECONDS * rate:
            raise ValueError(f"reverb: ir has {ir.size} taps (1 to {REVERB_MAX_IR_SECONDS} s = {REVERB_MAX_IR_SECONDS * rate} at {rate} Hz)")
        if not np.all(np.isfinite(ir)):
            raise ValueError("reverb: ir taps must be finite")
        mix = float(np.float32(_keyed_params("reverb", {"mix": spec.get("mix", REVERB_PRESETS["room"]["mix"])}, REVERB_RANGES,
                                             REVERB_PRESETS, "room")["mix"]))
        return {"ir": ir, "mix": mix}
    p = {k: float(np.float32(v)) for k, v in _keyed_params("reverb", spec, REVERB_RANGES, REVERB_PRESETS, "room").items()}
    if p["seed"] != int(p["seed"]):
        raise ValueError(f"reverb: seed={p['seed']:g} must be an integer")
    p["seed"] = int(p["seed"])
    return dict(ir=reverb_ir(p["rt60"], p["predelay"], p["seed"], rate), **p)


# the bed's parameters with their ranges; `offset` is checked against the bed's length, and seed / length belong to
# the pink preset
BED_RANGES = {"level": (-60.0, -10.0), "duck": (0.0, 40.0), "threshold": (-60.0, 0.0), "attack": (0.5, 200.0),
              "release": (5.0, 5000.0), "fade_in": (0.0, 5000.0), "tail": (0.0, 10000.0), "xfade": (0.0, 1000.0),
              "offset": (0.0, 600.0)}
BED_DEFAULTS = {"level": -30.0, "duck": 12.0, "threshold": -40.0, "attack": 10.0, "release": 500.0, "fade_in": 250.0,
                "tail": 1000.0, "xfade": 50.0, "offset": 0.0}
BED_PINK_RANGES = {"seed": (0.0, float(2 ** 24)), "length": (0.5, 600.0)}
BED_PINK_DEFAULTS = {"seed": 0.0, "length": 8.0}
BED_MAX_SECONDS = 600
BED_MAX_BEDS = 8
# the keys a bank's beds may differ in: every other one is a parameter of the call
_BED_OWN = ("audio", "audio_rate", "level", "seed", "length")


def pink_bed(seed: int, seconds: float, rate: int) -> np.ndarray:
    """The `pink` preset's bed (float32 [round(seconds rate)]): white Gaussian noise default_rng(seed) shaped to a 1/f
    power spectrum in the frequency domain (bin k scaled by 1 / sqrt(k), DC removed), scaled to unit RMS in float64 and
    cast once.  The shaping is circular, so the bed loops without a seam of its own."""
    n = int(round(float(seconds) * rate))
    X = np.fft.rfft(np.random.default_rng(int(seed)).standard_normal(n))
    k = np.arange(X.size)
    X[0] = 0.0
    X[1:] /= np.sqrt(k[1:])
    v = np.fft.irfft(X, n)
    return (v / np.sqrt(np.mean(v * v))).astype(np.float32)


def bed_params(spec, rate: int) -> dict:
    """The bed of a `spec` at the chain rate `rate` (an integer in [8000, 192000] and a multiple of 10, where the bed's
    loudness is measured): {audio: float32, audio_rate, level, duck, threshold, attack, release, fade_in, tail, xfade,
    offset (float32 values), Nb: samples at `rate`, Fi, Tt, C, o: fade_in, tail, xfade and offset in samples at `rate`
    (rint)}.  `spec` is the preset `pink` with comma-separated key=value pairs after it (`pink,seed=3,duck=18`: seeded
    pink noise of `length` s, default 8, see `pink_bed`), or a dict that gives `audio` (a mono float array at
    `audio_rate`, default `rate`; any ratio the resampler takes, each reduced term at most 1024) or leaves it out for
    the pink preset.  level LUFS in [-60, -10] (default -30), duck dB in [0, 40] (12), threshold dBFS in [-60, 0] (-40),
    attack ms in [0.5, 200] (10), release ms in [5, 5000] (500), fade_in ms in [0, 5000] (250), tail ms in [0, 10000]
    (1000), xfade ms in [0, 1000] (50) with 2 C below the bed's samples, offset s in [0, the bed's length) (0).  The bed
    lasts 0.5 s at `rate` to 600 s.  Raises ValueError naming the key."""
    _check_rate("bed", rate)
    rate = int(rate)
    if rate % 10:
        raise ValueError(f"bed: rate {rate} must be a multiple of 10 (the bed's loudness is measured at it)")
    if isinstance(spec, str):
        head, *items = [t.strip() for t in spec.split(",")]
        if head.lower() != "pink":
            raise ValueError(f"bed: a string spec is the preset 'pink' with key=value pairs after it, got {head!r} "
                             "(pass a dict with audio= for a bed of your own)")
        given = {}
        for item in items:
            key, eq, val = item.partition("=")
            if not eq:
                raise ValueError(f"bed: {item!r} is not key=value (keys {', '.join([*BED_RANGES, *BED_PINK_RANGES])})")
            given[key.strip().lower()] = val.strip()
    elif isinstance(spec, dict):
        given = dict(spec)
    else:
        raise ValueError(f"bed: a spec is a string or a dict, got {type(spec).__name__}")
    audio, audio_rate = given.pop("audio", None), given.pop("audio_rate", None)
    pink = audio is None
    if pink and audio_rate is not None:
        raise ValueError("bed: audio_rate= goes with audio=")
    ranges = dict(BED_RANGES, **(BED_PINK_RANGES if pink else {}))
    p = _keyed_params("bed", given, ranges, {"pink": dict(BED_DEFAULTS, **(BED_PINK_DEFAULTS if pink else {}))}, "pink")
    if pink:
        if p["seed"] != int(p["seed"]):
            raise ValueError(f"bed: seed={p['seed']:g} must be an integer")
        p["seed"] = int(p["seed"])
        audio, audio_rate = pink_bed(p["seed"], p["length"], rate), rate
    else:
        try:
            audio = np.ascontiguousarray(np.asarray(audio, np.float64).astype(np.float32))
        except (TypeError, ValueError):
            raise ValueError("bed: audio= must be an array of numbers") from None
        if audio.ndim != 1:
            raise ValueError(f"bed: audio must be mono [N], got {audio.shape}")
        if not np.all(np.isfinite(audio)):
            raise ValueError("bed: audio samples must be finite")
        try:
            audio_rate = rate if audio_rate is None else int(audio_rate)
            up, down = resample_ratio(audio_rate, rate)
        except (TypeError, ValueError):
            raise ValueError(f"bed: audio_rate={audio_rate!r} must be a positive integer") from None
        if max(up, down) > 1024:
            raise ValueError(f"bed: audio_rate {audio_rate} -> {rate} reduces to {up}/{down} (at most 1024 each)")
    nb = resample_length(audio.size, audio_rate, rate)
    if not (2 * nb >= rate and audio.size <= BED_MAX_SECONDS * audio_rate):
        raise ValueError(f"bed: audio lasts {audio.size / audio_rate:g} s (0.5 s at {rate} Hz to {BED_MAX_SECONDS} s)")
    n = {k: int(np.rint(p[k] * rate / 1000.0)) for k in ("fade_in", "tail", "xfade")}
    o = int(np.rint(p["offset"] * rate))
    if 2 * n["xfade"] >= nb:
        raise ValueError(f"bed: xfade={p['xfade']:g} ms makes 2 x {n['xfade']} samples, not below the bed's {nb}")
    if o >= nb:
        raise ValueError(f"bed: offset={p['offset']:g} s lies past the bed's {nb / rate:g} s")
    return dict(audio=audio, audio_rate=audio_rate, **p, Nb=nb, Fi=n["fade_in"], Tt=n["tail"], C=n["xfade"], o=o)


def bed_specs(spec, rate: int) -> list:
    """`bed_params` of a spec or of a list of 1 to 8 specs (a bank), which may differ only in their audio, level and
    pink seed and length"""
    specs = list(spec) if isinstance(spec, (list, tuple)) else [spec]
    if not 1 <= len(specs) <= BED_MAX_BEDS:
        raise ValueError(f"bed: {len(specs)} beds (1 to {BED_MAX_BEDS})")
    ps = [bed_params(s, rate) for s in specs]
    shared = [k for k in BED_RANGES if k not in _BED_OWN]
    for i, q in enumerate(ps[1:], 1):
        for k in shared:
            if q[k] != ps[0][k]:
                raise ValueError(f"bed: bed {i} has {k}={q[k]:g} and bed 0 {k}={ps[0][k]:g} (the beds of a bank share every "
                                 f"key but {', '.join(_BED_OWN)})")
        if 2 * ps[0]["C"] >= q["Nb"] or ps[0]["o"] >= q["Nb"]:
            raise ValueError(f"bed: bed {i}'s {q['Nb']} samples do not hold the xfade and offset")
    return ps


class BedBank(NamedTuple):
    """The prepared beds of a bank on the device (Engine.prepare_beds): each resampled to `rate` and scaled to its level."""
    audio: "object"          # float32 CUDA tensor [sum of lengths], bed k at offsets[k]
    offsets: np.ndarray      # int64 [K]
    lengths: np.ndarray      # int32 [K]
    params: list             # bed_params of each bed
    rate: int

    def args(self) -> tuple:
        """the bank and call parameters of vtts_bed_* after the rate: bank, offsets, lengths, K, duck, threshold, attack,
        release, fade_in, tail, xfade, offset"""
        p = self.params[0]
        return (_ptr(self.audio), _ptr(self.offsets), _ptr(self.lengths), len(self.params), p["duck"], p["threshold"],
                p["attack"], p["release"], p["Fi"], p["Tt"], p["C"], p["o"])

    def index(self, bed, n: int) -> np.ndarray:
        """int32 [n]: a bank entry for every row, or one per row, each in [-1, K)"""
        a = np.asarray(bed)
        if a.dtype.kind not in "iu" and not (a.dtype.kind == "f" and np.all(np.isfinite(a)) and np.all(a == np.round(a))):
            raise ValueError(f"bed index must be integers, got {bed!r}")
        a = np.full(n, a, np.int64) if a.ndim == 0 else a.reshape(-1).astype(np.int64)
        if a.shape != (n,):
            raise ValueError(f"bed index: one value or one per row ({n}), got {np.shape(bed)}")
        if np.any((a < -1) | (a >= len(self.params))):
            raise ValueError(f"bed index must lie in [-1, {len(self.params) - 1}], got {bed!r}")
        return a.astype(np.int32)


WATERMARK_MAX_STRENGTH = 0.3
WATERMARK_STRENGTH = 0.1                           # the default strength
WATERMARK_ALIGNED_THRESHOLD = 5.0                  # P(z >= 5) <= exp(-12.5) = 3.7e-6 for audio without the key
WATERMARK_SEARCH_THRESHOLD = 6.5                   # 1024 offsets: P(max z >= 6.5) <= 1024 exp(-21.1) = 7e-7
WATERMARK_MAX_KEYS = 4096                          # keys per detect call


def _watermark_key(v) -> int:
    """an integer in [0, 2^64) (a bool, a float or a string of anything else raises ValueError)"""
    if isinstance(v, (bool, np.bool_)) or isinstance(v, (float, np.floating)):
        raise ValueError(f"watermark: key {v!r} must be an integer in [0, 2^64)")
    try:
        k = int(v, 0) if isinstance(v, str) else int(v)
    except (TypeError, ValueError):
        raise ValueError(f"watermark: key {v!r} must be an integer in [0, 2^64)") from None
    if not 0 <= k < 2 ** 64:
        raise ValueError(f"watermark: key {k} must be an integer in [0, 2^64)")
    return k


def watermark_params(spec) -> dict:
    """{key: int, strength: float32 value} of a watermark `spec`: a bare integer key (an int or a string such as
    "12345" or "0x3039"), comma-separated `key=…,strength=…`, or a dict of them.  The key is an integer in [0, 2^64);
    strength lies in [0, 0.3] (default 0.1; 0 leaves the audio exactly as it is).  Raises ValueError naming the key."""
    if isinstance(spec, dict):
        given = dict(spec)
    elif isinstance(spec, str) and "=" in spec:
        given = {}
        for part in spec.split(","):
            k, eq, v = part.partition("=")
            k = k.strip().lower()
            if not eq or not k:
                raise ValueError(f"watermark: {part.strip()!r} is not key=value")
            given[k] = v.strip()
    else:
        given = {"key": spec}
    extra = set(given) - {"key", "strength"}
    if extra:
        raise ValueError(f"watermark: unknown key {sorted(extra)[0]!r} (keys key, strength)")
    if "key" not in given:
        raise ValueError("watermark: key= is required")
    key = _watermark_key(given["key"])
    try:
        eps = float(given.get("strength", WATERMARK_STRENGTH))
    except (TypeError, ValueError):
        raise ValueError(f"watermark: strength={given['strength']!r} must be a number") from None
    if not 0.0 <= np.float32(eps) <= np.float32(WATERMARK_MAX_STRENGTH):      # NaN fails too; as the library compares
        raise ValueError(f"watermark: strength={eps:g} must lie in [0, {WATERMARK_MAX_STRENGTH:g}]")
    return {"key": key, "strength": float(np.float32(eps))}


def watermark_keys(keys) -> np.ndarray:
    """uint64 [K] of one key or a list of 1 to 4096 keys, each an integer in [0, 2^64)"""
    ks = [keys] if np.ndim(keys) == 0 else list(np.asarray(keys, object).ravel())
    if not 1 <= len(ks) <= WATERMARK_MAX_KEYS:
        raise ValueError(f"watermark: {len(ks)} keys (1 to {WATERMARK_MAX_KEYS})")
    return np.array([_watermark_key(k) for k in ks], np.uint64)


ENCODINGS = {"pcm16": 0, "ulaw": 1, "alaw": 2}       # vtts_encoding
ENCODING_DTYPES = {"pcm16": np.int16, "ulaw": np.uint8, "alaw": np.uint8}


def encoding_name(encoding) -> str:
    """the name of a wire encoding ('pcm16', 'ulaw' or 'alaw'; anything else raises ValueError)"""
    if encoding not in ENCODINGS:
        if isinstance(encoding, str) and encoding.split(",")[0] == "flac":
            raise ValueError(f"encoding {encoding!r}: FLAC codes frames, not samples; use Engine.encode_flac")
        raise ValueError(f"encoding {encoding!r} must be one of {', '.join(ENCODINGS)}")
    return encoding


FLAC_BLOCKS = (256, 512, 1024, 2048, 4096)
FLAC_HEADER_BYTES = 42


def flac_rate(rate) -> int:
    """`rate` if a FLAC frame header can state it (vtts_flac_rate_code: a table rate, kHz <= 255, Hz <= 65535, tens of Hz
    <= 655350)"""
    r = int(rate)
    if r != rate or not 0 < r < 2**31 or _lib.load().vtts_flac_rate_code(r) < 0:
        raise ValueError(f"flac: rate {rate} has no frame-header code (kHz <= 255, Hz <= 65535 or tens of Hz <= 655350)")
    return r


def flac_block(block) -> int:
    if block not in FLAC_BLOCKS:
        raise ValueError(f"flac: block {block} must be one of {', '.join(map(str, FLAC_BLOCKS))}")
    return int(block)


def flac_params(spec) -> dict:
    """{'block': N} of a FLAC spec: 'flac' (block 4096) or 'flac,block=N' with N in FLAC_BLOCKS (ValueError otherwise)"""
    parts = str(spec).split(",") if isinstance(spec, str) else [None]
    if parts[0] != "flac":
        raise ValueError(f"flac spec {spec!r} must be 'flac' or 'flac,block=N'")
    out = {"block": 4096}
    for kv in parts[1:]:
        k, eq, v = kv.partition("=")
        if k.strip() != "block" or not eq:
            raise ValueError(f"flac spec {spec!r}: unknown setting {kv!r} (block=N)")
        try:
            out["block"] = flac_block(int(v))
        except ValueError:
            raise ValueError(f"flac spec {spec!r}: block must be one of {', '.join(map(str, FLAC_BLOCKS))}") from None
    return out


def flac_bound(S: int, block: int = 4096) -> int:
    """bytes per row that no FLAC stream of a row of S samples exceeds (vtts_flac_bound)"""
    return int(_lib.load().vtts_flac_bound(int(S), flac_block(block)))


class WatermarkDetection(NamedTuple):
    z: np.ndarray          # float32 [B, K] (or [K] for one row): the detection score
    offset: np.ndarray     # int32, same shape: where sample 0 sits in the mark's 65536-sample period at 16 kHz
    detected: np.ndarray   # bool, same shape: z at or above the mode's threshold


def _check_rate(what: str, rate):
    try:
        r = float(rate)
    except (TypeError, ValueError):
        r = None
    if r is None or not (8000 <= r <= 192000 and r == int(r)):
        raise ValueError(f"{what}: rate {rate} must be an integer in [8000, 192000]")


def _keyed_params(what: str, spec, ranges: dict, presets: dict, default: str = "voice") -> dict:
    """the float32 values of a `spec` (a preset name, comma-separated key=value pairs, or a dict) over `ranges`, keys
    left out taking presets[default]; every value must lie in its range.  Raises ValueError naming the key."""
    if isinstance(spec, str):
        given = {}
        s = spec.strip().lower()
        if s not in presets:
            for item in s.split(","):
                key, eq, val = item.strip().partition("=")
                if not eq:
                    raise ValueError(f"{what}: {item.strip()!r} is not key=value (keys {', '.join(ranges)}) "
                                     f"or a preset ({', '.join(presets)})")
                given[key.strip()] = val.strip()
    elif isinstance(spec, dict):
        given = dict(spec)
    else:
        raise ValueError(f"{what}: a spec is a string or a dict, got {type(spec).__name__}")
    out = dict(presets[s] if isinstance(spec, str) and s in presets else presets[default])
    for key, val in given.items():
        if key not in ranges:
            raise ValueError(f"{what}: unknown key {key!r} (keys {', '.join(ranges)})")
        try:
            v = float(np.float32(float(val)))
        except (TypeError, ValueError):
            raise ValueError(f"{what}: {key}={val!r} is not a number") from None
        lo, hi = ranges[key]
        if not (np.isfinite(v) and lo <= v <= hi):
            raise ValueError(f"{what}: {key}={val} must lie in [{lo:g}, {hi:g}]")
        out[key] = v
    for key, v in out.items():       # the preset's values too: a range may depend on the rate
        lo, hi = ranges[key]
        if not lo <= v <= hi:
            raise ValueError(f"{what}: {key}={v:g} (the {default} preset's) must lie in [{lo:g}, {hi:g}] at this rate")
    return out


def _ptr(a):
    if a is None:
        return None
    if isinstance(a, np.ndarray):
        return a.ctypes.data
    return a.data_ptr()  # torch tensor


def _np(a, dtype, shape=None, what="array"):
    a = np.ascontiguousarray(np.asarray(a), dtype=dtype)
    if shape is not None and tuple(a.shape) != tuple(shape):
        raise ValueError(f"{what}: expected shape {tuple(shape)}, got {tuple(a.shape)}")
    return a


def _wav_rows(wav, lengths=None):
    """(x f32 [B,S], lengths int32 [B] or None, one) of a one-shot host call: a host [S] or [B,S] array as rows, its
    row lengths, and whether it was a single row"""
    x = _np(wav, np.float32)
    one = x.ndim == 1
    x = x[None] if one else x
    if x.ndim != 2:
        raise ValueError(f"wav must be [S] or [B,S], got {np.shape(wav)}")
    return x, None if lengths is None else _np(lengths, np.int32, (x.shape[0],), "lengths"), one


def _out_tensor(out, shape, device, what="out"):
    """`out` checked to be a contiguous float32 tensor of `shape`, or a new one on `device`"""
    import torch
    if out is None:
        return torch.empty(shape, dtype=torch.float32, device=device)
    if tuple(out.shape) != shape or out.dtype != torch.float32 or not out.is_contiguous() or out.device != torch.device(device):
        raise ValueError(f"{what} must be contiguous float32 [{', '.join(map(str, shape))}] on {device}")
    return out


def _torch_code_dtype(encoding: str):
    import torch
    return torch.int16 if encoding == "pcm16" else torch.uint8


def _code_tensor(out, shape, encoding: str, device):
    """`out` checked to be a contiguous code tensor of `shape` for `encoding`, or a new one on `device`"""
    import torch
    dt = _torch_code_dtype(encoding)
    if out is None:
        return torch.empty(shape, dtype=dt, device=device)
    if tuple(out.shape) != shape or out.dtype != dt or not out.is_contiguous() or out.device != torch.device(device):
        raise ValueError(f"out must be contiguous {dt} [{', '.join(map(str, shape))}] on {device}")
    return out


def _dev_rows(x_t, out, stream, width=None):
    """(B, S, out, CUDA stream) of a one-shot device call on x_t, a contiguous float32 CUDA tensor [B,S]: `out` checked
    or made as [B, width] (default S), and the caller's stream or else the current one"""
    import torch
    assert x_t.is_cuda and x_t.dtype == torch.float32 and x_t.is_contiguous() and x_t.dim() == 2
    B, S = x_t.shape
    out = _out_tensor(out, (B, S if width is None else width), x_t.device)
    return B, S, out, torch.cuda.current_stream(x_t.device).cuda_stream if stream is None else stream


class Engine:
    """A context on one H100.  Not thread-safe (like the C context)."""

    def __init__(self, device: int = 0):
        self.lib = _lib.load()
        self.device = int(device)
        h = _lib.c_ctx()
        rc = self.lib.vtts_create(self.device, C.byref(h))
        if rc != 0:
            msg = self.lib.vtts_last_error(None)
            raise _lib.VttsError(rc, msg.decode() if msg else "?")
        self.h = h
        self._hifigan_key = None
        self._acoustic_key = None
        self._duration_key = None
        self._mel_fb = None         # host copy of the filterbank on the device (None: none loaded)
        self._denoise_bias = None   # default denoiser bias of the loaded generator in the current mode (denoiser_bias)
        self._reverb_irs = {}       # (string spec, rate, device) -> (IR on the device, mix) of reverb_forward
        self._bed_banks = {}        # (string spec(s), rate) -> BedBank of mix_bed / mix_bed_forward

    def close(self):
        if getattr(self, "h", None):
            self.lib.vtts_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _ck(self, rc):
        _lib.check(self.h, rc)

    # ---- info ----
    def device_info(self) -> dict:
        sm, ma, mi, hb = C.c_int(), C.c_int(), C.c_int(), C.c_int64()
        self._ck(self.lib.vtts_device_info(self.h, C.byref(sm), C.byref(ma), C.byref(mi), C.byref(hb)))
        return dict(sm_count=sm.value, cc=(ma.value, mi.value), hbm_bytes=hb.value)

    def launch_count(self) -> int:
        return int(self.lib.vtts_launch_count(self.h))

    def last_stage_ms(self, stage: int) -> float:
        ms = C.c_float()
        self._ck(self.lib.vtts_last_stage_ms(self.h, stage, C.byref(ms)))
        return float(ms.value)

    def set_precision(self, mode) -> None:
        """'fp32' (strict, FMA pipe), 'bf16x3' (wgmma tensor cores, split-bf16, fp32 accumulate; the default) or 'fp16'
        (fast generator: one fp16 product per operand pair, fp32 accumulate, waveform L-inf <= 3e-3 against float64 on
        synthetic weights; every other model runs as in 'bf16x3')."""
        m = PRECISIONS.get(mode, mode)
        self._ck(self.lib.vtts_set_precision(self.h, int(m)))
        self._denoise_bias = None

    def debug_conv1d(self, precision, x_t, w_t, bias_t, k, dil, pre_slope=1.0, resid_t=None, len_t=None):
        """Test hook: one conv layer on torch CUDA tensors through either arithmetic path."""
        import torch
        B, T, Cin = x_t.shape
        Cout = w_t.shape[2]
        out = torch.empty((B, T, Cout), dtype=torch.float32, device=x_t.device)
        m = PRECISIONS.get(precision, precision)
        self._ck(self.lib.vtts_debug_conv1d(self.h, int(m), _ptr(x_t), _ptr(w_t), _ptr(bias_t), _ptr(resid_t), _ptr(len_t),
                                            B, T, Cin, Cout, int(k), int(dil), float(pre_slope), _ptr(out)))
        return out

    POST_ACTS = {"none": 0, "tanh": 1, "relu": 2}

    def debug_conv_dispatch(self, precision, xs, ws, biases, k, dil=1, bns=None, resids=None, post_act="none", len_t=None, outs=None):
        """Test hook: len(xs) convs of one shape through the shared conv dispatcher of the acoustic and duration models,
        on torch CUDA tensors.  xs[p] [B,T,Cin], ws[p] [k,Cin,Cout], biases[p] [Cout], bns[p] None or [4,Cout] (scale,
        offset, mean, var), resids[p] None or [B,T,Cout]; post_act 'none', 'tanh' or 'relu'.  Writes outs[p] [B,T,Cout]
        (allocated when not given) except the rows at or past len_t[b], and returns outs."""
        import torch
        n = len(xs)
        B, T, Cin = xs[0].shape
        Cout = ws[0].shape[2]
        if outs is None:
            outs = [torch.empty((B, T, Cout), dtype=torch.float32, device=xs[0].device) for _ in range(n)]

        def arr(ts):
            return None if ts is None else (C.c_void_p * n)(*[_ptr(t) for t in ts])

        m = PRECISIONS.get(precision, precision)
        self._ck(self.lib.vtts_debug_conv_dispatch(self.h, int(m), n, arr(xs), arr(ws), arr(biases), arr(bns), arr(resids), arr(outs),
                                                   _ptr(len_t), B, T, Cin, Cout, int(k), int(dil), self.POST_ACTS[post_act]))
        return outs

    def debug_pair(self, x_t, w1_t, b1_t, w2_t, b2_t, k, dil, slope=0.1, len_t=None):
        """Test hook: one fused ResBlock pair on torch CUDA tensors (tensor-core path; fp16 operands when the engine is
        in 'fp16', bf16x3 otherwise)."""
        import torch
        B, T, Cc = x_t.shape
        out = torch.empty_like(x_t)
        self._ck(self.lib.vtts_debug_pair(self.h, _ptr(x_t), _ptr(w1_t), _ptr(b1_t), _ptr(w2_t), _ptr(b2_t), _ptr(len_t),
                                          B, T, Cc, int(k), int(dil), float(slope), _ptr(out)))
        return out

    HIFIGAN_LAYERS = 18   # 0 conv_pre, 1..4 ConvTranspose of stage i - 1, 5 + 3i + m ResBlock step (i, m), 17 conv_post

    def debug_hifigan_layer(self, layer, xs, outs, n_frames_t=None, T=None):
        """Test hook (vtts_debug_hifigan_layer): exactly one layer of the generator forward on torch CUDA tensors, with
        the loaded weights, the engine's precision mode and fused-pair setting.  xs: one tensor (layers 0 and 1) or three
        (the chains of a stage), [B, rows, C]; outs: one tensor (three for the ResBlock steps 5..16), written in place
        except the rows at or past n_frames_t[b] times the stage's rows per mel frame.  T (mel frames) defaults to the
        rows of xs[0] divided by the stage's rows per mel frame."""
        scale = [1, 1, 8, 64, 128] + [8] * 3 + [64] * 3 + [128] * 3 + [256] * 3 + [256]
        B, rows = xs[0].shape[:2]
        if T is None:
            T = rows // scale[layer]
        arr = lambda ts: (C.c_void_p * len(ts))(*[_ptr(t) for t in ts])  # noqa: E731
        self._ck(self.lib.vtts_debug_hifigan_layer(self.h, int(layer), arr(xs), arr(outs), _ptr(n_frames_t), int(B), int(T)))
        return outs

    PAIR_KERNELS = {"smem": 0, "tmem": 1, "smem2": 2}

    def set_fused_pairs(self, on: bool, kind: str | None = None):
        """Run the C <= 64 ResBlock pairs in the fused pair kernel (off: two tensor-core conv launches per pair).
        kind selects its form: "smem2" 256-row tiles (the default), "tmem" the same with conv2's A operand in registers
        (register-A wgmma), "smem" 128-row tiles."""
        flags = 0x200 | ((1 if on else 0) << 10)
        if kind is not None:
            flags |= 0x800 | (self.PAIR_KERNELS[kind] << 12)
        self._ck(self.lib.vtts_debug_tc_stats(self.h, flags, None))
        self._denoise_bias = None   # the generator's output (and so the default bias) may change in its last bits

    def tc_stats(self, enable=True):
        """Per-CTA stall counters of the last tensor-core conv launch (see vtts_debug_tc_stats)."""
        out = np.zeros((256, 16), np.int64)
        self._ck(self.lib.vtts_debug_tc_stats(self.h, 1 if enable else 0, _ptr(out)))
        return out

    SUBSTAGES = {1: "acoustic.encoder", 2: "acoustic.upsample", 3: "acoustic.cond_gemm", 4: "acoustic.decoder_scan",
                 5: "acoustic.projection", 6: "acoustic.postnet", 9: "hifigan.conv_pre", 10: "hifigan.stage0", 11: "hifigan.stage1",
                 12: "hifigan.stage2", 13: "hifigan.stage3", 14: "hifigan.conv_post", 17: "teacher.encoder_upsample",
                 18: "teacher.prenet_hoisted_gemm", 19: "teacher.zoneout_scan", 20: "teacher.projection_postnet"}

    def substages(self, enable=True) -> dict:
        """Per-kernel-group device times (ms) of the forward calls since the previous call (vtts_debug_substages);
        `enable` switches the event recording on/off for the following calls."""
        out = np.zeros(24, np.float32)
        self._ck(self.lib.vtts_debug_substages(self.h, 1 if enable else 0, _ptr(out)))
        return {name: float(out[i]) for i, name in self.SUBSTAGES.items() if out[i] > 0}

    # ---- weights ----
    def _load(self, fn, pack, src):
        blob = pack(src) if isinstance(src, dict) else src
        n = int(blob.size if isinstance(blob, np.ndarray) else blob.numel())
        if isinstance(blob, np.ndarray):
            blob = _np(blob, np.float32)
        self._ck(fn(self.h, _ptr(blob), n))

    def load_hifigan(self, params, key=None):
        """params: Haiku-layout dict, a packed float32 numpy blob, or a torch CUDA
        tensor holding the blob (e.g. received through an NCCL broadcast)."""
        self._load(self.lib.vtts_load_hifigan, weights.pack_hifigan, params)
        self._hifigan_key = key if key is not None else object()
        self._denoise_bias = None

    def load_acoustic(self, ckpt, key=None):
        self._load(self.lib.vtts_load_acoustic, weights.pack_acoustic, ckpt)
        self._acoustic_key = key if key is not None else object()

    def load_duration(self, ckpt, key=None):
        """ckpt: the duration checkpoint dict (params/aux), a packed numpy blob, or a torch CUDA tensor."""
        self._load(self.lib.vtts_load_duration, weights.pack_duration, ckpt)
        self._duration_key = key if key is not None else object()

    def broadcast_weights(self, nccl_comm, root: int, is_root: bool, stream=None):
        """vtts_broadcast_weights: the root's loaded models reach every rank's context by one grouped ncclBroadcast.
        `nccl_comm`: an ncclComm_t as ctypes.c_void_p / int (e.g. parallel.NcclComm(...).handle)."""
        self._ck(self.lib.vtts_broadcast_weights(self.h, nccl_comm, int(root), 1 if is_root else 0, stream))
        self._denoise_bias = None
        if not is_root:
            self._hifigan_key = self._acoustic_key = self._duration_key = object()

    def load_mel_filterbank(self, fb=None):
        """The filterbank f32 [80,513] of `melspec` and `melspec_forward` (by default the Slaney bank of
        weights.mel_filterbank(), what MelFilter(16000, 1024, 80) builds).  `gta` always uses the default bank."""
        fb = _np(weights.mel_filterbank() if fb is None else fb, np.float32, (config.MEL_DIM, config.N_FFT // 2 + 1), "filterbank").copy()
        self._mel_fb = None
        self._ck(self.lib.vtts_load_mel_filterbank(self.h, _ptr(fb), fb.shape[0], fb.shape[1]))
        self._mel_fb = fb

    # ---- host-buffer calls -----------------------------------------------------------
    def mel2wave(self, mel, n_frames=None, out=None) -> np.ndarray:
        """mel f32 [B,T,80] -> wav f32 [B,256T] (Generator.__call__, hifigan/model.py:109-125)."""
        mel = _np(mel, np.float32)
        if mel.ndim != 3 or mel.shape[2] != config.MEL_DIM:
            raise ValueError(f"mel must be [B,T,{config.MEL_DIM}], got {mel.shape}")
        B, T, _ = mel.shape
        nf = None if n_frames is None else _np(n_frames, np.int32, (B,), "n_frames")
        if out is not None and (out.shape != (B, T * config.HOP) or out.dtype != np.float32 or not out.flags.c_contiguous):
            raise ValueError(f"out must be C-contiguous float32 {(B, T * config.HOP)}")
        wav = out if out is not None else np.empty((B, T * config.HOP), np.float32)
        self._ck(self.lib.vtts_mel2wave_host(self.h, _ptr(mel), _ptr(nf), B, T, _ptr(wav)))
        return wav

    # receptive field of the generator in mel frames, one side: conv_pre 3 + ups_0 1 + stage-0 ResBlocks 60/8 +
    # stage 1 60/64 + stage 2 60/128 + stage 3 60/256 + ups/conv_post crumbs = 13.3 (hifigan/model.py:44-51,109-125)
    STREAM_HALO = 16

    def mel2wave_stream(self, mel, chunk_frames: int = 32, halo: int | None = None):
        """Chunked vocoding of ONE utterance for low first-audio latency (SURVEY.md §8f row 4): yields the waveform
        in pieces of `chunk_frames` mel frames.  Each piece is computed from its frames plus `halo` frames of
        context on both sides (recomputed, not carried), so the concatenation equals `mel2wave(mel)` exactly:
        every output sample sees its full receptive field, and samples inside the halo are discarded."""
        mel = _np(mel, np.float32)
        if mel.ndim == 3:
            if mel.shape[0] != 1:
                raise ValueError("mel2wave_stream takes one utterance ([T,80] or [1,T,80])")
            mel = mel[0]
        if mel.ndim != 2 or mel.shape[1] != config.MEL_DIM:
            raise ValueError(f"mel must be [T,{config.MEL_DIM}], got {mel.shape}")
        halo = self.STREAM_HALO if halo is None else int(halo)
        if chunk_frames < 1 or halo < 0:
            raise ValueError("chunk_frames >= 1 and halo >= 0 required")
        T = mel.shape[0]
        for t0 in range(0, T, chunk_frames):
            t1 = min(T, t0 + chunk_frames)
            a, b = max(0, t0 - halo), min(T, t1 + halo)
            wav = self.mel2wave(mel[None, a:b])[0]
            yield wav[(t0 - a) * config.HOP: (t1 - a) * config.HOP]

    def open_vocoder_stream(self, max_streams: int, max_chunk_frames: int) -> "VocoderStream":
        """Stateful streaming generator with `max_streams` independent slots (vtts_vocoder_stream_*): push each slot's
        new mel frames as they arrive and get back every waveform frame whose receptive field is complete.  Each push
        costs only the frames it brings; the emitted audio equals `mel2wave` of the whole mel bit for bit (same
        precision mode, fused pairs off).  Needs the generator weights and the 'bf16x3' or 'fp16' mode."""
        return VocoderStream(self, max_streams, max_chunk_frames)

    def open_acoustic_stream(self, max_streams: int, max_chunk_frames: int, max_frames: int, max_tokens: int, seed=None, rng=None,
                             masks: bool = False) -> "AcousticStream":
        """Streaming acoustic model with `max_streams` (<= 128) independent slots (vtts_acoustic_stream_*): `begin`
        starts utterances in free slots, each `push` advances every open slot by up to `max_chunk_frames` decoder steps
        in one scan launch and returns the mel frames that are final.  Each utterance's frames equal `predict_mel` of
        that utterance alone bit for bit.  Dropout, fixed for the stream: `masks=True` (MASK, masks given to `begin`),
        else `seed` (SEED, slot s draws as row s of `predict_mel(seed=)`), else `rng` (REFERENCE), else off."""
        return AcousticStream(self, max_streams, max_chunk_frames, max_frames, max_tokens, seed=seed, rng=rng, masks=masks)

    def open_tts_stream(self, max_streams: int, max_chunk_frames: int, max_frames: int, max_tokens: int = 1024, seed=None,
                        rng=None, output_rate=None, denoise=None, meter=False, semitones=None, tempo=None, limit=None,
                        gain_db=0.0, eq=None, compress=None, deess=None, reverb=None, watermark=None,
                        encoding=None, bed=None, max_joined_frames=None, formant=None) -> "TtsStream":
        """Text-to-speech per slot as a stream: one acoustic stream feeding one vocoder stream, the mel never leaving the
        device.  `begin(slot, tokens)` plans the utterance as `tts` does; each `step()` returns the new audio per slot.
        With fused pairs off a slot's audio equals `tts` of the same tokens bit for bit.
        `begin(..., more=True)` keeps the slot open after its sentence, and `append(slot, tokens)` adds the next one (a
        voice agent's text arrives a sentence at a time): the slot's audio is then `tts_joined` of its sentences, one
        utterance through every stage, bit for bit.  `max_frames` and `max_tokens` bound one sentence;
        `max_joined_frames` (default `max_frames`) bounds the frames a slot vocodes over all its sentences, and sizes the
        meter's history.  `output_rate`: a resample
        stream follows the vocoder on the device and `step()` returns samples at that rate, equal to `resample` of the
        `tts` audio bit for bit.  `denoise`: a strength; a denoise stream with the default bias (`denoiser_bias()`) sits
        between the vocoder and the resampler, and the audio equals `denoise` of the `tts` audio (then resampled) bit for
        bit.  `semitones`: a pitch-shift stream follows the denoiser (before the resampler) with this shift as every slot's
        default (`begin(..., semitones=)` overrides it per slot), and the audio equals `pitch_shift` of the (denoised)
        `tts` audio bit for bit.  `formant`: the pitch-shift stream (on with `semitones` or `formant`) moves the formants
        by this many semitones as every slot's default (`begin(..., formant=)` overrides it per slot; 0 keeps them), and
        the audio equals `pitch_shift(..., formant=)` bit for bit.  `tempo`: a time-stretch stream follows the pitch shifter (before the resampler) with this
        tempo as every slot's default (`begin(..., tempo=)` overrides it per slot), and the audio equals `time_stretch` of
        the (denoised, pitch-shifted) `tts` audio bit for bit.  `limit=CEILING_DBTP`: a limiter stream follows the
        resampler, at the output rate (a multiple of 10), with pre-gain `gain_db` as every slot's default
        (`begin(..., gain_db=)` overrides it per slot); its audio equals `limit` of the unlimited stream audio bit for bit.
        `eq`: an equalizer spec or sos array (`eq_sections`), designed at the output rate; an equalizer stream follows the
        resampler (before the limiter and the meter) and the audio equals `equalize` of the (resampled) `tts` audio bit
        for bit.  It releases every sample it receives, so it adds no delay.
        `compress`: a compressor spec (`compressor_params`); a compressor stream follows the equalizer (before the
        limiter and the meter) at the output rate, and the audio equals `compress` of the (resampled, equalized) `tts`
        audio bit for bit.  It also adds no delay.
        `deess`: a de-esser spec (`deesser_params`); a de-esser stream follows the compressor (before the limiter and the
        meter) at the output rate, and the audio equals `deess` of the (resampled, equalized, compressed) `tts` audio bit
        for bit.  It also adds no delay.
        `reverb`: a reverb spec (`reverb_params`, presets and keys); a reverb stream follows the de-esser (before the
        limiter and the meter) at the output rate, and the audio equals `reverb` of the (resampled, ..., de-essed) `tts`
        audio bit for bit.  It holds back up to 511 samples until the next block of 512 is complete.
        `bed`: a bed spec or a list of up to 8 (`bed_specs`); a bed stream follows the reverb (before the limiter and the
        meter) at the output rate, its bank prepared once here, and each slot's audio equals `mix_bed` of the
        (resampled, ..., reverberated) `tts` audio with the slot's bank entry (`begin(..., bed=)`, default 0, -1 for
        none) bit for bit.  It adds no delay; a slot's last step also returns its `tail`.
        `watermark`: a watermark spec (`watermark_params`: a key, or key=…,strength=…); a watermark stream follows the
        time stretcher (before the resampler) at 16 kHz, and the audio equals `watermark` of the (denoised, shifted,
        stretched) `tts` audio bit for bit.  Every slot carries the same key.  It holds back up to 1023 samples.
        `encoding`: 'pcm16', 'ulaw' or 'alaw'; after the meter the last stage's buffer is encoded on the device
        (`encode_forward` over the whole buffer) and `step()` copies and returns those codes (2 or 1 bytes per sample
        instead of 4), equal to `encode` of the float audio bit for bit.
        'flac' or 'flac,block=N': a per-slot FLAC stream (FlacStream) runs after the meter, and `step()` copies the
        per-slot (offset, count) table and then only the packed bytes, returning {slot: bytes}.
        `meter=True`: a loudness meter runs last, on what `step()` returns at the output rate (a
        multiple of 10), and `TtsStream.meter()` gives each stepped slot's readings, read back in the step's one
        synchronisation.  Needs the 'bf16x3' or 'fp16' mode (the vocoder stream has no strict fp32 path)."""
        return TtsStream(self, max_streams, max_chunk_frames, max_frames, max_tokens, seed=seed, rng=rng, output_rate=output_rate,
                         denoise=denoise, meter=meter, semitones=semitones, tempo=tempo, limit=limit, gain_db=gain_db, eq=eq,
                         compress=compress, deess=deess, reverb=reverb, watermark=watermark, encoding=encoding, bed=bed,
                         max_joined_frames=max_joined_frames, formant=formant)

    def tts_plan(self, tokens, lengths=None, silence_duration=-1.0):
        """vtts_tts_plan: the duration half of `tts` for token rows [B,L].  Returns (durations in seconds [B,L], durations
        in frames [B,L], acoustic frames n_frames [B], frames kept after the trailing-silence trim n_emit [B])."""
        tokens = _np(tokens, np.int32)
        if tokens.ndim != 2:
            raise ValueError("tokens must be [B,L]")
        B, L = tokens.shape
        lens = None if lengths is None else _np(lengths, np.int32, (B,), "lengths")
        sec = np.empty((B, L), np.float32)
        frames = np.empty((B, L), np.float32)
        nf = np.empty(B, np.int32)
        ne = np.empty(B, np.int32)
        self._ck(self.lib.vtts_tts_plan(self.h, _ptr(tokens), _ptr(lens), B, L, float(silence_duration), _ptr(sec), _ptr(frames),
                                        _ptr(nf), _ptr(ne)))
        return sec, frames, nf, ne

    def get_precision(self) -> int:
        return int(self.lib.vtts_get_precision(self.h))

    def _acoustic_args(self, tokens, dur_frames, lengths, n_frames, masks, seed, rng=None):
        ref_seed = None if rng is None else _rng_seed(rng, masks, seed)
        tokens = _np(tokens, np.int32)
        if tokens.ndim != 2:
            raise ValueError("tokens must be [B,L]")
        B, L = tokens.shape
        dur = _np(dur_frames, np.float32, (B, L), "durations")
        lens = None if lengths is None else _np(lengths, np.int32, (B,), "lengths")
        if n_frames is None:
            from .nat.text2mel import frame_count
            nf = np.array([frame_count(dur[b, : (L if lens is None else lens[b])]) for b in range(B)], np.int32)
        else:
            nf = _np(n_frames, np.int32, (B,), "n_frames")
        N = int(nf.max())
        if N < 1:
            raise ValueError("durations sum to less than one frame")
        if ref_seed is not None:
            return tokens, dur, lens, nf, N, None, DROPOUT_REFERENCE, ref_seed
        if masks is not None:
            mode = DROPOUT_MASK
            masks = _np(masks, np.uint8)
            if masks.shape[0] != B or masks.shape[1] < N or masks.shape[2:] != (2, config.PRENET_DIM):
                raise ValueError(f"masks must be uint8 [B,>=N,2,256], got {masks.shape}")
            masks = np.ascontiguousarray(masks[:, :N])
        elif seed is not None:
            mode = DROPOUT_SEED
        else:
            mode = DROPOUT_OFF
        return tokens, dur, lens, nf, N, masks, mode, int(seed or 0)

    @staticmethod
    def _call_seed(mode, seed, chunk):
        # SEED gives every 128-row chunk its own key; the REFERENCE draws do not depend on the row, so every chunk
        # shares the checkpoint's key
        return seed if mode == DROPOUT_REFERENCE else _chunk_seed(seed, chunk)

    def predict_mel(self, tokens, dur_frames, lengths=None, n_frames=None, masks=None, seed=None, rng=None) -> np.ndarray:
        """AcousticModel.inference for a (ragged) batch: tokens int [B,L], durations in FRAMES
        [B,L] -> mel f32 [B,N,80] with N = max_b n_frames[b] (rows past n_frames[b] are 0).
        Dropout (live at inference in the reference): `masks` uint8 [B,N,2,256] keep-masks,
        else `seed` for the on-device threefry stream, else `rng` (the checkpoint's uint32[2]) for the reference's own
        mask stream drawn on the device (every row gets the masks of the reference run on that row alone), else off."""
        tokens, dur, lens, nf, N, masks, mode, seed = self._acoustic_args(tokens, dur_frames, lengths, n_frames, masks, seed, rng)
        B, L = tokens.shape
        mel = np.empty((B, N, config.MEL_DIM), np.float32)
        for b0 in range(0, B, MAX_ACOUSTIC_ROWS):
            b1 = min(B, b0 + MAX_ACOUSTIC_ROWS)
            sl = slice(b0, b1)
            out = np.empty((b1 - b0, N, config.MEL_DIM), np.float32)
            self._ck(self.lib.vtts_predict_mel_host(
                self.h, _ptr(tokens[sl]), _ptr(None if lens is None else lens[sl]), _ptr(dur[sl]), _ptr(nf[sl]),
                _ptr(None if masks is None else np.ascontiguousarray(masks[sl])), mode, self._call_seed(mode, seed, b0 // MAX_ACOUSTIC_ROWS),
                b1 - b0, L, N, _ptr(out)))
            mel[sl] = out
        return mel

    def predict_duration(self, tokens, lengths=None) -> np.ndarray:
        """DurationModel.__call__ (nat/model.py:64-70) for a (ragged) batch: tokens int [B,L] -> predicted
        durations in SECONDS f32 [B,L] (0 past lengths[b]); row b equals the reference run on row b alone."""
        tokens = _np(tokens, np.int32)
        if tokens.ndim != 2:
            raise ValueError("tokens must be [B,L]")
        B, L = tokens.shape
        lens = None if lengths is None else _np(lengths, np.int32, (B,), "lengths")
        out = np.empty((B, L), np.float32)
        for b0 in range(0, B, MAX_ACOUSTIC_ROWS):
            b1 = min(B, b0 + MAX_ACOUSTIC_ROWS)
            o = np.empty((b1 - b0, L), np.float32)
            self._ck(self.lib.vtts_predict_duration_host(
                self.h, _ptr(np.ascontiguousarray(tokens[b0:b1])), _ptr(None if lens is None else np.ascontiguousarray(lens[b0:b1])),
                b1 - b0, L, _ptr(o)))
            out[b0:b1] = o
        return out

    @staticmethod
    def pinned_empty(shape, dtype=np.float32) -> np.ndarray:
        """numpy array backed by page-locked host memory.  Passed as `out=` to synthesize / mel2wave the
        library copies D2H straight into it (no staging copy, no page faults of a fresh array).
        The pinned allocation lives exactly as long as the array (or any view of it)."""
        import weakref
        import torch
        t = torch.empty(tuple(shape), dtype=getattr(torch, np.dtype(dtype).name), pin_memory=True)
        a = t.numpy()
        key = a.ctypes.data
        Engine._pinned_keepalive[key] = t            # the tensor owns the memory ...
        weakref.finalize(a, Engine._pinned_keepalive.pop, key, None)   # ... and is dropped with the array
        return a

    _pinned_keepalive: dict = {}

    def synthesize(self, tokens, dur_frames, lengths=None, n_frames=None, masks=None, seed=None, return_mel=False, out=None, rng=None):
        """predict_mel -> mel2wave with the mel staying on the device.  Returns wav [B,256N]
        (and mel [B,N,80] if return_mel).  `out`: optional preallocated float32 [B,256N] result array
        (ideally from `pinned_empty`); it is validated and written in every path (rows land directly in it).
        In SEED mode row r of a call draws the device stream keyed by (seed, r, frame): an utterance's masks depend on
        its row index, not on the padded frame count of the batch; MASK / OFF / `rng` (REFERENCE) modes are position
        independent."""
        tokens, dur, lens, nf, N, masks, mode, seed = self._acoustic_args(tokens, dur_frames, lengths, n_frames, masks, seed, rng)
        B, L = tokens.shape
        if out is not None and (out.shape != (B, N * config.HOP) or out.dtype != np.float32 or not out.flags.c_contiguous):
            raise ValueError(f"out must be C-contiguous float32 {(B, N * config.HOP)}")
        wav = out if out is not None else np.empty((B, N * config.HOP), np.float32)
        mel = np.empty((B, N, config.MEL_DIM), np.float32) if return_mel else None
        for b0 in range(0, B, MAX_ACOUSTIC_ROWS):
            b1 = min(B, b0 + MAX_ACOUSTIC_ROWS)
            sl = slice(b0, b1)
            # row slices of C-contiguous arrays are contiguous: the library writes straight into the result
            self._ck(self.lib.vtts_synthesize_host(
                self.h, _ptr(tokens[sl]), _ptr(None if lens is None else lens[sl]), _ptr(dur[sl]), _ptr(nf[sl]),
                _ptr(None if masks is None else np.ascontiguousarray(masks[sl])), mode, self._call_seed(mode, seed, b0 // MAX_ACOUSTIC_ROWS),
                b1 - b0, L, N, _ptr(None if mel is None else mel[sl]), _ptr(wav[sl])))
        return (wav, mel) if return_mel else wav

    def tts(self, tokens, lengths=None, silence_duration=-1.0, seed=None, max_frames=None, rng=None):
        """Token rows -> waveforms in ONE library call (vtts_tts_host): duration model, the duration fix-ups of
        text2mel.py:88-97, acoustic model, trailing-silence trim (:99-102) and generator, the mel never leaving
        the device.  tokens int [B,L] (rows padded to L), lengths int [B].  Returns (list of f32 waveforms,
        durations_sec f32 [B,L]).  Dropout: `seed` for the on-device counter stream (keyed by row index), else `rng`
        (the checkpoint's uint32[2]) for the reference's own stream (each row as the reference run on it alone), else off."""
        ref_seed = None if rng is None else _rng_seed(rng, seed)
        tokens = _np(tokens, np.int32)
        if tokens.ndim != 2:
            raise ValueError("tokens must be [B,L]")
        B, L = tokens.shape
        if B > MAX_ACOUSTIC_ROWS:
            raise ValueError(f"tts: at most {MAX_ACOUSTIC_ROWS} rows per call")
        lens = None if lengths is None else _np(lengths, np.int32, (B,), "lengths")
        dur = np.empty((B, L), np.float32)
        nf = np.zeros(B, np.int32)
        nmax = C.c_int32(0)
        cap = int(max_frames) if max_frames else max(16, int(L * 0.12 * config.SAMPLE_RATE / config.HOP))
        mode = DROPOUT_SEED if seed is not None else DROPOUT_OFF
        if ref_seed is not None:
            mode, seed = DROPOUT_REFERENCE, ref_seed
        for _ in range(2):
            wav = np.empty(B * cap * config.HOP, np.float32)
            rc = self.lib.vtts_tts_host(self.h, _ptr(tokens), _ptr(lens), B, L, float(silence_duration), mode, int(seed or 0),
                                        cap, _ptr(dur), _ptr(nf), C.byref(nmax), _ptr(wav))
            if rc == 0 or not (0 < cap < nmax.value):
                break
            cap = int(nmax.value)       # buffer too small: the call reported the size it needs
        self._ck(rc)
        n = int(nmax.value)
        wav = wav[: B * n * config.HOP].reshape(B, n * config.HOP)
        return [wav[b, : int(nf[b]) * config.HOP].copy() for b in range(B)], dur

    def tts_joined(self, texts, silence_duration=-1.0, seed=None, rng=None, max_frames=None):
        """Texts of several sentences -> one waveform per text, in ONE library call (vtts_tts_joined_host).  `texts` is a
        list of texts, each a list of 1-D token rows (its sentences).  Every sentence is planned and run through the
        acoustic model as `tts` runs it alone; the frames it keeps after its trailing-silence trim are joined in order
        and the generator runs once per text, so a text sounds as one utterance with no seam to hear.  Any number of
        sentences per call (the acoustic model runs 128 rows per launch).  Returns (list of f32 waveforms, list of int64
        arrays: each sentence's first sample in its text's waveform at 16 kHz).  Dropout as `tts`: `seed` (row r draws
        as row r of `predict_mel(seed=)` on the same rows), else `rng`, else off."""
        ref_seed = None if rng is None else _rng_seed(rng, seed)
        rows, bounds = [], [0]
        for i, text in enumerate(texts):
            sent = [np.asarray(r) for r in text]
            if not sent:
                raise ValueError(f"tts_joined: text {i} has no sentence")
            for r in sent:
                if r.ndim != 1 or r.size < 1 or not np.issubdtype(r.dtype, np.integer):
                    raise ValueError(f"tts_joined: every sentence of text {i} must be a non-empty 1-D row of token ids")
            rows += sent
            bounds.append(len(rows))
        if not rows:
            raise ValueError("tts_joined: no texts")
        B, G, L = len(rows), len(bounds) - 1, max(r.size for r in rows)
        tokens = np.zeros((B, L), np.int32)
        lens = np.array([r.size for r in rows], np.int32)
        for b, r in enumerate(rows):
            tokens[b, : r.size] = r
        gs = np.asarray(bounds, np.int32)
        dur = np.empty((B, L), np.float32)
        starts = np.zeros(B, np.int32)
        nf = np.zeros(G, np.int32)
        nmax = C.c_int32(0)
        text_tokens = int(np.add.reduceat(lens, gs[:-1]).max())
        cap = int(max_frames) if max_frames else max(16, int(text_tokens * 0.12 * config.SAMPLE_RATE / config.HOP))
        mode = DROPOUT_SEED if seed is not None else DROPOUT_OFF
        if ref_seed is not None:
            mode, seed = DROPOUT_REFERENCE, ref_seed
        for _ in range(2):
            wav = np.empty(G * cap * config.HOP, np.float32)
            rc = self.lib.vtts_tts_joined_host(self.h, _ptr(tokens), _ptr(lens), B, L, _ptr(gs), G, float(silence_duration), mode,
                                               int(seed or 0), cap, _ptr(dur), _ptr(starts), _ptr(nf), C.byref(nmax), _ptr(wav))
            if rc == 0 or not (0 < cap < nmax.value):
                break
            cap = int(nmax.value)       # buffer too small: the call reported the size it needs
        self._ck(rc)
        n = int(nmax.value)
        wav = wav[: G * n * config.HOP].reshape(G, n * config.HOP)
        return ([wav[g, : int(nf[g]) * config.HOP].copy() for g in range(G)],
                [starts[gs[g]: gs[g + 1]].astype(np.int64) * config.HOP for g in range(G)])

    def synthesize_many(self, utterances, seed=None, masks=None, max_pad_frac=0.08, max_rows=32, rng=None):
        """Mixed-length workload (BASELINE configs[4]): `utterances` is a list of (tokens list[int],
        durations_in_frames f32[L]).  They are bucketed by frame count so that padding stays below
        `max_pad_frac`, each bucket runs as one ragged batch, and the waveforms come back in input order
        (list of np.float32 [256*n_frames_i]).  Row i of any bucket equals utterance i run alone (with `rng`, the
        reference's own dropout stream, that includes its masks)."""
        from .nat.text2mel import frame_count
        from .parallel import bucket_by_length
        if rng is not None:
            _rng_seed(rng, masks, seed)
        nfs = [frame_count(d) for _, d in utterances]
        out = [None] * len(utterances)
        for bucket in bucket_by_length(nfs, max_pad_frac, max_rows):
            Lmax = max(len(utterances[i][0]) for i in bucket)
            tok = np.zeros((len(bucket), Lmax), np.int32)
            dur = np.zeros((len(bucket), Lmax), np.float32)
            lens = np.zeros(len(bucket), np.int32)
            for r, i in enumerate(bucket):
                t, d = utterances[i]
                tok[r, : len(t)] = t
                dur[r, : len(t)] = d
                lens[r] = len(t)
            nf = np.asarray([nfs[i] for i in bucket], np.int32)
            m = None if masks is None else np.stack([np.asarray(masks[i])[: nf.max()] if np.asarray(masks[i]).shape[0] >= nf.max()
                                                     else np.pad(np.asarray(masks[i]), ((0, nf.max() - np.asarray(masks[i]).shape[0]), (0, 0), (0, 0)))
                                                     for i in bucket])
            wav = self.synthesize(tok, dur, lengths=lens, n_frames=nf, masks=m, seed=seed, rng=rng)
            for r, i in enumerate(bucket):
                out[i] = wav[r, : nfs[i] * config.HOP].copy()
        return out

    def _tf_masks(self, B, N, keep_masks, zone_masks, seed, rng=None):
        """(keep, zone, mode, seed) of a teacher-forced call."""
        if rng is not None:
            return None, None, DROPOUT_REFERENCE, _rng_seed(rng, keep_masks, zone_masks, seed)
        if keep_masks is not None or zone_masks is not None:
            if keep_masks is None or zone_masks is None:
                raise ValueError("keep_masks and zone_masks must be given together")
            km = _np(keep_masks, np.uint8, (B, N, 2, config.PRENET_DIM), "keep_masks")
            zm = _np(zone_masks, np.uint8, (B, N, 4, config.ACOUSTIC_DECODER_DIM), "zone_masks")
            return km, zm, DROPOUT_MASK, 0
        return None, None, (DROPOUT_SEED if seed is not None else DROPOUT_OFF), int(seed or 0)

    def teacher_forced(self, tokens, dur_frames, mels_in, lengths=None, n_frames=None, keep_masks=None, zone_masks=None, seed=None,
                       rng=None):
        """AcousticModel.__call__ (nat/model.py:146-169, is_training=False): tokens int [B,L], durations in frames
        [B,L], mels_in f32 [B,N,80] (ground truth shifted by one frame) -> (mel1, mel2) f32 [B,N,80].
        keep_masks uint8 [B,N,2,256] / zone_masks uint8 [B,N,4,512] (1 = keep previous state), else `seed` for the
        on-device stream, else `rng` (the checkpoint's uint32[2]) for the reference's own whole-batch draws on the
        device (= jaxrng.teacher_forced_masks(rng, B, N)), else both off.  Host buffers; the device work is
        vtts_acoustic_teacher_forward."""
        import torch
        tokens = _np(tokens, np.int32)
        B, L = tokens.shape
        mels_in = _np(mels_in, np.float32)
        N = mels_in.shape[1]
        if mels_in.shape != (B, N, config.MEL_DIM):
            raise ValueError(f"mels_in must be [B,N,{config.MEL_DIM}]")
        if B > MAX_ACOUSTIC_ROWS:
            raise ValueError(f"teacher_forced: at most {MAX_ACOUSTIC_ROWS} rows per call")
        km, zm, mode, seed = self._tf_masks(B, N, keep_masks, zone_masks, seed, rng)
        dev = torch.device("cuda", self.device)
        up = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to(dev)   # noqa: E731
        t_tok, t_dur, t_in = up(tokens), up(_np(dur_frames, np.float32, (B, L), "durations")), up(mels_in)
        t_len = up(None if lengths is None else _np(lengths, np.int32, (B,), "lengths"))
        t_nf = up(None if n_frames is None else _np(n_frames, np.int32, (B,), "n_frames"))
        t_km, t_zm = up(km), up(zm)
        m1 = torch.empty((B, N, config.MEL_DIM), dtype=torch.float32, device=dev)
        m2 = torch.empty_like(m1)
        st = torch.cuda.current_stream(dev).cuda_stream
        self._ck(self.lib.vtts_acoustic_teacher_forward(self.h, _ptr(t_tok), _ptr(t_len), _ptr(t_dur), _ptr(t_nf), _ptr(t_in), _ptr(t_km),
                                                        _ptr(t_zm), mode, seed, B, L, N, _ptr(m1), _ptr(m2), st))
        torch.cuda.synchronize(dev)
        return m1.cpu().numpy(), m2.cpu().numpy()

    def gta(self, wav_i16, tokens, dur_sec, lengths=None, wav_lengths=None, keep_masks=None, zone_masks=None, seed=None, return_gt=False,
            rng=None):
        """forward_fn of nat/gta.py:28-44 in one library call: int16 wavs [B,S] + aligned phonemes -> mel2_hat
        f32 [B,S/256,80] (rows past wav_lengths[b]//256 are 0).  Masks as in `teacher_forced`.  The ground-truth mel
        (returned first with return_gt) is MelFilter(16000, 1024, 80)(wav / 2**15) with the default filterbank, as the
        reference builds its own MelFilter (gta.py:29-31), whatever bank `load_mel_filterbank` last loaded; that bank
        stays loaded for `melspec`."""
        wav = np.ascontiguousarray(np.asarray(wav_i16))
        if wav.dtype != np.int16 or wav.ndim != 2:
            raise ValueError("wav_i16 must be int16 [B,S]")
        B, S = wav.shape
        tokens = _np(tokens, np.int32)
        if tokens.ndim != 2 or tokens.shape[0] != B:
            raise ValueError("tokens must be [B,L]")
        L = tokens.shape[1]
        if B > MAX_ACOUSTIC_ROWS:
            raise ValueError(f"gta: at most {MAX_ACOUSTIC_ROWS} rows per call")
        N = S // config.HOP
        km, zm, mode, seed = self._tf_masks(B, N, keep_masks, zone_masks, seed, rng)
        lens = None if lengths is None else _np(lengths, np.int32, (B,), "lengths")
        wl = None if wav_lengths is None else _np(wav_lengths, np.int32, (B,), "wav_lengths")
        dur = _np(dur_sec, np.float32, (B, L), "durations")
        gt = np.empty((B, N, config.MEL_DIM), np.float32) if return_gt else None
        out = np.empty((B, N, config.MEL_DIM), np.float32)
        kept = self._mel_fb
        swap = kept is None or not np.array_equal(kept, weights.mel_filterbank())
        if swap:
            self.load_mel_filterbank()
        try:
            self._ck(self.lib.vtts_gta_host(self.h, _ptr(wav), _ptr(wl), _ptr(tokens), _ptr(lens), _ptr(dur), _ptr(km), _ptr(zm), mode, seed,
                                            B, L, S, _ptr(gt), _ptr(out)))
        finally:
            if swap and kept is not None:
                self.load_mel_filterbank(kept)
        return (out, gt) if return_gt else out

    def melspec(self, wav) -> np.ndarray:
        """MelFilter.__call__ (nat/dsp.py:115-128): wav f32 [B,S] -> log-mel [B,S/256,80], with the filterbank
        `load_mel_filterbank` last loaded (the default bank if none)."""
        if self._mel_fb is None:
            self.load_mel_filterbank()
        wav = _np(wav, np.float32)
        assert wav.ndim == 2, "MelFilter expects [B,S] (dsp.py:118)"
        B, S = wav.shape
        mel = np.empty((B, S // config.HOP, config.MEL_DIM), np.float32)
        self._ck(self.lib.vtts_melspec_host(self.h, _ptr(wav), B, S, _ptr(mel)))
        return mel

    def debug_read(self, name: str, shape) -> np.ndarray:
        out = np.empty(shape, np.float32)
        self._ck(self.lib.vtts_debug_read(self.h, name.encode(), _ptr(out), out.size))
        return out

    # ---- device-pointer calls (torch tensors as memory containers) --------------------
    def hifigan_forward(self, mel_t, n_frames_t=None, out=None, stream=None):
        import torch
        assert mel_t.is_cuda and mel_t.dtype == torch.float32 and mel_t.is_contiguous()
        B, T, _ = mel_t.shape
        if out is None:
            out = torch.empty((B, T * config.HOP), dtype=torch.float32, device=mel_t.device)
        st = torch.cuda.current_stream(mel_t.device).cuda_stream if stream is None else stream
        self._ck(self.lib.vtts_hifigan_forward(self.h, _ptr(mel_t), _ptr(n_frames_t), B, T, _ptr(out), st))
        return out

    def debug_dropout_masks(self, kind, rng, B, N) -> np.ndarray:
        """Test hook (vtts_debug_dropout_masks): the masks the `rng` (REFERENCE) mode applies, drawn on the device.
        kind 0: autoregressive prenet masks uint8 [N,2,256]; kind 1: teacher-forced (keep [B,N,2,256], zone [B,N,4,512])."""
        seed = _rng_seed(rng)
        nk = (1 if kind == 0 else B) * N * 2 * config.PRENET_DIM
        nz = 0 if kind == 0 else B * N * 4 * config.ACOUSTIC_DECODER_DIM
        out = np.empty(nk + nz, np.uint8)
        self._ck(self.lib.vtts_debug_dropout_masks(self.h, int(kind), seed, int(B), int(N), _ptr(out)))
        if kind == 0:
            return out.reshape(N, 2, config.PRENET_DIM)
        return out[:nk].reshape(B, N, 2, config.PRENET_DIM), out[nk:].reshape(B, N, 4, config.ACOUSTIC_DECODER_DIM)

    def acoustic_forward(self, tokens_t, dur_t, N, lengths_t=None, n_frames_t=None, masks_t=None, seed=None, out=None, stream=None,
                         rng=None):
        """vtts_acoustic_forward on torch CUDA tensors, stream-ordered.  Dropout: masks_t, else seed, else rng (the
        reference's own stream drawn on the device), else off."""
        import torch
        assert tokens_t.is_cuda and tokens_t.dtype == torch.int32 and dur_t.dtype == torch.float32
        B, L = tokens_t.shape
        if out is None:
            out = torch.empty((B, N, config.MEL_DIM), dtype=torch.float32, device=tokens_t.device)
        mode = DROPOUT_MASK if masks_t is not None else (DROPOUT_SEED if seed is not None else DROPOUT_OFF)
        if rng is not None:
            mode, seed = DROPOUT_REFERENCE, _rng_seed(rng, masks_t, seed)
        st = torch.cuda.current_stream(tokens_t.device).cuda_stream if stream is None else stream
        self._ck(self.lib.vtts_acoustic_forward(self.h, _ptr(tokens_t), _ptr(lengths_t), _ptr(dur_t), _ptr(n_frames_t),
                                                _ptr(masks_t), mode, int(seed or 0), B, L, int(N), _ptr(out), st))
        return out

    def duration_forward(self, tokens_t, lengths_t=None, out=None, stream=None):
        import torch
        assert tokens_t.is_cuda and tokens_t.dtype == torch.int32 and tokens_t.is_contiguous()
        B, L = tokens_t.shape
        if out is None:
            out = torch.empty((B, L), dtype=torch.float32, device=tokens_t.device)
        st = torch.cuda.current_stream(tokens_t.device).cuda_stream if stream is None else stream
        self._ck(self.lib.vtts_duration_forward(self.h, _ptr(tokens_t), _ptr(lengths_t), B, L, _ptr(out), st))
        return out

    def melspec_forward(self, wav_t, out=None, stream=None):
        """vtts_melspec on torch CUDA tensors, stream-ordered: wav_t f32 [B,S] -> log-mel [B,S/256,80], as `melspec`."""
        import torch
        assert wav_t.is_cuda and wav_t.dtype == torch.float32 and wav_t.is_contiguous() and wav_t.dim() == 2
        B, S = wav_t.shape
        out = _out_tensor(out, (B, S // config.HOP, config.MEL_DIM), wav_t.device)
        if self._mel_fb is None:
            self.load_mel_filterbank()
        st = torch.cuda.current_stream(wav_t.device).cuda_stream if stream is None else stream
        self._ck(self.lib.vtts_melspec(self.h, _ptr(wav_t), B, S, _ptr(out), st))
        return out

    # ---- resampling to an output rate (vtts_resample*: scipy.signal.resample_poly with its defaults, fp32) ----
    def resample(self, wav, out_rate: int, in_rate: int = config.SAMPLE_RATE, lengths=None) -> np.ndarray:
        """Host arrays: wav f32 [S] or [B,S] at `in_rate` -> [ceil(S * up / down)] or [B, that] at `out_rate`, where up /
        down is out_rate / in_rate in lowest terms (each <= 1024).  lengths int [B]: row b holds lengths[b] samples,
        and its outputs past ceil(lengths[b] * up / down) are 0.  Equals scipy.signal.resample_poly(x, up, down) up to
        fp32 rounding; in_rate == out_rate is a copy."""
        x, lens, one = _wav_rows(wav, lengths)
        if x.shape[1] < 1:
            raise ValueError(f"wav must be [S] or [B,S], got {np.shape(wav)}")
        B, S = x.shape
        y = np.empty((B, resample_length(S, in_rate, out_rate)), np.float32)
        self._ck(self.lib.vtts_resample_host(self.h, _ptr(x), _ptr(lens), B, S, int(in_rate), int(out_rate), _ptr(y)))
        return y[0] if one else y

    def resample_forward(self, x_t, out_rate: int, in_rate: int = config.SAMPLE_RATE, lengths_t=None, out=None, stream=None):
        """vtts_resample on torch CUDA tensors, stream-ordered: x_t f32 [B,S] -> [B, ceil(S * up / down)]; lengths_t
        int32 CUDA [B] or None."""
        B, S, out, st = _dev_rows(x_t, out, stream, resample_length(x_t.shape[-1], in_rate, out_rate))
        self._ck(self.lib.vtts_resample(self.h, _ptr(x_t), _ptr(lengths_t), B, S, int(in_rate), int(out_rate), _ptr(out), st))
        return out

    def open_resample_stream(self, max_streams: int, max_chunk_samples: int, out_rate: int,
                             in_rate: int = config.SAMPLE_RATE) -> "ResampleStream":
        """Streaming resampler with `max_streams` independent slots (vtts_resample_stream_*): each slot carries its
        filter history across pushes, so its outputs, concatenated, equal `resample` of its whole input bit for bit.
        An output is emitted as soon as every input it reads has arrived (at most `lookahead` samples after its own
        time); END emits the rest."""
        return ResampleStream(self, max_streams, max_chunk_samples, out_rate, in_rate)

    # ---- bias denoiser (vtts_denoise*: STFT spectral subtraction of the vocoder's bias spectrum, fp32) ----
    def denoiser_bias(self, mel=None) -> np.ndarray:
        """The denoiser's bias beta [513]: |X_0|, the magnitude spectrum of frame 0 of the loaded generator's output in
        the current precision mode, for `mel` ([T,80] or [1,T,80]) or by default an all-zero mel [1, 88, 80].  The
        default is computed on first use and kept until the generator or the precision mode changes."""
        import torch
        default = mel is None
        if default and self._denoise_bias is not None:
            return self._denoise_bias.copy()
        m = np.zeros((1, DENOISE_BIAS_FRAMES, config.MEL_DIM), np.float32) if default else _np(mel, np.float32)
        if m.ndim == 2:
            m = m[None]
        if m.ndim != 3 or m.shape[0] != 1 or m.shape[2] != config.MEL_DIM:
            raise ValueError(f"mel must be [T,{config.MEL_DIM}] or [1,T,{config.MEL_DIM}], got {np.shape(mel)}")
        wav = torch.from_numpy(self.mel2wave(m)[0]).to(torch.device("cuda", self.device))
        out = torch.empty(DENOISE_BINS, dtype=torch.float32, device=wav.device)
        st = torch.cuda.current_stream(wav.device).cuda_stream
        self._ck(self.lib.vtts_denoise_bias(self.h, _ptr(wav), int(wav.numel()), _ptr(out), st))
        beta = out.cpu().numpy()
        if default:
            self._denoise_bias = beta.copy()
        return beta

    def _bias_arg(self, bias) -> np.ndarray:
        b = self.denoiser_bias() if bias is None else _np(bias, np.float32, (DENOISE_BINS,), "bias")
        if not (np.all(np.isfinite(b)) and np.all(b >= 0)):
            raise ValueError("bias values must be finite and >= 0")
        return b

    def denoise(self, wav, strength: float, lengths=None, bias=None) -> np.ndarray:
        """Host arrays: wav f32 [S] or [B,S] -> the same shape with strength * bias subtracted from every STFT magnitude
        (n_fft 1024, hop 256, Hann, reflect-padded centered frames), phase kept; rows of <= 512 samples are copied.
        lengths int [B] in [0, S]: row b holds lengths[b] samples and its outputs past them are 0.  bias f32 [513]
        (default: `denoiser_bias()`)."""
        strength = _strength(strength)
        x, lens, one = _wav_rows(wav, lengths)
        B, S = x.shape
        if S == 0 or B == 0:
            return (x[0] if one else x).copy()          # nothing to transform: empty rows are short rows
        b = self._bias_arg(bias)
        y = np.empty((B, S), np.float32)
        self._ck(self.lib.vtts_denoise_host(self.h, _ptr(x), _ptr(lens), B, S, strength, _ptr(b), _ptr(y)))
        return y[0] if one else y

    def denoise_forward(self, x_t, strength: float, lengths_t=None, bias_t=None, out=None, stream=None):
        """vtts_denoise on torch CUDA tensors, stream-ordered: x_t f32 [B,S] -> [B,S]; lengths_t int32 CUDA [B] or None;
        bias_t f32 CUDA [513] or None (`denoiser_bias()`)."""
        import torch
        strength = _strength(strength)
        B, S, out, st = _dev_rows(x_t, out, stream)
        if bias_t is None:
            bias_t = torch.from_numpy(self._bias_arg(None)).to(x_t.device)
        elif tuple(bias_t.shape) != (DENOISE_BINS,) or bias_t.dtype != torch.float32 or not bias_t.is_contiguous():
            raise ValueError(f"bias_t must be contiguous float32 [{DENOISE_BINS}]")
        self._ck(self.lib.vtts_denoise(self.h, _ptr(x_t), _ptr(lengths_t), B, S, strength, _ptr(bias_t), _ptr(out), st))
        return out

    def open_denoise_stream(self, max_streams: int, max_chunk_samples: int, strength: float, bias=None) -> "DenoiseStream":
        """Streaming denoiser with `max_streams` independent slots (vtts_denoise_stream_*), strength and bias fixed:
        each slot's outputs, concatenated, equal `denoise` of its whole input bit for bit.  An output is emitted once the
        frames covering it are final (at most 1023 samples after its own time); END emits the rest."""
        return DenoiseStream(self, max_streams, max_chunk_samples, strength, bias)

    # ---- pitch shift (vtts_pitch_shift*: a peak-locked phase vocoder on the denoiser's STFT, fp32, double phases) ----
    def pitch_shift(self, wav, semitones, lengths=None, formant=None) -> np.ndarray:
        """Host arrays: wav f32 [S] or [B,S] -> the same shape, every spectral peak's region moved by the ratio
        fp32(2^(s / 12)) with its phase kept coherent across frames (n_fft 1024, hop 256); the timing of every sample is
        kept.  semitones: a scalar or one value per row, finite and in [-12, 12]; rows with 0 and rows of <= 512 samples
        are copied.  lengths int [B] in [0, S]: row b holds lengths[b] samples and its outputs past them are 0.
        formant (vtts_voice_shift): None, the formants move with the pitch; else a scalar or one value per row, finite
        and in [-12, 12], the shift of the spectral envelope in semitones whatever the pitch does (0 keeps the voice's
        formants where they are); rows with semitones 0 and formant 0 are copied."""
        x, lens, one = _wav_rows(wav, lengths)
        B, S = x.shape
        sem = SEMITONES.rows(semitones, B)
        fmt = None if formant is None else FORMANT.rows(formant, B)
        if S == 0 or B == 0:
            return (x[0] if one else x).copy()          # nothing to transform: empty rows are short rows
        y = np.empty((B, S), np.float32)
        if fmt is None:
            self._ck(self.lib.vtts_pitch_shift_host(self.h, _ptr(x), _ptr(lens), B, S, _ptr(sem), _ptr(y)))
        else:
            self._ck(self.lib.vtts_voice_shift_host(self.h, _ptr(x), _ptr(lens), B, S, _ptr(sem), _ptr(fmt), _ptr(y)))
        return y[0] if one else y

    def pitch_shift_forward(self, x_t, semitones, lengths_t=None, out=None, stream=None, formant=None):
        """vtts_pitch_shift (vtts_voice_shift with `formant`, as `pitch_shift` takes it) on torch CUDA tensors,
        stream-ordered: x_t f32 [B,S] -> [B,S] (not x_t); semitones a scalar or one host value per row; lengths_t int32
        CUDA [B] or None."""
        B, S, out, st = _dev_rows(x_t, out, stream)
        sem = SEMITONES.rows(semitones, B)
        if formant is None:
            self._ck(self.lib.vtts_pitch_shift(self.h, _ptr(x_t), _ptr(lengths_t), B, S, _ptr(sem), _ptr(out), st))
        else:
            fmt = FORMANT.rows(formant, B)
            self._ck(self.lib.vtts_voice_shift(self.h, _ptr(x_t), _ptr(lengths_t), B, S, _ptr(sem), _ptr(fmt), _ptr(out), st))
        return out

    def debug_pitch_decisions(self, x_t, semitones, lengths_t=None) -> np.ndarray:
        """Test hook (vtts_debug_pitch_decisions): int32 [B, S // 256 + 1, 513], the device's peak flags (bit 0) and the
        side of the princarg cut each peak's phase deviation took (bit 1: negative) for `pitch_shift_forward` of the
        same arguments."""
        import torch
        B, S = x_t.shape
        sem = SEMITONES.rows(semitones, B)
        out = torch.empty((B, S // config.HOP + 1, DENOISE_BINS), dtype=torch.int32, device=x_t.device)
        st = torch.cuda.current_stream(x_t.device).cuda_stream
        self._ck(self.lib.vtts_debug_pitch_decisions(self.h, _ptr(x_t), _ptr(lengths_t), B, S, _ptr(sem), _ptr(out), st))
        return out.cpu().numpy()

    def open_pitch_shift_stream(self, max_streams: int, max_chunk_samples: int) -> "PitchShiftStream":
        """Streaming pitch shifter with `max_streams` independent slots (vtts_pitch_shift_stream_*): a slot's shift is
        given with BEGIN and fixed until END, and its outputs, concatenated, equal `pitch_shift` of its whole input bit
        for bit.  Outputs are released on the denoise stream's schedule (at most 1023 samples after their own time)."""
        return PitchShiftStream(self, max_streams, max_chunk_samples)

    def open_voice_shift_stream(self, max_streams: int, max_chunk_samples: int) -> "VoiceShiftStream":
        """The pitch-shift stream with a formant shift per slot (vtts_voice_shift_stream_push): `semitones=` and
        `formant=` with BEGIN, fixed until END; a slot's outputs, concatenated, equal `pitch_shift(..., formant=)` of its
        whole input bit for bit.  Schedule and lookahead are the pitch-shift stream's."""
        return VoiceShiftStream(self, max_streams, max_chunk_samples)

    # ---- time stretch (vtts_time_stretch*: the pitch shifter's phase vocoder with analysis frames at 256 t alpha) ----
    def time_stretch_length(self, n: int, tempo: float) -> int:
        """M = floor(n / alpha + 0.5) (in double, alpha the fp32 tempo): the samples `time_stretch` makes of n"""
        m = int(self.lib.vtts_time_stretch_length(int(n), float(TEMPO.rows(tempo, 1)[0])))
        if m < 0:
            raise ValueError(f"time_stretch_length: n={n} must be >= 0")
        return m

    def time_stretch(self, wav, tempo, lengths=None) -> np.ndarray:
        """Host arrays: wav f32 [S] -> [M], or [B,S] -> [B, max_b M_b], played `tempo` times as fast with the pitch kept
        (a peak-locked phase vocoder, n_fft 1024, synthesis hop 256); M_b = floor(n_b / tempo_b + 0.5) and row b is zero
        past M_b.  tempo: a scalar or one value per row, finite and in [0.5, 2]; rows at 1 and rows of <= 512 samples
        give their first min(n, M) samples.  lengths int [B] in [0, S]: row b holds lengths[b] samples."""
        x, lens, one = _wav_rows(wav, lengths)
        B, S = x.shape
        tp = TEMPO.rows(tempo, B)
        n = np.full(B, S) if lens is None else lens
        Sy = max((self.time_stretch_length(int(n[b]), tp[b]) for b in range(B)), default=0)
        if S == 0 or B == 0 or Sy == 0:
            y = np.zeros((B, Sy), np.float32)
            for b in range(B):
                k = min(int(n[b]), Sy)
                y[b, :k] = x[b, :k]                     # nothing to transform: empty rows are short rows
            return y[0] if one else y
        y = np.empty((B, Sy), np.float32)
        self._ck(self.lib.vtts_time_stretch_host(self.h, _ptr(x), _ptr(lens), B, S, _ptr(tp), _ptr(y), Sy))
        return y[0] if one else y

    def time_stretch_forward(self, x_t, tempo, lengths_t=None, out=None, stream=None):
        """vtts_time_stretch on torch CUDA tensors, stream-ordered: x_t f32 [B,S] -> [B, Sy] (not x_t), Sy = out's width or
        max_b time_stretch_length(S, tempo_b); tempo a scalar or one host value per row; lengths_t int32 CUDA [B] or None."""
        import torch
        assert x_t.is_cuda and x_t.dtype == torch.float32 and x_t.is_contiguous() and x_t.dim() == 2
        B, S = x_t.shape
        tp = TEMPO.rows(tempo, B)
        if out is None:
            out = _out_tensor(None, (B, max(self.time_stretch_length(S, a) for a in tp)), x_t.device)
        elif out.dim() != 2 or out.shape[0] != B or out.shape[1] < 1 or out.dtype != torch.float32 or not out.is_contiguous():
            raise ValueError(f"out must be contiguous float32 [{B}, Sy >= 1]")
        st = torch.cuda.current_stream(x_t.device).cuda_stream if stream is None else stream
        self._ck(self.lib.vtts_time_stretch(self.h, _ptr(x_t), _ptr(lengths_t), B, S, _ptr(tp), _ptr(out), int(out.shape[1]), st))
        return out

    def debug_time_stretch_decisions(self, x_t, tempo, lengths_t=None) -> np.ndarray:
        """Test hook (vtts_debug_time_stretch_decisions): int32 [B, T_max, 513], T_max = max_b time_stretch_length(S,
        tempo_b) // 256 + 1, the device's peak flags (bit 0) and princarg sides (bit 1: negative), as
        `debug_pitch_decisions` encodes them, for `time_stretch_forward` of the same arguments."""
        import torch
        B, S = x_t.shape
        tp = TEMPO.rows(tempo, B)
        T = max(self.time_stretch_length(S, a) for a in tp) // config.HOP + 1
        out = torch.empty((B, T, DENOISE_BINS), dtype=torch.int32, device=x_t.device)
        st = torch.cuda.current_stream(x_t.device).cuda_stream
        self._ck(self.lib.vtts_debug_time_stretch_decisions(self.h, _ptr(x_t), _ptr(lengths_t), B, S, _ptr(tp), _ptr(out), st))
        return out.cpu().numpy()

    def open_time_stretch_stream(self, max_streams: int, max_chunk_samples: int) -> "TimeStretchStream":
        """Streaming time stretcher with `max_streams` independent slots (vtts_time_stretch_stream_*): a slot's tempo is
        given with BEGIN and fixed until END, and its outputs, concatenated, equal `time_stretch` of its whole input bit
        for bit.  An output is released once every synthesis frame overlapping it is synthesized; END releases the rest."""
        return TimeStretchStream(self, max_streams, max_chunk_samples)

    # ---- loudness (vtts_loudness*: ITU-R BS.1770-4 gated loudness and true peak, fp32) ----
    def loudness(self, wav, rate: int = config.SAMPLE_RATE, lengths=None) -> "Loudness":
        """Host arrays: wav f32 [S] or [B,S] at `rate` (a multiple of 10 in [8000, 192000]) -> Loudness of float32 [B]
        arrays (scalars for a 1-D input): integrated, momentary and short-term loudness in LUFS (-inf where undefined) and
        the true peak in dBTP (4x oversampled by resample_poly).  lengths int [B] in [0, S]."""
        rate = _loudness_rate(rate)
        x, lens, one = _wav_rows(wav, lengths)
        B, S = x.shape
        out = np.full((B, 4), -np.inf, np.float32)
        if B and S:                                # empty rows measure as silence
            self._ck(self.lib.vtts_loudness_host(self.h, _ptr(x), _ptr(lens), B, S, rate, _ptr(out)))
        cols = [out[:, i] for i in range(4)]
        return Loudness(*(c[0] for c in cols)) if one else Loudness(*cols)

    def normalize_loudness(self, wav, target: float, rate: int = config.SAMPLE_RATE, true_peak=None, lengths=None, limit=False,
                           lookahead_ms: float = 5.0, release_ms: float = 100.0):
        """Host arrays: (y, gain_db).  y = wav * fp32(10^(g / 20)) per row with g = target - integrated loudness, at most
        true_peak - the true peak when a ceiling (dBTP, in [-20, 0]) is given; rows measuring -inf are copied (g = 0) and
        outputs past lengths[b] are 0.  target in [-70, 0] LUFS.
        limit=True (needs true_peak): reach the target and hold the ceiling with the limiter instead of lowering the
        gain: measure, limit at g = target - L, measure the result L_y, limit again at g + (target - L_y); gain_db is that
        final g (vtts_loudness_normalize_limited)."""
        rate = _loudness_rate(rate)
        target, ceiling = _loudness_target(target, true_peak)
        if limit:
            if true_peak is None:
                raise ValueError("normalize_loudness(limit=True) needs a true_peak ceiling")
            _limit_args(ceiling, rate, lookahead_ms, release_ms)
        x, lens, one = _wav_rows(wav, lengths)
        B, S = x.shape
        y = x.copy()
        g = np.zeros(B, np.float32)
        if B and S and limit:
            self._ck(self.lib.vtts_loudness_normalize_limited_host(self.h, _ptr(x), _ptr(lens), B, S, rate, target, ceiling,
                                                                   float(lookahead_ms), float(release_ms), _ptr(y), _ptr(g)))
        elif B and S:
            self._ck(self.lib.vtts_loudness_normalize_host(self.h, _ptr(x), _ptr(lens), B, S, rate, target, ceiling, _ptr(y), _ptr(g)))
        return (y[0], g[0]) if one else (y, g)

    def loudness_forward(self, x_t, rate: int = config.SAMPLE_RATE, lengths_t=None, out=None, stream=None):
        """vtts_loudness on torch CUDA tensors, stream-ordered: x_t f32 [B,S] -> f32 [B,4] (integrated, momentary,
        short-term LUFS, true peak dBTP); lengths_t int32 CUDA [B] or None."""
        rate = _loudness_rate(rate)
        B, S, out, st = _dev_rows(x_t, out, stream, 4)
        self._ck(self.lib.vtts_loudness(self.h, _ptr(x_t), _ptr(lengths_t), B, S, rate, _ptr(out), st))
        return out

    def normalize_loudness_forward(self, x_t, target: float, rate: int = config.SAMPLE_RATE, true_peak=None, lengths_t=None, out=None,
                                   gain_db=None, stream=None, limit=False, lookahead_ms: float = 5.0, release_ms: float = 100.0):
        """vtts_loudness_normalize (limit=True: vtts_loudness_normalize_limited, see normalize_loudness) on torch CUDA
        tensors, stream-ordered and without a host synchronisation: returns (y [B,S], gain_db [B]).  `out` may be x_t
        (in place)."""
        rate = _loudness_rate(rate)
        target, ceiling = _loudness_target(target, true_peak)
        if limit:
            if true_peak is None:
                raise ValueError("normalize_loudness_forward(limit=True) needs a true_peak ceiling")
            _limit_args(ceiling, rate, lookahead_ms, release_ms)
        B, S, out, st = _dev_rows(x_t, out, stream)
        gain_db = _out_tensor(gain_db, (B,), x_t.device, "gain_db")
        if limit:
            self._ck(self.lib.vtts_loudness_normalize_limited(self.h, _ptr(x_t), _ptr(lengths_t), B, S, rate, target, ceiling,
                                                              float(lookahead_ms), float(release_ms), _ptr(out), _ptr(gain_db), st))
        else:
            self._ck(self.lib.vtts_loudness_normalize(self.h, _ptr(x_t), _ptr(lengths_t), B, S, rate, target, ceiling, _ptr(out),
                                                      _ptr(gain_db), st))
        return out, gain_db

    def open_loudness_meter(self, max_streams: int, max_chunk_samples: int, rate: int = config.SAMPLE_RATE,
                            max_seconds: int = 600) -> "LoudnessMeter":
        """Streaming loudness meter with `max_streams` independent slots (vtts_loudness_stream_*): after every push a
        slot's integrated, momentary and short-term readings equal `loudness` of what it has received, bit for bit; its
        true peak lags `lookahead` samples and equals the one-shot value after END.  A slot holds up to `max_seconds`."""
        return LoudnessMeter(self, max_streams, max_chunk_samples, rate, max_seconds)

    # ---- limiter (vtts_limit*: lookahead true-peak limiter, fp32) ----
    def limit(self, wav, ceiling: float = -1.0, rate: int = config.SAMPLE_RATE, gain_db=0.0, lookahead_ms: float = 5.0,
              release_ms: float = 100.0, lengths=None):
        """Host arrays: (y, reduction_db).  wav f32 [S] or [B,S] at `rate` (a multiple of 10 in [8000, 192000]) times the
        pre-gain gain_db (a scalar or one per row, in [-70, 70] dB), held under `ceiling` dBTP (in [-20, 0]) by a
        lookahead limiter: the gain dips ahead of every 4x-oversampled peak over `lookahead_ms` (in [1, 20]) and
        recovers with `release_ms` (in [1, 2000]).  reduction_db: the deepest gain reduction per row (<= 0).  Rows whose
        peaks stay under the ceiling come back exactly as wav times the pre-gain.  lengths int [B] in [0, S]."""
        ceiling, rate, lookahead_ms, release_ms = _limit_args(ceiling, rate, lookahead_ms, release_ms)
        x, lens, one = _wav_rows(wav, lengths)
        B, S = x.shape
        g = GAIN_DB.rows(gain_db, B)
        y = np.zeros((B, S), np.float32)
        red = np.zeros(B, np.float32)
        if B and S:
            self._ck(self.lib.vtts_limit_host(self.h, _ptr(x), _ptr(lens), _ptr(g), B, S, rate, ceiling, lookahead_ms, release_ms, _ptr(y),
                                              _ptr(red)))
        return (y[0], red[0]) if one else (y, red)

    def limit_forward(self, x_t, ceiling: float = -1.0, rate: int = config.SAMPLE_RATE, gain_db=0.0, lookahead_ms: float = 5.0,
                      release_ms: float = 100.0, lengths_t=None, out=None, reduction_db=None, stream=None):
        """vtts_limit on torch CUDA tensors, stream-ordered and without a host synchronisation: returns (y [B,S],
        reduction_db [B]).  gain_db: a host scalar or [B] (validated as in `limit`), or a float32 CUDA tensor [B] read on
        the device.  `out` may be x_t (in place)."""
        import torch
        ceiling, rate, lookahead_ms, release_ms = _limit_args(ceiling, rate, lookahead_ms, release_ms)
        B, S, out, st = _dev_rows(x_t, out, stream)
        if isinstance(gain_db, torch.Tensor):
            if tuple(gain_db.shape) != (B,) or gain_db.dtype != torch.float32 or not gain_db.is_cuda or not gain_db.is_contiguous():
                raise ValueError(f"gain_db must be a contiguous float32 CUDA tensor [{B}] or host values")
            g_t = gain_db
        else:
            g_t = torch.from_numpy(GAIN_DB.rows(gain_db, B)).to(x_t.device, non_blocking=False)
        reduction_db = _out_tensor(reduction_db, (B,), x_t.device, "reduction_db")
        self._ck(self.lib.vtts_limit(self.h, _ptr(x_t), _ptr(lengths_t), _ptr(g_t), B, S, rate, ceiling, lookahead_ms, release_ms,
                                     _ptr(out), _ptr(reduction_db), st))
        return out, reduction_db

    def limiter_stream_lookahead(self, rate: int, lookahead_ms: float = 5.0) -> int:
        """inputs past sample t a limiter stream needs before it releases t: W + 19, W = max(1, rint(lookahead_ms rate / 1000))"""
        _, rate, lookahead_ms, _ = _limit_args(-1.0, rate, lookahead_ms, 100.0)
        return int(self.lib.vtts_limiter_stream_lookahead(rate, lookahead_ms))

    def open_limiter_stream(self, max_streams: int, max_chunk_samples: int, rate: int = config.SAMPLE_RATE, ceiling: float = -1.0,
                            lookahead_ms: float = 5.0, release_ms: float = 100.0) -> "LimiterStream":
        """Streaming limiter with `max_streams` independent slots (vtts_limiter_stream_*): a slot's pre-gain is given with
        BEGIN; its outputs, concatenated, equal `limit` of its whole input bit for bit.  Sample t is released once
        `lookahead` more samples have arrived; END releases the rest."""
        return LimiterStream(self, max_streams, max_chunk_samples, rate, ceiling, lookahead_ms, release_ms)

    # ---- equalizer (vtts_eq*: a cascade of second-order sections, fp32) ----
    def equalize(self, wav, eq, rate: int = config.SAMPLE_RATE, lengths=None) -> np.ndarray:
        """Host arrays: wav f32 [S] or [B,S] at `rate` through the equalizer `eq` (a spec or an sos array, see
        `eq_sections`), equal to scipy.signal.sosfilt of each row from zero state up to fp32 rounding; not clipped.
        lengths int [B] in [0, S]: outputs past lengths[b] are 0."""
        sos = eq_sections(eq, rate)
        x, lens, one = _wav_rows(wav, lengths)
        B, S = x.shape
        y = np.zeros((B, S), np.float32)
        if B and S:
            self._ck(self.lib.vtts_eq_host(self.h, _ptr(x), _ptr(lens), B, S, _ptr(sos), sos.shape[0], _ptr(y)))
        return y[0] if one else y

    def equalize_forward(self, x_t, eq, rate: int = config.SAMPLE_RATE, lengths_t=None, out=None, stream=None):
        """vtts_eq on torch CUDA tensors, stream-ordered and without a host synchronisation: x_t f32 [B,S] -> [B,S];
        lengths_t int32 CUDA [B] or None.  `out` may be x_t (in place)."""
        sos = eq_sections(eq, rate)
        B, S, out, st = _dev_rows(x_t, out, stream)
        self._ck(self.lib.vtts_eq(self.h, _ptr(x_t), _ptr(lengths_t), B, S, _ptr(sos), sos.shape[0], _ptr(out), st))
        return out

    def open_eq_stream(self, max_streams: int, max_chunk_samples: int, eq, rate: int = config.SAMPLE_RATE) -> "EqStream":
        """Streaming equalizer with `max_streams` independent slots (vtts_eq_stream_*): every push releases every sample
        it brings (no lookahead), and a slot's outputs, concatenated, equal `equalize` of its whole input bit for bit."""
        return EqStream(self, max_streams, max_chunk_samples, eq, rate)

    # ---- compressor (vtts_compress*: feed-forward soft-knee compressor, fp32) ----
    def compress(self, wav, spec="voice", rate: int = config.SAMPLE_RATE, lengths=None):
        """Host arrays: (y, reduction_db).  wav f32 [S] or [B,S] at `rate` through the compressor `spec` (see
        `compressor_params`): a soft-knee gain computer on the log level, a smooth decoupled peak detector (release, then
        attack) and the makeup gain.  reduction_db: the deepest gain reduction per row (<= 0, makeup excluded).  Rows
        that stay below the knee come back exactly as wav times the makeup factor.  lengths int [B] in [0, S]: outputs
        past lengths[b] are 0."""
        p = compressor_params(spec, rate)
        x, lens, one = _wav_rows(wav, lengths)
        B, S = x.shape
        y = np.zeros((B, S), np.float32)
        red = np.zeros(B, np.float32)
        if B and S:
            self._ck(self.lib.vtts_compress_host(self.h, _ptr(x), _ptr(lens), B, S, int(rate), *p.values(), _ptr(y), _ptr(red)))
        return (y[0], red[0]) if one else (y, red)

    def compress_forward(self, x_t, spec="voice", rate: int = config.SAMPLE_RATE, lengths_t=None, out=None, reduction_db=None,
                         stream=None):
        """vtts_compress on torch CUDA tensors, stream-ordered and without a host synchronisation: returns (y [B,S],
        reduction_db [B]), both on the device.  lengths_t int32 CUDA [B] or None.  `out` may be x_t (in place)."""
        p = compressor_params(spec, rate)
        B, S, out, st = _dev_rows(x_t, out, stream)
        reduction_db = _out_tensor(reduction_db, (B,), x_t.device, "reduction_db")
        self._ck(self.lib.vtts_compress(self.h, _ptr(x_t), _ptr(lengths_t), B, S, int(rate), *p.values(), _ptr(out), _ptr(reduction_db), st))
        return out, reduction_db

    def open_compressor_stream(self, max_streams: int, max_chunk_samples: int, spec="voice",
                               rate: int = config.SAMPLE_RATE) -> "CompressorStream":
        """Streaming compressor with `max_streams` independent slots (vtts_compressor_stream_*): every push releases every
        sample it brings (no lookahead), and a slot's outputs, concatenated, equal `compress` of its whole input bit for
        bit."""
        return CompressorStream(self, max_streams, max_chunk_samples, spec, rate)

    # ---- de-esser (vtts_deess*: split-band sibilance compressor, fp32) ----
    def deess(self, wav, spec="voice", rate: int = config.SAMPLE_RATE, lengths=None):
        """Host arrays: (y, reduction_db).  wav f32 [S] or [B,S] at `rate` through the de-esser `spec` (see
        `deesser_params`): the compressor's detector keyed by the band above the crossover `freq` (the second-order
        Butterworth high-pass h of `equalize`), and y = x - (1 - g) h, so only that band is turned down, by at most
        `range` dB.  reduction_db: the deepest reduction of the band per row (<= 0).  Rows whose high band stays below the
        knee come back exactly as wav.  lengths int [B] in [0, S]: outputs past lengths[b] are 0."""
        p = deesser_params(spec, rate)
        x, lens, one = _wav_rows(wav, lengths)
        B, S = x.shape
        y = np.zeros((B, S), np.float32)
        red = np.zeros(B, np.float32)
        if B and S:
            self._ck(self.lib.vtts_deess_host(self.h, _ptr(x), _ptr(lens), B, S, int(rate), *p.values(), _ptr(y), _ptr(red)))
        return (y[0], red[0]) if one else (y, red)

    def deess_forward(self, x_t, spec="voice", rate: int = config.SAMPLE_RATE, lengths_t=None, out=None, reduction_db=None,
                      stream=None):
        """vtts_deess on torch CUDA tensors, stream-ordered and without a host synchronisation: returns (y [B,S],
        reduction_db [B]), both on the device.  lengths_t int32 CUDA [B] or None.  `out` may be x_t (in place)."""
        p = deesser_params(spec, rate)
        B, S, out, st = _dev_rows(x_t, out, stream)
        reduction_db = _out_tensor(reduction_db, (B,), x_t.device, "reduction_db")
        self._ck(self.lib.vtts_deess(self.h, _ptr(x_t), _ptr(lengths_t), B, S, int(rate), *p.values(), _ptr(out), _ptr(reduction_db), st))
        return out, reduction_db

    def open_deesser_stream(self, max_streams: int, max_chunk_samples: int, spec="voice",
                            rate: int = config.SAMPLE_RATE) -> "DeesserStream":
        """Streaming de-esser with `max_streams` independent slots (vtts_deesser_stream_*): every push releases every
        sample it brings (no lookahead), and a slot's outputs, concatenated, and its reduction equal `deess` of its whole
        input bit for bit."""
        return DeesserStream(self, max_streams, max_chunk_samples, spec, rate)

    # ---- convolution reverb (vtts_reverb*: partitioned overlap-save FIR, fp32) ----
    def reverb(self, wav, spec="room", rate: int = config.SAMPLE_RATE, lengths=None) -> np.ndarray:
        """Host array y: wav f32 [S] or [B,S] at `rate` through the reverb `spec` (see `reverb_params`): y = (1 - mix) x
        + mix (h * x), the causal convolution with the IR h from zero state, its tail past each row's end not emitted.
        mix = 0 returns wav exactly.  lengths int [B] in [0, S]: outputs past lengths[b] are 0."""
        p = reverb_params(spec, rate)
        x, lens, one = _wav_rows(wav, lengths)
        B, S = x.shape
        y = np.zeros((B, S), np.float32)
        if B and S:
            ir = p["ir"]
            self._ck(self.lib.vtts_reverb_host(self.h, _ptr(x), _ptr(lens), B, S, int(rate), _ptr(ir), ir.size, p["mix"], _ptr(y)))
        return y[0] if one else y

    def reverb_forward(self, x_t, spec="room", rate: int = config.SAMPLE_RATE, lengths_t=None, out=None, stream=None):
        """vtts_reverb on torch CUDA tensors, stream-ordered: returns y [B,S] on the device.  lengths_t int32 CUDA [B] or
        None.  `out` may be x_t (in place).  The IR is copied to the device before the launches (once per string spec
        and rate: it is kept for later calls)."""
        import torch
        B, S, out, st = _dev_rows(x_t, out, stream)
        key = (spec, int(rate), x_t.device) if isinstance(spec, str) else None
        cached = self._reverb_irs.get(key) if key else None
        if cached is None:
            p = reverb_params(spec, rate)
            cached = (torch.from_numpy(p["ir"]).to(x_t.device), p["mix"])
            if key:
                self._reverb_irs[key] = cached
        ir_t, mix = cached
        self._ck(self.lib.vtts_reverb(self.h, _ptr(x_t), _ptr(lengths_t), B, S, int(rate), _ptr(ir_t), ir_t.numel(), mix, _ptr(out), st))
        return out

    def open_reverb_stream(self, max_streams: int, max_chunk_samples: int, spec="room",
                           rate: int = config.SAMPLE_RATE) -> "ReverbStream":
        """Streaming reverb with `max_streams` independent slots (vtts_reverb_stream_*): before END a slot that has
        received p samples has emitted 512 floor(p / 512), and a slot's outputs, concatenated, equal `reverb` of its
        whole input bit for bit."""
        return ReverbStream(self, max_streams, max_chunk_samples, spec, rate)

    # ---- background bed (vtts_bed*: a looped bed ducked by the compressor's detector on the voice, fp32) ----
    def prepare_beds(self, bed, rate: int = config.SAMPLE_RATE) -> BedBank:
        """The bank of a bed spec or a list of up to 8 (`bed_specs`) prepared on the device once: each bed resampled from
        its audio_rate to `rate` (vtts_resample) and scaled to its integrated loudness `level` (vtts_loudness_normalize;
        a silent bed stays silent).  A BedBank passes through unchanged (its rate must be `rate`)."""
        import torch
        if isinstance(bed, BedBank):
            if bed.rate != int(rate):
                raise ValueError(f"bed: the bank was prepared at {bed.rate} Hz, not {rate}")
            return bed
        ps = bed_specs(bed, rate)
        lengths = np.array([p["Nb"] for p in ps], np.int32)
        offsets = np.concatenate([[0], np.cumsum(lengths[:-1], dtype=np.int64)]).astype(np.int64)
        dev = torch.device("cuda", self.device)
        audio = torch.empty(int(lengths.sum()), dtype=torch.float32, device=dev)
        for p, o, n in zip(ps, offsets, lengths):
            row = audio[int(o):int(o) + int(n)].view(1, -1)
            a = torch.from_numpy(p["audio"]).to(dev).view(1, -1)
            if p["audio_rate"] != int(rate):
                a = self.resample_forward(a, int(rate), p["audio_rate"])
            self.normalize_loudness_forward(a, p["level"], int(rate), out=row)
        torch.cuda.current_stream(dev).synchronize()
        return BedBank(audio, offsets, lengths, ps, int(rate))

    def _bed_bank(self, bed, rate) -> BedBank:
        """prepare_beds, kept for later calls when the spec is a string or a list of strings"""
        key = None
        if isinstance(bed, str) or (isinstance(bed, (list, tuple)) and all(isinstance(b, str) for b in bed)):
            key = (bed if isinstance(bed, str) else tuple(bed), int(rate))
        bank = self._bed_banks.get(key) if key else None
        if bank is None:
            bank = self.prepare_beds(bed, rate)
            if key:
                self._bed_banks[key] = bank
        return bank

    def mix_bed(self, wav, bed="pink", rate: int = config.SAMPLE_RATE, lengths=None, index=0):
        """Host arrays: (y, reduction_db).  wav f32 [S] or [B,S] at `rate` over the bed `bed` (a spec, a list of up to 8
        or a BedBank, see `bed_params` and `prepare_beds`): the bank entry `index` (one for every row or one per row, -1
        for none) looped from its offset with an equal-power crossfade at the seam, under a raised-cosine fade-in, ducked
        by up to `duck` dB while the voice is above the threshold (the compressor's detector, ratio 20, knee 6 dB), and
        carried `tail` ms past each row's end, where the voice is silent, the bed swells back and a raised-cosine fade
        brings it to zero.  y is [B, S + tail samples]: row b holds n[b] + tail samples (n[b] as wav without a bed), then
        zeros; a single row comes back as [S + tail] ([S] without a bed).  reduction_db: the deepest duck per row (<= 0).
        lengths int [B] in [0, S]."""
        bank = self._bed_bank(bed, rate)
        x, lens, one = _wav_rows(wav, lengths)
        B, S = x.shape
        idx = bank.index(index, B)
        W = S + bank.params[0]["Tt"]
        if B and not S:                            # empty rows still carry the bed's tail
            x, lens = np.zeros((B, 1), np.float32), np.zeros(B, np.int32)
        y = np.zeros((B, x.shape[1] + bank.params[0]["Tt"]), np.float32)
        red = np.zeros(B, np.float32)
        if B:
            self._ck(self.lib.vtts_bed_mix_host(self.h, _ptr(x), _ptr(lens), B, x.shape[1], int(rate), *bank.args()[:4], _ptr(idx),
                                                *bank.args()[4:], _ptr(y), _ptr(red)))
        y = y[:, :W]
        if one:
            return (y[0] if idx[0] >= 0 else y[0, :S]), red[0]
        return y, red

    def mix_bed_forward(self, x_t, bed="pink", rate: int = config.SAMPLE_RATE, lengths_t=None, index=0, out=None, reduction_db=None,
                        stream=None):
        """vtts_bed_mix on torch CUDA tensors, stream-ordered and without a host synchronisation: returns (y [B, S + tail],
        reduction_db [B]), both on the device, as `mix_bed`.  lengths_t int32 CUDA [B] or None; `index` host values.
        The bank is prepared once per string spec and rate and kept for later calls."""
        bank = self._bed_bank(bed, rate)
        B, S, out, st = _dev_rows(x_t, out, stream, x_t.shape[1] + bank.params[0]["Tt"])
        idx = bank.index(index, B)
        reduction_db = _out_tensor(reduction_db, (B,), x_t.device, "reduction_db")
        self._ck(self.lib.vtts_bed_mix(self.h, _ptr(x_t), _ptr(lengths_t), B, S, int(rate), *bank.args()[:4], _ptr(idx),
                                       *bank.args()[4:], _ptr(out), _ptr(reduction_db), st))
        return out, reduction_db

    def open_bed_stream(self, max_streams: int, max_chunk_samples: int, bed="pink", rate: int = config.SAMPLE_RATE) -> "BedStream":
        """Streaming bed with `max_streams` independent slots (vtts_bed_stream_*): a slot's bank entry is given with
        BEGIN (`bed=`, default 0, -1 for none); every push releases every sample it brings, the push with END also the
        tail, and a slot's outputs, concatenated, and its reduction equal `mix_bed` of its whole input bit for bit."""
        return BedStream(self, max_streams, max_chunk_samples, bed, rate)

    # ---- watermark (vtts_watermark*: a keyed spread-spectrum mark on the denoiser's STFT, fp32) ----
    def watermark(self, wav, spec, lengths=None) -> np.ndarray:
        """Host array y: wav f32 [S] or [B,S] at 16 kHz marked with the key of `spec` (see `watermark_params`): every
        STFT bin from 312 to 3422 Hz scaled by 1 +- strength after the key's chip pattern.  strength 0 and rows of <= 512
        samples return wav exactly.  lengths int [B] in [0, S]: outputs past lengths[b] are 0."""
        p = watermark_params(spec)
        x, lens, one = _wav_rows(wav, lengths)
        B, S = x.shape
        y = np.zeros((B, S), np.float32)
        if B and S:
            self._ck(self.lib.vtts_watermark_host(self.h, _ptr(x), _ptr(lens), B, S, p["key"], p["strength"], _ptr(y)))
        return y[0] if one else y

    def watermark_forward(self, x_t, spec, lengths_t=None, out=None, stream=None):
        """vtts_watermark on torch CUDA tensors, stream-ordered: x_t f32 [B,S] at 16 kHz -> [B,S] (not x_t itself);
        lengths_t int32 CUDA [B] or None."""
        p = watermark_params(spec)
        B, S, out, st = _dev_rows(x_t, out, stream)
        self._ck(self.lib.vtts_watermark(self.h, _ptr(x_t), _ptr(lengths_t), B, S, p["key"], p["strength"], _ptr(out), st))
        return out

    def open_watermark_stream(self, max_streams: int, max_chunk_samples: int, spec) -> "WatermarkStream":
        """Streaming watermark with `max_streams` independent slots (vtts_watermark_stream_*), key and strength fixed:
        each slot's outputs, concatenated, equal `watermark` of its whole input bit for bit, on the denoise stream's
        schedule (at most 1023 samples of lookahead)."""
        return WatermarkStream(self, max_streams, max_chunk_samples, spec)

    def detect_watermark(self, wav, keys, rate: int = config.SAMPLE_RATE, lengths=None, search: bool = True) -> WatermarkDetection:
        """Scores host audio wav f32 [S] or [B,S] at `rate` against every key of `keys` (one or up to 4096 integers).
        search=True: the largest score over the 1024 offsets of the mark's period, so a crop is found wherever it
        starts; search=False: the score at offset 0, for audio that starts where the mark started.  `detected` is
        z >= 6.5 (search) or z >= 5 (aligned); for audio without the key these are crossed with probability at most
        7e-7 and 3.7e-6 per row and key.  Returns (z, offset, detected), each [B,K] (or [K] for one row)."""
        rate = _output_rate(rate)
        ks = watermark_keys(keys)
        x, lens, one = _wav_rows(wav, lengths)
        B, S = x.shape
        K = ks.size
        z = np.zeros((B, K), np.float32)
        off = np.zeros((B, K), np.int32)
        if B and S:
            self._ck(self.lib.vtts_watermark_detect_host(self.h, _ptr(x), _ptr(lens), B, S, rate, _ptr(ks), K, int(bool(search)),
                                                         _ptr(z), _ptr(off)))
        det = z >= (WATERMARK_SEARCH_THRESHOLD if search else WATERMARK_ALIGNED_THRESHOLD)
        return WatermarkDetection(z[0], off[0], det[0]) if one else WatermarkDetection(z, off, det)

    def detect_watermark_forward(self, x_t, keys, rate: int = config.SAMPLE_RATE, lengths_t=None, search: bool = True,
                                 stream=None) -> WatermarkDetection:
        """vtts_watermark_detect on torch CUDA tensors, stream-ordered: x_t f32 [B,S] at `rate`; keys a uint64 CUDA
        tensor [K] (torch.uint64) or host keys, copied to the device.  Returns (z f32 [B,K], offset int32 [B,K], detected
        bool [B,K]) as CUDA tensors."""
        import torch
        rate = _output_rate(rate)
        if not (isinstance(keys, torch.Tensor) and keys.is_cuda):
            keys = torch.from_numpy(watermark_keys(keys)).to(x_t.device)
        if keys.dtype != torch.uint64 or keys.dim() != 1 or not keys.is_contiguous() or not 1 <= keys.numel() <= WATERMARK_MAX_KEYS:
            raise ValueError(f"keys must be a contiguous uint64 tensor of 1 to {WATERMARK_MAX_KEYS} keys")
        B, S, z, st = _dev_rows(x_t, None, stream, keys.numel())
        off = torch.empty((B, keys.numel()), dtype=torch.int32, device=x_t.device)
        self._ck(self.lib.vtts_watermark_detect(self.h, _ptr(x_t), _ptr(lengths_t), B, S, rate, _ptr(keys), keys.numel(), int(bool(search)),
                                                _ptr(z), _ptr(off), st))
        return WatermarkDetection(z, off, z >= (WATERMARK_SEARCH_THRESHOLD if search else WATERMARK_ALIGNED_THRESHOLD))

    # ---- wire encodings (vtts_encode / vtts_decode: PCM-16, G.711 mu-law and A-law, bit-exact) ----
    def encode(self, wav, encoding, lengths=None) -> np.ndarray:
        """Codes of host audio wav f32 [S] or [B,S] in `encoding` (see `encoding_name`): np.int16 for 'pcm16' (as
        synthesizer.float_to_pcm16, NaN as 0), np.uint8 G.711 codes for 'ulaw' and 'alaw'; the same shape.  lengths int
        [B] in [0, S]: outputs past lengths[b] are the code of 0."""
        enc = encoding_name(encoding)
        x, lens, one = _wav_rows(wav, lengths)
        B, S = x.shape
        y = np.zeros((B, S), ENCODING_DTYPES[enc])
        if B and S:
            self._ck(self.lib.vtts_encode_host(self.h, _ptr(x), _ptr(lens), B, S, ENCODINGS[enc], _ptr(y)))
        return y[0] if one else y

    def encode_forward(self, x_t, encoding, lengths_t=None, out=None, stream=None):
        """vtts_encode on torch CUDA tensors, stream-ordered: x_t f32 [B,S] -> an int16 ('pcm16') or uint8 tensor [B,S]
        (`out`, contiguous, of that dtype and shape, or a new one); lengths_t int32 CUDA [B] or None."""
        import torch
        enc = encoding_name(encoding)
        assert x_t.is_cuda and x_t.dtype == torch.float32 and x_t.is_contiguous() and x_t.dim() == 2
        B, S = x_t.shape
        out = _code_tensor(out, (B, S), enc, x_t.device)
        st = torch.cuda.current_stream(x_t.device).cuda_stream if stream is None else stream
        self._ck(self.lib.vtts_encode(self.h, _ptr(x_t), _ptr(lengths_t), B, S, ENCODINGS[enc], _ptr(out), st))
        return out

    def decode(self, codes, encoding, lengths=None) -> np.ndarray:
        """Host float32 audio of codes [S] or [B,S] in `encoding` (int16 for 'pcm16', uint8 otherwise): the G.711
        expansion to int16 (or the int16 itself) over 32767, as synthesizer.read_wav scales.  Outputs past lengths[b]
        are 0."""
        enc = encoding_name(encoding)
        c = np.ascontiguousarray(codes)
        if c.dtype != ENCODING_DTYPES[enc]:
            raise ValueError(f"{enc} codes must be {np.dtype(ENCODING_DTYPES[enc]).name}, got {c.dtype}")
        one = c.ndim == 1
        c = c[None] if one else c
        if c.ndim != 2:
            raise ValueError(f"codes must be [S] or [B,S], got {np.shape(codes)}")
        B, S = c.shape
        lens = None if lengths is None else _np(lengths, np.int32, (B,), "lengths")
        y = np.zeros((B, S), np.float32)
        if B and S:
            self._ck(self.lib.vtts_decode_host(self.h, _ptr(c), _ptr(lens), B, S, ENCODINGS[enc], _ptr(y)))
        return y[0] if one else y

    def decode_forward(self, c_t, encoding, lengths_t=None, out=None, stream=None):
        """vtts_decode on torch CUDA tensors, stream-ordered: codes c_t [B,S] (int16 for 'pcm16', uint8 otherwise) -> f32
        [B,S]; lengths_t int32 CUDA [B] or None."""
        import torch
        enc = encoding_name(encoding)
        if not (c_t.is_cuda and c_t.is_contiguous() and c_t.dim() == 2 and c_t.dtype == _torch_code_dtype(enc)):
            raise ValueError(f"{enc} codes must be a contiguous {_torch_code_dtype(enc)} CUDA tensor [B,S]")
        B, S = c_t.shape
        out = _out_tensor(out, (B, S), c_t.device)
        st = torch.cuda.current_stream(c_t.device).cuda_stream if stream is None else stream
        self._ck(self.lib.vtts_decode(self.h, _ptr(c_t), _ptr(lengths_t), B, S, ENCODINGS[enc], _ptr(out), st))
        return out


    # ---- FLAC (vtts_flac_encode: lossless frames of the PCM-16 codes, oracle/flac_oracle.py byte for byte) ----
    def encode_flac(self, wav, rate=config.SAMPLE_RATE, lengths=None, block=4096):
        """Native FLAC streams (mono, 16 bits, streamable subset) of host audio wav f32 [S] or [B,S] at `rate`: bytes
        for [S], a list of bytes per row for [B,S].  The samples are the PCM-16 codes of `encode(wav, 'pcm16')`, so a
        decoder gives those back exactly.  lengths int [B] in [0, S]: row b holds its first lengths[b] samples."""
        rate, block = flac_rate(rate), flac_block(block)
        x, lens, one = _wav_rows(wav, lengths)
        B, S = x.shape
        out = []
        if B:
            pitch = flac_bound(S, block)
            y = np.empty((B, pitch), np.uint8)
            nb = np.zeros(B, np.int32)
            self._ck(self.lib.vtts_flac_encode_host(self.h, _ptr(x) if S else None, _ptr(lens), B, S, rate, block, _ptr(y),
                                                    pitch, _ptr(nb)))
            out = [y[b, : nb[b]].tobytes() for b in range(B)]
        return out[0] if one else out

    def open_flac_stream(self, max_streams: int, max_chunk_samples: int, rate=config.SAMPLE_RATE, block=4096) -> "FlacStream":
        """Per-slot FLAC streams (FlacStream): push samples as they arrive, get each slot's finished frames."""
        return FlacStream(self, max_streams, max_chunk_samples, rate, block)

    def encode_flac_forward(self, x_t, rate=config.SAMPLE_RATE, lengths_t=None, block=4096, out=None, stream=None):
        """vtts_flac_encode on torch CUDA tensors, stream-ordered: x_t f32 [B,S] -> (uint8 [B, flac_bound(S, block)],
        int32 nbytes [B]): row b's stream is out[b, :nbytes[b]], and nothing past it is written.  `out`: a contiguous
        uint8 CUDA tensor [B, >= the bound] (its row stride is the pitch) or None."""
        import torch
        rate, block = flac_rate(rate), flac_block(block)
        assert x_t.is_cuda and x_t.dtype == torch.float32 and x_t.is_contiguous() and x_t.dim() == 2
        B, S = x_t.shape
        bound = flac_bound(S, block)
        if out is None:
            out = torch.empty((B, bound), dtype=torch.uint8, device=x_t.device)
        elif not (out.is_cuda and out.dtype == torch.uint8 and out.dim() == 2 and out.shape[0] == B and out.shape[1] >= bound
                  and out.is_contiguous()):
            raise ValueError(f"out must be a contiguous uint8 CUDA tensor [{B}, >= {bound}]")
        nbytes = torch.empty(B, dtype=torch.int32, device=x_t.device)
        st = torch.cuda.current_stream(x_t.device).cuda_stream if stream is None else stream
        self._ck(self.lib.vtts_flac_encode(self.h, _ptr(x_t), _ptr(lengths_t), B, S, rate, block, _ptr(out), out.shape[1],
                                           _ptr(nbytes), st))
        return out, nbytes


class Loudness(NamedTuple):
    integrated: np.ndarray     # LUFS (gated, BS.1770-4)
    momentary: np.ndarray      # LUFS, the last 400 ms block
    short_term: np.ndarray     # LUFS, the last 3 s
    true_peak: np.ndarray      # dBTP


def _loudness_rate(rate) -> int:
    r = int(rate)
    if r != rate or r % 10 or not 8000 <= r <= 192000:
        raise ValueError(f"loudness: rate {rate} must be a multiple of 10 in [8000, 192000] (100 ms a whole number of samples)")
    return r


def _loudness_target(target, true_peak):
    """(target, ceiling) as vtts_loudness_normalize takes them: ceiling +inf for none"""
    t = float(target)
    if not -70.0 <= t <= 0.0:
        raise ValueError(f"loudness target {target} LUFS must lie in [-70, 0]")
    if true_peak is None:
        return t, float("inf")
    c = float(true_peak)
    if not (np.isfinite(c) and -20.0 <= c <= 0.0):
        raise ValueError(f"true-peak ceiling {true_peak} dBTP must be finite and lie in [-20, 0]")
    return t, c


def _limit_args(ceiling, rate, lookahead_ms, release_ms):
    """(ceiling, rate, lookahead_ms, release_ms) as vtts_limit takes them, each checked"""
    c = float(ceiling)
    if not (np.isfinite(c) and -20.0 <= c <= 0.0):
        raise ValueError(f"limiter ceiling {ceiling} dBTP must be finite and lie in [-20, 0]")
    r = _loudness_rate(rate)
    a, rel = float(lookahead_ms), float(release_ms)
    if not (np.isfinite(a) and 1.0 <= a <= 20.0):
        raise ValueError(f"limiter lookahead {lookahead_ms} ms must lie in [1, 20]")
    if not (np.isfinite(rel) and 1.0 <= rel <= 2000.0):
        raise ValueError(f"limiter release {release_ms} ms must lie in [1, 2000]")
    return c, r, a, rel


def _gain_db(v, n: int) -> np.ndarray:
    """float32 [n]: a scalar pre-gain for every row, or one per row, each finite and in [-70, 70] dB"""
    return GAIN_DB.rows(v, n)


STREAM_BEGIN, STREAM_END = 1, 2


class _SlotStream:
    """What every per-slot stream handle shares: the library handle `h` of one stream of `eng`'s context, the marshalling
    of a push (zero padding of short chunks, the BEGIN / END flag bits, the n_new / flags arrays, the device-buffer checks,
    the CUDA stream, the per-slot BEGIN parameters), the push itself and the lifecycle.  A subclass opens its stream and
    declares its kind, its input, its output width and its BEGIN parameters."""
    _kind = ""       # the library's vtts_<kind>_push[_host] pushes and vtts_<kind>_destroy closes the stream
    _push_kind = ""  # the push's own kind where it differs from _kind
    _x = "x"         # the input's name in error messages
    _row = ()        # shape of one input element past [S, F]: () for samples, (80,) for mel frames
    _scale = 1       # output samples per unit of n_out
    _params = ()     # the _BeginParams a push takes for the slots it begins, in the push's argument order
    _carried = ()    # per _param: the attribute holding each slot's value since its BEGIN
    h = None

    def __init__(self, eng: Engine, max_streams: int, max_chunk: int):
        self.eng = eng
        self.max_streams, self._chunk = int(max_streams), int(max_chunk)
        for p, name in zip(self._params, self._carried):
            setattr(self, name, np.full(self.max_streams, p.neutral, np.float32))

    @property
    def _width(self):
        """outputs per slot of a push's output buffer"""
        return self.out_pitch

    def _create(self, fn, *args, pitch=False):
        """calls vtts_<kind>_create(ctx, *args, &h[, &pitch]); sets `h` and, with pitch, `out_pitch`"""
        h, p = C.c_void_p(), C.c_int()
        self.eng._ck(fn(self.eng.h, *args, C.byref(h), *((C.byref(p),) if pitch else ())))
        self.h = h
        if pitch:
            self.out_pitch = int(p.value)   # outputs per slot of a push's output buffer

    def _host_in(self, x, n_new, begin, end):
        """(x f32 [S, F, *row] zero-padded, n_new int32 [S], flags uint8 [S]) of a host push"""
        S, F, row = self.max_streams, self._chunk, self._row
        x = _np(x, np.float32)
        if x.ndim != 2 + len(row) or x.shape[0] != S or x.shape[1] > F or x.shape[2:] != row:
            raise ValueError(f"{self._x} must be [{S}, <= {F}{''.join(f', {d}' for d in row)}], got {x.shape}")
        if x.shape[1] < F:
            x = np.concatenate([x, np.zeros((S, F - x.shape[1]) + row, np.float32)], axis=1)
        flags = np.zeros(S, np.uint8)
        if begin is not None:
            flags |= np.asarray(begin, bool).astype(np.uint8) * STREAM_BEGIN
        if end is not None:
            flags |= np.asarray(end, bool).astype(np.uint8) * STREAM_END
        return (x,) + self._args(n_new, flags)

    def _args(self, n_new, flags):
        S = self.max_streams
        return _np(n_new, np.int32, (S,), "n_new"), _np(flags, np.uint8, (S,), "flags")

    def _device_in(self, x_t, out_t, n_new, flags, stream):
        """(n_new int32 [S], flags uint8 [S], CUDA stream) of a device push, after checking both buffers"""
        import torch
        for t, name, shape in ((x_t, self._x + "_t", (self.max_streams, self._chunk) + self._row),
                               (out_t, "out_t", (self.max_streams, self._width))):
            if tuple(t.shape) != shape or t.dtype != torch.float32 or not t.is_contiguous():
                raise ValueError(f"{name} must be contiguous float32 [{', '.join(map(str, shape))}]")
        st = torch.cuda.current_stream(x_t.device).cuda_stream if stream is None else stream
        return self._args(n_new, flags) + (st,)

    def _values(self, flags, vs) -> tuple:
        """per BEGIN parameter, float32 [S]: the push's value (a scalar or [S]) in `vs` for the slots it begins and each
        slot's carried value elsewhere, which the library checks is unchanged; None for an optional parameter left out
        (the slots that begin take its neutral value)"""
        return tuple(self._value(p, name, flags, v) for p, name, v in zip(self._params, self._carried, vs))

    def _value(self, p, carried, flags, v):
        out = getattr(self, carried).copy()
        begin = (flags & STREAM_BEGIN) != 0
        v = p.default if v is None else v
        if v is None and p.optional:
            return None
        if begin.any():
            if v is None:
                raise ValueError(f"{p.name}= is required for the slots a push begins")
            g = np.asarray(v, np.float32)
            g = np.full(out.size, g, np.float32) if g.ndim == 0 else g
            if g.shape != (out.size,):
                raise ValueError(f"{p.name}: one value or one per slot ({out.size}), got {np.shape(v)}")
            out[begin] = g[begin]
        if p.host_check:
            _per_row(out, out.size, p.name, p.lo, p.hi, shown=v)
        return out

    def _outs(self):
        """the push call's outputs after y: n_out int32 [S] (a subclass adds its own)"""
        return (np.zeros(self.max_streams, np.int32),)

    def _result(self, y, outs, host: bool):
        """what a push returns: each slot's new outputs (host) or n_out (device)"""
        return self._rows(y, outs[0], self._scale) if host else outs[0]

    def _push(self, host: bool, x, n, f, values, y, outs, st=None):
        fn = getattr(self.eng.lib, f"vtts_{self._push_kind or self._kind}_push" + ("_host" if host else ""))
        self.eng._ck(fn(self.eng.h, self.h, _ptr(x), _ptr(n), _ptr(f), *map(_ptr, values), _ptr(y), *map(_ptr, outs),
                        *(() if host else (st,))))
        begin = (f & STREAM_BEGIN) != 0
        for p, name, v in zip(self._params, self._carried, values):
            getattr(self, name)[begin] = p.neutral if v is None else v[begin]
        return self._result(y, outs, host)

    def _push_host(self, x, n_new, begin, end, *vs):
        x, n, f = self._host_in(x, n_new, begin, end)
        values = self._values(f, vs)
        y = np.empty((self.max_streams, self._width), np.float32)
        return self._push(True, x, n, f, values, y, self._outs())

    def _push_device(self, x_t, n_new, flags, out_t, stream, *vs, dev=()):
        """`dev`: the stream's own device outputs after n_out"""
        n, f, st = self._device_in(x_t, out_t, n_new, flags, stream)
        values = self._values(f, vs)
        return self._push(False, x_t, n, f, values, out_t, self._outs(*dev), st)

    def push(self, x, n_new, begin=None, end=None) -> list:
        """x f32 [S, <= max_chunk_samples] (samples past n_new[s] ignored), n_new int [S], begin / end bool [S] or None.
        Returns one float32 array per slot with the samples it emits now."""
        return self._push_host(x, n_new, begin, end)

    def push_device(self, x_t, n_new, flags, out_t, stream=None) -> np.ndarray:
        """Device buffers: x_t f32 CUDA [S, max_chunk_samples], out_t f32 CUDA [S, out_pitch]; n_new int [S] and flags
        uint8 [S] (bit0 BEGIN, bit1 END) on the host.  Stream-ordered; returns n_out int32 [S] (outputs slot s got at the
        start of its row of out_t)."""
        return self._push_device(x_t, n_new, flags, out_t, stream)

    def _rows(self, y, n_out, scale=1):
        return [y[s, : int(n_out[s]) * scale].copy() for s in range(self.max_streams)]

    def close(self):
        if getattr(self, "h", None) and getattr(self.eng, "h", None):
            self.eng._ck(getattr(self.eng.lib, f"vtts_{self._kind}_destroy")(self.eng.h, self.h))
        self.h = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class VocoderStream(_SlotStream):
    """Handle of a streaming generator (Engine.open_vocoder_stream): push mel f32 [S, F', 80], get 256 samples per
    frame.  A slot that has received P frames since BEGIN has emitted max(0, P - lookahead) frames; a push with END
    emits the rest.  `push_device` takes out_t [S, wav_ld] and returns n_out in frames."""
    _kind, _x, _row, _scale = "vocoder_stream", "mel", (config.MEL_DIM,), config.HOP

    def __init__(self, eng: Engine, max_streams: int, max_chunk_frames: int):
        super().__init__(eng, max_streams, max_chunk_frames)
        self.max_chunk_frames = self._chunk
        self.lookahead = int(eng.lib.vtts_vocoder_stream_lookahead())
        self.wav_ld = config.HOP * (self.max_chunk_frames + self.lookahead)   # samples per slot of the output buffer
        self._create(eng.lib.vtts_vocoder_stream_create, self.max_streams, self.max_chunk_frames)

    @property
    def _width(self):
        return self.wav_ld

    def push(self, mel, n_new, begin=None, end=None) -> list:
        """mel f32 [S,F',80] (F' <= max_chunk_frames; rows past n_new[s] ignored), n_new int [S], begin / end bool [S]
        or None.  Returns one float32 array per slot with the samples it emits now (256 per frame)."""
        return self._push_host(mel, n_new, begin, end)

    def push_device(self, mel_t, n_new, flags, out_t, stream=None) -> np.ndarray:
        """Device buffers: mel_t f32 CUDA [S,F,80], out_t f32 CUDA [S, 256*(F+lookahead)]; n_new int [S] and flags
        uint8 [S] (bit0 BEGIN, bit1 END) on the host.  Stream-ordered; returns n_out int32 [S] (frames slot s got at
        the start of its row of out_t)."""
        return self._push_device(mel_t, n_new, flags, out_t, stream)


class ResampleStream(_SlotStream):
    """Handle of a streaming resampler (Engine.open_resample_stream).  Before END a slot that has received P samples
    has emitted min(ceil(P up / down), max(0, floor((P up - 1 - half) / down) + 1)) outputs, half = 10 max(up, down);
    a push with END emits the rest."""
    _kind = "resample_stream"

    def __init__(self, eng: Engine, max_streams: int, max_chunk_samples: int, out_rate: int, in_rate: int = config.SAMPLE_RATE):
        super().__init__(eng, max_streams, max_chunk_samples)
        self.max_chunk_samples = self._chunk
        self.in_rate, self.out_rate = int(in_rate), int(out_rate)
        resample_ratio(self.in_rate, self.out_rate)
        self._create(eng.lib.vtts_resample_stream_create, self.max_streams, self.max_chunk_samples, self.in_rate, self.out_rate, pitch=True)
        self.lookahead = int(eng.lib.vtts_resample_stream_lookahead(self.in_rate, self.out_rate))


class DenoiseStream(_SlotStream):
    """Handle of a streaming denoiser (Engine.open_denoise_stream).  Before END a slot that has received P samples has
    emitted min(P, 256 max(0, floor(P / 256) - 3)) outputs; a push with END emits the rest."""
    _kind = "denoise_stream"

    def __init__(self, eng: Engine, max_streams: int, max_chunk_samples: int, strength: float, bias=None):
        super().__init__(eng, max_streams, max_chunk_samples)
        self.max_chunk_samples = self._chunk
        self.strength = _strength(strength)
        self.bias = eng._bias_arg(bias)
        self._create(eng.lib.vtts_denoise_stream_create, self.max_streams, self.max_chunk_samples, self.strength, _ptr(self.bias),
                     pitch=True)
        self.lookahead = int(eng.lib.vtts_denoise_stream_lookahead())


class PitchShiftStream(_SlotStream):
    """Handle of a streaming pitch shifter (Engine.open_pitch_shift_stream): `semitones=` with BEGIN.  Before END a slot
    that has received P samples has emitted min(P, 256 max(0, floor(P / 256) - 3)) outputs; a push with END emits the
    rest.  `shift` holds each slot's shift since its BEGIN."""
    _kind, _params, _carried = "pitch_shift_stream", (SEMITONES,), ("shift",)

    def __init__(self, eng: Engine, max_streams: int, max_chunk_samples: int):
        super().__init__(eng, max_streams, max_chunk_samples)
        self.max_chunk_samples = self._chunk
        self._create(eng.lib.vtts_pitch_shift_stream_create, self.max_streams, self.max_chunk_samples, pitch=True)
        self.lookahead = int(eng.lib.vtts_pitch_shift_stream_lookahead())

    def push(self, x, n_new, begin=None, end=None, semitones=None) -> list:
        """As `_SlotStream.push`, with semitones: a scalar or [S], read for the slots that begin."""
        return self._push_host(x, n_new, begin, end, semitones)

    def push_device(self, x_t, n_new, flags, out_t, semitones=None, stream=None) -> np.ndarray:
        """As `_SlotStream.push_device`, with semitones (host scalar or [S], read for the slots that begin)."""
        return self._push_device(x_t, n_new, flags, out_t, stream, semitones)


class VoiceShiftStream(PitchShiftStream):
    """Handle of a streaming voice shifter (Engine.open_voice_shift_stream): the pitch-shift stream with `semitones=`
    and `formant=` with BEGIN.  `formant` holds each slot's formant shift since its BEGIN (NaN: the formants follow the
    pitch, as a push that leaves `formant=` out begins its slots)."""
    _push_kind, _params, _carried = "voice_shift_stream", (SEMITONES, FORMANT), ("shift", "formant")

    def push(self, x, n_new, begin=None, end=None, semitones=None, formant=None) -> list:
        """As `_SlotStream.push`, with semitones and formant: each a scalar or [S], read for the slots that begin."""
        return self._push_host(x, n_new, begin, end, semitones, formant)

    def push_device(self, x_t, n_new, flags, out_t, semitones=None, formant=None, stream=None) -> np.ndarray:
        """As `_SlotStream.push_device`, with semitones and formant (host scalars or [S], read for the slots that begin)."""
        return self._push_device(x_t, n_new, flags, out_t, stream, semitones, formant)


class TimeStretchStream(_SlotStream):
    """Handle of a streaming time stretcher (Engine.open_time_stretch_stream): `tempo=` with BEGIN.  Before END a slot at
    tempo alpha that has scanned Q frames (frame t once rint(256 t alpha) + 512 <= P, P > 512) has released
    max(0, 256 Q - 511) outputs (all P at tempo 1); a push with END releases the rest.  `tempo` holds each slot's tempo
    since its BEGIN."""
    _kind, _params, _carried = "time_stretch_stream", (TEMPO,), ("tempo",)

    def __init__(self, eng: Engine, max_streams: int, max_chunk_samples: int):
        super().__init__(eng, max_streams, max_chunk_samples)
        self.max_chunk_samples = self._chunk
        self._create(eng.lib.vtts_time_stretch_stream_create, self.max_streams, self.max_chunk_samples, pitch=True)
        self.lookahead = int(eng.lib.vtts_time_stretch_stream_lookahead())

    def push(self, x, n_new, begin=None, end=None, tempo=None) -> list:
        """As `_SlotStream.push`, with tempo: a scalar or [S], read for the slots that begin."""
        return self._push_host(x, n_new, begin, end, tempo)

    def push_device(self, x_t, n_new, flags, out_t, tempo=None, stream=None) -> np.ndarray:
        """As `_SlotStream.push_device`, with tempo (host scalar or [S], read for the slots that begin)."""
        return self._push_device(x_t, n_new, flags, out_t, stream, tempo)


class LoudnessMeter(_SlotStream):
    """Handle of a streaming loudness meter (Engine.open_loudness_meter).  Every push returns every slot's readings
    [S,4] (`push_device`: fills out_t [S,4] and returns it): integrated, momentary, short-term LUFS and true peak dBTP of
    the samples it has received since BEGIN."""
    _kind, _width = "loudness_stream", 4

    def __init__(self, eng: Engine, max_streams: int, max_chunk_samples: int, rate: int = config.SAMPLE_RATE, max_seconds: int = 600):
        super().__init__(eng, max_streams, max_chunk_samples)
        self.max_chunk_samples = self._chunk
        self.rate, self.max_seconds = _loudness_rate(rate), int(max_seconds)
        self._create(eng.lib.vtts_loudness_stream_create, self.max_streams, self.max_chunk_samples, self.rate, self.max_seconds)
        self.lookahead = int(eng.lib.vtts_loudness_stream_lookahead(self.rate))

    def _outs(self):
        return ()

    def _result(self, y, outs, host: bool):
        return y


class _ReductionStream(_SlotStream):
    """A stream handle that also reports each slot's gain reduction so far: `reduction_db` after a host push, the
    required reduction_t f32 CUDA [S] of a device push."""

    def _outs(self, *dev):
        """a host push: n_out and a new host reduction array; a device push: n_out and reduction_t, which must be a tensor"""
        import torch
        if not dev:
            return super()._outs() + (np.empty(self.max_streams, np.float32),)
        (red,) = dev
        if (not isinstance(red, torch.Tensor) or tuple(red.shape) != (self.max_streams,) or red.dtype != torch.float32
                or not red.is_contiguous()):
            raise ValueError(f"reduction_t must be a contiguous float32 tensor [{self.max_streams}]")
        return super()._outs() + (red,)

    def _result(self, y, outs, host: bool):
        if host:
            self.reduction_db = outs[1]
        return super()._result(y, outs, host)


class LimiterStream(_ReductionStream):
    """Handle of a streaming limiter (Engine.open_limiter_stream): `gain_db=` with BEGIN (default 0 dB).  Before END a slot that has received P samples has released
    max(0, P - lookahead) outputs; a push with END releases the rest.  After every host push `reduction_db` holds each
    slot's deepest reduction over what it has released since BEGIN; `gain_db` holds each slot's pre-gain."""
    _kind, _params, _carried = "limiter_stream", (GAIN_DB,), ("gain_db",)

    def __init__(self, eng: Engine, max_streams: int, max_chunk_samples: int, rate: int = config.SAMPLE_RATE, ceiling: float = -1.0,
                 lookahead_ms: float = 5.0, release_ms: float = 100.0):
        super().__init__(eng, max_streams, max_chunk_samples)
        self.max_chunk_samples = self._chunk
        self.ceiling, self.rate, self.lookahead_ms, self.release_ms = _limit_args(ceiling, rate, lookahead_ms, release_ms)
        self._create(eng.lib.vtts_limiter_stream_create, self.max_streams, self.max_chunk_samples, self.rate, self.ceiling,
                     self.lookahead_ms, self.release_ms, pitch=True)
        self.lookahead = int(eng.lib.vtts_limiter_stream_lookahead(self.rate, self.lookahead_ms))
        self.reduction_db = np.zeros(self.max_streams, np.float32)   # host pushes: each slot's reduction so far

    def push(self, x, n_new, begin=None, end=None, gain_db=None) -> list:
        """As `_SlotStream.push`, with gain_db: a scalar or [S], read for the slots that begin (default 0 dB)."""
        return self._push_host(x, n_new, begin, end, gain_db)

    def push_device(self, x_t, n_new, flags, out_t, reduction_t, gain_db=None, stream=None) -> np.ndarray:
        """As `_SlotStream.push_device`, with reduction_t f32 CUDA [S] (each slot's reduction so far, written on the
        device) and gain_db (host scalar or [S], read for the slots that begin, default 0 dB)."""
        return self._push_device(x_t, n_new, flags, out_t, stream, gain_db, dev=(reduction_t,))


class EqStream(_SlotStream):
    """Handle of a streaming equalizer (Engine.open_eq_stream).  Every push releases every sample it brings:
    n_out = n_new (`push_device`: out_t may be x_t)."""
    _kind = "eq_stream"
    lookahead = 0

    def __init__(self, eng: Engine, max_streams: int, max_chunk_samples: int, eq, rate: int = config.SAMPLE_RATE):
        super().__init__(eng, max_streams, max_chunk_samples)
        self.max_chunk_samples = self.out_pitch = self._chunk
        self.sos = eq_sections(eq, rate)
        self._create(eng.lib.vtts_eq_stream_create, self.max_streams, self.max_chunk_samples, _ptr(self.sos), self.sos.shape[0])


class CompressorStream(_ReductionStream):
    """Handle of a streaming compressor (Engine.open_compressor_stream).  Every push releases every sample it brings:
    n_out = n_new (`push_device`: out_t may be x_t).  After every host push `reduction_db` holds each slot's deepest
    reduction over what it has released since BEGIN."""
    _kind = "compressor_stream"
    lookahead = 0

    def __init__(self, eng: Engine, max_streams: int, max_chunk_samples: int, spec="voice", rate: int = config.SAMPLE_RATE):
        super().__init__(eng, max_streams, max_chunk_samples)
        self.max_chunk_samples = self.out_pitch = self._chunk
        self.params, self.rate = compressor_params(spec, rate), int(rate)
        self._create(eng.lib.vtts_compressor_stream_create, self.max_streams, self.max_chunk_samples, self.rate, *self.params.values())
        self.reduction_db = np.zeros(self.max_streams, np.float32)   # host pushes: each slot's reduction so far

    def push_device(self, x_t, n_new, flags, out_t, reduction_t, stream=None) -> np.ndarray:
        """As `_SlotStream.push_device`, with reduction_t f32 CUDA [S] (each slot's reduction so far, written on the
        device)."""
        return self._push_device(x_t, n_new, flags, out_t, stream, dev=(reduction_t,))


class DeesserStream(_ReductionStream):
    """Handle of a streaming de-esser (Engine.open_deesser_stream).  Every push releases every sample it brings:
    n_out = n_new (`push_device`: out_t may be x_t).  After every host push `reduction_db` holds each slot's deepest
    reduction of its high band over what it has released since BEGIN."""
    _kind = "deesser_stream"
    lookahead = 0

    def __init__(self, eng: Engine, max_streams: int, max_chunk_samples: int, spec="voice", rate: int = config.SAMPLE_RATE):
        super().__init__(eng, max_streams, max_chunk_samples)
        self.max_chunk_samples = self.out_pitch = self._chunk
        self.params, self.rate = deesser_params(spec, rate), int(rate)
        self._create(eng.lib.vtts_deesser_stream_create, self.max_streams, self.max_chunk_samples, self.rate, *self.params.values())
        self.reduction_db = np.zeros(self.max_streams, np.float32)   # host pushes: each slot's reduction so far

    def push_device(self, x_t, n_new, flags, out_t, reduction_t, stream=None) -> np.ndarray:
        """As `_SlotStream.push_device`, with reduction_t f32 CUDA [S] (each slot's reduction so far, written on the
        device)."""
        return self._push_device(x_t, n_new, flags, out_t, stream, dev=(reduction_t,))


class ReverbStream(_SlotStream):
    """Handle of a streaming reverb (Engine.open_reverb_stream).  Before END a slot that has received p samples has
    emitted 512 floor(p / 512) outputs (`lookahead` = 511); a push with END emits the rest."""
    _kind = "reverb_stream"

    def __init__(self, eng: Engine, max_streams: int, max_chunk_samples: int, spec="room", rate: int = config.SAMPLE_RATE):
        super().__init__(eng, max_streams, max_chunk_samples)
        self.max_chunk_samples = self._chunk
        self.params, self.rate = reverb_params(spec, rate), int(rate)
        ir = self.params["ir"]
        self._create(eng.lib.vtts_reverb_stream_create, self.max_streams, self.max_chunk_samples, self.rate, _ptr(ir), ir.size,
                     self.params["mix"], pitch=True)
        self.lookahead = int(eng.lib.vtts_reverb_stream_lookahead())


class BedStream(_ReductionStream):
    """Handle of a streaming bed (Engine.open_bed_stream): `bed=` with BEGIN, the slot's bank entry (default 0, -1 for
    none).  Every push releases every sample it brings, and the push with END also the slot's `tail` samples
    (n_out = n_new, + tail at END with a bed; out_pitch = max_chunk_samples + tail).  After every host push
    `reduction_db` holds each slot's deepest duck over what it has released since BEGIN; `bed` holds each slot's entry."""
    _kind, _params, _carried = "bed_stream", (BED,), ("bed",)
    lookahead = 0

    def __init__(self, eng: Engine, max_streams: int, max_chunk_samples: int, bed="pink", rate: int = config.SAMPLE_RATE):
        super().__init__(eng, max_streams, max_chunk_samples)
        self.max_chunk_samples = self._chunk
        self.rate = int(rate)
        self.bank = eng.prepare_beds(bed, self.rate)    # held: the stream reads it until it closes
        self.tail = self.bank.params[0]["Tt"]
        self.bed = np.full(self.max_streams, -1, np.int32)
        self._create(eng.lib.vtts_bed_stream_create, self.max_streams, self.max_chunk_samples, self.rate, *self.bank.args(), pitch=True)
        self.reduction_db = np.zeros(self.max_streams, np.float32)   # host pushes: each slot's reduction so far

    def _values(self, flags, vs) -> tuple:
        """(int32 [S],): the push's entry `vs[0]` (default 0; one or one per slot) for the slots it begins, each slot's
        own elsewhere"""
        (v,) = vs
        out = self.bed.copy()
        begin = (flags & STREAM_BEGIN) != 0
        if begin.any():
            out[begin] = self.bank.index(BED.default if v is None else v, out.size)[begin]
        return (out,)

    def push(self, x, n_new, begin=None, end=None, bed=None) -> list:
        """As `_SlotStream.push`, with bed: a bank entry or one per slot, read for the slots that begin (default 0)."""
        return self._push_host(x, n_new, begin, end, bed)

    def push_device(self, x_t, n_new, flags, out_t, reduction_t, bed=None, stream=None) -> np.ndarray:
        """As `_SlotStream.push_device`, with reduction_t f32 CUDA [S] (each slot's reduction so far, written on the
        device) and bed (host, read for the slots that begin, default 0)."""
        return self._push_device(x_t, n_new, flags, out_t, stream, bed, dev=(reduction_t,))


class WatermarkStream(_SlotStream):
    """Handle of a streaming watermark (Engine.open_watermark_stream).  Before END a slot that has received P samples
    has emitted min(P, 256 max(0, floor(P / 256) - 3)) outputs; a push with END emits the rest."""
    _kind = "watermark_stream"

    def __init__(self, eng: Engine, max_streams: int, max_chunk_samples: int, spec):
        super().__init__(eng, max_streams, max_chunk_samples)
        self.max_chunk_samples = self._chunk
        self.params = watermark_params(spec)
        self._create(eng.lib.vtts_watermark_stream_create, self.max_streams, self.max_chunk_samples, self.params["key"],
                     self.params["strength"], pitch=True)
        self.lookahead = int(eng.lib.vtts_watermark_stream_lookahead())


def flac_stream_frames(p: int, block: int, end: bool = False) -> int:
    """frames a FLAC stream slot has emitted after p samples since BEGIN: floor(p / block), ceil(p / block) once END"""
    return -(-int(p) // block) if end else int(p) // block


class FlacStream(_SlotStream):
    """Handle of a per-slot FLAC stream (Engine.open_flac_stream).  A slot's bytes from BEGIN to END are
    `Engine.encode_flac` of its samples with STREAMINFO's total samples and min / max frame size 0 ("unknown"): the
    stream header with BEGIN, then each frame once its block of samples has arrived, and the short last frame with END
    (flac_stream_frames).  `push` returns one `bytes` per slot; `push_device` writes every slot's bytes packed into out_t
    (uint8 [out_bytes]) and their (offset, count) into tbl_t (int32 [S, 2])."""
    _kind = "flac_stream"

    def __init__(self, eng: Engine, max_streams: int, max_chunk_samples: int, rate=config.SAMPLE_RATE, block=4096):
        super().__init__(eng, max_streams, max_chunk_samples)
        self.max_chunk_samples = self._chunk
        self.rate, self.block = flac_rate(rate), flac_block(block)
        h, nb = C.c_void_p(), C.c_int64()
        eng._ck(eng.lib.vtts_flac_stream_create(eng.h, self.max_streams, self._chunk, self.rate, self.block, C.byref(h),
                                                C.byref(nb)))
        self.h, self.out_bytes = h, int(nb.value)

    def push(self, x, n_new, begin=None, end=None) -> list:
        """x f32 [S, <= max_chunk_samples], n_new int [S], begin / end bool [S] or None; one `bytes` per slot"""
        x, n, f = self._host_in(x, n_new, begin, end)
        y = np.empty(self.out_bytes, np.uint8)
        tbl = np.zeros((self.max_streams, 2), np.int32)
        self.eng._ck(self.eng.lib.vtts_flac_stream_push_host(self.eng.h, self.h, _ptr(x), _ptr(n), _ptr(f), _ptr(y), _ptr(tbl)))
        return [y[o:o + c].tobytes() for o, c in tbl]

    def push_device(self, x_t, n_new, flags, out_t, tbl_t, stream=None):
        """x_t f32 CUDA [S, max_chunk_samples], out_t uint8 CUDA [out_bytes], tbl_t int32 CUDA [S, 2]; n_new and flags
        on the host.  Stream-ordered."""
        import torch
        S, F = self.max_streams, self._chunk
        if tuple(x_t.shape) != (S, F) or x_t.dtype != torch.float32 or not x_t.is_contiguous():
            raise ValueError(f"x_t must be contiguous float32 [{S}, {F}]")
        if tuple(out_t.shape) != (self.out_bytes,) or out_t.dtype != torch.uint8:
            raise ValueError(f"out_t must be uint8 [{self.out_bytes}]")
        if tuple(tbl_t.shape) != (S, 2) or tbl_t.dtype != torch.int32 or not tbl_t.is_contiguous():
            raise ValueError(f"tbl_t must be contiguous int32 [{S}, 2]")
        n, f = self._args(n_new, flags)
        st = torch.cuda.current_stream(x_t.device).cuda_stream if stream is None else stream
        self.eng._ck(self.eng.lib.vtts_flac_stream_push(self.eng.h, self.h, _ptr(x_t), _ptr(n), _ptr(f), _ptr(out_t), _ptr(tbl_t),
                                                        st))


def reverb_stream_emitted(p: int, end: bool = False) -> int:
    """outputs a reverb stream slot has emitted after receiving p samples: 512 floor(p / 512), or p once END is pushed"""
    return int(p) if end else 512 * (int(p) // 512)


def acoustic_stream_schedule(n_frames: int, n_emit: int | None, chunk: int, lookahead: int = 10) -> list:
    """Frames an acoustic stream slot emits per push: it scans min(n_frames, n_emit + lookahead) frames, `chunk` per
    push; after P frames scanned it has emitted min(n_emit, max(0, P - lookahead)), and its last push emits the rest."""
    n_emit = n_frames if n_emit is None else n_emit
    end = min(n_frames, n_emit + lookahead)
    P, E, out = 0, 0, []
    while P < end:
        P = min(end, P + chunk)
        e = n_emit if P == end else min(n_emit, max(0, P - lookahead))
        out.append(e - E)
        E = e
    return out


class AcousticStream(_SlotStream):
    """Handle of a streaming acoustic model (Engine.open_acoustic_stream)."""
    _kind = "acoustic_stream"

    def __init__(self, eng: Engine, max_streams: int, max_chunk_frames: int, max_frames: int, max_tokens: int, seed=None, rng=None,
                 masks: bool = False):
        super().__init__(eng, max_streams, max_chunk_frames)
        self.max_chunk_frames = self._chunk
        self.max_frames, self.max_tokens = int(max_frames), int(max_tokens)
        if rng is not None:
            self.mode, self.seed = DROPOUT_REFERENCE, _rng_seed(rng, seed, True if masks else None)
        elif masks:
            if seed is not None:
                raise ValueError("masks=True selects MASK mode; it cannot be combined with seed=")
            self.mode, self.seed = DROPOUT_MASK, 0
        else:
            self.mode, self.seed = (DROPOUT_SEED if seed is not None else DROPOUT_OFF), int(seed or 0)
        self.lookahead = int(eng.lib.vtts_acoustic_stream_lookahead())
        self.out_frames = self.max_chunk_frames + self.lookahead   # frames per slot of a push's output buffer
        self.open = np.zeros(self.max_streams, bool)               # host mirror of the library's slot state
        self._left = np.zeros(self.max_streams, np.int64)          # pushes left per open slot
        h = C.c_void_p()
        eng._ck(eng.lib.vtts_acoustic_stream_create(eng.h, self.max_streams, self.max_chunk_frames, self.max_frames, self.max_tokens,
                                                    self.mode, self.seed, C.byref(h)))
        self.h = h

    def begin(self, slots, tokens, dur_frames, lengths=None, n_frames=None, n_emit=None, masks=None):
        """Start one utterance per entry of `slots` (closed slots): tokens int [nb,L], durations in frames [nb,L],
        lengths / n_frames as for `predict_mel`, n_emit int [nb] (frames to emit, <= n_frames; default all), masks uint8
        [nb,>=N,2,256] in MASK mode."""
        slots = _np(np.atleast_1d(slots), np.int32)
        if (masks is not None) != (self.mode == DROPOUT_MASK):
            raise ValueError("masks are given to begin exactly when the stream was opened with masks=True")
        tokens, dur, lens, nf, N, masks, _, _ = self.eng._acoustic_args(tokens, dur_frames, lengths, n_frames, masks, None)
        nb, L = tokens.shape
        if slots.shape != (nb,):
            raise ValueError(f"slots must hold one slot per token row ({nb}), got {slots.shape}")
        ne = None if n_emit is None else _np(n_emit, np.int32, (nb,), "n_emit")
        self.eng._ck(self.eng.lib.vtts_acoustic_stream_begin(self.eng.h, self.h, nb, _ptr(slots), _ptr(tokens), _ptr(lens), _ptr(dur),
                                                             _ptr(nf), _ptr(ne), _ptr(masks), L))
        for i, s in enumerate(slots):
            self.open[s] = True
            self._left[s] = len(acoustic_stream_schedule(int(nf[i]), None if ne is None else int(ne[i]), self.max_chunk_frames,
                                                         self.lookahead))

    def _advance(self):
        """slots that close with this push"""
        closing = self.open & (self._left == 1)
        self._left[self.open] -= 1
        self.open &= ~closing
        return closing

    def push(self) -> list:
        """Advance every open slot; returns one float32 [n, 80] array per slot with the frames it emits now."""
        S = self.max_streams
        mel = np.empty((S, self.out_frames, config.MEL_DIM), np.float32)
        n_out = np.zeros(S, np.int32)
        self.eng._ck(self.eng.lib.vtts_acoustic_stream_push_host(self.eng.h, self.h, _ptr(mel), _ptr(n_out)))
        self._advance()
        return [mel[s, : int(n_out[s])].copy() for s in range(S)]

    def push_device(self, out_t, stream=None) -> np.ndarray:
        """Device output: out_t f32 CUDA [S, F + lookahead, 80].  Stream-ordered; returns n_out int32 [S] (frames slot s
        got at the start of its row of out_t)."""
        import torch
        S = self.max_streams
        if tuple(out_t.shape) != (S, self.out_frames, config.MEL_DIM) or out_t.dtype != torch.float32 or not out_t.is_contiguous():
            raise ValueError(f"out_t must be contiguous float32 [{S}, {self.out_frames}, {config.MEL_DIM}]")
        n_out = np.zeros(S, np.int32)
        st = torch.cuda.current_stream(out_t.device).cuda_stream if stream is None else stream
        self.eng._ck(self.eng.lib.vtts_acoustic_stream_push(self.eng.h, self.h, _ptr(out_t), _ptr(n_out), st))
        self._advance()
        return n_out


def _output_rate(rate) -> int:
    """an output rate the resampler reaches from 16 kHz (reduced ratio at most 1024 each way)"""
    up, down = resample_ratio(config.SAMPLE_RATE, rate)
    if max(up, down) > 1024:
        raise ValueError(f"output rate {rate}: {config.SAMPLE_RATE} -> {rate} reduces to {up}/{down} (at most 1024 each)")
    return int(rate)


class OptionError(ValueError):
    """A bad AudioChain option; `option` is its keyword."""

    def __init__(self, option: str, msg: str):
        super().__init__(msg)
        self.option = option


class AudioChain:
    """The audio stages after the vocoder, their options validated, in the one order every caller runs them: denoise,
    pitch shift, time stretch and watermark at 16 kHz, then resample, equalize, compress, de-ess, reverb, bed, limit
    (or normalize loudness) and meter at the output rate.  The bed sits under the limiter and the meter, so it counts in
    the program loudness and stays under the true-peak ceiling; its tail makes each row `tail` samples longer.  The
    watermark is the last 16 kHz stage, after everything that moves time or pitch.  `encoding` ('pcm16', 'ulaw' or 'alaw') turns the float audio into the codes of that wire format
    last, after the meter; it has no state, so it is not a stream stage (TtsStream encodes its last buffer itself).
    'flac' or 'flac,block=N' makes `run` return a FLAC stream of the PCM-16 codes (Engine.encode_flac at the output rate).
    `run` applies the chain to one waveform with the one-shot host calls; `streams` opens it as stream stages.  `loudness` (a target in LUFS, reached under `true_peak`, or under the limiter's ceiling with `limit`) has no
    streaming form, and `meter` only measures, so `run` leaves the audio as it is for it.  Raises OptionError (a
    ValueError naming the option) for an option out of range."""

    def __init__(self, denoise=None, semitones=None, tempo=None, output_rate=None, eq=None, limit=None, gain_db=0.0,
                 loudness=None, true_peak=None, meter=False, compress=None, deess=None, reverb=None, watermark=None,
                 encoding=None, bed=None, formant=None):
        def checked(option, check, *args):
            try:
                return check(*args)
            except ValueError as e:
                raise OptionError(option, str(e)) from None

        self.output_rate = None if output_rate is None else checked("output_rate", _output_rate, output_rate)
        self.rate = self.output_rate or config.SAMPLE_RATE
        self.denoise = None if denoise is None else checked("denoise", _strength, denoise)
        self.semitones = None if semitones is None else float(checked("semitones", SEMITONES.rows, semitones, 1)[0])
        # the formant shift of the pitch stage (which runs when semitones or formant is given; None follows the pitch)
        self.formant = None if formant is None else float(checked("formant", FORMANT.rows, formant, 1)[0])
        self.tempo = None if tempo is None else float(checked("tempo", TEMPO.rows, tempo, 1)[0])
        self.watermark = None if watermark is None else checked("watermark", watermark_params, watermark)
        self.eq = None if eq is None else checked("eq", eq_sections, eq, self.rate)
        self.compress = None if compress is None else checked("compress", compressor_params, compress, self.rate)
        self.deess = None if deess is None else checked("deess", deesser_params, deess, self.rate)
        if reverb is not None:
            checked("reverb", reverb_params, reverb, self.rate)
        self.reverb = reverb           # the spec: the stages synthesize its IR where they open
        self.bed = None if bed is None else checked("bed", bed_specs, bed, self.rate)
        self._bed_spec, self._banks = bed, {}   # the bank is prepared once per engine, where a stage first runs or opens
        self.limit = None if limit is None else checked("limit", _limit_args, limit, self.rate, 5.0, 100.0)[0]
        self.gain_db = float(checked("gain_db", GAIN_DB.rows, gain_db, 1)[0]) if limit is not None else 0.0
        self.loudness = self.true_peak = None
        if loudness is not None:
            self.loudness, self.true_peak = checked("loudness", _loudness_target, loudness, self.limit if limit is not None else true_peak)
        if meter or loudness is not None:
            checked("meter" if loudness is None else "loudness", _loudness_rate, self.rate)
        self.meter = bool(meter)
        self.encoding = self.flac = None
        if isinstance(encoding, str) and encoding.split(",")[0] == "flac":
            self.flac = checked("encoding", flac_params, encoding)
            checked("encoding", flac_rate, self.rate)
            self.encoding = "flac"
        elif encoding is not None:
            self.encoding = checked("encoding", encoding_name, encoding)

    def _stages(self):
        """(TtsStream attribute, one-shot call or None, stream factory or None) of each stage that is on, in order"""
        r = self.rate
        stages = (
            (self.denoise is not None, "dn", lambda e, w: e.denoise(w, self.denoise),
             lambda e, S, p, sec: DenoiseStream(e, S, p, self.denoise)),
            (self.semitones is not None or self.formant is not None, "ps",
             lambda e, w: e.pitch_shift(w, self.semitones or 0.0, formant=self.formant),
             lambda e, S, p, sec: PitchShiftStream(e, S, p) if self.formant is None else VoiceShiftStream(e, S, p)),
            (self.tempo is not None, "ts", lambda e, w: e.time_stretch(w, self.tempo), lambda e, S, p, sec: TimeStretchStream(e, S, p)),
            (self.watermark is not None, "wm", lambda e, w: e.watermark(w, self.watermark),
             lambda e, S, p, sec: WatermarkStream(e, S, p, self.watermark)),
            (self.output_rate is not None, "rs", lambda e, w: e.resample(w, self.output_rate),
             lambda e, S, p, sec: ResampleStream(e, S, p, self.output_rate)),
            (self.eq is not None, "eq", lambda e, w: e.equalize(w, self.eq, r), lambda e, S, p, sec: EqStream(e, S, p, self.eq, r)),
            (self.compress is not None, "cp", lambda e, w: e.compress(w, self.compress, r)[0],
             lambda e, S, p, sec: CompressorStream(e, S, p, self.compress, r)),
            (self.deess is not None, "ds", lambda e, w: e.deess(w, self.deess, r)[0], lambda e, S, p, sec: DeesserStream(e, S, p, self.deess, r)),
            (self.reverb is not None, "rv", lambda e, w: e.reverb(w, self.reverb, r), lambda e, S, p, sec: ReverbStream(e, S, p, self.reverb, r)),
            (self.bed is not None, "bd", lambda e, w: e.mix_bed(w, self._bank(e), r)[0],
             lambda e, S, p, sec: BedStream(e, S, p, self._bank(e), r)),
            (self.loudness is not None, "lm",
             lambda e, w: e.normalize_loudness(w, self.loudness, r, true_peak=self.true_peak, limit=self.limit is not None)[0], None),
            (self.loudness is None and self.limit is not None, "lm", lambda e, w: e.limit(w, self.limit, r, self.gain_db)[0],
             lambda e, S, p, sec: LimiterStream(e, S, p, r, self.limit)),
            (self.meter, "mt", None, lambda e, S, p, sec: LoudnessMeter(e, S, p, r, sec)),
        )
        return [s[1:] for s in stages if s[0]]

    def _bank(self, eng: Engine) -> BedBank:
        if eng not in self._banks:
            self._banks[eng] = eng.prepare_beds(self._bed_spec, self.rate)
        return self._banks[eng]

    def run(self, eng: Engine, wav) -> np.ndarray:
        """the one-shot host calls of every stage on `wav` ([S] or [B,S] at 16 kHz), in order, then `Engine.encode`
        with `encoding` (float32 audio without one; FLAC stream bytes, or a list of them for [B,S], with 'flac')"""
        for _, call, _ in self._stages():
            if call is not None:
                wav = call(eng, wav)
        if self.flac is not None:
            return eng.encode_flac(wav, self.rate, block=self.flac["block"])
        return wav if self.encoding is None else eng.encode(wav, self.encoding)

    def streams(self, eng: Engine, max_streams: int, pitch: int, max_frames: int):
        """Opens the stream stages in order, yielding (TtsStream attribute, handle) as each opens: the first takes
        `pitch` samples per slot and push, each next one the previous one's output width; a meter slot holds the audio of
        `max_frames` vocoder frames, slowed down at most 1 / MIN_TEMPO times by the time stretcher."""
        if self.loudness is not None:
            raise ValueError("loudness normalization has no streaming form (use limit= and gain_db=, or meter=True)")
        slow = int(1 / MIN_TEMPO) if self.tempo is not None else 1
        seconds = -(-int(max_frames) * config.HOP * slow // config.SAMPLE_RATE) + 1
        if self.bed is not None:
            seconds += -(-self.bed[0]["Tt"] // self.rate)       # the bed's tail
        for name, _, make in self._stages():
            st = make(eng, max_streams, pitch, seconds)
            yield name, st
            pitch = getattr(st, "out_pitch", pitch)


# the open_tts_stream option of each stage's BEGIN parameter
_OPENED_WITH = {"semitones": "semitones", "formant": "formant", "tempo": "tempo", "gain_db": "limit", "bed": "bed"}


class TtsStream:
    """Handle of a text-to-speech stream (Engine.open_tts_stream): an acoustic stream of max_chunk_frames F feeding a
    vocoder stream of F + the acoustic lookahead frames per push, then the stream stages of the AudioChain of the
    options, each taking the previous one's output buffer, with a loudness meter of the audio `step()` returns last."""

    def __init__(self, eng: Engine, max_streams: int, max_chunk_frames: int, max_frames: int, max_tokens: int, seed=None, rng=None,
                 output_rate=None, denoise=None, meter=False, semitones=None, tempo=None, limit=None, gain_db=0.0, eq=None,
                 compress=None, deess=None, reverb=None, watermark=None, encoding=None, bed=None, max_joined_frames=None,
                 formant=None):
        import torch
        self.max_joined_frames = int(max_frames if max_joined_frames is None else max_joined_frames)
        if self.max_joined_frames < 1:
            raise ValueError(f"max_joined_frames must be >= 1, got {self.max_joined_frames}")
        if eng.get_precision() == PRECISION_FP32:
            raise ValueError("the tts stream needs the 'bf16x3' or 'fp16' mode (the vocoder stream has no strict fp32 path)")
        self._chain = AudioChain(denoise=denoise, semitones=semitones, tempo=tempo, output_rate=output_rate, eq=eq, limit=limit,
                                 gain_db=gain_db, meter=meter, compress=compress, deess=deess, reverb=reverb,
                                 watermark=watermark, encoding=encoding, bed=bed, formant=formant)
        self.eng = eng
        self.rs = self.dn = self.ps = self.ts = self.wm = self.eq = self.cp = self.ds = self.rv = self.bd = self.lm = self.mt = None
        S = max_streams
        self._built = []   # every stream handle, in construction order
        try:
            self.ac = AcousticStream(eng, S, max_chunk_frames, max_frames, max_tokens, seed=seed, rng=rng)
            self._built.append(self.ac)
            self.voc = VocoderStream(eng, S, self.ac.out_frames)
            self._built.append(self.voc)
            for name, st in self._chain.streams(eng, S, self.voc.wav_ld, self.max_joined_frames):
                self._built.append(st)
                setattr(self, name, st)
        except Exception:
            self.close()
            raise
        dev = torch.device("cuda", eng.device)
        self._mel = torch.zeros((S, self.ac.out_frames, config.MEL_DIM), dtype=torch.float32, device=dev)
        self._wav = torch.zeros((S, self.voc.wav_ld), dtype=torch.float32, device=dev)
        # (handle, device output buffer, extra push arguments) of the stages after the vocoder; a stage's BEGIN
        # parameter is the array of each slot's utterance value, set by `begin`
        self._stages = []
        for st in self._built[2:]:
            kw = {p.name: np.full(S, p.neutral, np.float32) for p in st._params}
            if isinstance(st, _ReductionStream):
                kw["reduction_t"] = torch.zeros(S, dtype=torch.float32, device=dev)
            self._stages.append((st, torch.zeros((S, st._width), dtype=torch.float32, device=dev), kw))
        self._mout_h = None if self.mt is None else torch.zeros((S, 4), dtype=torch.float32).pin_memory()
        # the codes of the last audio buffer (the meter's input), the one buffer `step` copies to the host when encoding
        last = ([b for st, b, _ in self._stages if st is not self.mt] or [self._wav])[-1]
        self._codes = self._flac = None
        if self._chain.flac is not None:
            # FLAC is a stateful last stage: a slot's frames leave as its blocks complete
            self._flac = FlacStream(eng, S, last.shape[1], self._chain.rate, self._chain.flac["block"])
            self._built.append(self._flac)
            self._flac_out = torch.zeros(self._flac.out_bytes, dtype=torch.uint8, device=dev)
            self._flac_tbl = torch.zeros((S, 2), dtype=torch.int32, device=dev)
            self._empty_out = b""
        elif self._chain.encoding is not None:
            self._codes = _code_tensor(None, tuple(last.shape), self._chain.encoding, dev)
        if self._flac is None:
            self._empty_out = np.zeros(0, np.float32 if self._codes is None else ENCODING_DTYPES[self._chain.encoding])
        self._meter = {}
        self._fresh = np.zeros(max_streams, bool)   # begun, no acoustic push yet: the next vocoder push carries BEGIN
        self._empty = set()                         # begun with nothing left after the trim: reported empty at the next step
        # a slot's utterance, from `begin` until END is pushed: live; another sentence may be appended: more; the
        # sentence on the acoustic stream ends the utterance: last; what is planned and not started yet, in order (a
        # (tokens, frames, n_frames, n_emit, last) sentence, or None where the utterance ends without one): queue;
        # frames vocoded over all its sentences: joined; begin's silence_duration: sil
        self._live = np.zeros(max_streams, bool)
        self._more = np.zeros(max_streams, bool)
        self._last = np.zeros(max_streams, bool)
        self._queue = [[] for _ in range(max_streams)]
        self._joined = np.zeros(max_streams, np.int64)
        self._sil = np.full(max_streams, -1.0)

    @property
    def max_streams(self):
        return self.ac.max_streams

    def _plan(self, slot: int, tokens, silence_duration, joined: int, queued: bool):
        """tts_plan of one sentence for `slot`: (tokens [1,L], frames, n_frames, n_emit); raises ValueError if it would
        take the slot past max_joined_frames, or, for a sentence `queued` to start later, if the acoustic stream would
        refuse it then"""
        tok = _np(tokens, np.int32).reshape(1, -1)
        if queued and tok.shape[1] > self.ac.max_tokens:
            raise ValueError(f"tts stream: {tok.shape[1]} tokens, the stream takes at most max_tokens={self.ac.max_tokens} per sentence")
        _, frames, nf, ne = self.eng.tts_plan(tok, silence_duration=silence_duration)
        if nf[0] < 1:
            raise ValueError("tts stream: predicted durations sum to less than one frame")
        if queued and nf[0] > self.ac.max_frames:
            raise ValueError(f"tts stream: {int(nf[0])} frames, the stream takes at most max_frames={self.ac.max_frames} per sentence")
        if joined + int(ne[0]) > self.max_joined_frames:
            raise ValueError(f"tts stream: slot {slot} would vocode {joined + int(ne[0])} frames, more than "
                             f"max_joined_frames={self.max_joined_frames}")
        return tok, frames, nf, ne

    def begin(self, slot: int, tokens, silence_duration=-1.0, semitones=None, tempo=None, gain_db=None, bed=None, more=False,
              formant=None):
        """Start `tokens` (one row of phoneme ids) in a free slot: durations, the text2mel fix-ups and the trim are
        planned exactly as `Engine.tts` plans them (vtts_tts_plan).  `semitones` and `tempo` override the stream's shift
        and tempo for this utterance, `gain_db` the limiter's pre-gain, `bed` the bank entry of the stream's beds (default
        0, -1 for none), `formant` the formant shift (a stream opened with formant=).  `more=True` keeps the slot open after this sentence for `append` (or `finish`); every sentence
        of the slot keeps these values.  Returns the number of frames the slot will vocode."""
        slot = int(slot)
        if self._live[slot] or slot in self._empty:
            raise ValueError(f"slot {slot} is still open")
        given = {"semitones": semitones, "formant": formant, "tempo": tempo, "gain_db": gain_db, "bed": bed}
        values = []   # (a stage's per-slot array, this utterance's value)
        for st, _, kw in self._stages:
            if st is self.bd:
                v = given.pop("bed")
                values.append((kw["bed"], int(st.bank.index(BED.default if v is None else v, 1)[0])))
            else:
                for p in st._params:
                    v, dflt = given.pop(p.name), getattr(self._chain, p.name)
                    values.append((kw[p.name], (p.neutral if dflt is None else dflt) if v is None else float(p.rows(v, 1)[0])))
        for name, v in given.items():
            if v is not None:
                raise ValueError(f"the stream was opened without {_OPENED_WITH[name]}= (no stage takes {name}=)")
        tok, frames, nf, ne = self._plan(slot, tokens, silence_duration, 0, queued=False)
        if ne[0] == 0 and not more:
            self._empty.add(slot)
            return 0
        if ne[0] > 0:
            self.ac.begin([slot], tok, frames, n_frames=nf, n_emit=ne)
        self._live[slot], self._more[slot], self._last[slot] = True, bool(more), not more
        self._fresh[slot] = True
        self._joined[slot], self._sil[slot] = int(ne[0]), float(silence_duration)
        for a, v in values:
            a[slot] = v
        return int(ne[0])

    def append(self, slot: int, tokens, more=False):
        """Add the next sentence to a slot whose last `begin` or `append` had more=True.  It is planned now (with
        begin's silence_duration), so errors surface here, and queued: it starts on the acoustic stream at the first
        step where the slot's previous sentence has made its last acoustic push.  The vocoder and every stage see the
        sentences as one utterance (no flags between them, every state carried), so the slot's audio is `tts_joined` of
        its sentences.  `more=False` makes it the last.  Returns the number of frames it will vocode."""
        slot = int(slot)
        if not self._more[slot]:
            raise ValueError(f"slot {slot} takes no more sentences (begin it with more=True; append after more=False "
                             f"or finish is not possible)")
        tok, frames, nf, ne = self._plan(slot, tokens, self._sil[slot], int(self._joined[slot]), queued=True)
        self._joined[slot] += int(ne[0])
        self._more[slot] = bool(more)
        if ne[0] > 0:
            self._queue[slot].append((tok, frames, nf, ne, not more))
        elif not more:
            self._queue[slot].append(None)
        return int(ne[0])

    def finish(self, slot: int):
        """End a slot that still takes sentences (open or waiting) without another one: END goes out in the step after
        its queued sentences have made their last acoustic push."""
        slot = int(slot)
        if not self._more[slot]:
            raise ValueError(f"slot {slot} takes no more sentences: nothing to finish")
        self._more[slot] = False
        self._queue[slot].append(None)

    def busy(self) -> np.ndarray:
        """bool [S]: slots with an utterance still running, including a slot waiting for its next sentence"""
        b = self._live.copy()
        for s in self._empty:
            b[s] = True
        return b

    def _start_queued(self) -> np.ndarray:
        """starts the next queued sentence of every slot whose acoustic side is closed; returns the slots whose
        utterance ends without another sentence (END in this step)"""
        end_now = np.zeros(self.max_streams, bool)
        for s in np.flatnonzero(self._live & ~self.ac.open):
            if not self._queue[s]:
                continue
            item = self._queue[s].pop(0)
            if item is None:
                end_now[s] = True
                continue
            tok, frames, nf, ne, last = item
            self.ac.begin([int(s)], tok, frames, n_frames=nf, n_emit=ne)
            self._last[s] = last
        return end_now

    def step(self) -> dict:
        """One acoustic push into a device buffer, then one vocoder push of the frames it emitted (BEGIN on a slot's
        first push, END on its last sentence's last one); one synchronisation.  Returns {slot: float32 samples} for every
        slot that was running (possibly empty), or {slot: codes} (int16 or uint8, `Engine.encode` of those samples) when
        the stream was opened with `encoding`, or {slot: bytes} with 'flac' (the FLAC stream of the slot's samples, the
        stream header with its first step and each frame once its block is complete, the short last frame at its end); a slot whose utterance finished this step is free afterwards.
        A slot waiting for its next sentence gets an empty array, and its vocoder and stages get no frames and no flags:
        each keeps its lookahead (the vocoder's 13 frames, a stage's held samples) until the next sentence or `finish`.
        That held audio is the cost of a seamless join."""
        end_now = self._start_queued()
        never = end_now & self._fresh          # every sentence planned zero frames: nothing was ever pushed
        live = self._live.copy()
        self._live &= ~never
        active = self.ac.open.copy()
        closing_before = active.copy()
        n_out = self.ac.push_device(self._mel) if active.any() else np.zeros(self.max_streams, np.int32)
        closed = closing_before & ~self.ac.open
        end = (closed & self._last) | (end_now & ~never)
        flags = (self._fresh & active).astype(np.uint8) * STREAM_BEGIN | end.astype(np.uint8) * STREAM_END
        pushed = active | end
        self._live &= ~end
        out = {s: (self._empty_out.copy() if self._flac is None else b"") for s in sorted(self._empty | set(np.flatnonzero(live).tolist()))}
        self._empty = set()
        if pushed.any():
            n_wav = self.voc.push_device(self._mel, n_out, flags, self._wav)
            n_wav = n_wav * config.HOP
            src = self._wav
            for st, buf, kw in self._stages:
                r = st.push_device(src, n_wav, flags, buf, **kw)
                if st is self.mt:
                    self._mout_h.copy_(buf, non_blocking=True)   # ready once the blocking copy below returns
                else:
                    n_wav, src = r, buf
            if self._flac is not None:
                self._flac.push_device(src, n_wav, flags, self._flac_out, self._flac_tbl)
                tbl = self._flac_tbl.cpu().numpy()        # the per-slot (offset, count), then only the bytes produced
                total = int(tbl[:, 1].sum())
                data = self._flac_out[:total].cpu().numpy().tobytes() if total else b""
                for s in np.flatnonzero(pushed):
                    o, c = tbl[s]
                    out[int(s)] = data[o:o + c]
            else:
                if self._codes is not None:
                    src = self.eng.encode_forward(src, self._chain.encoding, out=self._codes)
                wav = src.cpu().numpy()
                for s in np.flatnonzero(pushed):
                    out[int(s)] = wav[s, : int(n_wav[s])].copy()
            if self.mt is not None:
                m = self._mout_h.numpy()
                self._meter = {int(s): tuple(float(v) for v in m[s]) for s in np.flatnonzero(pushed)}
        self._fresh &= ~active
        return out

    def meter(self) -> dict:
        """{slot: (integrated, momentary, short_term, true_peak)} of the audio each slot stepped last has produced since
        its BEGIN (meter=True): equal to `Engine.loudness` of that audio, bit for bit, once the slot's last step ran."""
        if self.mt is None:
            raise ValueError("the stream was opened without meter=True")
        return dict(self._meter)

    def close(self):
        for st in reversed(getattr(self, "_built", [])):
            st.close()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()


_engines: dict = {}
_lock = threading.Lock()


def get_engine(device: int | None = None) -> Engine:
    """Process-wide engine per device (LOCAL_RANK by default under torchrun)."""
    import os
    if device is None:
        device = int(os.environ.get("LOCAL_RANK", "0"))
    with _lock:
        if device not in _engines:
            _engines[device] = Engine(device)
        return _engines[device]
