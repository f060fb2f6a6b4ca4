"""Command line front end, mirroring vietTTS/synthesizer.py (`python -m viettts_b200.synthesizer`).

Same flags as the reference (--text --output --sample-rate --silence-duration --lexicon-file) and the same
pipeline (synthesizer.py:34-39): normalise -> text2mel -> mel2wave -> 16-bit PCM WAV.  Two additions that the
GPU path makes worthwhile: `--text-file` synthesises one utterance per input line as ragged batches through a
single library call per batch (`Engine.tts`), and the WAV writer is built in (the reference needs `soundfile`).
`--precision fp16` runs the generator in the fast fp16 mode (Engine.set_precision) for either input.
`--output-rate R` resamples the audio on the device (Engine.resample) and writes R in the header; `--sample-rate` keeps
the reference's meaning, the header rate of the unchanged 16 kHz samples.  `--denoise S` removes the generator's bias
hiss on the device (Engine.denoise, strength S, the default bias) at 16 kHz, before any resampling.  `--pitch P` shifts
the voice by P semitones on the device (Engine.pitch_shift) at 16 kHz, after --denoise and before any resampling.
`--loudness L`
normalizes every output to L LUFS (ITU-R BS.1770-4, Engine.normalize_loudness) at the rate it is written, after
--denoise and --output-rate, under a true-peak ceiling (`--true-peak`, default -1 dBTP as EBU R128 asks).
"""
from __future__ import annotations

import re
import struct
import unicodedata
from argparse import ArgumentParser
from pathlib import Path

import numpy as np

from . import config

_SIL = config.SPECIAL_PHONEMES[config.SIL_INDEX]

# synthesizer.py:21-32 as an ordered rewrite table (applied after NFKC + lower + strip)
_REWRITES = (
    (re.compile(r"[\n.,:]+"), f" {_SIL} "),        # sentence punctuation and newlines become a silence token
    (re.compile(r'"'), " "),
    (re.compile(r"\s+"), " "),
    (re.compile(r"[.,:;?!]+"), f" {_SIL} "),
    (re.compile(r"[ ]+"), " "),
    (re.compile(f"( {_SIL}+)+ "), f" {_SIL} "),    # runs of silence tokens collapse to one
)


def nat_normalize_text(text: str) -> str:
    text = unicodedata.normalize("NFKC", text).lower().strip()
    for pattern, repl in _REWRITES:
        text = pattern.sub(repl, text)
    return text.strip()


def float_to_pcm16(wave) -> np.ndarray:
    """libsndfile's float -> PCM_16 conversion (what `soundfile.write(path, float_array, sr)` stores in a .wav):
    round-to-nearest-even of x * 0x7FFF; samples are clipped to the int16 range instead of wrapping."""
    x = np.asarray(wave, np.float32).astype(np.float64) * 32767.0
    return np.clip(np.rint(x), -32768, 32767).astype("<i2")


def write_wav(path, wave, sample_rate: int = config.SAMPLE_RATE) -> None:
    """Mono 16-bit PCM RIFF/WAVE file with the canonical 44-byte header (synthesizer.py:39)."""
    pcm = float_to_pcm16(np.ravel(wave))
    data = pcm.tobytes()
    header = b"RIFF" + struct.pack("<I", 36 + len(data)) + b"WAVE"
    header += b"fmt " + struct.pack("<IHHIIHH", 16, 1, 1, int(sample_rate), int(sample_rate) * 2, 2, 16)
    header += b"data" + struct.pack("<I", len(data))
    with open(path, "wb") as f:
        f.write(header + data)


def read_wav(path):
    """Inverse of write_wav for tests: (float32 wave in [-1,1), sample_rate)."""
    raw = Path(path).read_bytes()
    assert raw[:4] == b"RIFF" and raw[8:12] == b"WAVE" and raw[12:16] == b"fmt "
    fmt, ch, sr, _, _, bits = struct.unpack("<HHIIHH", raw[20:36])
    assert (fmt, ch, bits) == (1, 1, 16) and raw[36:40] == b"data"
    n = struct.unpack("<I", raw[40:44])[0]
    return np.frombuffer(raw[44:44 + n], "<i2").astype(np.float32) / 32767.0, sr


def synthesize_lines(lines, lexicon_file, silence_duration=-1.0, seed=None, max_rows=32, engine=None, rng=None):
    """Batched text -> list of waveforms (input order).  Lines are sorted by token count and cut into batches of
    at most `max_rows` rows so the padding inside a batch stays small; every batch is one `Engine.tts` call.
    Dropout: `rng` (the checkpoint's uint32[2], `text2mel.checkpoint_rng()`) draws the reference's own mask stream on
    the device, so each line sounds as it does alone through `text2mel`; otherwise the on-device counter stream keyed
    by `seed` (default: the checkpoint's rng words), whose masks depend on the line's row in its batch."""
    from .nat import text2mel as t2m
    from .hifigan.mel2wave import load_generator
    engine = t2m.load_duration(engine)
    _, ck_seed = t2m.load_acoustic(engine)
    if seed is None and rng is None:
        seed = ck_seed          # default stream key: the checkpoint's rng words
    load_generator(engine)
    toks = [t2m.text2tokens(nat_normalize_text(line), lexicon_file) for line in lines]
    order = sorted(range(len(toks)), key=lambda i: len(toks[i]))
    out = [None] * len(toks)
    for s in range(0, len(order), max_rows):
        idx = order[s:s + max_rows]
        L = max(len(toks[i]) for i in idx)
        tok = np.zeros((len(idx), L), np.int32)
        lens = np.zeros(len(idx), np.int32)
        for r, i in enumerate(idx):
            tok[r, : len(toks[i])] = toks[i]
            lens[r] = len(toks[i])
        waves, _ = engine.tts(tok, lens, silence_duration=silence_duration, seed=seed, rng=rng)
        for r, i in enumerate(idx):
            out[i] = waves[r]
    return out


def main(argv=None) -> int:
    parser = ArgumentParser(description="H100-native vietTTS synthesizer")
    parser.add_argument("--text", type=str)
    parser.add_argument("--text-file", type=Path, default=None, help="one utterance per line; outputs <output stem>_NNNN.wav")
    parser.add_argument("--output", default="clip.wav", type=Path)
    parser.add_argument("--sample-rate", default=None, type=int,
                        help="rate written in the WAV header (default 16000); as in the reference it does not change the "
                             "samples, which stay at the model's 16 kHz -- use --output-rate to resample")
    parser.add_argument("--output-rate", default=None, type=int,
                        help="resample the audio on the device to this rate (scipy.signal.resample_poly with its defaults) "
                             "and write it in the header")
    parser.add_argument("--denoise", default=None, type=float, metavar="STRENGTH",
                        help="subtract STRENGTH times the generator's bias spectrum (its output for an all-zero mel) from the "
                             "STFT magnitude of the 16 kHz audio on the device, before any --output-rate resampling; >= 0")
    parser.add_argument("--pitch", default=None, type=float, metavar="SEMITONES",
                        help="shift the voice's pitch by this many semitones on the device (a peak-locked phase vocoder that "
                             "keeps the timing), in [-12, 12]; at 16 kHz, after --denoise and before --output-rate")
    parser.add_argument("--loudness", default=None, type=float, metavar="LUFS",
                        help="normalize every output (each --text-file line separately) to this integrated loudness, "
                             "ITU-R BS.1770-4, in [-70, 0]; measured on the device at the output rate, after --denoise and "
                             "--output-rate (e.g. -23 broadcast, -16 podcasts)")
    parser.add_argument("--true-peak", default=None, type=float, metavar="DBTP",
                        help="with --loudness: the true-peak ceiling in dBTP, in [-20, 0] (default -1.0, EBU R128); the gain is "
                             "lowered until the 4x-oversampled peak stays below it")
    parser.add_argument("--silence-duration", default=-1, type=float)
    parser.add_argument("--lexicon-file", default=None)
    parser.add_argument("--seed", default=None, type=int,
                        help="prenet dropout: key of the on-device counter stream; default = the checkpoint's rng "
                             "(--text: the reference's own JAX/Haiku mask stream, drawn on the device; --text-file: the "
                             "counter stream keyed by those words, see --reference-dropout)")
    parser.add_argument("--reference-dropout", action="store_true",
                        help="with --text-file: draw the reference's own JAX/Haiku mask stream from the checkpoint's rng "
                             "for every line, so each line's audio is the --text audio of that line (not with --seed)")
    parser.add_argument("--precision", default=None, choices=["bf16x3", "fp16", "fp32"],
                        help="conv arithmetic (default bf16x3, the library default): bf16x3 = fp32-class split-bf16 tensor-core "
                             "products; fp16 = fast generator, one fp16 product per operand pair (waveform within ~1e-3 of "
                             "bf16x3), every other model as bf16x3; fp32 = strict FMA pipe")
    args = parser.parse_args(argv)
    if args.reference_dropout and args.text_file is None:
        parser.error("--reference-dropout applies to --text-file (--text always uses the reference's stream)")
    if args.reference_dropout and args.seed is not None:
        parser.error("--reference-dropout and --seed select different dropout streams; give one")
    if args.denoise is not None and not (np.isfinite(args.denoise) and args.denoise >= 0):
        parser.error(f"--denoise {args.denoise}: the strength must be finite and >= 0")
    if args.pitch is not None and not (np.isfinite(args.pitch) and abs(args.pitch) <= 12.0):
        parser.error(f"--pitch {args.pitch}: the shift must be finite and lie in [-12, 12] semitones")
    if args.output_rate is not None:
        if args.sample_rate is not None and args.sample_rate != args.output_rate:
            parser.error("--sample-rate only labels the 16 kHz samples and --output-rate resamples them; they disagree")
        from .engine import resample_ratio
        try:
            up, down = resample_ratio(config.SAMPLE_RATE, args.output_rate)
        except ValueError as e:
            parser.error(f"--output-rate: {e}")
        if max(up, down) > 1024:
            parser.error(f"--output-rate {args.output_rate}: {config.SAMPLE_RATE} -> {args.output_rate} reduces to {up}/{down} "
                         "(at most 1024 each)")
    if args.true_peak is not None and args.loudness is None:
        parser.error("--true-peak is the ceiling of --loudness normalization; give --loudness too")
    if args.loudness is not None:
        from .engine import _loudness_rate, _loudness_target
        if args.true_peak is None:
            args.true_peak = -1.0
        try:
            _loudness_target(args.loudness, args.true_peak)
            _loudness_rate(args.output_rate or config.SAMPLE_RATE)
        except ValueError as e:
            parser.error(f"--loudness: {e}")
    header_rate = args.output_rate or args.sample_rate or config.SAMPLE_RATE
    lexicon = args.lexicon_file if args.lexicon_file is not None else config.LEXICON_FILE
    if args.precision is not None:
        from .engine import get_engine
        get_engine().set_precision(args.precision)      # the engine both the --text and the --text-file paths use

    def to_output_rate(waves):
        from .engine import get_engine
        if args.denoise is not None:
            waves = [get_engine().denoise(w, args.denoise) for w in waves]
        if args.pitch is not None:
            waves = [get_engine().pitch_shift(w, args.pitch) for w in waves]
        if args.output_rate is not None:
            waves = [get_engine().resample(w, args.output_rate) for w in waves]
        if args.loudness is not None:
            rate = args.output_rate or config.SAMPLE_RATE
            waves = [get_engine().normalize_loudness(w, args.loudness, rate, true_peak=args.true_peak)[0] for w in waves]
        return waves

    if args.text_file is not None:
        lines = [ln for ln in args.text_file.read_text().splitlines() if ln.strip()]
        rng = None
        if args.reference_dropout:
            from .nat.text2mel import checkpoint_rng
            rng = checkpoint_rng()
        waves = to_output_rate(synthesize_lines(lines, lexicon, args.silence_duration, seed=args.seed, rng=rng))
        for i, w in enumerate(waves):
            fn = args.output.with_name(f"{args.output.stem}_{i:04d}{args.output.suffix or '.wav'}")
            print("writing output to file", fn)
            write_wav(fn, w, header_rate)
        return 0

    if args.text is None:
        parser.error("--text or --text-file is required")
    from .hifigan.mel2wave import mel2wave
    from .nat.text2mel import text2mel
    text = nat_normalize_text(args.text)
    print("Normalized text input:", text)
    mel = text2mel(text, lexicon, args.silence_duration, seed=args.seed)
    wave = to_output_rate([np.ravel(mel2wave(mel))])[0]
    print("writing output to file", args.output)
    write_wav(args.output, wave, header_rate)
    return 0


if __name__ == "__main__":
    raise SystemExit(main())
