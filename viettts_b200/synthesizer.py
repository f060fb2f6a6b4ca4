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
`--formant F` moves the voice's formants by F semitones whatever the pitch does, in the same stage (with or without
--pitch): `--pitch 4 --formant 0` is a higher voice from the same throat, `--formant -3` alone a deeper throat.
`--tempo T` plays the speech T times as fast with its pitch kept (Engine.time_stretch) at 16 kHz, after --pitch and
before any resampling.
`--loudness L`
normalizes every output to L LUFS (ITU-R BS.1770-4, Engine.normalize_loudness) at the rate it is written, after
--denoise and --output-rate, under a true-peak ceiling (`--true-peak`, default -1 dBTP as EBU R128 asks).
`--limiter` holds that ceiling with a lookahead true-peak limiter (Engine.limit) instead of lowering the gain: with
--loudness the target is reached (Engine.normalize_loudness(limit=True)), without it every output is limited to
--true-peak at the rate it is written, after --output-rate.
`--eq SPEC` equalizes every output on the device (Engine.equalize: high / low-pass, shelves, peaking and notch bands,
or the `telephone` preset) at the rate it is written, after --output-rate and before --loudness / --limiter.
`--compress SPEC` lowers the dynamic range of every output on the device (Engine.compress: a soft-knee feed-forward
compressor, the `voice` preset or key=value settings) at the rate it is written, after --eq and before --loudness /
--limiter, so the limiter only catches what the compressor leaves.
`--deess SPEC` turns down harsh sibilants of every output on the device (Engine.deess: the band above a crossover,
only while it is loud) at the rate it is written, after --compress and before --loudness / --limiter.
`--reverb SPEC` places every output in a synthetic room on the device (Engine.reverb: a convolution with a decaying
noise impulse response, the `room` or `hall` preset or key=value settings) at the rate it is written, after --deess and
before --loudness / --limiter.
`--bed FILE.wav[,key=value…]` mixes a background bed under every output on the device (Engine.mix_bed: a mono or stereo
PCM-16 file, stereo averaged, or `pink` noise, looped with a crossfaded seam, ducked under the voice and carried on for
a tail) at the rate it is written, after --reverb and before --loudness / --limiter, so the bed counts in the loudness
and stays under the ceiling.
`--watermark SPEC` marks every output with a key on the device (Engine.watermark: a keyed spread-spectrum mark, a bare
integer key or key=…,strength=…) at 16 kHz, after --tempo and before any resampling; `python -m viettts_b200.watermark
detect --key K FILE.wav` checks a written file for it.
`--encoding E` encodes every output on the device (Engine.encode) at the rate it is written, after every other stage,
and writes that WAVE format: `pcm16` (the same bytes as without the flag), `ulaw` or `alaw` (8-bit G.711, format 7 or
6, the wire format of telephony, e.g. with `--output-rate 8000 --eq telephone`).  `--encoding flac[,block=N]` writes a
native FLAC file instead (Engine.encode_flac: lossless, the PCM-16 samples of `pcm16`, in about half the bytes on speech).
`--split-sentences` splits `--text` and each `--text-file` line at its sentence ends (split_sentences) and synthesizes
the sentences as one joined utterance (Engine.tts_joined): a long text runs as a batch of short rows instead of one long
scan, with one waveform, one output file, as before.
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


# WAVE format tag and bits per sample of each wire encoding (Engine.encode)
WAV_FORMATS = {"pcm16": (1, 16), "ulaw": (7, 8), "alaw": (6, 8)}


def write_wav(path, wave, sample_rate: int = config.SAMPLE_RATE, encoding=None) -> None:
    """Mono RIFF/WAVE file.  Without `encoding`: float audio quantized by float_to_pcm16 into 16-bit PCM with the
    canonical 44-byte header (synthesizer.py:39).  With `encoding`, `wave` holds codes already encoded in it
    (Engine.encode): 'pcm16' int16 samples under the same 44-byte header; 'ulaw' (format 7) or 'alaw' (format 6) uint8
    codes under an 18-byte fmt chunk (cbSize 0, 8 bits, block align 1, byte rate = rate) and a fact chunk holding the
    sample count, as non-PCM WAVE files carry."""
    rate = int(sample_rate)
    if encoding is None:
        codes, encoding = float_to_pcm16(np.ravel(wave)), "pcm16"
    else:
        if encoding not in WAV_FORMATS:
            raise ValueError(f"encoding {encoding!r} must be one of {', '.join(WAV_FORMATS)}")
        codes = np.ravel(wave)
        want = np.int16 if encoding == "pcm16" else np.uint8
        if codes.dtype != want:
            raise ValueError(f"{encoding} samples must be {np.dtype(want).name}, got {codes.dtype}")
    fmt, bits = WAV_FORMATS[encoding]
    data = codes.astype("<i2" if bits == 16 else np.uint8).tobytes()
    if fmt == 1:
        chunks = b"fmt " + struct.pack("<IHHIIHH", 16, 1, 1, rate, rate * 2, 2, 16)
    else:
        chunks = b"fmt " + struct.pack("<IHHIIHHH", 18, fmt, 1, rate, rate, 1, 8, 0)
        chunks += b"fact" + struct.pack("<II", 4, codes.size)
    chunks += b"data" + struct.pack("<I", len(data)) + data + b"\0" * (len(data) % 2)   # chunks are word aligned
    with open(path, "wb") as f:
        f.write(b"RIFF" + struct.pack("<I", 4 + len(chunks)) + b"WAVE" + chunks)


def read_wav_codes(path, stereo: bool = False):
    """(codes, sample_rate, encoding) of a mono WAVE file in one of the wire encodings: int16 samples for 'pcm16'
    (format 1, 16 bits), uint8 codes for 'ulaw' (format 7) and 'alaw' (format 6, both 8 bits).  With `stereo` a
    2-channel PCM-16 file is read too, as int16 [N, 2].  Chunks other than fmt and data are skipped.  Raises ValueError
    for anything else."""
    raw = Path(path).read_bytes()
    if raw[:4] != b"RIFF" or raw[8:12] != b"WAVE":
        raise ValueError(f"{path}: not a RIFF/WAVE file")
    pos, fmt = 12, None
    while pos + 8 <= len(raw):
        cid, size = raw[pos:pos + 4], struct.unpack("<I", raw[pos + 4:pos + 8])[0]
        body = raw[pos + 8:pos + 8 + size]
        if cid == b"fmt " and size >= 16:
            fmt = struct.unpack("<HHIIHH", body[:16])
        elif cid == b"data":
            if fmt is None:
                raise ValueError(f"{path}: data before the fmt chunk")
            tag, ch, sr, _, _, bits = fmt
            enc = next((e for e, f in WAV_FORMATS.items() if f == (tag, bits)), None)
            two = stereo and ch == 2 and enc == "pcm16"
            if (ch != 1 and not two) or enc is None:
                raise ValueError(f"{path}: format {tag}, {ch} channels, {bits} bits (mono PCM-16, mu-law or A-law"
                                 + (", or stereo PCM-16)" if stereo else ")"))
            codes = np.frombuffer(body, "<i2" if bits == 16 else np.uint8).astype(np.int16 if bits == 16 else np.uint8)
            return (codes[: codes.size // 2 * 2].reshape(-1, 2) if two else codes), sr, enc
        pos += 8 + size + size % 2
    raise ValueError(f"{path}: no data chunk")


def read_wav(path):
    """Inverse of write_wav for tests: (float32 wave in [-1,1), sample_rate) of a 16-bit PCM file."""
    codes, sr, encoding = read_wav_codes(path)
    assert encoding == "pcm16"
    return codes.astype(np.float32) / 32767.0, sr


def read_bed_wav(path):
    """(float32 mono samples, sample_rate) of a PCM-16 WAVE file for a background bed: a stereo file is downmixed by
    averaging its two channels (in float64, cast once); samples scale as read_wav's, by 1 / 32767."""
    codes, sr, enc = read_wav_codes(path, stereo=True)
    if enc != "pcm16":
        raise ValueError(f"{path}: a bed is a PCM-16 file, got {enc}")
    v = codes.astype(np.float64)
    v = v.mean(axis=1) if v.ndim == 2 else v
    return (v / 32767.0).astype(np.float32), sr


def bed_arg(arg: str):
    """The bed spec of a `--bed` value: `pink[,key=value…]` as it is, or `FILE.wav[,key=value…]` as a dict holding the
    file's samples (read_bed_wav) and rate and the keys after it.  Raises ValueError for a file it cannot read."""
    head, *items = [t.strip() for t in arg.split(",")]
    if head.lower() == "pink":
        return arg
    try:
        audio, rate = read_bed_wav(head)
    except OSError as e:
        raise ValueError(f"cannot read {head}: {e.strerror or e}") from None
    spec = {"audio": audio, "audio_rate": rate}
    for item in items:
        key, eq, val = item.partition("=")
        if not eq or key.strip() in ("audio", "audio_rate"):
            raise ValueError(f"{item!r} is not key=value over the bed's keys")
        spec[key.strip().lower()] = val.strip()
    return spec


_SENTENCE_END = re.compile(r"[.!?…]+(?=\s|$)|\n")


def split_sentences(text: str) -> list:
    """The sentences of a raw text: it is split after each run of `.`, `!`, `?` or `…` followed by whitespace or the
    end (so `3.5` stays whole), and at newlines; the run itself is dropped, and so is a piece with no letter or digit.
    Each piece then goes through nat_normalize_text and text2tokens as a whole text does, so two joined sentences have
    one silence token between them (the next one's leading sil) where the whole text had the punctuation's one."""
    return [p for p in _SENTENCE_END.split(text) if any(ch.isalnum() for ch in p)]


def _load_models(engine):
    """the engine with the duration, acoustic and generator checkpoints loaded, and the acoustic checkpoint's rng words"""
    from .nat import text2mel as t2m
    from .hifigan.mel2wave import load_generator
    engine = t2m.load_duration(engine)
    _, ck_seed = t2m.load_acoustic(engine)
    load_generator(engine)
    return engine, ck_seed


def synthesize_joined(texts, lexicon_file, silence_duration=-1.0, seed=None, rng=None, engine=None):
    """`texts` split into sentences (split_sentences; a text without one is taken whole) -> one `Engine.tts_joined`
    call -> one waveform per text, in order"""
    from .nat import text2mel as t2m
    sentences = [split_sentences(t) or [t] for t in texts]
    toks = [[t2m.text2tokens(nat_normalize_text(s), lexicon_file) for s in sent] for sent in sentences]
    waves, _ = engine.tts_joined(toks, silence_duration=silence_duration, seed=seed, rng=rng)
    return waves


def synthesize_lines(lines, lexicon_file, silence_duration=-1.0, seed=None, max_rows=32, engine=None, rng=None, split_sentences=False):
    """Batched text -> list of waveforms (input order).  Lines are sorted by token count and cut into batches of
    at most `max_rows` rows so the padding inside a batch stays small; every batch is one `Engine.tts` call.
    Dropout: `rng` (the checkpoint's uint32[2], `text2mel.checkpoint_rng()`) draws the reference's own mask stream on
    the device, so each line sounds as it does alone through `text2mel`; otherwise the on-device counter stream keyed
    by `seed` (default: the checkpoint's rng words), whose masks depend on the line's row in its batch.
    `split_sentences`: each line is split into its sentences and joined back into one utterance (`Engine.tts_joined`),
    `max_rows` lines per call."""
    from .nat import text2mel as t2m
    engine, ck_seed = _load_models(engine)
    if seed is None and rng is None:
        seed = ck_seed          # default stream key: the checkpoint's rng words
    toks = [t2m.text2tokens(nat_normalize_text(line), lexicon_file) for line in lines]
    order = sorted(range(len(toks)), key=lambda i: len(toks[i]))
    out = [None] * len(toks)
    for s in range(0, len(order), max_rows):
        idx = order[s:s + max_rows]
        if split_sentences:
            for i, w in zip(idx, synthesize_joined([lines[i] for i in idx], lexicon_file, silence_duration, seed, rng, engine)):
                out[i] = w
            continue
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


# the command-line flag of each AudioChain option the CLI sets
_FLAGS = {"denoise": "--denoise", "semitones": "--pitch", "formant": "--formant", "tempo": "--tempo", "output_rate": "--output-rate", "eq": "--eq",
          "limit": "--limiter", "loudness": "--loudness", "compress": "--compress",
          "deess": "--deess", "reverb": "--reverb", "watermark": "--watermark", "encoding": "--encoding", "bed": "--bed"}


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
    parser.add_argument("--formant", default=None, type=float, metavar="SEMITONES",
                        help="move the voice's formants (its spectral envelope) by this many semitones on the device, in "
                             "[-12, 12], independently of --pitch (0 keeps them where they are while --pitch moves the "
                             "pitch); in the --pitch stage")
    parser.add_argument("--tempo", default=None, type=float, metavar="T",
                        help="speak T times as fast with the pitch kept (a peak-locked phase-vocoder time stretch on the "
                             "device), in [0.5, 2]; at 16 kHz, after --pitch and before --output-rate")
    parser.add_argument("--loudness", default=None, type=float, metavar="LUFS",
                        help="normalize every output (each --text-file line separately) to this integrated loudness, "
                             "ITU-R BS.1770-4, in [-70, 0]; measured on the device at the output rate, after --denoise and "
                             "--output-rate (e.g. -23 broadcast, -16 podcasts)")
    parser.add_argument("--true-peak", default=None, type=float, metavar="DBTP",
                        help="with --loudness: the true-peak ceiling in dBTP, in [-20, 0] (default -1.0, EBU R128); the gain is "
                             "lowered until the 4x-oversampled peak stays below it")
    parser.add_argument("--limiter", action="store_true",
                        help="hold the --true-peak ceiling (default -1 dBTP) with a lookahead limiter on the device (5 ms "
                             "lookahead, 100 ms release): with --loudness the target is reached instead of the gain being "
                             "lowered; without it every output is limited at the output rate, after --output-rate")
    parser.add_argument("--eq", default=None, metavar="SPEC",
                        help="equalize every output on the device at the output rate, after --output-rate and before "
                             "--loudness / --limiter: comma-separated bands hp:F[:ORDER], lp:F[:ORDER], ls:F:GAIN[:S], "
                             "hs:F:GAIN[:S], pk:F:Q:GAIN, notch:F:Q, or 'telephone' (hp:300:4,lp:3400:4, the 300-3400 Hz "
                             "band); at most 8 second-order sections in all")
    parser.add_argument("--compress", default=None, metavar="SPEC",
                        help="compress the dynamic range of every output on the device at the output rate, after --eq and "
                             "before --loudness / --limiter: 'voice' (-24 dBFS threshold, 3:1, 6 dB knee, 5 ms attack, 80 ms "
                             "release, 0 dB makeup) or comma-separated threshold=, ratio=, knee=, attack=, release=, makeup= "
                             "(keys left out keep the voice values)")
    parser.add_argument("--deess", default=None, metavar="SPEC",
                        help="de-ess every output on the device at the output rate, after --compress and before --loudness / "
                             "--limiter: only the band above the crossover is turned down, only while it is loud. 'voice' "
                             "(5000 Hz crossover, -30 dBFS threshold, 4:1, 6 dB knee, 1 ms attack, 60 ms release, 12 dB range; "
                             "needs an output rate of at least 11112 Hz) or comma-separated freq=, threshold=, ratio=, knee=, "
                             "attack=, release=, range= (keys left out keep the voice values)")
    parser.add_argument("--reverb", default=None, metavar="SPEC",
                        help="add a synthetic room to every output on the device at the output rate, after --deess and "
                             "before --loudness / --limiter: 'room' (rt60 0.35 s, 8 ms predelay, mix 0.15), 'hall' (rt60 "
                             "1.8 s, 25 ms predelay, mix 0.22) or comma-separated rt60=, predelay=, mix=, seed= (keys left "
                             "out keep the room values)")
    parser.add_argument("--bed", default=None, metavar="FILE.wav[,KEY=VALUE...]",
                        help="mix a background bed under every output on the device at the output rate, after --reverb and "
                             "before --loudness / --limiter: a mono or stereo PCM-16 WAV file (stereo is averaged; any rate "
                             "the resampler reaches) or 'pink' (seeded pink noise, seed=, length= s), looped with a crossfade, "
                             "ducked under the voice and carried on for a tail; keys level= LUFS (-30), duck= dB (12), "
                             "threshold= dBFS (-40), attack= ms (10), release= ms (500), fade_in= ms (250), tail= ms (1000), "
                             "xfade= ms (50), offset= s (0)")
    parser.add_argument("--watermark", default=None, metavar="SPEC",
                        help="mark every output with a key on the device at 16 kHz, after --tempo and before --output-rate: "
                             "an integer key in [0, 2^64) or key=K,strength=S (S in [0, 0.3], default 0.1); "
                             "`python -m viettts_b200.watermark detect --key K FILE.wav` detects it")
    parser.add_argument("--encoding", default=None, metavar="{pcm16,ulaw,alaw,flac[,block=N]}",
                        help="encode every output on the device at the output rate, after every other stage, and write it "
                             "in that WAVE format: pcm16 (16-bit PCM, the default file), ulaw or alaw (8-bit G.711, e.g. "
                             "with --output-rate 8000 --eq telephone for telephony); or flac (a native FLAC file of the "
                             "pcm16 samples, lossless; block=256/512/1024/2048/4096 samples per frame, default 4096)")
    parser.add_argument("--split-sentences", action="store_true",
                        help="split --text, and each --text-file line, at its sentence ends (. ! ? … before a space or the end, "
                             "and newlines), run the sentences as separate rows and join their frames into one utterance "
                             "before the vocoder (Engine.tts_joined): long texts run as a batch of short rows")
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
    if args.output_rate is not None and args.sample_rate is not None and args.sample_rate != args.output_rate:
        parser.error("--sample-rate only labels the 16 kHz samples and --output-rate resamples them; they disagree")
    if args.true_peak is not None and args.loudness is None and not args.limiter:
        parser.error("--true-peak is the ceiling of --loudness normalization or of --limiter; give one of them too")
    from .engine import AudioChain, OptionError
    ceiling = -1.0 if args.true_peak is None else args.true_peak
    try:
        bed = None if args.bed is None else bed_arg(args.bed)
    except ValueError as e:
        parser.error(f"--bed: {e}")
    try:
        chain = AudioChain(denoise=args.denoise, semitones=args.pitch, formant=args.formant, tempo=args.tempo, output_rate=args.output_rate,
                           eq=args.eq,
                           limit=ceiling if args.limiter else None, loudness=args.loudness, true_peak=ceiling, compress=args.compress,
                           deess=args.deess, reverb=args.reverb, watermark=args.watermark, encoding=args.encoding, bed=bed)
    except OptionError as e:
        parser.error(f"{_FLAGS[e.option]}: {e}")
    header_rate = args.output_rate or args.sample_rate or config.SAMPLE_RATE
    lexicon = args.lexicon_file if args.lexicon_file is not None else config.LEXICON_FILE
    if args.precision is not None:
        from .engine import get_engine
        get_engine().set_precision(args.precision)      # the engine both the --text and the --text-file paths use

    def to_output_rate(waves):
        from .engine import get_engine
        return [chain.run(get_engine(), w) for w in waves]

    def write(path, w):
        if chain.flac is not None:
            Path(path).write_bytes(w)     # chain.run gave the FLAC stream
        else:
            write_wav(path, w, header_rate, encoding=chain.encoding)

    if args.text_file is not None:
        lines = [ln for ln in args.text_file.read_text().splitlines() if ln.strip()]
        rng = None
        if args.reference_dropout:
            from .nat.text2mel import checkpoint_rng
            rng = checkpoint_rng()
        waves = to_output_rate(synthesize_lines(lines, lexicon, args.silence_duration, seed=args.seed, rng=rng,
                                                split_sentences=args.split_sentences))
        for i, w in enumerate(waves):
            suffix = args.output.suffix or (".flac" if chain.flac is not None else ".wav")
            fn = args.output.with_name(f"{args.output.stem}_{i:04d}{suffix}")
            print("writing output to file", fn)
            write(fn, w)
        return 0

    if args.text is None:
        parser.error("--text or --text-file is required")
    if args.split_sentences:
        from .engine import get_engine
        from .nat.text2mel import checkpoint_rng
        engine, _ = _load_models(get_engine())
        rng = checkpoint_rng() if args.seed is None else None
        wave = to_output_rate(synthesize_joined([args.text], lexicon, args.silence_duration, seed=args.seed, rng=rng, engine=engine))[0]
        print("writing output to file", args.output)
        write(args.output, wave)
        return 0
    from .hifigan.mel2wave import mel2wave
    from .nat.text2mel import text2mel
    text = nat_normalize_text(args.text)
    print("Normalized text input:", text)
    mel = text2mel(text, lexicon, args.silence_duration, seed=args.seed)
    wave = to_output_rate([np.ravel(mel2wave(mel))])[0]
    print("writing output to file", args.output)
    write(args.output, wave)
    return 0


if __name__ == "__main__":
    raise SystemExit(main())
