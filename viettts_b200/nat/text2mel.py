"""Drop-in for vietTTS/nat/text2mel.py: `predict_mel` (:61-82), `predict_duration` (:22-34),
`text2tokens` (:37-58), `load_lexicon` (:16-19) and `text2mel` (:85-103).

`predict_mel(tokens, durations)`: tokens list[int] (length L), durations f32
[1,L] in SECONDS; reads assets/infore/nat/acoustic_latest_ckpt.pickle (keys
step/params/aux/rng/optim_state) and returns mel f32 [1,N,80] with
N = int(sum(durations*16000/256)).

Dropout: the reference applies prenet dropout at inference with the
checkpoint's `rng` through Haiku's split chain on JAX's threefry generator
(nat/model.py:95-100,132).  That is a pure function of the two rng words, so by
default `predict_mel` has the device draw exactly the keep-masks the reference
would draw (the library's REFERENCE dropout mode: sample-wise parity with the JAX
path, classic threefry layout; `viettts_b200.jaxrng` states the same function in
numpy).  `seed=` selects the library's own on-device counter stream instead,
`masks=` (uint8 [1,N,2,256]) supplies masks explicitly, and `dropout=False` is
the deterministic mode."""
from __future__ import annotations

import os

import numpy as np

from .. import config
from ..engine import get_engine
from ..weights import load_pickle

CKPT_FILE = config.ACOUSTIC_CKPT
DURATION_CKPT_FILE = config.DURATION_CKPT


def _file_key(path):
    st = os.stat(path)
    return (str(path), st.st_mtime_ns, st.st_size)


_rng_words = {}
_rng_keys = {}


def load_acoustic(engine=None, ckpt_file=None):
    """Loads the checkpoint into the engine once per file version; returns (engine, rng words as one uint64)."""
    engine = engine or get_engine()
    ckpt_file = ckpt_file or CKPT_FILE
    key = _file_key(ckpt_file)
    if engine._acoustic_key != key or key not in _rng_words:
        dic = load_pickle(ckpt_file)
        engine.load_acoustic(dic, key=key)
        rng = np.asarray(dic.get("rng", [0, 42])).astype(np.uint64).ravel()
        _rng_words[key] = int((int(rng[0]) << 32) | int(rng[-1]))
        _rng_keys[key] = np.array([rng[0], rng[-1]], np.uint32)
    return engine, _rng_words.get(key, 42)


def checkpoint_rng(ckpt_file=None) -> np.ndarray:
    """The checkpoint's `rng` (text2mel.py:69), uint32[2]; the acoustic checkpoint must have been loaded."""
    key = _file_key(ckpt_file or CKPT_FILE)
    if key not in _rng_keys:
        load_acoustic(ckpt_file=ckpt_file)
    return _rng_keys[key]


def frame_count(frames) -> int:
    """The acoustic frame count of one utterance, `int(sum(durations))` of text2mel.py:79, from its float32 per-token
    durations in frames: summed in float64 in token order, rounded to float32 once, then truncated.  This is the
    library's one definition (vtts_tts_plan, so `Engine.tts` and the TTS stream, computes the same).  For any realistic
    row the float64 sum is exact, so it does not depend on the order of the terms; a float32 sum does, and near an
    integer it can land one frame off."""
    f = np.asarray(frames, np.float32).ravel()
    total = float(np.cumsum(f, dtype=np.float64)[-1]) if f.size else 0.0
    return int(np.float32(total))


def seconds_to_frames(durations):
    """text2mel.py:78-79: durations * sample_rate / (n_fft // 4) in float32, and the frame count (`frame_count`)."""
    d = (np.asarray(durations, np.float32) * np.float32(config.SAMPLE_RATE)) / np.float32(config.N_FFT // 4)
    return d, frame_count(d)


def predict_mel(tokens, durations, masks=None, dropout=True, seed=None):
    engine, _ = load_acoustic()
    d, n_frames = seconds_to_frames(durations)
    tokens = np.array(tokens, dtype=np.int32)[None, :]
    d = d.reshape(1, -1)
    if not dropout:
        return engine.predict_mel(tokens, d, n_frames=[n_frames])
    if masks is None and seed is None:
        # the reference's own stream, drawn on the device: hk.next_rng_key() chain from the checkpoint rng, two [1,256]
        # draws per frame
        return engine.predict_mel(tokens, d, n_frames=[n_frames], rng=checkpoint_rng())
    return engine.predict_mel(tokens, d, n_frames=[n_frames], masks=masks, seed=seed if masks is None else None)


# ---------------------------------------------------------------------------
# duration model + text front-end glue (the callers of predict_mel, SURVEY.md §8f row 1)
# ---------------------------------------------------------------------------
def load_duration(engine=None, ckpt_file=None):
    engine = engine or get_engine()
    ckpt_file = ckpt_file or DURATION_CKPT_FILE
    key = _file_key(ckpt_file)
    if engine._duration_key != key:
        engine.load_duration(load_pickle(ckpt_file), key=key)
    return engine


def predict_duration(tokens):
    """text2mel.py:22-34: tokens list[int] -> predicted durations f32 [1,L] in seconds
    (DurationModel(is_training=False) on a batch of one, lengths = [len(tokens)])."""
    engine = load_duration()
    tok = np.array(tokens, dtype=np.int32)[None, :]
    return engine.predict_duration(tok, lengths=np.array([len(tokens)], np.int32))


def load_lexicon(fn):
    """text2mel.py:16-19: one `word<TAB>phoneme phoneme ...` entry per line, lower-cased."""
    table = {}
    with open(fn, "r") as f:
        for line in f.readlines():
            word, phones = line.lower().strip().split("\t")
            table[word] = phones
    return table


def text2tokens(text, lexicon_fn):
    """text2mel.py:37-58.  sil at both ends; a special phoneme maps to its own id; a lexicon word to its
    phoneme ids followed by the word-end id; an unknown word is spelled letter by letter (unknown letters
    dropped) followed by the word-end id."""
    phonemes = config.PHONEMES
    index = {p: i for i, p in enumerate(phonemes)}
    lexicon = load_lexicon(lexicon_fn)
    tokens = [config.SIL_INDEX]
    for word in text.strip().lower().split():
        if word in config.SPECIAL_PHONEMES:
            tokens.append(index[word])
            continue
        if word in lexicon:
            tokens.extend(phonemes.index(ph) for ph in lexicon[word].split())   # ValueError on an unknown phoneme, as the reference
        else:
            tokens.extend(index[ch] for ch in word if ch in index)
        tokens.append(config.WORD_END_INDEX)
    tokens.append(config.SIL_INDEX)
    return tokens


def adjust_durations(tokens, durations, silence_duration=-1.0):
    """text2mel.py:88-97: silence tokens are clipped from below at `silence_duration`, word ends last 0 s."""
    tok = np.asarray(tokens)[None, :]
    d = np.asarray(durations, np.float32)
    d = np.where(tok == config.SIL_INDEX, np.clip(d, silence_duration, None), d)
    d = np.where(tok == config.WORD_END_INDEX, np.float32(0.0), d)
    return d.astype(np.float32)


def text2mel(text, lexicon_fn=None, silence_duration=-1.0, masks=None, dropout=True, seed=None):
    """text2mel.py:85-103: text -> tokens -> durations -> mel f32 [1,N',80]; the frames of the trailing
    silence token are cut (`:99-102`)."""
    tokens = text2tokens(text, lexicon_fn if lexicon_fn is not None else config.LEXICON_FILE)
    durations = adjust_durations(tokens, predict_duration(tokens), silence_duration)
    mels = predict_mel(tokens, durations, masks=masks, dropout=dropout, seed=seed)
    if tokens[-1] == config.SIL_INDEX:
        end_silence = float(durations[0, -1])
        silence_frame = int(end_silence * config.SAMPLE_RATE / (config.N_FFT // 4))
        mels = mels[:, : (mels.shape[1] - silence_frame)]
    return mels
