"""Ground-truth-aligned mel generation, the device side of vietTTS/nat/gta.py.

The reference's `generate_gta` (gta.py:47-77) iterates a TextGrid/wav data loader (out of scope: training data
plumbing) and for every batch calls `forward_fn` (gta.py:28-44) and stores `mel[idx, :l].T` as `<name>.npy`
with l = wav_length // 256.  `forward_fn` + the save loop are provided here on top of `Engine.gta`
(one `vtts_gta_host` call per batch: MelFilter -> shift -> teacher-forced acoustic model)."""
from __future__ import annotations

from pathlib import Path

import numpy as np

from .. import config
from .text2mel import checkpoint_rng, load_acoustic


def forward_fn(wavs, phonemes, lengths, durations, wav_lengths=None, keep_masks=None, zone_masks=None, seed=None, engine=None):
    """gta.py:28-44.  wavs int16 [B,S]; phonemes int [B,L]; lengths int [B]; durations f32 [B,L] SECONDS.
    Returns mel2_hat f32 [B,S/256,80] over the FULL padded length: like the reference's `forward_fn_`, the model never
    sees `wav_lengths` (the postnet runs over all S/256 frames; gta.py:70-76 only slices `mel[idx, :l]` when saving),
    so `wav_lengths` is accepted for signature compatibility and used by `save_batch` alone.
    Masks: `keep_masks`/`zone_masks` explicitly, else `seed` for the library's on-device stream, else (default) the
    masks the reference itself draws from the checkpoint's rng (Haiku split chain, whole-batch draws), drawn on the
    device."""
    engine, _ = load_acoustic(engine)
    if keep_masks is None and seed is None:
        return engine.gta(wavs, phonemes, durations, lengths=lengths, wav_lengths=None, rng=checkpoint_rng())
    return engine.gta(wavs, phonemes, durations, lengths=lengths, wav_lengths=None, keep_masks=keep_masks,
                      zone_masks=zone_masks, seed=seed)


def save_batch(out_dir, names, mel, wav_lengths):
    """gta.py:70-76: one `<name>.npy` per utterance holding mel[:l].T ([80, l]), l = wav_length // hop."""
    out_dir = Path(out_dir)
    out_dir.mkdir(parents=True, exist_ok=True)
    files = []
    for idx, fn in enumerate(names):
        l = int(wav_lengths[idx]) // config.HOP
        file = out_dir / f"{fn}.npy"
        np.save(file, mel[idx, :l].T)
        files.append(file)
    return files


def generate_gta(batches, out_dir, **kw):
    """`batches` yields (names, wavs, wav_lengths, phonemes, lengths, durations) -- what the reference's
    load_textgrid_wav(..., "gta") produces per step."""
    written = []
    for names, wavs, wav_lengths, phonemes, lengths, durations in batches:
        mel = forward_fn(wavs, phonemes, lengths, durations, wav_lengths=wav_lengths, **kw)
        written += save_batch(out_dir, names, mel, wav_lengths)
    return written
