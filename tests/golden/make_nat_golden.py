"""Golden vectors for the NAT / duration / GTA / MelFilter path, produced by EXECUTING THE REFERENCE'S OWN SOURCE
FILES (`vietTTS/nat/{model,text2mel,gta,dsp}.py` of a checkout named by VIETTTS_REFERENCE, unmodified) on the synthetic Haiku-layout
checkpoints, with `tests/refshim` standing in for the third-party libraries that cannot be installed here
(jax, dm-haiku, librosa: see tests/refshim/README.md and profiles/r2_ref_deps_probe_*.json).

What this pins: every line of the reference's wiring (it runs as written) and its Haiku parameter naming (a wrong
name or shape in the checkpoint layout raises).  What it does not pin: the third-party primitives, which the shim
restates (cross-checked elsewhere against torch operators).

Run with a reference checkout:   VIETTTS_REFERENCE=<path> python tests/golden/make_nat_golden.py
Writes tests/golden/nat_ref_*.npz (float32 outputs of float64 arithmetic; masks bit-packed).
"""
from __future__ import annotations

import os
import pickle
import sys
import tempfile
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
REPO = HERE.parents[1]
REF = Path(os.environ.get("VIETTTS_REFERENCE", "vietTTS-reference"))   # a checkout of NTT123/vietTTS
sys.path.insert(0, str(REPO / "tests" / "refshim"))   # jax / haiku / librosa stand-ins FIRST
sys.path.insert(1, str(REF))
sys.path.insert(2, str(REPO))

import jax  # noqa: E402  (the shim)
import haiku as hk  # noqa: E402  (the shim)

assert "refshim" in jax.__file__ and "refshim" in hk.__file__

from vietTTS.nat import gta as ref_gta  # noqa: E402  -- reference source files, unmodified
from vietTTS.nat import model as ref_model  # noqa: E402
from vietTTS.nat import text2mel as ref_t2m  # noqa: E402
from vietTTS.nat.config import FLAGS, AcousticInput  # noqa: E402
from vietTTS.nat.dsp import MelFilter  # noqa: E402

from viettts_b200 import synthetic  # noqa: E402


def record():
    jax.random.RECORD = []
    return jax.random.RECORD


def pack(m):
    m = np.asarray(m, np.uint8)
    return np.packbits(m.reshape(-1)), np.array(m.shape, np.int64)


def keep_masks_from_steps(rec, B, N):
    """inference: 2 draws of shape [B,256] per frame, in frame order -> uint8 [B,N,2,256]."""
    assert len(rec) == 2 * N, (len(rec), N)
    out = np.zeros((B, N, 2, 256), np.uint8)
    for i, (shape, p, m) in enumerate(rec):
        assert shape == (B, 256) and p == 0.5
        out[:, i // 2, i % 2] = m
    return out


def main():
    ack = synthetic.acoustic_ckpt(1234)
    duk = synthetic.duration_ckpt(1234)
    tmp = Path(tempfile.mkdtemp())
    with open(tmp / "acoustic_latest_ckpt.pickle", "wb") as f:
        pickle.dump(ack, f)
    with open(tmp / "duration_latest_ckpt.pickle", "wb") as f:
        pickle.dump(duk, f)
    FLAGS.ckpt_dir = tmp

    # ---- A: predict_mel (text2mel.py:61-82), one utterance ------------------------------------------------
    tokens, dur = synthetic.utterance(7, n_phonemes=40, seconds=1.9)
    rec = record()
    mel = np.asarray(ref_t2m.predict_mel(tokens, dur))            # [1,N,80]
    N = mel.shape[1]
    d32 = (dur * np.float32(16000)) / np.float32(256)
    assert N == int(np.sum(d32, dtype=np.float32)), "n_frames must not depend on f32/f64 rounding for this fixture"
    keep = keep_masks_from_steps(rec, 1, N)
    kb, ks = pack(keep)
    np.savez_compressed(HERE / "nat_ref_predict_mel.npz", tokens=np.asarray(tokens, np.int32), durations_sec=dur,
                        mel=mel.astype(np.float32), keep_bits=kb, keep_shape=ks, rng=ack["rng"])
    print("A predict_mel", mel.shape, float(np.abs(mel).mean()))

    # ---- B: AcousticModel.inference with B=2 (model.py:123-144): batch layout of the mask draws -----------
    rng = np.random.default_rng(11)
    L, N2 = 24, 60
    tk2 = rng.integers(4, 93, size=(2, L)).astype(np.int32)
    du2 = rng.uniform(0.5, 4.5, size=(2, L)).astype(np.float32)
    du2 *= (N2 + 0.4) / du2.sum(axis=1, keepdims=True)

    @hk.transform_with_state
    def fwd(tokens, durations, n_frames):
        return ref_model.AcousticModel(is_training=False).inference(tokens, durations, n_frames)

    rec = record()
    mel2, st = fwd.apply(ack["params"], ack["aux"], ack["rng"], tk2, du2, N2)
    keep2 = keep_masks_from_steps(rec, 2, N2)
    kb, ks = pack(keep2)
    np.savez_compressed(HERE / "nat_ref_inference_b2.npz", tokens=tk2, durations_frames=du2, n_frames=np.int64(N2),
                        mel=np.asarray(mel2, np.float32), attn=np.asarray(st["acoustic_model"]["attn"], np.float32),
                        keep_bits=kb, keep_shape=ks, rng=ack["rng"])
    print("B inference B=2", mel2.shape)

    # ---- C: predict_duration (text2mel.py:22-34) -------------------------------------------------------------
    jax.random.RECORD = None
    dsec = np.asarray(ref_t2m.predict_duration(tokens))            # [1,L]
    np.savez_compressed(HERE / "nat_ref_duration.npz", tokens=np.asarray(tokens, np.int32), durations_sec=dsec.astype(np.float32))
    print("C predict_duration", dsec.shape, float(dsec.mean()))

    # ---- D: text2mel (text2mel.py:85-103): text -> tokens -> durations -> fix-ups -> mel -> trailing-silence trim --
    text = "xin chào thế giới sp tiếng việt"
    lex = HERE / "lexicon_small.txt"
    rec = record()
    melD = np.asarray(ref_t2m.text2mel(text, lex, 0.2))
    tokD = ref_t2m.text2tokens(text, lex)
    n_rec = len(rec) // 2
    keepD = keep_masks_from_steps(rec, 1, n_rec)
    kb, ks = pack(keepD)
    np.savez_compressed(HERE / "nat_ref_text2mel.npz", text=np.array(text), tokens=np.asarray(tokD, np.int32),
                        silence_duration=np.float32(0.2), mel=melD.astype(np.float32), n_frames_model=np.int64(n_rec),
                        keep_bits=kb, keep_shape=ks)
    print("D text2mel", melD.shape, "model frames", n_rec, "tokens", len(tokD))

    # ---- E: GTA forward_fn_ (gta.py:28-41) + MelFilter (dsp.py:104-128), ragged batch ------------------------
    rng = np.random.default_rng(5)
    B, Lg, S = 2, 24, 16384                      # 64 frames
    lengths = np.array([24, 17], np.int32)
    tkg = rng.integers(4, 93, size=(B, Lg)).astype(np.int32)
    dug = rng.uniform(0.02, 0.08, size=(B, Lg)).astype(np.float32)
    for b in range(B):
        tkg[b, lengths[b]:] = 0
        dug[b, lengths[b]:] = 0.0
    wav_len = np.array([S, 11000], np.int32)
    t = np.arange(S) / 16000.0
    wav = np.zeros((B, S), np.float64)
    for b in range(B):
        for f0, a in ((180.0 + 40 * b, 0.3), (1250.0, 0.1), (3100.0 + 500 * b, 0.05)):
            wav[b] += a * np.sin(2 * np.pi * f0 * t + b)
        wav[b] += 0.02 * rng.standard_normal(S)
        wav[b, wav_len[b]:] = 0.0
    wav_i16 = np.clip(np.round(wav * 32767), -32768, 32767).astype(np.int16)
    inp = AcousticInput(tkg, lengths, dug, wav_i16, wav_len, None)
    rec = record()
    mel2_hat = np.asarray(ref_gta.forward_fn_(ack["params"], ack["aux"], ack["rng"], inp))
    Ng = mel2_hat.shape[1]
    assert len(rec) == 6 and rec[0][0] == (B, Ng, 256) and rec[2][0] == (B, Ng, 512) and rec[2][1] == 0.1
    keepg = np.stack([rec[0][2], rec[1][2]], axis=2)                      # [B,N,2,256] prenet keep masks
    zoneg = np.stack([rec[2][2], rec[3][2], rec[4][2], rec[5][2]], axis=2)   # [B,N,4,512]: h0, c0, h1, c1 (1 = keep previous)
    jax.random.RECORD = None
    logmel = np.asarray(MelFilter(FLAGS.sample_rate, FLAGS.n_fft, FLAGS.mel_dim, FLAGS.fmin, FLAGS.fmax)(
        wav_i16.astype(np.float32) / (2 ** 15)))

    # mel1 as well (AcousticModel.__call__ returns both; forward_fn_ keeps only mel2): same rng -> same masks
    @hk.transform_with_state
    def val_net(x):
        return ref_model.AcousticModel(is_training=False)(x)

    inp_mels = np.concatenate((np.zeros((B, 1, 80), np.float32), logmel[:, :-1, :]), axis=1)
    (mel1, mel2b), _ = val_net.apply(ack["params"], ack["aux"], ack["rng"],
                                      inp._replace(mels=inp_mels, durations=dug * FLAGS.sample_rate / (FLAGS.n_fft // 4)))
    assert np.abs(np.asarray(mel2b) - mel2_hat).max() == 0.0
    kb, ks = pack(keepg)
    zb, zs = pack(zoneg)
    np.savez_compressed(HERE / "nat_ref_gta.npz", tokens=tkg, lengths=lengths, durations_sec=dug, wav_i16=wav_i16,
                        wav_lengths=wav_len, logmel=logmel.astype(np.float32), mel1=np.asarray(mel1, np.float32),
                        mel2=mel2_hat.astype(np.float32), keep_bits=kb, keep_shape=ks, zone_bits=zb, zone_shape=zs,
                        rng=ack["rng"])
    print("E gta", mel2_hat.shape, "logmel", logmel.shape)


if __name__ == "__main__":
    main()
