"""CPU restatement of AcousticModel.inference.  Test infrastructure only.

Pinned to golden vectors produced by executing the reference's own source files on numpy stand-ins
for jax / haiku (tests/refshim, tests/golden/make_nat_golden.py, tests/test_reference_goldens.py): the
WIRING below is held to the reference at float64; the dm-haiku / jax primitives it relies on are
restated (jax / dm-haiku cannot be installed where this project is tested)
and cross-checked against torch operators.  float64 mode is the arbiter for the float32 CUDA path.

  TokenEncoder.__call__      vietTTS/nat/model.py:26-47
  AcousticModel.prenet       vietTTS/nat/model.py:95-100
  AcousticModel.upsample     vietTTS/nat/model.py:102-111
  AcousticModel.postnet      vietTTS/nat/model.py:113-121
  AcousticModel.inference    vietTTS/nat/model.py:123-144
  predict_mel                vietTTS/nat/text2mel.py:61-82
  DurationModel.__call__     vietTTS/nat/model.py:49-70
  AcousticModel.__call__     vietTTS/nat/model.py:146-169   (teacher forced, zoneout)
  forward_fn_ (GTA)          vietTTS/nat/gta.py:28-41
  text2mel post-processing   vietTTS/nat/text2mel.py:85-103

dm-haiku semantics used (not vendored in the reference, setup.py:6-19):
  hk.LSTM            z=[x,h]W+b; i,g,f,o=split(z,4); c'=sigmoid(f+1)c+sigmoid(i)tanh(g); h'=sigmoid(o)tanh(c')
  deep_rnn_with_skip_connections   layer1 input = concat(x, out0); output = concat(out0,out1)
  hk.BatchNorm(eval) (x-mean_ema.average)*scale*rsqrt(var_ema.average+1e-5)+offset
  hk.Conv1D          NWC, w[K,Cin,Cout], SAME zero padding
  hk.dropout         keep*x/(1-rate); the keep mask is an explicit INPUT here
                     (the reference draws it from the checkpoint's rng, model.py:97,99)
  hk.ResetCore       state zeroed where reset is True, before the core runs
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

A = "acoustic_model/~/"
T = A + "token_encoder/~/"


def _t(a, dtype):
    return torch.as_tensor(np.asarray(a)).to(dtype)


def conv1d_same(x, w, b):
    K = w.shape[0]
    y = F.conv1d(x.transpose(1, 2), w.permute(2, 1, 0).contiguous(), b, padding=(K - 1) // 2)
    return y.transpose(1, 2)


def batchnorm_eval(x, P, S, name, dtype):
    scale = _t(P[name]["scale"], dtype)
    offset = _t(P[name]["offset"], dtype)
    mean = _t(S[name + "/~/mean_ema"]["average"], dtype)
    var = _t(S[name + "/~/var_ema"]["average"], dtype)
    inv = scale * torch.rsqrt(var + 1e-5)
    return (x - mean) * inv + offset


def lstm_step(x, h, c, w, b):
    """hk.LSTM.__call__"""
    z = torch.cat([x, h], dim=-1) @ w + b
    i, g, f, o = torch.chunk(z, 4, dim=-1)
    f = torch.sigmoid(f + 1)
    c = f * c + torch.sigmoid(i) * torch.tanh(g)
    h = torch.sigmoid(o) * torch.tanh(c)
    return h, c


def token_encoder(P, S, tokens, lengths, dtype=torch.float32, T=T):
    """model.py:26-47 with is_training=False.  tokens int [B,L]; lengths int [B].
    Returns [B,L,2D].  `T` is the Haiku module prefix (acoustic or duration model's encoder)."""
    tokens = torch.as_tensor(np.asarray(tokens)).long()
    lengths = torch.as_tensor(np.asarray(lengths)).long()
    x = _t(P[T + "embed"]["embeddings"], dtype)[tokens]
    for i in range(3):
        sfx = "" if i == 0 else f"_{i}"
        cw = P[T + "conv1_d" + sfx]
        x = conv1d_same(x, _t(cw["w"], dtype), _t(cw["b"], dtype))
        x = torch.relu(batchnorm_eval(x, P, S, T + "batch_norm" + sfx, dtype))
    B, L, D = x.shape
    mask = torch.arange(L)[None, :] >= (lengths[:, None] - 1)  # model.py:37
    wf, bf = _t(P[T + "lstm/linear"]["w"], dtype), _t(P[T + "lstm/linear"]["b"], dtype)
    wb, bb = _t(P[T + "lstm_1/linear"]["w"], dtype), _t(P[T + "lstm_1/linear"]["b"], dtype)
    h = x.new_zeros(B, D)
    c = x.new_zeros(B, D)
    fwd = []
    for t in range(L):
        h, c = lstm_step(x[:, t], h, c, wf, bf)
        fwd.append(h)
    h = x.new_zeros(B, D)
    c = x.new_zeros(B, D)
    bwd = [None] * L
    for t in range(L - 1, -1, -1):  # flipped sequence, model.py:40-44
        r = mask[:, t][:, None]
        h = torch.where(r, torch.zeros_like(h), h)  # ResetCore
        c = torch.where(r, torch.zeros_like(c), c)
        h, c = lstm_step(x[:, t], h, c, wb, bb)
        bwd[t] = h
    return torch.cat([torch.stack(fwd, 1), torch.stack(bwd, 1)], dim=-1)


def upsample(x, durations, n_frames: int):
    """model.py:102-111.  x [B,L,D]; durations [B,L] in frames."""
    ruler = torch.arange(0, n_frames, dtype=x.dtype)[None, :]
    end_pos = torch.cumsum(durations, dim=1)
    mid_pos = end_pos - durations / 2
    d2 = torch.square(mid_pos[:, None, :] - ruler[:, :, None]) / 10.0
    w = torch.softmax(-d2, dim=-1)
    return torch.einsum("BLT,BTD->BLD", w, x), w


def prenet(P, x, keep, dtype):
    """model.py:95-100.  keep: None (dropout off, scale 1) or bool [B,2,256]."""
    w1 = _t(P[A + "linear_1"]["w"], dtype)
    w2 = _t(P[A + "linear_2"]["w"], dtype)
    x = torch.relu(x @ w1)
    if keep is not None:
        x = keep[:, 0].to(dtype) * x / 0.5
    x = torch.relu(x @ w2)
    if keep is not None:
        x = keep[:, 1].to(dtype) * x / 0.5
    return x


def decode(P, cond, masks=None, dtype=torch.float32):
    """The hk.dynamic_unroll(loop_fn) of model.py:129-142.  cond [B,N,512];
    masks uint8 [B,N,2,256] keep-masks or None.  Returns pre-postnet mel [B,N,80]."""
    B, N, _ = cond.shape
    w0, b0 = _t(P[A + "lstm/linear"]["w"], dtype), _t(P[A + "lstm/linear"]["b"], dtype)
    w1, b1 = _t(P[A + "lstm_1/linear"]["w"], dtype), _t(P[A + "lstm_1/linear"]["b"], dtype)
    wo, bo = _t(P[A + "linear"]["w"], dtype), _t(P[A + "linear"]["b"], dtype)
    H = w0.shape[1] // 4
    mel = cond.new_zeros(B, wo.shape[1])
    h0 = cond.new_zeros(B, H)
    c0 = cond.new_zeros(B, H)
    h1 = cond.new_zeros(B, H)
    c1 = cond.new_zeros(B, H)
    if masks is not None:
        masks = torch.as_tensor(np.asarray(masks)).bool()
    out = []
    for t in range(N):
        p = prenet(P, mel, None if masks is None else masks[:, t], dtype)
        x = torch.cat([cond[:, t], p], dim=-1)
        h0, c0 = lstm_step(x, h0, c0, w0, b0)
        h1, c1 = lstm_step(torch.cat([x, h0], dim=-1), h1, c1, w1, b1)
        mel = torch.cat([h0, h1], dim=-1) @ wo + bo
        out.append(mel)
    return torch.stack(out, 1)


def postnet(P, S, mel, dtype=torch.float32):
    """model.py:113-121 with is_training=False."""
    x = mel
    for i in range(5):
        sfx = "" if i == 0 else f"_{i}"
        cw = P[A + "conv1_d" + sfx]
        x = conv1d_same(x, _t(cw["w"], dtype), _t(cw["b"], dtype))
        if i < 4:
            x = torch.tanh(batchnorm_eval(x, P, S, A + "batch_norm" + sfx, dtype))
    return x


def inference(ckpt, tokens, durations_frames, n_frames: int, masks=None, dtype=torch.float32, taps=None):
    """AcousticModel.inference (model.py:123-144).  tokens [B,L]; durations [B,L]
    in frames; like the reference, `lengths=[L]` for every row."""
    P, S = ckpt["params"], ckpt["aux"]
    tokens = np.asarray(tokens)
    B, L = tokens.shape
    with torch.no_grad():
        enc = token_encoder(P, S, tokens, np.full((B,), L), dtype)
        cond, attn = upsample(enc, _t(durations_frames, dtype), n_frames)
        x = decode(P, cond, masks, dtype)
        res = postnet(P, S, x, dtype)
        if taps is not None:
            taps.update(enc=enc, cond=cond, attn=attn, pre=x, res=res)
        return x + res


def frame_count(frames):
    """n_frames = int(sum(durations)) of text2mel.py:79 for one row of float32 frame durations: the sum in float64,
    term by term in token order, rounded to float32 once, truncated.  The reference's `jnp.sum` leaves the order to
    XLA; the float64 sum of float32 terms is exact for any realistic row, so this count does not depend on it."""
    total = 0.0
    for f in np.asarray(frames, np.float32).ravel().tolist():
        total += f
    return int(np.float32(total))


def seconds_to_frames(durations_sec):
    """text2mel.py:78-79: float32 `durations * 16000 / 256`, n_frames = frame_count."""
    d = (np.asarray(durations_sec, np.float32) * np.float32(16000)) / np.float32(256)
    return d, frame_count(d)


def predict_mel(ckpt, tokens, durations_sec, masks=None, dtype=torch.float32):
    """predict_mel (text2mel.py:61-82) minus the pickle load; returns np [N,80]."""
    d, n = seconds_to_frames(durations_sec)
    mel = inference(ckpt, np.asarray(tokens, np.int32)[None, :], d, n, masks, dtype)
    return mel[0].numpy()


def inference_ragged(ckpt, tokens_list, dur_frames_list, masks_list=None, dtype=torch.float32):
    """Definition of batched semantics (SURVEY.md §7 H4): row b of a batch equals
    the reference run on row b alone, unpadded.  Returns list of np [N_b,80]."""
    outs = []
    for b, (tk, d) in enumerate(zip(tokens_list, dur_frames_list)):
        d = np.asarray(d, np.float32)[None, :]
        n = frame_count(d)
        m = None if masks_list is None else np.asarray(masks_list[b])[None, :n]
        outs.append(inference(ckpt, np.asarray(tk, np.int32)[None, :], d, n, m, dtype)[0].numpy())
    return outs


# ---------------------------------------------------------------------------
# DurationModel (model.py:49-70) and the text2mel glue around it (text2mel.py:85-103)
# ---------------------------------------------------------------------------
DM = "duration_model/~/"


def gelu_tanh(x):
    """jax.nn.gelu with its default approximate=True (model.py:61 passes the bare function)."""
    return 0.5 * x * (1.0 + torch.tanh(np.sqrt(2.0 / np.pi) * (x + 0.044715 * x ** 3)))


def softplus(x):
    """jax.nn.softplus = logaddexp(x, 0)."""
    return torch.clamp(x, min=0) + torch.log1p(torch.exp(-torch.abs(x)))


def duration_model(ckpt, tokens, lengths, dtype=torch.float32):
    """DurationModel(is_training=False)(DurationInput(tokens, lengths, None)), model.py:64-70.
    tokens int [B,L]; lengths int [B] -> durations in seconds [B,L] (every position, as the reference)."""
    P, S = ckpt["params"], ckpt["aux"]
    with torch.no_grad():
        x = token_encoder(P, S, tokens, lengths, dtype, T=DM + "token_encoder/~/")
        l1, l2 = P[DM + "linear"], P[DM + "linear_1"]
        x = gelu_tanh(x @ _t(l1["w"], dtype) + _t(l1["b"], dtype))
        x = (x @ _t(l2["w"], dtype) + _t(l2["b"], dtype)).squeeze(-1)
        return softplus(x).numpy()


def predict_duration(ckpt, tokens, dtype=torch.float32):
    """text2mel.py:22-34: one utterance, lengths = [len(tokens)] -> [1,L] seconds."""
    tok = np.asarray(tokens, np.int32)[None, :]
    return duration_model(ckpt, tok, np.array([tok.shape[1]], np.int32), dtype)


def adjust_durations(tokens, durations, silence_duration=-1.0, sil_index=0, word_end_index=3):
    """text2mel.py:88-97: sil tokens are clipped from below at `silence_duration`, word-end tokens get 0."""
    tok = np.asarray(tokens)[None, :]
    d = np.asarray(durations, np.float32)
    d = np.where(tok == sil_index, np.clip(d, silence_duration, None), d)
    d = np.where(tok == word_end_index, np.float32(0.0), d)
    return d.astype(np.float32)


def trim_end_silence(tokens, durations, mel, sil_index=0):
    """text2mel.py:99-102: drop the frames of the trailing silence token."""
    if tokens[-1] == sil_index:
        end_silence = float(durations[0, -1])
        silence_frame = int(end_silence * 16000 / 256)
        mel = mel[:, : (mel.shape[1] - silence_frame)]
    return mel


# ---------------------------------------------------------------------------
# teacher-forced pass with zoneout (model.py:146-169) and the GTA forward (gta.py:28-41)
# ---------------------------------------------------------------------------
def teacher_forced(ckpt, tokens, lengths, durations_frames, mels_in, keep_masks=None, zone_masks=None, dtype=torch.float32):
    """AcousticModel(is_training=False).__call__(AcousticInput(...)).  tokens int [B,L]; lengths int [B];
    durations [B,L] in frames; mels_in [B,N,80] = ground truth shifted by one frame (the caller does the shift,
    gta.py:34-36).  keep_masks uint8 [B,N,2,256] (prenet dropout keep) or None; zone_masks uint8 [B,N,4,512] in the
    state-tree order (layer0.hidden, layer0.cell, layer1.hidden, layer1.cell), 1 = keep previous state
    (`s1 * m + s2 * (1 - m)`, model.py:157-159), or None.  Both mask sets are explicit INPUTS here; the reference
    draws them from hk.next_rng_key().  Returns (mel1, mel2) = (projection, projection + postnet) as numpy [B,N,80]."""
    P, S = ckpt["params"], ckpt["aux"]
    with torch.no_grad():
        mels_in = _t(mels_in, dtype)
        N = mels_in.shape[1]
        enc = token_encoder(P, S, tokens, lengths, dtype)
        cond, _ = upsample(enc, _t(durations_frames, dtype), N)
        x = torch.cat([cond, tf_prenet(P, mels_in, keep_masks, dtype)], dim=-1)
        mel1 = project(P, zoneout_decode(P, x, zone_masks, dtype), dtype)
        mel2 = mel1 + postnet(P, S, mel1, dtype)
        return mel1.numpy(), mel2.numpy()


def tf_prenet(P, mels_in, keep=None, dtype=torch.float32):
    """The prenet of the teacher-forced pass over whole sequences (model.py:95-100,149).  mels_in [B,N,80] (any float
    array); keep uint8 [B,N,2,256] or None (dropout off, scale 1).  Returns p2 [B,N,256]."""
    with torch.no_grad():
        x = _t(mels_in, dtype)
        w1 = _t(P[A + "linear_1"]["w"], dtype)
        w2 = _t(P[A + "linear_2"]["w"], dtype)
        km = None if keep is None else torch.as_tensor(np.asarray(keep)).bool()
        x = torch.relu(x @ w1)
        if km is not None:
            x = km[:, :, 0].to(dtype) * x / 0.5
        x = torch.relu(x @ w2)
        if km is not None:
            x = km[:, :, 1].to(dtype) * x / 0.5
        return x


def zoneout_decode(P, x, zone=None, dtype=torch.float32):
    """The zoneout decoder of the teacher-forced pass (model.py:150-166): x [B,N,768] = [cond | p2] (any float array);
    zone uint8 [B,N,4,512] in the state-tree order (layer0.hidden, layer0.cell, layer1.hidden, layer1.cell), 1 = keep
    the previous state (`s1 * m + s2 * (1 - m)`, model.py:157-159), or None.  Returns the decoder output [B,N,1024] =
    [h0 | h1], the cores' new (un-zoned) hidden states."""
    with torch.no_grad():
        x = _t(x, dtype)
        B, N, _ = x.shape
        w0, b0 = _t(P[A + "lstm/linear"]["w"], dtype), _t(P[A + "lstm/linear"]["b"], dtype)
        w1, b1 = _t(P[A + "lstm_1/linear"]["w"], dtype), _t(P[A + "lstm_1/linear"]["b"], dtype)
        H = w0.shape[1] // 4
        h0 = x.new_zeros(B, H); c0 = x.new_zeros(B, H); h1 = x.new_zeros(B, H); c1 = x.new_zeros(B, H)
        zm = None if zone is None else torch.as_tensor(np.asarray(zone)).bool()
        outs = []
        for t in range(N):
            nh0, nc0 = lstm_step(x[:, t], h0, c0, w0, b0)
            nh1, nc1 = lstm_step(torch.cat([x[:, t], nh0], dim=-1), h1, c1, w1, b1)   # skip connection feeds the NEW h0
            outs.append(torch.cat([nh0, nh1], dim=-1))                                 # decoder output = un-zoned states
            if zm is None:
                h0, c0, h1, c1 = nh0, nc0, nh1, nc1
            else:
                h0 = torch.where(zm[:, t, 0], h0, nh0); c0 = torch.where(zm[:, t, 1], c0, nc0)
                h1 = torch.where(zm[:, t, 2], h1, nh1); c1 = torch.where(zm[:, t, 3], c1, nc1)
        return torch.stack(outs, 1)


def project(P, hout, dtype=torch.float32):
    """The output projection (model.py:167): hout [B,N,1024] (any float array) -> mel1 [B,N,80]."""
    with torch.no_grad():
        return _t(hout, dtype) @ _t(P[A + "linear"]["w"], dtype) + _t(P[A + "linear"]["b"], dtype)


def gta_forward(ckpt, wav_i16, tokens, lengths, durations_sec, keep_masks=None, zone_masks=None, dtype=torch.float32):
    """forward_fn_ (gta.py:28-41) for one padded batch: int16 wavs [B,S] -> (ground-truth mel, mel2_hat)."""
    from . import mel_oracle
    wav = np.asarray(wav_i16).astype(np.float32) / np.float32(2 ** 15)
    mels = mel_oracle.mel_filter(wav)
    inp = np.concatenate([np.zeros_like(mels[:, :1]), mels[:, :-1]], axis=1)
    frames = (np.asarray(durations_sec, np.float32) * np.float32(16000)) / np.float32(256)
    _, mel2 = teacher_forced(ckpt, tokens, lengths, frames, inp, keep_masks, zone_masks, dtype)
    return mels, mel2
