"""CPU restatement of the Haiku HiFiGAN generator.  Test infrastructure only.

Follows the reference's vietTTS/hifigan/model.py line by line, in the NWC layout
and with the Haiku parameter layout of hk_hifi.pickle:

  get_padding      model.py:8-10
  ResBlock1        model.py:13-51
  Generator        model.py:77-125

hk.Conv1D / hk.Conv1DTranspose are dm-haiku library modules (not vendored); their
arithmetic is restated here from the published semantics (SURVEY.md appendix A)
and PINNED against the reference's importable torch implementation
(vietTTS/hifigan/torch_model.py) through tests/golden/make_golden.py.

All functions take/return torch CPU tensors; `dtype` float32 is the parity mode,
float64 the arbiter.
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

LRELU_SLOPE = 0.1  # model.py:5
UPSAMPLE_RATES = [8, 8, 2, 2]
UPSAMPLE_KERNELS = [16, 16, 4, 4]
RB_KERNELS = [3, 7, 11]
RB_DILATIONS = [1, 3, 5]


def get_padding(kernel_size: int, dilation: int = 1) -> int:
    """model.py:8-10"""
    return int((kernel_size * dilation - dilation) / 2)


def _t(a, dtype):
    return torch.as_tensor(np.asarray(a)).to(dtype)


def conv1d_nwc(x, w, b, dilation: int = 1, pad: int | None = None):
    """hk.Conv1D: y[b,t,o] = bias[o] + sum_j sum_i xpad[b, t + j*d, i] * w[j,i,o].

    x [B,T,Cin]; w Haiku layout [K,Cin,Cout]; zero pad `pad` both sides
    (default SAME for odd K = get_padding)."""
    K = w.shape[0]
    if pad is None:
        pad = get_padding(K, dilation)
    y = F.conv1d(x.transpose(1, 2), w.permute(2, 1, 0).contiguous(), b, padding=pad, dilation=dilation)
    return y.transpose(1, 2)


def conv1d_transpose_nwc(x, w, b, stride: int):
    """hk.Conv1DTranspose(padding="SAME"): zero-insert by `stride`, pad
    (K+stride-2) split ceil/floor, correlate with the stored kernel w[K,Cout,Cin]
    without flipping (SURVEY.md appendix A; model.py:87-95)."""
    B, L, Cin = x.shape
    K = w.shape[0]
    xd = x.new_zeros(B, (L - 1) * stride + 1, Cin)
    xd[:, ::stride] = x
    pad_len = K + stride - 2
    a = (pad_len + 1) // 2
    bpad = pad_len - a
    xd = F.pad(xd.transpose(1, 2), (a, bpad))
    y = F.conv1d(xd, w.permute(1, 2, 0).contiguous(), b)  # weight [Cout,Cin,K], correlation
    assert y.shape[-1] == L * stride
    return y.transpose(1, 2)


def resblock1(x, p, prefix: str, k: int, dtype, taps: dict | None = None, tag: str = ""):
    """model.py:44-51.  If `taps` is a dict, the input of step m is stored as taps[f"{tag}_{m}"] and the output as
    taps[f"{tag}_3"]."""
    for m, d in enumerate(RB_DILATIONS):
        if taps is not None:
            taps[f"{tag}_{m}"] = x
        c1 = p[f"{prefix}/~/convs1_{m}"]
        c2 = p[f"{prefix}/~/convs2_{m}"]
        xt = F.leaky_relu(x, LRELU_SLOPE)
        xt = conv1d_nwc(xt, _t(c1["w"], dtype), _t(c1["b"], dtype), dilation=d)
        xt = F.leaky_relu(xt, LRELU_SLOPE)
        xt = conv1d_nwc(xt, _t(c2["w"], dtype), _t(c2["b"], dtype), dilation=1)
        x = xt + x
    if taps is not None:
        taps[f"{tag}_3"] = x
    return x


def generator_forward(params: dict, mel, dtype=torch.float32, taps: dict | None = None):
    """Generator.__call__ (model.py:109-125).  mel [B,T,80] -> wav [B,256T].

    If `taps` is a dict, intermediate activations are stored in it
    ("pre", "ups_i", "stage_i"; "rb_i_j_m": the input of ResBlock step m of chain j of stage i, m = 3 its output)."""
    x = _t(mel, dtype)
    g = "generator/~/"
    p0 = params[g + "conv1_d"]
    x = conv1d_nwc(x, _t(p0["w"], dtype), _t(p0["b"], dtype), pad=3)
    if taps is not None:
        taps["pre"] = x
    for i, u in enumerate(UPSAMPLE_RATES):
        x = F.leaky_relu(x, LRELU_SLOPE)
        pu = params[g + f"ups_{i}"]
        x = conv1d_transpose_nwc(x, _t(pu["w"], dtype), _t(pu["b"], dtype), u)
        if taps is not None:
            taps[f"ups_{i}"] = x
        xs = None
        for j, k in enumerate(RB_KERNELS):
            r = resblock1(x, params, g + f"res_block1_{i * 3 + j}", k, dtype, taps, f"rb_{i}_{j}")
            xs = r if xs is None else xs + r
        x = xs / 3
        if taps is not None:
            taps[f"stage_{i}"] = x
    x = F.leaky_relu(x)  # default slope 0.01, model.py:122
    pp = params[g + "conv1_d_1"]
    x = conv1d_nwc(x, _t(pp["w"], dtype), _t(pp["b"], dtype), pad=3)
    x = torch.tanh(x)
    return x.squeeze(-1)


def mel2wave(params: dict, mel, dtype=torch.float32) -> np.ndarray:
    """mel2wave.py:20-41 minus the file I/O: forward, squeeze, to numpy."""
    with torch.no_grad():
        wav = generator_forward(params, mel, dtype)
    return np.squeeze(wav.numpy())
