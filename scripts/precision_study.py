"""CPU emulation of the dense-contraction arithmetic modes on the whole HiFiGAN generator.

Every conv / transposed conv of the oracle is replaced by a version that rounds its operands the way a mode does,
multiplies the rounded operands in float64 (exact products) and rounds each layer output to fp32 -- i.e. the only
error modelled is the operand rounding, which is what distinguishes the modes.  Reported: waveform error against a
float64 run of the same network.

    python scripts/precision_study.py [T_frames]
"""
import sys
from pathlib import Path

import numpy as np
import torch

REPO = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(REPO))
from oracle import hifigan_oracle as ho  # noqa: E402
from viettts_b200 import synthetic  # noqa: E402


def _bf16(x):
    return x.to(torch.float32).to(torch.bfloat16).to(torch.float64)


def _tf32(x):
    i = x.to(torch.float32).view(torch.int32)
    i = (i + 0x1000) & ~0x1FFF           # round to 10 mantissa bits (nearest, ties away)
    return i.view(torch.float32).to(torch.float64)


FP16_MAX = 65504.0


def _fp16(x):
    # saturating, like the kernels' conversions (cvt.rn.satfinite): a value past the fp16 range becomes +-65504, not inf
    return x.to(torch.float32).clamp(-FP16_MAX, FP16_MAX).to(torch.float16).to(torch.float64)


def split(x, rnd, terms):
    """x -> [x0, x1, ...] with x0 = rnd(x), x1 = rnd(x - x0), ..."""
    out, rest = [], x.to(torch.float64)
    for _ in range(terms):
        p = rnd(rest)
        out.append(p)
        rest = rest - p
    return out


MODES = {
    # name: (rounding, operand terms, products kept as (i, j) index pairs of the a / w terms)
    "fp32": (None, 1, None),
    "bf16x1": (_bf16, 1, [(0, 0)]),
    "tf32x1": (_tf32, 1, [(0, 0)]),
    "fp16x1": (_fp16, 1, [(0, 0)]),
    "bf16x3": (_bf16, 2, [(0, 0), (0, 1), (1, 0)]),
    "tf32x3": (_tf32, 2, [(0, 0), (0, 1), (1, 0)]),
    "bf16x6": (_bf16, 3, [(0, 0), (0, 1), (1, 0), (1, 1), (0, 2), (2, 0)]),
}


def run(params, mel, mode):
    rnd, terms, pairs = MODES[mode]
    conv0, convt0 = ho.conv1d_nwc, ho.conv1d_transpose_nwc

    def conv(x, w, b, dilation=1, pad=None):
        if rnd is None:
            return conv0(x.to(torch.float32), w.to(torch.float32), b.to(torch.float32), dilation, pad).to(torch.float64)
        xs, ws = split(x, rnd, terms), split(w, rnd, terms)
        acc = None
        for i, j in pairs:
            y = conv0(xs[i], ws[j], torch.zeros_like(b, dtype=torch.float64), dilation, pad)
            acc = y if acc is None else acc + y
        return (acc + b.to(torch.float64)).to(torch.float32).to(torch.float64)

    def convt(x, w, b, stride):
        if rnd is None:
            return convt0(x.to(torch.float32), w.to(torch.float32), b.to(torch.float32), stride).to(torch.float64)
        xs, ws = split(x, rnd, terms), split(w, rnd, terms)
        acc = None
        for i, j in pairs:
            y = convt0(xs[i], ws[j], torch.zeros_like(b, dtype=torch.float64), stride)
            acc = y if acc is None else acc + y
        return (acc + b.to(torch.float64)).to(torch.float32).to(torch.float64)

    ho.conv1d_nwc, ho.conv1d_transpose_nwc = conv, convt
    try:
        with torch.no_grad():
            return ho.generator_forward(params, mel, torch.float64).numpy()
    finally:
        ho.conv1d_nwc, ho.conv1d_transpose_nwc = conv0, convt0


def study(T=24, modes=tuple(MODES)):
    params = synthetic.hifigan_params(1234)
    mel = synthetic.mel_input(0, 1, T)
    with torch.no_grad():
        ref = ho.generator_forward(params, mel, torch.float64).numpy()
    out = {}
    for m in modes:
        e = run(params, mel, m) - ref
        out[m] = (float(np.abs(e).max()), float(np.sqrt(np.mean(e ** 2))))
    return out


if __name__ == "__main__":
    T = int(sys.argv[1]) if len(sys.argv) > 1 else 24
    print(f"{'mode':8s} {'waveform L-inf':>15s} {'RMS':>10s}   (generator, T={T} frames, vs float64)")
    for m, (linf, rms) in study(T).items():
        print(f"{m:8s} {linf:15.1e} {rms:10.1e}")
