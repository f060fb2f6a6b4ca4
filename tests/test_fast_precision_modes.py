"""The fast fp16 generator mode (VTTS_PRECISION_FP16) and its stated tolerance, from the CPU emulation of operand rounding
(scripts/precision_study.py): one fp16 product per operand pair, saturating conversions, fp32 accumulate.

The waveform tolerance of the mode, L-inf <= 3e-3 and RMS <= 6e-4 against float64, is about 3x the emulated error of the
whole generator on the synthetic weights; tests/test_gpu_fp16_generator.py holds the kernels to it.  The per-layer bound
of that file (normalised L-inf <= 1e-3) is checked here to be at least 3x the emulated error of the same layers."""
import importlib.util
from pathlib import Path

import numpy as np
import torch

REPO = Path(__file__).resolve().parents[1]
FAST_WAV_LINF, FAST_WAV_RMS = 3e-3, 6e-4      # the tolerance of tests/test_gpu_fp16_generator.py
LAYER_NLINF = 1e-3                              # max |err| / max |ref| of one conv or fused pair, same file


def _study():
    spec = importlib.util.spec_from_file_location("precision_study", REPO / "scripts" / "precision_study.py")
    ps = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ps)
    return ps


def test_fp16_meets_the_fast_tolerance_and_matches_tf32():
    ps = _study()
    r = ps.study(T=12, modes=("bf16x1", "tf32x1", "fp16x1"))
    linf, rms = r["fp16x1"]
    assert linf <= FAST_WAV_LINF / 2.5 and rms <= FAST_WAV_RMS / 2.2, r    # the tolerance keeps >= 2x headroom
    # fp16 and tf32 keep the same 11 significand bits: the same error; bf16 keeps 8
    assert linf <= 1.2 * r["tf32x1"][0] and rms <= 1.2 * r["tf32x1"][1], r
    assert 4 * linf <= r["bf16x1"][0] and 4 * rms <= r["bf16x1"][1], r


def test_fp16_rounding_saturates():
    ps = _study()
    x = torch.tensor([1e6, -1e6, 65519.0, 1.0 + 2.0 ** -12, np.nan], dtype=torch.float64)
    y = ps._fp16(x)
    assert y[0] == 65504.0 and y[1] == -65504.0 and y[2] == 65504.0
    assert y[3] == 1.0 and torch.isnan(y[4])


def _conv(x, w, b, k, dil):
    f = torch.nn.functional
    return f.conv1d(x.transpose(1, 2), w.permute(2, 1, 0).contiguous(), b, padding=(k - 1) * dil // 2, dilation=dil).transpose(1, 2)


def test_layer_bound_has_headroom_over_the_emulation():
    """The inputs of the GPU layer tests (same seeds and shapes); the emulated operand rounding must stay below a third of
    the bound."""
    ps = _study()
    f = torch.nn.functional
    worst_conv = worst_pair = 0.0
    for C in (32, 64, 128, 256):
        for k in (3, 7, 11):
            for dil in (1, 3, 5):
                rng = np.random.default_rng(C * 100 + k * 10 + dil)
                B, T = 2, 600
                x = torch.from_numpy(rng.standard_normal((B, T, C)).astype(np.float32)).double()
                w = torch.from_numpy((rng.standard_normal((k, C, C)) / np.sqrt(k * C)).astype(np.float32)).double()
                b = torch.from_numpy((rng.standard_normal(C) * 0.1).astype(np.float32)).double()
                res = torch.from_numpy(rng.standard_normal((B, T, C)).astype(np.float32)).double()
                xa = f.leaky_relu(x, 0.1)
                ref = _conv(xa, w, b, k, dil) + res
                emu = _conv(ps._fp16(xa), ps._fp16(w), b, k, dil) + res
                worst_conv = max(worst_conv, float((emu - ref).abs().max() / ref.abs().max()))
                if C > 64:
                    continue
                rng = np.random.default_rng(C * 1000 + k * 10 + dil)
                B, T = 3, 700
                x = torch.from_numpy(rng.standard_normal((B, T, C)).astype(np.float32)).double()
                w1 = torch.from_numpy((rng.standard_normal((k, C, C)) / np.sqrt(k * C)).astype(np.float32)).double()
                w2 = torch.from_numpy((rng.standard_normal((k, C, C)) / np.sqrt(k * C)).astype(np.float32)).double()
                b1 = torch.from_numpy((rng.standard_normal(C) * 0.1).astype(np.float32)).double()
                b2 = torch.from_numpy((rng.standard_normal(C) * 0.1).astype(np.float32)).double()

                def pair(rnd):
                    y = f.leaky_relu(_conv(rnd(f.leaky_relu(x, 0.1)), rnd(w1), b1, k, dil), 0.1)
                    return _conv(rnd(y), rnd(w2), b2, k, 1) + x

                ref, emu = pair(lambda v: v), pair(ps._fp16)
                worst_pair = max(worst_pair, float((emu - ref).abs().max() / ref.abs().max()))
    print(f"emulated normalised L-inf: conv {worst_conv:.2e}, fused pair {worst_pair:.2e}")
    assert 3 * worst_conv <= LAYER_NLINF and 3 * worst_pair <= LAYER_NLINF, (worst_conv, worst_pair)
