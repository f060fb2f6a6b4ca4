"""CPU: the per-layer bounds of tests/test_gpu_generator_layers.py against an emulation of each arithmetic mode, on the base
case of every generator layer (same seeds and shapes as the GPU test).

Each emulation rounds the operands as the kernels do and multiplies them exactly (float64):
  fp32    the FP32 kernel (csrc/conv1d.cu): one fp32 fma per (16-channel chunk, tap, channel) in that order, a
          ConvTranspose as its u two-tap output phases;
  bf16x3  hi.hi + hi.lo + lo.hi of the bf16 hi/lo split;
  fp16    one product of saturated fp16 operands;
and rounds every layer output to fp32.  Each TOL must stay 4x above its mode's emulated error; and the bounds must see
what they guard against: plain bf16 (the lo terms dropped) in one problem of a launch exceeds the bf16x3 bound 10x, and
bf16 operands exceed the fp16 bound."""
import importlib.util
from pathlib import Path

import numpy as np
import torch

import test_gpu_generator_layers as gl
from oracle import hifigan_oracle as ho

REPO = Path(__file__).resolve().parents[1]
_spec = importlib.util.spec_from_file_location("precision_study", REPO / "scripts" / "precision_study.py")
ps = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(ps)
CPU = torch.device("cpu")


def split_conv(mode):
    """a conv of gl.reference's signature with the operand rounding of a precision_study mode, output rounded to fp32"""
    rnd, terms, pairs = ps.MODES[mode]

    def conv(x, w, b, dil=1, pad=None, stride=None):
        xs, ws = ps.split(x, rnd, terms), ps.split(w, rnd, terms)
        y = sum(gl.exact_conv(xs[i], ws[j], None, dil, pad, stride) for i, j in pairs)
        return (y + b).float().double()
    return conv


def _fp32_taps(x, w, in_off, dil):
    """out[t] = sum_j sum_i x[t + in_off + j*dil, i] w[j, i, :], x [B, L, Cin] (zero outside), w [k, Cin, Cout]: one fp32
    fma per (16-channel chunk, tap, channel), in that order"""
    B, L, cin = x.shape
    k = w.shape[0]
    lo = max(0, -in_off)
    hi = max(0, in_off + (k - 1) * dil)
    xp = torch.nn.functional.pad(x, (0, 0, lo, hi))
    acc = torch.zeros(B, L, w.shape[2], dtype=torch.float32)
    for c in range(0, cin, 16):
        for j in range(k):
            s = lo + in_off + j * dil
            for i in range(c, c + 16):
                acc = (acc.double() + xp[:, s : s + L, i : i + 1] * w[j, i]).float()
    return acc.double()


def fp32_conv(x, w, b, dil=1, pad=None, stride=None):
    if stride is None:
        pad = ho.get_padding(w.shape[0], dil) if pad is None else pad
        return (_fp32_taps(x, w, -pad, dil) + b).float().double()
    # the u output phases of the transposed conv (csrc/hifigan.cu repack_ups_kernel): phase r reads taps j0 + q*u at
    # input rows tau + e + q
    K, u = w.shape[0], stride
    a = (K + u - 2 + 1) // 2
    B, L, _ = x.shape
    y = torch.empty(B, L * u, w.shape[1], dtype=torch.float64)
    for r in range(u):
        j0 = (a - r) % u
        e = (r + j0 - a) // u
        wr = torch.stack([w[j0].T, w[j0 + u].T])
        y[:, r::u] = (_fp32_taps(x, wr, e, 1) + b).float().double()
    return y


EMULATIONS = {"fp32": fp32_conv, "bf16x3": split_conv("bf16x3"), "fp16": split_conv("fp16x1"), "bf16x1": split_conv("bf16x1")}


def first_problem(L, a):
    """the outputs of the launch's first problem in one output tensor: conv_pre's first N = 256 tile, the ConvTranspose's
    first output phase (a ResBlock step's problems are its chains, one output each)"""
    if L.kind == "pre":
        return a[..., :256]
    if L.kind == "ups":
        return a[:, :: ho.UPSAMPLE_RATES[L.stage]]
    return a


def normalised(refs, emus, L=None):
    """worst |emulated - float64| / S over the outputs (L given: over the first problem only)"""
    pairs = list(zip(refs, emus))[:1] if L is not None else zip(refs, emus)
    worst = 0.0
    for (ref, s, _), (y, _, _) in pairs:
        err = (y - ref).abs() / s.clamp_min(1e-30)
        worst = max(worst, float((first_problem(L, err) if L is not None else err).max()))
    return worst


def test_bounds_have_headroom_over_the_emulation(hifigan_params):
    worst = {m: 0.0 for m in gl.MODES}
    low = {"bf16x1 one problem": np.inf, "bf16x1 vs fp16": np.inf}
    report = []
    for L in gl.LAYERS:
        xs = gl.random_inputs(L, 1, gl.BASE_T, gl.layer_seed(L, "base"))
        xs = [torch.from_numpy(x) for x in xs]
        with torch.no_grad():
            refs = gl.reference(L, hifigan_params, xs, None, CPU)
            row = {}
            for mode in gl.MODES:
                # conv_post is strict fp32 in every mode
                conv = EMULATIONS["fp32" if L.kind == "post" else mode]
                row[mode] = normalised(refs, gl.reference(L, hifigan_params, xs, None, CPU, conv))
                worst[mode] = max(worst[mode], row[mode])
            if L.kind != "post":
                emu = gl.reference(L, hifigan_params, xs, None, CPU, EMULATIONS["bf16x1"])
                row["bf16x1 one problem"] = normalised(refs, emu, L)
                row["bf16x1 vs fp16"] = normalised(refs, emu)
                for k in low:
                    low[k] = min(low[k], row[k])
        report.append(f"{L.name}: " + " ".join(f"{k} {v:.2e}" for k, v in row.items()))
    print("emulated max |err| / S:\n  " + "\n  ".join(report))
    for mode in gl.MODES:
        assert 4 * worst[mode] <= gl.TOL[mode], (mode, worst[mode], gl.TOL[mode])
    assert low["bf16x1 one problem"] >= 10 * gl.TOL["bf16x3"], low
    assert low["bf16x1 vs fp16"] > gl.TOL["fp16"], low
