"""CPU side of tests/test_gpu_duration_stages.py: where its duration-head bound comes from, what it separates, and the
one frame-count definition.

The head (`duration_head_kernel`, one warp per token) is emulated in fp32 in its own order: lane l holds elements
8l..8l+7 of the hidden row, forms gelu (tanh form) of each and accumulates the eight products with w2 in order by fused
multiply-adds; an xor-shuffle tree over 16, 8, 4, 2, 1 sums the lanes; b2 is added and softplus is fmaxf(s, 0) +
log1pf(expf(-|s|)).  It is fed the float64 oracle's hidden rows of every GPU case, rounded to float32, and compared
with the float64 head of the same rows in HEAD_TOL's unit.  Wrong variants of the head, evaluated in float64, must
exceed the bound by at least 10x; the one that cannot is reported, not loosened away."""
import numpy as np
import pytest
import torch
from scipy.special import erf

from oracle import nat_oracle as no
from test_gpu_duration_stages import (E2E_UNITS, HEAD_TOL, boundary_silence_duration, cases, e2e_ref, enc_ref,
                                      f32_frame_count, head_ref, head_weights, hidden_ref, silence_frames)
from viettts_b200 import synthetic


@pytest.fixture(scope="module")
def ckpt():
    return synthetic.duration_ckpt(1234)


@pytest.fixture(scope="module")
def hidden(ckpt):
    """float32 hidden rows [n,256] of every token of every GPU stage case (each row alone, as on the GPU)"""
    out = []
    for _, rows in cases():
        for e in enc_ref(ckpt, rows):
            out.append(hidden_ref(ckpt, e)[0])
    return np.concatenate(out).astype(np.float32)


def emulate_head(ckpt, y):
    """duration_head_kernel in fp32, in its own order, for y float32 [n,256] -> durations [n]"""
    _, _, w2, b2 = head_weights(ckpt)
    w = w2.numpy().astype(np.float32)
    f = np.float32
    x = y.astype(np.float32)
    g = f(0.5) * x * (f(1) + np.tanh(f(0.7978845608028654) * (x + f(0.044715) * x * x * x)))
    lane = (g[:, 0::8] * w[0::8]).astype(np.float32)                       # [n,32], lane l: element 8l
    for k in range(1, 8):                                                   # fmaf: one rounding per step
        lane = (g[:, k::8].astype(np.float64) * w[k::8] + lane).astype(np.float32)
    for o in (16, 8, 4, 2, 1):
        lane = lane + lane[:, np.arange(32) ^ o]
    s = lane[:, 0] + f(b2)
    return np.maximum(s, f(0)) + np.log1p(np.exp(-np.abs(s)))


def fp32_oracle_head(ckpt, y):
    _, _, w2, b2 = head_weights(ckpt)
    with torch.no_grad():
        g = no.gelu_tanh(torch.from_numpy(y))
        return no.softplus(g @ w2.float() + torch.tensor(b2, dtype=torch.float32)).numpy()


def units(ckpt, y, d):
    ref, unit = head_ref(ckpt, y)
    return np.abs(np.asarray(d, np.float64) - ref) / unit


def test_bound_has_headroom_over_the_emulation(ckpt, hidden):
    emu = units(ckpt, hidden, emulate_head(ckpt, hidden)).max()
    o32 = units(ckpt, hidden, fp32_oracle_head(ckpt, hidden)).max()
    print(f"head over {len(hidden)} tokens: emulation {emu:.2f} units, fp32 oracle {o32:.2f} units, bound {HEAD_TOL}")
    assert 4 * emu <= HEAD_TOL and 4 * o32 <= HEAD_TOL, (emu, o32)


def _gelu_erf(x):
    return 0.5 * x * (1.0 + torch.from_numpy(erf(x.numpy() / np.sqrt(2.0))))


WRONG = {
    "gelu erf form": dict(gelu=_gelu_erf),
    "b2 dropped": dict(bias=False),
    "w2 one lane block off": dict(w2_shift=8),
}


@pytest.mark.parametrize("name", list(WRONG))
def test_wrong_heads_exceed_the_bound_tenfold(ckpt, hidden, name):
    d, _ = head_ref(ckpt, hidden, **WRONG[name])
    worst = units(ckpt, hidden, d).max()
    print(f"{name}: {worst:.3g} units = {worst / HEAD_TOL:.3g} x the bound")
    assert worst >= 10 * HEAD_TOL, (name, worst)


def test_naive_softplus_cannot_be_separated(ckpt, hidden):
    """log(1 + exp(s)) cannot be told from the logaddexp form here.  The durations put s in about [-5.5, -1.8], where
    1 + e^s loses nothing in float64, so the float64 variant equals the definition to rounding.  As an fp32 kernel it
    would round 1 + e^s to float32: that exceeds the bound (the GPU check would catch it), but by less than 10x."""
    d64, _ = head_ref(ckpt, hidden, softplus=lambda s: torch.log(1 + torch.exp(s)))
    assert units(ckpt, hidden, d64).max() < 1e-3
    _, _, w2, b2 = head_weights(ckpt)
    with torch.no_grad():
        s = (no.gelu_tanh(torch.from_numpy(hidden).double()) @ w2 + b2).float()
        d32 = torch.log(1 + torch.exp(s)).numpy()
    worst = units(ckpt, hidden, d32).max()
    print(f"naive softplus in fp32: {worst:.3g} units = {worst / HEAD_TOL:.3g} x the bound")
    assert worst > HEAD_TOL


def test_end_to_end_bound_has_headroom_over_the_fp32_oracle(ckpt):
    """E2E_UNITS (tests/test_gpu_duration.py) against the plain fp32 oracle on that file's rows."""
    rows = [np.asarray(synthetic.utterance(s, n, None)[0], np.int32) for s, n in ((0, 100), (10, 57), (12, 23), (7, 14))]
    worst = 0.0
    for tk in rows + [np.zeros(10, np.int32)]:
        ref, unit = e2e_ref(ckpt, tk[None], np.array([len(tk)]))
        got = no.duration_model(ckpt, tk[None], np.array([len(tk)]), dtype=torch.float32)
        worst = max(worst, float((np.abs(got - ref) / unit).max()))
    print(f"end to end, fp32 oracle: {worst:.2f} units, bound {E2E_UNITS}")
    assert 4 * worst <= E2E_UNITS["fp32"] <= E2E_UNITS["bf16x3"] / 10


# ------------------------------------------------------------------------------------------------ frame count


def test_frame_count_definition():
    """sum in float64, round to float32 once, truncate: 111 tokens of fp32(0.36281073) s sum to 2516.99944 frames (a
    float32 sum gives 2517.0002), so the count is 2516."""
    from viettts_b200.nat import text2mel as t2m
    fr, n = no.seconds_to_frames(np.full((1, 111), 0.36281073, np.float32))
    assert abs(float(np.sum(fr, dtype=np.float64)) - 2516.99944) < 1e-4 and f32_frame_count(fr) == 2517
    assert n == 2516 and t2m.seconds_to_frames(np.full((1, 111), 0.36281073, np.float32))[1] == 2516
    assert no.frame_count([]) == 0 and no.frame_count([0.5, 0.25]) == 0 and no.frame_count([0.75, 0.25]) == 1


@pytest.mark.parametrize("seed", range(3))
def test_python_sites_agree_on_boundary_rows(seed):
    """Rows built as the GPU test builds its boundary row (silence predictions below the search range, silence_duration
    bisected to where the float64 sum crosses an integer, then stepped by ulps until the float32 count differs): the
    oracle, the drop-in text2mel's seconds_to_frames and predict_mel's default n_frames give one count."""
    from viettts_b200.engine import Engine
    from viettts_b200.nat import text2mel as t2m
    rng = np.random.default_rng(seed)
    raw = rng.uniform(0.01, 0.29, 111).astype(np.float32)
    sd = boundary_silence_duration(raw, 0.3, 0.32)
    fr = silence_frames(raw, sd)
    n = no.frame_count(fr)
    assert f32_frame_count(fr) != n, "the row must separate the two definitions"
    d = no.adjust_durations(np.zeros(111, np.int32), raw[None], sd)
    assert no.seconds_to_frames(d)[1] == n
    assert t2m.seconds_to_frames(t2m.adjust_durations([0] * 111, raw[None], float(sd)))[1] == n
    assert t2m.frame_count(fr) == n
    eng = Engine.__new__(Engine)                                           # _acoustic_args does not touch the device
    for lens in (None, [111]):
        nf = eng._acoustic_args(np.zeros((1, 111), np.int32), fr[None], lens, None, None, None)[3]
        assert nf.tolist() == [n]
