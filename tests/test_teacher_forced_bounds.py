"""CPU companion of tests/test_gpu_teacher_forced_stages.py: where its per-stage bounds come from, and what they catch.

Headroom: the bound of a stage must sit at least 4x above what plain fp32 arithmetic already costs on the same cases:
the fp32 oracle of the stage, fed the float64 input of the stage, against the float64 oracle, on every case the GPU
file compares with float64.  The stage bounds must also be tighter than the end-to-end mel check they replace.

Mutations: each wrong wiring of the pass, made in float64, must move its stage by at least 10x that stage's bound on
a case the GPU file runs, so a kernel with that mistake cannot pass."""
import numpy as np
import pytest
import torch

from helpers.threefry import zoneout_masks
from oracle import mel_oracle
from oracle import nat_oracle as no
from test_gpu_acoustic_scans import F64, LONG_CHECKED, MEL_LINF, N_MAX, SEED, cond_of, enc64, matrix_rows, postnet_rows
from test_gpu_teacher_forced_stages import (BOUND, DROPOUT, GTA_B, GTA_L, GTA_N, P2_TOL, SIZES, gta_case, gta_frames, l300_tf,
                                            long_tf, matrix_mels, p2_scale, plane_masks, short_rows, tf_masks)
from viettts_b200 import synthetic

F32 = torch.float32


def dec_in64(ckpt, rows, mels_in, keep, encs=None):
    """the float64 decoder input [cond | p2] of a batch ([B,N,768]; cond 0 past each row's n_frames)"""
    N = mels_in.shape[1]
    x = torch.zeros(len(rows), N, 768, dtype=F64)
    for b, (tk, d, n) in enumerate(rows):
        x[b, :n, :512] = cond_of(enc64(ckpt, tk) if encs is None else encs[b], d, n)
    x[:, :, 512:] = no.tf_prenet(ckpt["params"], mels_in, keep, F64)
    return x


def _linf(a, b, rows):
    return max(float((a[i, :n].double() - b[i, :n].double()).abs().max()) for i, (_, _, n) in enumerate(rows))


def emulate(ckpt, rows, x, zone):
    """worst fp32-vs-float64 error of dec_out, mel_pre and mel2, each stage fed its float64 input"""
    P = ckpt["params"]
    h64 = no.zoneout_decode(P, x, zone, F64)
    m64 = no.project(P, h64, F64)
    ns = [r[2] for r in rows]
    return dict(dec_out=_linf(no.zoneout_decode(P, x.float(), zone, F32), h64, rows),
                mel_pre=_linf(no.project(P, h64.float(), F32), m64, rows),
                mel2=max(float((a.double() - b).abs().max())
                         for a, b in zip(postnet_rows(ckpt, m64.float(), ns), postnet_rows(ckpt, m64, ns))))


def _cases(ckpt):
    """(name, rows, float64 decoder input, zone masks) of every case of the GPU file"""
    rows = matrix_rows()
    mels = matrix_mels()
    encs = [enc64(ckpt, r[0]) for r in rows]
    for dmode in DROPOUT:
        for B in (SIZES if dmode == "reference" else [128]):        # only the REFERENCE draws depend on B
            keep, zone = tf_masks(dmode, B, N_MAX)
            yield f"B={B} {dmode}", rows[:B], dec_in64(ckpt, rows[:B], mels[:B], keep, encs), zone
    for n in (1, 2, 3):
        r = short_rows(n)
        mels_n = synthetic.mel_input(50 + n, 40, n)                   # as test_short_sequences
        for dmode in DROPOUT:
            keep, zone = tf_masks(dmode, 40, n)
            yield f"N={n} {dmode}", r, dec_in64(ckpt, r, mels_n, keep), zone
    for which in range(4):
        keep, zone = plane_masks(which)
        yield f"plane {which}", rows[:40], dec_in64(ckpt, rows[:40], mels[:40], keep, encs), zone
    r, mels_l, keep, zone = l300_tf()
    yield "B=8 L=300", r, dec_in64(ckpt, r, mels_l, keep), zone
    r, mels_l, keep, zone = long_tf()
    idx = LONG_CHECKED
    r = [r[b] for b in idx]
    P, S = ckpt["params"], ckpt["aux"]
    with torch.no_grad():
        enc = no.token_encoder(P, S, np.stack([t[0] for t in r]), [100] * len(r), F64)
    yield "B=128 N=312", r, dec_in64(ckpt, r, mels_l[idx], keep[idx], list(enc)), zone[idx]
    wav, tok, dur_sec, _, nfs = gta_case()
    gt = mel_oracle.mel_filter(wav.astype(np.float32) / np.float32(2 ** 15))
    inp = np.concatenate([np.zeros_like(gt[:, :1]), gt[:, :-1]], axis=1)
    frames = gta_frames(dur_sec)
    r = [(tok[b], frames[b], int(nfs[b])) for b in range(GTA_B)]
    keep, zone = tf_masks("seed", GTA_B, GTA_N)
    assert tok.shape[1] == GTA_L
    yield "gta", r, dec_in64(ckpt, r, inp, keep), zone


def test_bounds_have_headroom_over_the_fp32_emulation(acoustic_ckpt):
    worst = dict(dec_out=0.0, mel_pre=0.0, mel2=0.0)
    for name, rows, x, zone in _cases(acoustic_ckpt):
        w = emulate(acoustic_ckpt, rows, x, zone)
        print(f"fp32 emulation {name}: " + " ".join(f"{k} {v:.2e}" for k, v in w.items()))
        worst = {k: max(worst[k], w[k]) for k in worst}
    print("fp32 emulation, worst: " + " ".join(f"{k} {v:.2e}" for k, v in worst.items()))
    for mode, bound in BOUND.items():
        for stage, emu in worst.items():
            assert 4 * emu <= bound[stage], (mode, stage, emu, bound[stage])
        assert bound["dec_out"] <= MEL_LINF / 4 and bound["mel_pre"] <= MEL_LINF / 4, bound


# ------------------------------------------------------------------------------------------------ mutations


def _decode_rewired(P, x, zone, mut):
    """zoneout_decode with one wiring mistake: LSTM1 fed the zoned h0 ("lstm1_zoned_h0"), or the decoder output taken
    after zoneout ("out_after_zoneout")"""
    w0, b0 = no._t(P[no.A + "lstm/linear"]["w"], F64), no._t(P[no.A + "lstm/linear"]["b"], F64)
    w1, b1 = no._t(P[no.A + "lstm_1/linear"]["w"], F64), no._t(P[no.A + "lstm_1/linear"]["b"], F64)
    B, N, _ = x.shape
    h0, c0, h1, c1 = (x.new_zeros(B, 512) for _ in range(4))
    zm = torch.as_tensor(zone).bool()
    outs = []
    for t in range(N):
        nh0, nc0 = no.lstm_step(x[:, t], h0, c0, w0, b0)
        zh0 = torch.where(zm[:, t, 0], h0, nh0)
        nh1, nc1 = no.lstm_step(torch.cat([x[:, t], zh0 if mut == "lstm1_zoned_h0" else nh0], dim=-1), h1, c1, w1, b1)
        zh1 = torch.where(zm[:, t, 2], h1, nh1)
        outs.append(torch.cat([zh0, zh1] if mut == "out_after_zoneout" else [nh0, nh1], dim=-1))
        h0, c0, h1, c1 = zh0, torch.where(zm[:, t, 1], c0, nc0), zh1, torch.where(zm[:, t, 3], c1, nc1)
    return torch.stack(outs, 1)


@pytest.fixture(scope="module")
def seed_case(acoustic_ckpt):
    """the B = 40 SEED case of the launch-edge matrix (two zoneout launches): rows, mels_in, keep, zone, float64
    decoder input and decoder output"""
    rows = matrix_rows()[:40]
    mels = matrix_mels()[:40]
    keep, zone = tf_masks("seed", 40, N_MAX)
    x = dec_in64(acoustic_ckpt, rows, mels, keep)
    with torch.no_grad():
        return rows, mels, keep, zone, x, no.zoneout_decode(acoustic_ckpt["params"], x, zone, F64)


def _zone_mutant(zone, mut, rows):
    z = np.array(zone)
    if mut == "swap_h_c":
        return z[:, :, [1, 0, 3, 2]]
    if mut == "swap_layers":
        return z[:, :, [2, 3, 0, 1]]
    if mut == "frame_late":
        z[:, 1:] = zone[:, :-1]
        z[:, 0] = 0
        return z
    if mut == "polarity_h0":
        z[:, :, 0] = 1 - z[:, :, 0]
        return z
    assert mut == "seed_launch_row"          # rows 32+ keyed by their row inside the zoneout launch
    return zoneout_masks(SEED, [b % 32 for b in range(len(rows))], zone.shape[1])


@pytest.mark.parametrize("mut", ["lstm1_zoned_h0", "out_after_zoneout", "swap_h_c", "swap_layers", "frame_late", "polarity_h0",
                                 "seed_launch_row"])
def test_decoder_mutations_exceed_the_bound(acoustic_ckpt, seed_case, mut):
    rows, _, _, zone, x, h = seed_case
    P = acoustic_ckpt["params"]
    with torch.no_grad():
        if mut in ("lstm1_zoned_h0", "out_after_zoneout"):
            hm = _decode_rewired(P, x, zone, mut)
        else:
            hm = no.zoneout_decode(P, x, _zone_mutant(zone, mut, rows), F64)
    lo = 32 if mut == "seed_launch_row" else 0
    err = _linf(hm[lo:], h[lo:], rows[lo:])
    bound = max(b["dec_out"] for b in BOUND.values())
    print(f"mutation {mut}: dec_out {err:.2e} = {err / bound:.0f} x the bound")
    assert err >= 10 * bound, (mut, err, bound)


def test_prenet_keep_scale_mutation_exceeds_the_bound(acoustic_ckpt, seed_case):
    """keep scale 1 instead of 1 / 0.5 in both prenet dropouts"""
    _, mels, keep, _, x, _ = seed_case
    P = acoustic_ckpt["params"]
    with torch.no_grad():
        km = torch.as_tensor(keep).double()
        a = km[:, :, 0] * torch.relu(torch.as_tensor(mels).double() @ no._t(P[no.A + "linear_1"]["w"], F64))
        pm = km[:, :, 1] * torch.relu(a @ no._t(P[no.A + "linear_2"]["w"], F64))
        s = p2_scale(P, mels, keep)
    ratio = float(((pm - x[:, :, 512:]).abs() / (max(P2_TOL.values()) * s).clamp_min(1e-300)).max())
    print(f"mutation keep scale 1: p2 {ratio:.0f} x the bound")
    assert ratio >= 10
