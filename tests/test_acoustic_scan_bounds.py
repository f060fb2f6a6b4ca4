"""CPU companion of tests/test_gpu_acoustic_scans.py: where its per-stage bounds come from, and the numpy restatement of
the device's SEED streams that it and the other GPU tests feed to the oracle.

The bound of a stage must sit at least 4x above what plain fp32 arithmetic already costs on the same utterances and
masks: the fp32 oracle of the stage, fed the float64 input of the stage, against the float64 oracle.  The matrix
batch (its 128 rows, in every dropout mode), the long B = 128 batch, the L = 300 batch and the L = 1400 row are
emulated, i.e. every row and mask set the GPU test compares."""
import numpy as np
import torch

from helpers import threefry
from test_gpu_acoustic_scans import (BOUND, DROPOUT, F64, LONG_CHECKED, MEL_LINF, N_MAX, SEED, _durations, cond_of, decode,
                                     enc64, keep_masks, l300_masks, l300_rows, long_masks, long_rows, matrix_rows)
from viettts_b200 import jaxrng, synthetic

F32 = torch.float32


def _linf(a, b):
    return float((a.double() - b.double()).abs().max())


def _emulate(ckpt, rows, masks_of):
    """worst fp32-vs-float64 error of each stage over the rows [(tokens, durations, n)], decoded as one batch per
    entry of masks_of (a list of keep-mask sets [B,N,2,256] or None)"""
    worst = dict(enc=0.0, cond=0.0, mel_pre=0.0)
    N = max(r[2] for r in rows)
    conds = torch.zeros(len(rows), N, 512, dtype=F64)
    for b, (tk, d, n) in enumerate(rows):
        e64 = enc64(ckpt, tk)
        worst["enc"] = max(worst["enc"], _linf(enc64(ckpt, tk, F32), e64))
        conds[b, :n] = cond_of(e64, d, n)
        worst["cond"] = max(worst["cond"], _linf(cond_of(e64, d, n, F32), conds[b, :n]))
    for masks in masks_of:
        p32, p64 = decode(ckpt, conds.float(), masks, F32), decode(ckpt, conds, masks)
        for b, (_, _, n) in enumerate(rows):
            worst["mel_pre"] = max(worst["mel_pre"], _linf(p32[b, :n], p64[b, :n]))
    return worst


def test_bounds_have_headroom_over_the_fp32_emulation(acoustic_ckpt):
    cases = {
        "matrix": _emulate(acoustic_ckpt, matrix_rows(), [keep_masks(m, 128, N_MAX) for m in DROPOUT]),
        "B=128 L=100 N=312": _emulate(acoustic_ckpt, [long_rows()[b] for b in LONG_CHECKED], [long_masks()[LONG_CHECKED]]),
    }
    rows = l300_rows()
    cases["B=8 L=300"] = _emulate(acoustic_ckpt, rows, [l300_masks(max(r[2] for r in rows))])
    rng = np.random.default_rng(1400)                    # the L = 1400 row of test_upsample_beyond_48k_shared_memory
    L, n = 1400, 280
    row = (rng.integers(0, 90, L).astype(np.int32), _durations(rng, L, n), n)
    cases["B=1 L=1400"] = _emulate(acoustic_ckpt, [row], [synthetic.dropout_masks(14, 1, n)])
    for name, w in cases.items():
        print(f"fp32 emulation {name}: " + " ".join(f"{k} {v:.2e}" for k, v in w.items()))
    for stage in ("enc", "cond", "mel_pre"):
        emu = max(w[stage] for w in cases.values())
        for mode, bound in BOUND.items():
            assert 4 * emu <= bound[stage], (stage, mode, emu, bound[stage])
    for bound in BOUND.values():
        assert bound["cond"] <= MEL_LINF / 10 and bound["mel_pre"] <= MEL_LINF / 4, bound


def test_threefry_helper_equals_jaxrng():
    """The tests' restatement of the device generator equals viettts_b200.jaxrng.threefry2x32, which
    tests/test_refshim_rng.py pins to the Random123 known answers."""
    rng = np.random.default_rng(0)
    for _ in range(4):
        k0, k1 = (int(v) for v in rng.integers(0, 2 ** 32, 2, dtype=np.uint64))
        c0, c1 = rng.integers(0, 2 ** 32, (2, 1000), dtype=np.uint64).astype(np.uint32)
        a = threefry.threefry2x32(k0, k1, c0, c1)
        b = jaxrng.threefry2x32(k0, k1, c0, c1)
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
    # Random123 known answer (20 rounds, key and counter all ones)
    o = threefry.threefry2x32(0xFFFFFFFF, 0xFFFFFFFF, np.uint32(0xFFFFFFFF), np.uint32(0xFFFFFFFF))
    assert (int(o[0]), int(o[1])) == (0x1CB996FC, 0xBB002BE7)


def test_seed_masks_follow_the_documented_counters():
    """prenet_keep_masks / zoneout_masks element by element against the counter words written out one at a time:
    prenet (frame, row << 12 | layer * 256 + unit) kept when o0 < 2^31; zoneout (frame, row << 12 | 512 + which * 512 +
    unit) kept when o0 < 429496730; keyed by the seed's low and high words."""
    rows, n = [0, 1, 31, 32, 127], 5
    keep = threefry.prenet_keep_masks(SEED, rows, n)
    zone = threefry.zoneout_masks(SEED, rows, n)
    assert keep.shape == (5, n, 2, 256) and zone.shape == (5, n, 4, 512)
    k0, k1 = SEED & 0xFFFFFFFF, SEED >> 32
    rng = np.random.default_rng(1)
    for _ in range(200):
        i, t = int(rng.integers(5)), int(rng.integers(n))
        layer, unit = int(rng.integers(2)), int(rng.integers(256))
        o0, _ = jaxrng.threefry2x32(k0, k1, np.uint32(t), np.uint32((rows[i] << 12) | (layer * 256 + unit)))
        assert keep[i, t, layer, unit] == (int(o0) < 2 ** 31)
        which, unit = int(rng.integers(4)), int(rng.integers(512))
        o0, _ = jaxrng.threefry2x32(k0, k1, np.uint32(t), np.uint32((rows[i] << 12) | (512 + which * 512 + unit)))
        assert zone[i, t, which, unit] == (int(o0) < 429496730)
    big = threefry.zoneout_masks(SEED, range(64), 20)
    assert 0.09 < big.mean() < 0.11 and 0.48 < threefry.prenet_keep_masks(SEED, range(64), 20).mean() < 0.52
    assert not np.array_equal(big[0], big[32])
