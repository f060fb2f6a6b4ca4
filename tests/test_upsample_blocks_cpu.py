"""The tensor-core ConvTranspose of the generator runs as one dense two-tap conv over blocks of u output rows
(csrc/hifigan.cu hg_ups).  This restates that form in float64 numpy, with the weights stacked the way
vtts_hifigan_prepare stacks them and the row bounds of the kernel's sub-row epilogue, and checks that it is the oracle's
ConvTranspose (hk.Conv1DTranspose "SAME"), for both shapes of the model: (u, K) = (8, 16) and (2, 4).  No GPU needed.

Block s covers output rows u*s - u/2 .. u*s + u/2 - 1 and reads input rows s - 1 and s; blocks s = 0..T.  Output row o
of a row with `valid` input rows is written iff 0 <= o < u * valid; rows of the first block before 0 (the end of the
previous batch row in memory) are never written."""
import numpy as np
import pytest
import torch

from oracle import hifigan_oracle as ho


def phase_weights(w, u):
    """w [K][Cout][Cin] -> per phase r: the input shift e_r and [2][Cin][Cout] (hifigan.cu repack_ups_kernel)"""
    K = w.shape[0]
    a = (K + u - 1) // 2
    out = []
    for r in range(u):
        j0 = (a - r) % u
        e = (r + j0 - a) // u
        assert (r + j0 - a) % u == 0
        out.append((e, np.stack([w[j0 + q * u].T for q in range(2)])))
    return out


def block_weights(w, u):
    """the stacked weights [2][Cin][u * Cout]: column block m is phase (m + u/2) mod u"""
    ph = phase_weights(w, u)
    return np.concatenate([ph[(m + u // 2) % u][1] for m in range(u)], axis=2)


def block_conv(x, w, b, u, valid, canary):
    """the block form over [B][T][Cin] with per-row valid input rows, into a [B][u*T][Cout] buffer of `canary` that is
    seen as [B*T][u*Cout] floats: the flat element offset of block s of row b is (b*T + s) * u*Cout - (u/2)*Cout"""
    B, T, Cin = x.shape
    Co = w.shape[1]
    wb = block_weights(w, u)
    bb = np.tile(b, u)
    flat = np.full(B * T * u * Co, canary)
    for bi in range(B):
        xs = np.zeros((T + 2, Cin))
        xs[1:valid[bi] + 1] = x[bi, :valid[bi]]               # xs[s] = x[s - 1], zero outside [0, valid)
        for s in range(T + 1):
            y = bb + xs[s] @ wb[0] + xs[s + 1] @ wb[1]
            for m in range(u):
                o = u * s - u // 2 + m                        # output row of column block m
                if 0 <= o < u * valid[bi]:
                    e = (bi * T + s) * u * Co - (u // 2) * Co + m * Co
                    flat[e:e + Co] = y[m * Co:(m + 1) * Co]
    return flat.reshape(B, u * T, Co)


def oracle(x, w, b, u, valid):
    xm = x.copy()
    for bi, n in enumerate(valid):
        xm[bi, n:] = 0.0
    y = ho.conv1d_transpose_nwc(torch.from_numpy(xm), torch.from_numpy(w), torch.from_numpy(b), u).numpy()
    return y


@pytest.mark.parametrize("u,K", [(8, 16), (2, 4)])
def test_phase_shifts(u, K):
    """phase r reads x[tau - 1 + q] for r < u/2 and x[tau + q] for r >= u/2: each block reads exactly two input rows"""
    w = np.zeros((K, 1, 1))
    assert [e for e, _ in phase_weights(w, u)] == [-1] * (u // 2) + [0] * (u // 2)


@pytest.mark.parametrize("u,K", [(8, 16), (2, 4)])
@pytest.mark.parametrize("T,valid", [(1, [1]), (5, [5, 3, 1, 4]), (6, [6, 1, 2, 5, 6])])
def test_block_form_is_the_conv_transpose(u, K, T, valid):
    """every output row below u * valid equals the oracle's; nothing else of the buffer is written (T = 1 has a single
    input row; valid < T ends the written rows in the middle of block `valid`)"""
    rng = np.random.default_rng(u * 100 + T)
    B, Cin, Co = len(valid), 12, 8
    x = rng.standard_normal((B, T, Cin))
    w = rng.standard_normal((K, Co, Cin))
    b = rng.standard_normal(Co)
    got = block_conv(x, w, b, u, valid, np.nan)
    ref = oracle(x, w, b, u, valid)
    for bi, n in enumerate(valid):
        np.testing.assert_allclose(got[bi, :u * n], ref[bi, :u * n], rtol=1e-12, atol=1e-12)
        assert np.isnan(got[bi, u * n:]).all(), (bi, n, "a row at or past u * valid was written")


@pytest.mark.parametrize("u,K", [(8, 16), (2, 4)])
def test_block_terms_in_phase_order(u, K):
    """a block column sums the same products in the same order as its phase: tap 0 is the phase's tap 0, so the
    tensor-core kernel's chunk-major, tap-0-then-1 accumulation is unchanged by the block form"""
    rng = np.random.default_rng(7)
    w = rng.standard_normal((K, 4, 3))
    ph = phase_weights(w, u)
    wb = block_weights(w, u)
    for m in range(u):
        r = (m + u // 2) % u
        np.testing.assert_array_equal(wb[:, :, m * 4:(m + 1) * 4], ph[r][1])
