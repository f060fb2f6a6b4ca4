"""GPU parity of the tensor-core (bf16x3) arithmetic path.

Layer level: wgmma conv vs float64 torch conv on the same inputs: L-inf <= 2e-4 on O(1) outputs
(bf16x3 split error ~2^-16 relative per product).  Generator level: same tolerances as the strict
fp32 path -- waveform L-inf <= 1e-4, RMS <= 1e-5 against the reference-pinned vectors."""
import numpy as np
import pytest
import torch

from oracle import hifigan_oracle as ho
from viettts_b200 import synthetic

pytestmark = pytest.mark.gpu
WAV_LINF, WAV_RMS = 1e-4, 1e-5
# forms of the fused pair kernel (Engine.set_fused_pairs): 256-row tiles (default), the same with conv2's A operand in
# registers, 128-row tiles
PAIR_KINDS = ["smem2", "tmem", "smem"]


@pytest.fixture(scope="module")
def eng(hifigan_params):
    from viettts_b200.engine import Engine
    e = Engine(0)
    e.load_hifigan(hifigan_params)
    e.set_precision("bf16x3")
    yield e
    e.close()


def _ref_conv(x, w, b, k, dil, slope, resid):
    xt = torch.nn.functional.leaky_relu(torch.from_numpy(x).double(), slope)
    wt = torch.from_numpy(w).double().permute(2, 1, 0).contiguous()
    y = torch.nn.functional.conv1d(xt.transpose(1, 2), wt, torch.from_numpy(b).double(), padding=(k - 1) * dil // 2, dilation=dil)
    return (y.transpose(1, 2) + torch.from_numpy(resid).double()).numpy()


@pytest.mark.parametrize("C", [32, 64, 128, 256])
@pytest.mark.parametrize("k,dil", [(3, 1), (3, 5), (7, 3), (11, 1), (11, 5)])
def test_layer_vs_float64(eng, C, k, dil):
    rng = np.random.default_rng(C * 100 + k * 10 + dil)
    B, T = 2, 600
    x = rng.standard_normal((B, T, C)).astype(np.float32)
    w = (rng.standard_normal((k, C, C)) / np.sqrt(k * C)).astype(np.float32)
    b = (rng.standard_normal(C) * 0.1).astype(np.float32)
    res = rng.standard_normal((B, T, C)).astype(np.float32)
    lens = np.array([T, 257], np.int32)
    dev = torch.device("cuda", 0)
    out = eng.debug_conv1d("bf16x3", torch.from_numpy(x).to(dev), torch.from_numpy(w).to(dev), torch.from_numpy(b).to(dev), k, dil, 0.1,
                           torch.from_numpy(res).to(dev), torch.from_numpy(lens).to(dev)).cpu().numpy()
    for bb in range(B):
        n = lens[bb]
        ref = _ref_conv(x[bb : bb + 1, :n], w, b, k, dil, 0.1, res[bb : bb + 1, :n])
        err = np.abs(out[bb, :n] - ref[0]).max()
        assert err < 2e-4, (C, k, dil, bb, err)


@pytest.mark.parametrize("tag", ["small", "t32"])
def test_generator_bf16x3_golden(eng, golden_dir, tag):
    g = np.load(golden_dir / f"hifigan_ref_{tag}.npz")
    wav = eng.mel2wave(g["mel"])
    err = np.abs(wav - g["wav"])
    rms = float(np.sqrt(np.mean(err**2)))
    print(f"[bf16x3 golden-{tag}] Linf={err.max():.3e} rms={rms:.3e}")
    assert err.max() <= WAV_LINF and rms <= WAV_RMS


def test_generator_bf16x3_ragged_and_config2(eng, hifigan_params):
    mel = synthetic.mel_input(3, 3, 40)
    nf = np.array([40, 23, 1], np.int32)
    wav = eng.mel2wave(mel, n_frames=nf)
    for b in range(3):
        ref = ho.mel2wave(hifigan_params, mel[b : b + 1, : nf[b]]).reshape(-1)
        err = np.abs(wav[b, : nf[b] * 256] - ref)
        assert err.max() <= WAV_LINF and np.sqrt(np.mean(err**2)) <= WAV_RMS
        assert np.all(wav[b, nf[b] * 256 :] == 0.0)
    mel = synthetic.mel_input(0, 1, 400)
    ref = ho.mel2wave(hifigan_params, mel).reshape(1, -1)
    err = np.abs(eng.mel2wave(mel) - ref)
    print(f"[bf16x3 config2] Linf={err.max():.3e} rms={np.sqrt(np.mean(err**2)):.3e}")
    assert err.max() <= WAV_LINF and np.sqrt(np.mean(err**2)) <= WAV_RMS


def test_generator_bf16x3_batch32_rows_independent(eng):
    mel = synthetic.mel_input(11, 32, 312)
    wav = eng.mel2wave(mel)
    assert np.isfinite(wav).all()
    alone = eng.mel2wave(mel[17:18])
    assert np.array_equal(alone[0], wav[17])


def _ref_pair(x, w1, b1, w2, b2, k, dil, slope):
    xt = torch.from_numpy(x).double()
    f = torch.nn.functional
    y = f.leaky_relu(xt, slope).transpose(1, 2)
    y = f.conv1d(y, torch.from_numpy(w1).double().permute(2, 1, 0).contiguous(), torch.from_numpy(b1).double(), padding=(k - 1) * dil // 2, dilation=dil)
    y = f.leaky_relu(y, slope)
    y = f.conv1d(y, torch.from_numpy(w2).double().permute(2, 1, 0).contiguous(), torch.from_numpy(b2).double(), padding=(k - 1) // 2)
    return (y.transpose(1, 2) + xt).numpy()


@pytest.mark.parametrize("ts", PAIR_KINDS)
@pytest.mark.parametrize("C", [32, 64])
@pytest.mark.parametrize("k,dil", [(3, 1), (3, 5), (7, 3), (11, 1), (11, 5)])
def test_fused_pair_vs_float64(eng, C, k, dil, ts):
    """Fused ResBlock pair, every form of tc_pair_kernel: row semantics (zero padding of BOTH convs at each row's true
    end)."""
    eng.set_fused_pairs(False, kind=ts)      # selects which pair kernel the debug hook runs; generator path unchanged
    rng = np.random.default_rng(C * 1000 + k * 10 + dil)
    B, T = 3, 700
    x = rng.standard_normal((B, T, C)).astype(np.float32)
    w1 = (rng.standard_normal((k, C, C)) / np.sqrt(k * C)).astype(np.float32)
    w2 = (rng.standard_normal((k, C, C)) / np.sqrt(k * C)).astype(np.float32)
    b1 = (rng.standard_normal(C) * 0.1).astype(np.float32)
    b2 = (rng.standard_normal(C) * 0.1).astype(np.float32)
    lens = np.array([T, 257, 3], np.int32)
    dev = torch.device("cuda", 0)
    t = lambda a: torch.from_numpy(a).to(dev)  # noqa: E731
    out = eng.debug_pair(t(x), t(w1), t(b1), t(w2), t(b2), k, dil, 0.1, t(lens)).cpu().numpy()
    for bb in range(B):
        n = lens[bb]
        ref = _ref_pair(x[bb : bb + 1, :n], w1, b1, w2, b2, k, dil, 0.1)
        err = np.abs(out[bb, :n] - ref[0]).max()
        assert err < 3e-4, (C, k, dil, bb, err)


@pytest.mark.parametrize("ts", PAIR_KINDS)
def test_fused_and_unfused_generator_agree(eng, hifigan_params, ts):
    mel = synthetic.mel_input(21, 2, 50)
    nf = np.array([50, 31], np.int32)
    eng.set_fused_pairs(True, kind=ts)
    a = eng.mel2wave(mel, n_frames=nf)
    eng.set_fused_pairs(False)
    b = eng.mel2wave(mel, n_frames=nf)
    assert np.abs(a - b).max() < 1e-4


def test_fused_pair_long_rows_many_tiles(eng):
    """More tiles than SMs (the persistent loop wraps, every ring changes phase many times) and a length that ends
    inside a tile; C = 32 and 64 at the generator's own kernel sizes."""
    dev = torch.device("cuda", 0)
    cases = [("smem2", 32, 7, 3), ("smem2", 64, 11, 5), ("smem2", 64, 3, 1), ("tmem", 32, 11, 5), ("tmem", 64, 7, 3),
             ("smem", 32, 3, 1), ("smem", 64, 11, 5)]
    for kind, C, k, dil in cases:
        eng.set_fused_pairs(False, kind=kind)
        rng = np.random.default_rng(C + k)
        B, T = 4, 9000
        x = rng.standard_normal((B, T, C)).astype(np.float32)
        w1 = (rng.standard_normal((k, C, C)) / np.sqrt(k * C)).astype(np.float32)
        w2 = (rng.standard_normal((k, C, C)) / np.sqrt(k * C)).astype(np.float32)
        b1 = (rng.standard_normal(C) * 0.1).astype(np.float32)
        b2 = (rng.standard_normal(C) * 0.1).astype(np.float32)
        lens = np.array([T, 8191, 4097, 130], np.int32)
        t = lambda a: torch.from_numpy(a).to(dev)  # noqa: E731
        out = eng.debug_pair(t(x), t(w1), t(b1), t(w2), t(b2), k, dil, 0.1, t(lens)).cpu().numpy()
        for bb in range(B):
            n = lens[bb]
            ref = _ref_pair(x[bb : bb + 1, :n], w1, b1, w2, b2, k, dil, 0.1)
            assert np.abs(out[bb, :n] - ref[0]).max() < 3e-4, (C, k, dil, bb)
