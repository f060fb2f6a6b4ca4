"""The ConvTranspose of each generator stage (vtts_debug_hifigan_layer layers 1..4) at ragged row lengths, into a
canary-filled buffer with guards before and after it.

The tensor-core modes run it as one conv over blocks of u output rows whose first block starts u/2 rows before a batch
row's output (csrc/hifigan.cu hg_ups), so a stray write lands at the end of the previous batch row or before the buffer.
Nothing outside rows [0, u * n_frames[b] * scale) of each batch row may be written, and every written row matches the
float64 Haiku layer within the bound of tests/test_gpu_generator_layers.py:  |got - ref| <= TOL * S + EPS * |ref|,  S the
root-sum-square of the products.  Lengths: a full row after a short one, a one-frame row, an odd one; T puts the rows of
stages 2 and 3 on a whole number of tiles, so the last block of a full row is a tile of its own."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import hifigan_oracle as ho

TOL = {"fp32": 3e-5, "bf16x3": 2e-4, "fp16": 5.5e-3}
EPS = 2.0 ** -21
SENTINEL = 0x7FC0DEAD
SCALE = [1, 8, 64, 128]
T = 40
LENS = [T, 1, 17, T]


@pytest.fixture(scope="module")
def eng(hifigan_params):
    from viettts_b200.engine import Engine
    e = Engine(0)
    e.load_hifigan(hifigan_params)
    yield e
    e.set_precision("bf16x3")
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["bf16x3", "fp16", "fp32"])
@pytest.mark.parametrize("stage", [0, 1, 2, 3])
def test_upsample_writes_only_valid_rows(eng, hifigan_params, stage, mode):
    dev = torch.device("cuda", 0)
    eng.set_precision(mode)
    u, C = ho.UPSAMPLE_RATES[stage], 512 >> stage
    Co, rows = C // 2, T * SCALE[stage]
    nx = 1 if stage == 0 else 3
    g = torch.Generator(device=dev).manual_seed(100 + stage)
    xs = [torch.randn((len(LENS), rows, C), device=dev, generator=g) for _ in range(nx)]
    for x in xs:
        for b, n in enumerate(LENS):
            x[b, n * SCALE[stage]:] = float("nan")    # rows at or past a row's length must read as zero
    lens_t = torch.tensor(LENS, dtype=torch.int32, device=dev)
    n = len(LENS) * rows * u * Co
    guard = 4 * u * Co
    buf = torch.empty(guard + n + guard, device=dev)
    buf.view(torch.int32).fill_(SENTINEL)
    out = buf[guard:guard + n].view(len(LENS), rows * u, Co)
    eng.debug_hifigan_layer(1 + stage, xs, [out], lens_t, T)

    bits = buf.view(torch.int32)
    assert (bits[:guard] == SENTINEL).all(), "written before the output"
    assert (bits[guard + n:] == SENTINEL).all(), "written after the output"
    p = hifigan_params[f"generator/~/ups_{stage}"]
    w = torch.as_tensor(np.asarray(p["w"]), dtype=torch.float64, device=dev)
    bias = torch.as_tensor(np.asarray(p["b"]), dtype=torch.float64, device=dev)
    for b, nf in enumerate(LENS):
        v_in, v_out = nf * SCALE[stage], nf * SCALE[stage] * u
        assert (out[b, v_out:].view(torch.int32) == SENTINEL).all(), (b, "a row at or past u * valid was written")
        xb = [x[b:b + 1, :v_in].double() for x in xs]
        phi = F.leaky_relu(xb[0] if nx == 1 else (xb[0] + xb[1] + xb[2]) / 3, ho.LRELU_SLOPE)
        ref = ho.conv1d_transpose_nwc(phi, w, bias, u)[0]
        s = ho.conv1d_transpose_nwc(phi * phi, w * w, None, u)[0].clamp_min(0).sqrt()
        err = (out[b, :v_out].double() - ref).abs()
        bound = TOL[mode] * s + EPS * ref.abs()
        assert torch.isfinite(out[b, :v_out]).all(), (b, "non-finite output")
        assert (err <= bound).all(), (b, f"worst |err| / S {float((err / s.clamp_min(1e-30)).max()):.3e} > {TOL[mode]:.0e}")
