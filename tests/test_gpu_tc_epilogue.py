"""The plain epilogue of tc_conv_kernel (bias + residual, staged through shared memory) at the row edges it handles.

Each ResBlock step of the four generator stages runs unfused (two tc_conv_kernel launches, conv2 with the residual),
so N = 256 / 128 / 64 / 32 each go through the staged epilogue, in bf16x3 and in fp16.  Row lengths end inside a
64-row block and inside a tile where the stage's rows per mel frame allow it (stage 1 has 64: its rows end on block
edges, inside a tile).  Outputs start as a sentinel with a guard behind them: rows at or past a row's length and the
guard must keep it, and the stored rows must match the strict fp32 path of the same layer."""
import numpy as np
import pytest
import torch

from viettts_b200 import synthetic

pytestmark = pytest.mark.gpu
SENTINEL = 0x7FC0DEAD
SCALE = [8, 64, 128, 256]          # rows per mel frame in stage i
TOL = {"bf16x3": 1e-3, "fp16": 3e-2}   # of the row's largest reference magnitude


@pytest.fixture(scope="module")
def eng():
    from viettts_b200.engine import Engine
    e = Engine(0)
    e.load_hifigan(synthetic.hifigan_params(1234))
    yield e
    e.close()


def _layer(eng, mode, layer, xs, lens_t, T, shape):
    eng.set_precision(mode)
    n = int(np.prod(shape))
    guard = 1024 * shape[2]
    bufs = [torch.empty(n + guard, dtype=torch.float32, device=xs[0].device) for _ in range(3)]
    for b in bufs:
        b.view(torch.int32).fill_(SENTINEL)
    outs = [b[:n].view(shape) for b in bufs]
    eng.debug_hifigan_layer(layer, xs, outs, lens_t, T)
    for b in bufs:
        assert (b[n:].view(torch.int32) == SENTINEL).all(), (mode, layer, "guard written")
    return outs


@pytest.mark.parametrize("mode", ["bf16x3", "fp16"])
@pytest.mark.parametrize("stage", [0, 1, 2, 3])
def test_staged_epilogue_row_edges(eng, mode, stage):
    dev = torch.device("cuda", 0)
    eng.set_fused_pairs(False)
    C = 512 >> (stage + 1)
    T = 7
    lens = np.array([T, 5, 3], np.int32)    # stage 0: 56, 40, 24 rows -- inside a 64-row block and a 128-row tile
    B, rows = len(lens), T * SCALE[stage]
    g = torch.Generator(device=dev).manual_seed(stage)
    xs = [torch.randn((B, rows, C), device=dev, generator=g) for _ in range(3)]
    lens_t = torch.from_numpy(lens).to(dev)
    valid = (torch.arange(rows, device=dev)[None, :] < lens_t[:, None] * SCALE[stage])[..., None].expand(B, rows, C)
    try:
        for m in range(3):
            layer = 5 + 3 * stage + m
            got = _layer(eng, mode, layer, xs, lens_t, T, (B, rows, C))
            ref = _layer(eng, "fp32", layer, xs, lens_t, T, (B, rows, C))
            for j in range(3):
                assert (got[j].view(torch.int32)[~valid] == SENTINEL).all(), (mode, layer, j, "a row at or past its length was written")
                for b in range(B):
                    nb = int(lens[b]) * SCALE[stage]
                    r, o = ref[j][b, :nb], got[j][b, :nb]
                    err = float((o - r).abs().max())
                    assert err <= TOL[mode] * float(r.abs().max()), (mode, layer, j, b, err)
    finally:
        eng.set_fused_pairs(True)
        eng.set_precision("bf16x3")
