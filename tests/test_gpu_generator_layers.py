"""Every launch of the HiFiGAN generator, one layer at a time, against a float64 Haiku layer, in all three arithmetic modes
and every form of the fused ResBlock pair.

The hook vtts_debug_hifigan_layer runs exactly one of the functions vtts_hifigan_run calls in order (conv_pre, the
ConvTranspose of stage i, ResBlock step m of stage i, conv_post) on caller buffers, with the loaded model's packed weights
and the context's mode and pair setting; test_layers_compose_to_the_forward checks that composing them is the forward.
So these tests reach what the waveform bounds let through: one problem, one output phase or one tile edge of one launch.

Reference: float64 on the checkpoint's own tensors through oracle/hifigan_oracle.py (conv1d_nwc, conv1d_transpose_nwc),
with zero padding at each row's true end.  Tolerance, per element, scale-free: with phi the layer's input activation
(identity, lrelu, or the 3-way mean then lrelu) and
    S = sqrt(conv(phi^2, w^2))      (the transposed conv for a ConvTranspose)
the root-sum-square of the layer's products, and E = |resid| + |ref| what the fp32 epilogue adds and rounds,
    |got - ref| <= TOL[mode] * S + EPS * E.
A ResBlock step carries conv1's bound through conv2 the same way (lrelu is 1-Lipschitz):
    S = S2 + sqrt(conv(S1^2, w2^2)).
conv_post is strict fp32 in every mode; it is bounded before its tanh (1-Lipschitz).
Operand rounding errors are independent per product, so a layer's error grows like S, whatever the layer's fan-in (k x
Cin = 14 .. 2816 here); the sum of |products| grows like the fan-in itself, and carried through |w2| it would loosen the
ResBlock bound by another factor of sqrt(fan-in), so that one TOL per mode could not both hold over bf16x3 and catch a
dropped bf16 lo plane (tests/test_generator_layer_bounds.py derives TOL from a CPU emulation of every mode)."""
import zlib
from collections import namedtuple

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import hifigan_oracle as ho
from viettts_b200 import synthetic

MODES = ("fp32", "bf16x3", "fp16")
TOL = {"fp32": 3e-5, "bf16x3": 2e-4, "fp16": 5.5e-3}
EPS = 2.0 ** -21                  # 8 fp32 ulps of each term the epilogue adds
SENTINEL = 0x7FC0DEAD             # NaN with a payload: the bits of every output element a layer must not write
WRAP_TILES = 4 * 132              # tensor-core tiles of a launch several times the SM count of an H100 SXM
SCALE = [1, 8, 64, 128, 256]      # rows per mel frame entering stage i (i = 4: conv_post)
G = "generator/~/"
BASE_T = 24                       # mel frames of the base case of every layer, also emulated on the CPU
RAGGED = [1, 2, 3, 4, 5, 7, 8, 9, 15, 16, 17, 31, 32, 33, 127, 128, 129]   # frames: a row end on, before and after every tile edge
DEFAULT_PAIRS = "smem2"

# one entry per layer id of vtts_debug_hifigan_layer: 0 conv_pre, 1 + i ConvTranspose of stage i, 5 + 3i + m ResBlock
# step (i, m), 17 conv_post.  nx / nout: buffers in and out; scale_in / scale_out: rows per mel frame.
Layer = namedtuple("Layer", "id name kind stage step cin cout nx nout scale_in scale_out")


def _layer(n):
    if n == 0:
        return Layer(0, "conv_pre", "pre", -1, -1, 80, 512, 1, 1, 1, 1)
    if n <= 4:
        i = n - 1
        C = 512 >> i
        return Layer(n, f"ups{i}", "ups", i, -1, C, C // 2, 1 if i == 0 else 3, 1, SCALE[i], SCALE[i + 1])
    if n <= 16:
        i, m = divmod(n - 5, 3)
        C = 512 >> (i + 1)
        return Layer(n, f"rb{i}.{m}", "rb", i, m, C, C, 3, 3, SCALE[i + 1], SCALE[i + 1])
    return Layer(17, "conv_post", "post", 4, -1, 32, 1, 3, 1, 256, 256)


LAYERS = [_layer(n) for n in range(18)]
FORWARD_ORDER = [0] + [n for i in range(4) for n in [1 + i] + [5 + 3 * i + m for m in range(3)]] + [17]


def configs(L):
    """(mode, pair form) of every run of layer L: the three modes with the default pair form; at the fused stages (C <= 64)
    also unfused, tmem and smem in bf16x3 and unfused in fp16 (fp16 operands exist for the default form only)"""
    out = [(m, DEFAULT_PAIRS) for m in MODES]
    if L.kind == "rb" and L.cin <= 64:
        out += [("bf16x3", "unfused"), ("bf16x3", "tmem"), ("bf16x3", "smem"), ("fp16", "unfused")]
    return out


def tc_rows(n):
    """rows per tensor-core conv tile: 64 x MW rows per consumer warpgroup, two warpgroups (csrc/tc_conv.cu launch_n)"""
    return 128 * (1 if n >= 256 else 2 if n == 128 else 4)


def launch_tiles(L, mode, pairs, B, T):
    """tiles of every tensor-core launch of one hook call (tc_conv.cu launch_cfg / launch_pair); [] on the FP32 path"""
    if mode == "fp32" or L.kind == "post":
        return []
    if L.kind == "pre":
        return [2 * B * -(-T // tc_rows(256))]                       # two N = 256 problems
    if L.kind == "ups":
        u = ho.UPSAMPLE_RATES[L.stage]
        return [u * B * -(-(T * L.scale_in) // tc_rows(L.cout))]     # u phases, in u / nph problems of nph phases
    rows = T * L.scale_out
    if L.cin <= 64 and pairs != "unfused":
        return [3 * B * -(-rows // ((128 if pairs == "smem" else 256) - 16))]   # pair tiles store R - 16 rows
    return [3 * B * -(-rows // tc_rows(L.cout))] * 2


def launches(L, mode, pairs):
    if mode == "fp32":
        return 2 if L.kind == "rb" else 1
    return max(1, len(launch_tiles(L, mode, pairs, 1, 1)))


def layer_seed(L, what):
    return zlib.crc32(f"{L.name}/{what}".encode())


# ------------------------------------------------------------------------------------------------ float64 reference


def _f64(a, dev):
    return torch.as_tensor(np.asarray(a), dtype=torch.float64, device=dev)


def valid_rows(B, rows, lens, scale, dev):
    """[B, rows, 1] mask of the rows below n_frames[b] * scale"""
    if lens is None:
        return torch.ones(B, rows, 1, dtype=torch.bool, device=dev)
    n = torch.as_tensor(np.asarray(lens), device=dev)[:, None] * scale
    return (torch.arange(rows, device=dev)[None, :] < n)[..., None]


def exact_conv(x, w, b, dil=1, pad=None, stride=None):
    """the float64 Haiku layer: hk.Conv1D (w [k,Cin,Cout]) or, with `stride`, hk.Conv1DTranspose (w [K,Cout,Cin])"""
    if stride is None:
        return ho.conv1d_nwc(x, w, b, dilation=dil, pad=pad)
    return ho.conv1d_transpose_nwc(x, w, b, stride)


def rss(x, w, dil=1, pad=None, stride=None):
    """S: the root-sum-square of the products of every output element"""
    return exact_conv(x * x, w * w, None, dil, pad, stride).clamp_min(0).sqrt()


def reference(L, params, xs, lens, dev, conv=exact_conv):
    """float64 layer L on inputs xs (rows at or past a row's length read as zero): one (ref, S, E) per output.
    `conv` computes every conv of the layer (the CPU tests pass emulations of the kernels' arithmetic)."""
    B, rows_in = xs[0].shape[:2]
    vin = valid_rows(B, rows_in, lens, L.scale_in, dev)
    xs = [torch.where(vin, torch.as_tensor(x, device=dev).double(), 0.0) for x in xs]
    if L.kind == "pre":
        p = params[G + "conv1_d"]
        w, b = _f64(p["w"], dev), _f64(p["b"], dev)
        y = conv(xs[0], w, b, pad=3)
        return [(y, rss(xs[0], w, pad=3), y.abs())]
    if L.kind == "ups":
        p = params[G + f"ups_{L.stage}"]
        w, b = _f64(p["w"], dev), _f64(p["b"], dev)
        phi = F.leaky_relu(xs[0] if L.nx == 1 else (xs[0] + xs[1] + xs[2]) / 3, ho.LRELU_SLOPE)
        u = ho.UPSAMPLE_RATES[L.stage]
        y = conv(phi, w, b, stride=u)
        return [(y, rss(phi, w, stride=u), y.abs())]
    if L.kind == "post":
        p = params[G + "conv1_d_1"]
        w, b = _f64(p["w"], dev), _f64(p["b"], dev)
        phi = F.leaky_relu((xs[0] + xs[1] + xs[2]) / 3, 0.01)
        y = conv(phi, w, b, pad=3)
        return [(y[..., 0], rss(phi, w, pad=3)[..., 0], torch.tanh(y[..., 0]).abs())]
    out = []
    vout = valid_rows(B, rows_in, lens, L.scale_out, dev)
    d = ho.RB_DILATIONS[L.step]
    for j in range(3):
        pre = G + f"res_block1_{3 * L.stage + j}/~/"
        c1, c2 = params[pre + f"convs1_{L.step}"], params[pre + f"convs2_{L.step}"]
        w1, b1, w2, b2 = (_f64(c1["w"], dev), _f64(c1["b"], dev), _f64(c2["w"], dev), _f64(c2["b"], dev))
        a1 = F.leaky_relu(xs[j], ho.LRELU_SLOPE)
        t = torch.where(vout, conv(a1, w1, b1, dil=d), 0.0)        # conv2 reads zeros past the row's end
        s1 = torch.where(vout, rss(a1, w1, dil=d), 0.0)
        a2 = F.leaky_relu(t, ho.LRELU_SLOPE)
        y = conv(a2, w2, b2) + xs[j]
        s = rss(a2, w2) + rss(s1, w2)
        out.append((y, s, xs[j].abs() + y.abs()))
    return out


def random_inputs(L, B, T, seed, lens=None):
    """float32 [B, T * scale_in, Cin] inputs of unit scale (the mel: the synthetic mel's -5 +- 2), NaN at and past a row's
    length"""
    rng = np.random.default_rng(seed)
    rows = T * L.scale_in
    if L.kind == "pre":
        xs = [synthetic.mel_input(seed, B, T)]
    else:
        xs = [rng.standard_normal((B, rows, L.cin), dtype=np.float32) for _ in range(L.nx)]
    if lens is not None:
        for x in xs:
            for b, n in enumerate(lens):
                x[b, n * L.scale_in:] = np.nan
    return xs


def oracle_inputs(L, taps):
    """the layer's own float64 input from the oracle run of a synthetic mel, cast to fp32"""
    if L.kind == "pre":
        return [taps["mel"]]
    if L.kind == "ups":
        if L.stage == 0:
            return [taps["pre"].float().numpy()]
        return [taps[f"rb_{L.stage - 1}_{j}_3"].float().numpy() for j in range(3)]
    if L.kind == "post":
        return [taps[f"rb_3_{j}_3"].float().numpy() for j in range(3)]
    return [taps[f"rb_{L.stage}_{j}_{L.step}"].float().numpy() for j in range(3)]


def oracle_taps(params, T=BASE_T, seed=5):
    mel = synthetic.mel_input(seed, 1, T)
    taps = {"mel": mel}
    with torch.no_grad():
        ho.generator_forward(params, mel, torch.float64, taps)
    return taps


# ---------------------------------------------------------------------------------------------------------------- GPU


@pytest.fixture(scope="module")
def eng(hifigan_params):
    from viettts_b200.engine import Engine
    e = Engine(0)
    e.load_hifigan(hifigan_params)
    yield e
    e.close()


@pytest.fixture(scope="module")
def taps(hifigan_params):
    return oracle_taps(hifigan_params)


def set_config(eng, mode, pairs):
    eng.set_precision(mode)
    if pairs == "unfused":
        eng.set_fused_pairs(False, kind=DEFAULT_PAIRS)
    else:
        eng.set_fused_pairs(True, kind=pairs)


def out_shape(L, B, T):
    return (B, T * L.scale_out) if L.kind == "post" else (B, T * L.scale_out, L.cout)


def run(eng, L, mode, pairs, xs_dev, lens_t, T):
    """one hook call into fresh sentinel-filled outputs, each followed by a guard of 1024 rows; checks the launch count,
    that no row at or past its length and no guard element is written (conv_post writes zeros there) and that every
    written value is finite.  Returns the outputs."""
    B = xs_dev[0].shape[0]
    shape = out_shape(L, B, T)
    n = int(np.prod(shape))
    guard = 1024 * (L.cout if L.kind != "post" else 1)
    bufs = [torch.empty(n + guard, dtype=torch.float32, device=xs_dev[0].device) for _ in range(L.nout)]
    for b in bufs:
        b.view(torch.int32).fill_(SENTINEL)
    outs = [b[:n].view(shape) for b in bufs]
    l0 = eng.launch_count()
    eng.debug_hifigan_layer(L.id, xs_dev, outs, lens_t, T)
    assert eng.launch_count() - l0 == launches(L, mode, pairs), (L.name, mode, pairs)
    lens = None if lens_t is None else lens_t.cpu().numpy()
    valid = valid_rows(B, T * L.scale_out, lens, L.scale_out, bufs[0].device)
    valid = valid[..., 0] if L.kind == "post" else valid.expand(shape)
    for b, o in zip(bufs, outs):
        assert torch.isfinite(o[valid]).all(), (L.name, mode, pairs, "non-finite output")
        if L.kind == "post":
            assert (o[~valid] == 0).all() and not torch.signbit(o[~valid]).any(), (L.name, mode, "conv_post must write +0 past a row")
        else:
            assert (o.view(torch.int32)[~valid] == SENTINEL).all(), (L.name, mode, pairs, "a row at or past its length was written")
        assert (b[n:].view(torch.int32) == SENTINEL).all(), (L.name, mode, pairs, "the guard after the output was written")
    return outs


def check(L, mode, outs, refs, lens, what):
    """the per-element bound on every valid element; returns the worst |err| / S"""
    worst = 0.0
    for p, (o, (ref, s, e)) in enumerate(zip(outs, refs)):
        B, rows = o.shape[:2]
        valid = valid_rows(B, rows, lens, L.scale_out, o.device)
        valid = valid[..., 0] if L.kind == "post" else valid.expand(o.shape)
        # conv_post: ref is the pre-activation; tanh is 1-Lipschitz, so its bound holds after the tanh
        err = (o.double() - (torch.tanh(ref) if L.kind == "post" else ref)).abs()
        err, s, e = err[valid], s[valid], e[valid]
        bad = err > TOL[mode] * s + EPS * e
        if bad.any():
            idx = torch.nonzero(valid)[bad.nonzero()[0, 0]].tolist()
            raise AssertionError(f"{what} {L.name} {mode} problem {p}: {int(bad.sum())} elements out of bound, first at "
                                 f"{idx}: |err| {float(err[bad][0]):.3e} > {TOL[mode]:.1e} * S {float(s[bad][0]):.3e}; "
                                 f"worst |err| / S {float((err / s.clamp_min(1e-30)).max()):.3e}")
        worst = max(worst, float((err / s.clamp_min(1e-30)).max()))
    return worst


def _bits_equal(xs, ys):
    return all(torch.equal(x.view(torch.int32), y.view(torch.int32)) for x, y in zip(xs, ys))


def wrap_T(L, mode, pairs, B):
    """the fewest mel frames that give every tensor-core launch of the layer more than WRAP_TILES tiles at batch B"""
    T = 1
    while min(launch_tiles(L, mode, pairs, B, T)) <= WRAP_TILES:
        T += 1
    return T


WORST = {}


@pytest.mark.gpu
@pytest.mark.parametrize("layer,mode,pairs", [(L.id, m, p) for L in LAYERS for m, p in configs(L)],
                         ids=[f"{L.name}-{m}-{p}" for L in LAYERS for m, p in configs(L)])
def test_layer_vs_float64(eng, hifigan_params, taps, layer, mode, pairs):
    """One layer in one mode and pair form: random inputs (base case), the oracle's own activations of a synthetic mel,
    a ragged batch with a row end at every tile edge, and (tensor-core paths) a launch of more than 4 x 132 tiles run
    twice for the same bits."""
    L = LAYERS[layer]
    dev = torch.device("cuda", 0)
    set_config(eng, mode, pairs)
    worst = {}
    try:
        cases = [("base", 1, BASE_T, None, random_inputs(L, 1, BASE_T, layer_seed(L, "base"))),
                 ("oracle", 1, BASE_T, None, oracle_inputs(L, taps)),
                 ("ragged", len(RAGGED), max(RAGGED), RAGGED, random_inputs(L, len(RAGGED), max(RAGGED), layer_seed(L, "ragged"), RAGGED))]
        tiles = launch_tiles(L, mode, pairs, 4, 1)
        if tiles:
            Tw = wrap_T(L, mode, pairs, 4)
            lw = [Tw, Tw - 1, 1, max(1, Tw // 2)]
            cases.append(("wrap", 4, Tw, lw, random_inputs(L, 4, Tw, layer_seed(L, "wrap"), lw)))
            assert min(launch_tiles(L, mode, pairs, 4, Tw)) > WRAP_TILES
        for what, B, T, lens, xs in cases:
            xs_dev = [torch.from_numpy(np.ascontiguousarray(x)).to(dev) for x in xs]
            lens_t = None if lens is None else torch.tensor(lens, dtype=torch.int32, device=dev)
            outs = run(eng, L, mode, pairs, xs_dev, lens_t, T)
            refs = reference(L, hifigan_params, xs_dev, lens, dev)
            worst[what] = check(L, mode, outs, refs, lens, what)
            if what == "wrap":
                again = run(eng, L, mode, pairs, xs_dev, lens_t, T)
                assert _bits_equal(outs, again), (L.name, mode, pairs, "the repeated launch gave other bits")
            del outs, refs, xs_dev
    finally:
        set_config(eng, "bf16x3", DEFAULT_PAIRS)
    WORST[(L.name, mode, pairs)] = worst
    print(f"[generator_layers] {L.name} {mode} {pairs}: worst |err| / S " + " ".join(f"{k} {v:.2e}" for k, v in worst.items())
          + f" (bound {TOL[mode]:.0e})")


@pytest.mark.gpu
@pytest.mark.parametrize("mode,pairs", [(m, DEFAULT_PAIRS) for m in MODES] + [("bf16x3", "unfused"), ("bf16x3", "tmem"),
                                                                              ("bf16x3", "smem"), ("fp16", "unfused")])
def test_layers_compose_to_the_forward(eng, mode, pairs):
    """Layers 0 -> 17 through the hook, on the buffers the forward would use, give the forward's waveform bit for bit: the
    hook runs the forward's own code, not a copy of it."""
    dev = torch.device("cuda", 0)
    mel = synthetic.mel_input(9, 3, 40)
    nf = np.array([40, 23, 1], np.int32)
    set_config(eng, mode, pairs)
    try:
        want = eng.mel2wave(mel, n_frames=nf)
        lens_t = torch.from_numpy(nf).to(dev)
        B, T = mel.shape[:2]
        x = [torch.from_numpy(mel).to(dev)]
        for L in (LAYERS[n] for n in FORWARD_ORDER):
            shape = out_shape(L, B, T)
            outs = [torch.zeros(shape, dtype=torch.float32, device=dev) for _ in range(L.nout)]
            eng.debug_hifigan_layer(L.id, x * 3 if L.kind == "rb" and L.step == 0 else x, outs, lens_t, T)
            x = outs                       # step 0 of a stage: the ConvTranspose output feeds all three chains
        got = x[0].cpu().numpy()
    finally:
        set_config(eng, "bf16x3", DEFAULT_PAIRS)
    assert np.array_equal(got.view(np.int32), want.view(np.int32)), (mode, pairs, float(np.abs(got - want).max()))


@pytest.mark.gpu
def test_bad_arguments_fail_cleanly(eng):
    """Rejected calls raise and write nothing: a layer id out of range, a missing chain, no frames."""
    from viettts_b200 import _lib
    dev = torch.device("cuda", 0)
    x = torch.zeros(1, 8, 512, device=dev)
    out = torch.full((1, 64, 256), 7.0, device=dev)
    for layer, xs, T in ((18, [x], 8), (-1, [x], 8), (2, [x, None, None], 1), (1, [x], 0)):
        with pytest.raises(_lib.VttsError):
            eng.debug_hifigan_layer(layer, xs, [out], None, T)
    assert (out == 7.0).all()
