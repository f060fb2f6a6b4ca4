"""The shared conv dispatcher (vtts_conv_dispatch), the path of every conv and hoisted GEMM of the acoustic, teacher-forced
and duration models, layer by layer against a float64 Haiku layer, in both arithmetic modes.

The hook vtts_debug_conv_dispatch packs, derives the BatchNorm inverses and dispatches exactly as the model's load and
run code do, so these tests reach what a single tensor-core launch does not: the split of Cout into N tiles of <= 256
columns, the partial last tile (Cout = 80), the cap of 8 problems per launch (two launches for the hoisted LSTM GEMMs),
the per-tile offsets of bias / BatchNorm / residual / output, the generic epilogue (eval BatchNorm, tanh, relu) and the
FP32 kernel's own epilogue.

Tolerance, per element, scale-free: with S = conv(|x|, |w|) in float64, inv the BatchNorm factor (1 without BatchNorm)
and E = |inv * mean| + |offset| + |resid| + |ref| the size of what the fp32 epilogue adds and rounds,
    |got - ref| <= TOL[mode] * |inv| * (S + |b|) + EPS * E.
test_bound_has_headroom_over_the_emulation derives TOL from a CPU emulation of each mode on the base case of every
entry (same seeds and shapes as here)."""
import re
import zlib
from collections import namedtuple
from pathlib import Path

import numpy as np
import pytest
import torch

REPO = Path(__file__).resolve().parents[1]
TOL = {"fp32": 2e-6, "bf16x3": 2e-5}
EPS = 2.0 ** -21                 # 8 fp32 ulps of each term the epilogue adds
SENTINEL = 0x7FC0DEAD            # NaN with a payload: the bits of every output element the dispatcher must not write
WRAP_TILES = 4 * 132             # tensor-core tiles of a launch several times the SM count of an H100 SXM
FP32_TM = 128                    # rows per CTA of the FP32 kernel for Cout > 64
CTX_MODE = "fp16"                # the context's own mode: every hook call must leave it so

# One entry per packing-table entry of csrc/nat.cu (`pk[PK_*] = {weight, k, Cin, Cout}`; the loop entries
# `pk[PK_ENC_CONV0 + i]` and `pk[PK_POST0 + i]` go by their first name), with the epilogue and batching of the run_convs
# call that uses it.  epi: "bn_relu" / "bn_tanh" (eval BatchNorm, then the activation), "resid" (+ residual), "zero_bias"
# (the bias-free prenet linears) or None (bias only).  ragged: B sequences with a length each; else one row of every
# token or frame of the batch (B = 1, no lengths).
Entry = namedtuple("Entry", "pk k cin cout nprob epi ragged")
TABLE = {
    "enc_conv": Entry(("PK_ENC_CONV0",), 3, 256, 256, 1, "bn_relu", True),      # PK_ENC_CONV0 + 0..2
    "enc_lstm": Entry(("PK_ENC_LSTM_F", "PK_ENC_LSTM_B"), 1, 256, 1024, 2, None, False),
    "dec_lstm": Entry(("PK_DEC_L0", "PK_DEC_L1"), 1, 512, 2048, 2, None, False),
    "tf_lstm": Entry(("PK_TF_L0", "PK_TF_L1"), 1, 768, 2048, 2, None, False),
    "pre1": Entry(("PK_PRE1",), 1, 80, 256, 1, "zero_bias", False),
    "pre2": Entry(("PK_PRE2",), 1, 256, 256, 1, "zero_bias", False),
    "proj": Entry(("PK_PROJ",), 1, 1024, 80, 1, None, True),
    "post0": Entry(("PK_POST0",), 5, 80, 512, 1, "bn_tanh", True),
    "post1": Entry(("PK_POST0",), 5, 512, 512, 1, "bn_tanh", True),             # PK_POST0 + 1..3
    "post4": Entry(("PK_POST0",), 5, 512, 80, 1, "resid", True),                # PK_POST0 + 4
    "du_fc1": Entry(("PK_DU_FC1",), 1, 512, 256, 1, None, False),
}
BASE_T = 600                     # the base case of every entry, also emulated on the CPU
POST_ACT = {"bn_relu": "relu", "bn_tanh": "tanh"}


def tile_n(cout):
    return 32 if cout <= 32 else 64 if cout <= 64 else 128 if cout <= 128 else 256


def tc_rows(cout):
    """rows per tensor-core tile: 64 x MW rows per consumer warpgroup, two warpgroups"""
    n = tile_n(cout)
    return 128 * (1 if n >= 256 else 2 if n == 128 else 4)


def tc_launches(e):
    """launches of one dispatch in bf16x3: full N tiles of every problem, 8 per launch, then the partial last tiles"""
    n = tile_n(e.cout)
    return -(-e.nprob * (e.cout // n) // 8) + (-(-e.nprob // 8) if e.cout % n else 0)


def base_seed(name):
    return zlib.crc32(name.encode())


Inputs = namedtuple("Inputs", "x w b bn resid")


def make_inputs(e, B, T, seed, lens=None, scale=1.0, tiny_var=False):
    """float32 numpy inputs of every problem.  Weights, biases and BatchNorm statistics differ per problem and per N tile,
    so a swapped tile or offset gives O(1) errors.  `scale` multiplies x, bias, BatchNorm mean and offset and the residual
    (the layer before its activation is homogeneous in them); rows at or past a length are NaN in x and resid."""
    rng = np.random.default_rng(seed)
    f32 = np.float32
    x, w, b, bn, resid = [], [], [], [], []
    for _ in range(e.nprob):
        x.append(rng.standard_normal((B, T, e.cin), dtype=f32) * f32(scale))
        w.append((rng.standard_normal((e.k, e.cin, e.cout)) / np.sqrt(e.k * e.cin)).astype(f32))
        b.append(np.zeros(e.cout, f32) if e.epi == "zero_bias" else (rng.standard_normal(e.cout) * 0.1 * scale).astype(f32))
        if e.epi in ("bn_relu", "bn_tanh"):
            var = np.full(e.cout, 1e-4) if tiny_var else rng.uniform(0.5, 1.5, e.cout)
            bn.append(np.stack([1.0 + 0.2 * rng.standard_normal(e.cout), 0.1 * scale * rng.standard_normal(e.cout),
                                0.1 * scale * rng.standard_normal(e.cout), var]).astype(f32))
        else:
            bn.append(None)
        resid.append(rng.standard_normal((B, T, e.cout), dtype=f32) * f32(scale) if e.epi == "resid" else None)
    if lens is not None:
        for b_ in range(B):
            for a in x + [r for r in resid if r is not None]:
                a[b_, lens[b_]:] = np.nan
    return Inputs(x, w, b, bn, resid)


def _conv(x, w):
    """SAME-padded conv of x [B,T,Cin] with a Haiku weight [k,Cin,Cout] (dilation 1, as every dispatcher call site)"""
    k = w.shape[0]
    if k == 1:
        return x @ w[0]
    return torch.nn.functional.conv1d(x.transpose(1, 2), w.permute(2, 1, 0), padding=(k - 1) // 2).transpose(1, 2)


def _valid(B, T, lens, device):
    if lens is None:
        return torch.ones(B, T, dtype=torch.bool, device=device)
    return torch.arange(T, device=device)[None, :] < torch.as_tensor(np.asarray(lens), device=device)[:, None]


def reference(e, inp, lens, device):
    """float64 Haiku layer per problem: (ref, A = |inv| (S + |b|), E), zero padding at each row's true length"""
    out = []
    for p in range(e.nprob):
        x = torch.from_numpy(inp.x[p]).to(device).double()
        B, T, _ = x.shape
        valid = _valid(B, T, lens, device)[..., None]
        x = torch.where(valid, x, 0.0)
        w = torch.from_numpy(inp.w[p]).to(device).double()
        b = torch.from_numpy(inp.b[p]).to(device).double()
        y = _conv(x, w) + b
        a = _conv(x.abs(), w.abs()) + b.abs()
        ep = torch.zeros_like(y)
        if inp.bn[p] is not None:
            scale, off, mean, var = torch.from_numpy(inp.bn[p]).to(device).double()
            inv = scale / torch.sqrt(var + 1e-5)
            y = (y - mean) * inv + off
            a = a * inv.abs()
            ep = ep + (inv * mean).abs() + off.abs()
        if e.epi == "bn_tanh":
            y = torch.tanh(y)
        elif e.epi == "bn_relu":
            y = torch.relu(y)
        if inp.resid[p] is not None:
            r = torch.where(valid, torch.from_numpy(inp.resid[p]).to(device).double(), 0.0)
            y = y + r
            ep = ep + r.abs()
        out.append((y, a, ep + y.abs()))
    return out


def cases(name):
    """(B, T, lens, seed) of one entry: the base case, lengths on every row-tile edge of both kernels, the bench shape of
    the k = 1 GEMMs (32 x 312 rows) and a tile count several times the SM count (the run-time tile scheduler wraps)"""
    e = TABLE[name]
    R = tc_rows(e.cout)
    edges = sorted({FP32_TM - 1, FP32_TM, FP32_TM + 1, R - 1, R, R + 1})
    seed = base_seed(name)
    out = [(1, BASE_T, [BASE_T] if e.ragged else None, seed)]
    for i, T in enumerate([1] + edges):
        out.append((1, T, [T] if e.ragged else None, seed + 1 + i))
    per_rowtile = e.nprob * -(-e.cout // tile_n(e.cout))
    if e.ragged:
        T = 2 * max(R, FP32_TM) + 37
        out.append((len(edges) + 2, T, [1] + edges + [T], seed + 20))
        if e.k == 1:
            out.append((32, 312, [312] * 31 + [97], seed + 21))
        T = -(-WRAP_TILES // (8 * per_rowtile)) * R - 45
        out.append((8, T, [T, T - 1, T - R, R + 1, T // 2, T, 1, T - 45], seed + 22))
    else:
        if e.k == 1:
            out.append((1, 32 * 312, None, seed + 21))
        out.append((1, -(-WRAP_TILES // per_rowtile) * R - 45, None, seed + 22))
    return out


# ---------------------------------------------------------------------------------------------------------------- CPU


def test_table_matches_the_packing_tables():
    """Every packed conv of the model has an entry here, with the packed shape; a new one cannot enter untested."""
    src = (REPO / "viettts_b200" / "csrc" / "nat.cu").read_text()
    names = set(re.findall(r"\bpk\[(PK_\w+)(?:\s*\+\s*i)?\]\s*=\s*\{", src))
    assert names == {n for e in TABLE.values() for n in e.pk}, names
    shapes = {}
    for n, k, cin, cout in re.findall(r"\bpk\[(PK_\w+)(?:\s*\+\s*i)?\]\s*=\s*\{[^{}\n]*?\],\s*(\d+),\s*(\d+),\s*(\d+)\}", src):
        shapes[n] = (int(k), int(cin), int(cout))
    # the literal shapes; the postnet loop computes its Cin / Cout (80 at its ends) and is checked through the call sites
    assert set(shapes) == names - {"PK_POST0"}, shapes
    for e in TABLE.values():
        for n in e.pk:
            if n in shapes:
                assert shapes[n] == (e.k, e.cin, e.cout), (n, shapes[n], e)
    assert "i == 0 ? 80 : 512, i == 4 ? 80 : 512" in src
    post = sorted((e.cin, e.cout) for e in TABLE.values() if e.pk == ("PK_POST0",))
    assert post == [(80, 512), (512, 80), (512, 512)]


def _emulate_fp32(x, w):
    """the FP32 kernel's arithmetic: one fp32 fma per (16-channel chunk, tap, channel) in that order (products of two
    fp32 values are exact in float64, so each step rounds once, as an fma does)"""
    k, cin, _ = w.shape
    xp = torch.nn.functional.pad(x[0], (0, 0, (k - 1) // 2, k - 1 - (k - 1) // 2))
    acc = torch.zeros(x.shape[1], w.shape[2], dtype=torch.float32)
    for c in range(0, cin, 16):
        for j in range(k):
            for i in range(c, c + 16):
                acc = (acc.double() + torch.outer(xp[j : j + x.shape[1], i], w[j, i])).float()
    return acc.double()[None]


def test_bound_has_headroom_over_the_emulation():
    """The base case of every entry: bf16x3's operand rounding (precision_study) stays 4x below its bound, bf16x1's
    rounding (the lo products dropped) exceeds the bound 10x, and the fp32 bound sits well above the FP32 kernel's
    accumulation error and well below the bf16x3 bound."""
    import importlib.util
    spec = importlib.util.spec_from_file_location("precision_study", REPO / "scripts" / "precision_study.py")
    ps = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ps)
    worst = {"bf16x3": 0.0, "bf16x1": np.inf, "fp32": 0.0}
    report = []
    for name, e in TABLE.items():
        B, T, lens, seed = cases(name)[0]
        inp = make_inputs(e, B, T, seed, lens)
        x = torch.from_numpy(inp.x[0]).double()
        w = torch.from_numpy(inp.w[0]).double()
        ref = _conv(x, w)
        a = _conv(x.abs(), w.abs()) + torch.from_numpy(inp.b[0]).double().abs()
        row = {}
        for mode in ("bf16x3", "bf16x1"):
            rnd, terms, pairs = ps.MODES[mode]
            xs, ws = ps.split(x, rnd, terms), ps.split(w, rnd, terms)
            y = sum(_conv(xs[i], ws[j]) for i, j in pairs)
            row[mode] = float(((y - ref).abs() / a).max())
        row["fp32"] = float(((_emulate_fp32(x, w) - ref).abs() / a).max())
        report.append(f"{name}: " + " ".join(f"{m} {v:.2e}" for m, v in row.items()))
        worst["bf16x3"] = max(worst["bf16x3"], row["bf16x3"])
        worst["bf16x1"] = min(worst["bf16x1"], row["bf16x1"])
        worst["fp32"] = max(worst["fp32"], row["fp32"])
    print("emulated max |err| / (S + |b|):\n  " + "\n  ".join(report))
    assert 4 * worst["bf16x3"] <= TOL["bf16x3"], worst
    assert worst["bf16x1"] >= 10 * TOL["bf16x3"], worst
    assert 4 * worst["fp32"] <= TOL["fp32"] <= TOL["bf16x3"] / 4, worst


# ---------------------------------------------------------------------------------------------------------------- GPU


@pytest.fixture(scope="module")
def eng():
    from viettts_b200.engine import Engine
    e = Engine(0)
    e.set_precision(CTX_MODE)
    yield e
    e.close()


def _dev(inp, device):
    return Inputs(*[[None if a is None else torch.from_numpy(a).to(device) for a in field] for field in inp])


def _row(dinp, r):
    """batch row r of device inputs, as a batch of one"""
    one = lambda ts: [None if t is None else t[r : r + 1] for t in ts]  # noqa: E731
    return dinp._replace(x=one(dinp.x), resid=one(dinp.resid))


def _ctx_mode():
    from viettts_b200.engine import PRECISIONS
    return PRECISIONS[CTX_MODE]


def run(eng, e, dinp, lens_t, mode):
    """one hook call into fresh sentinel-filled outputs, each followed by a guard of one row tile; checks the launch count,
    the context's mode, that no row at or past its length and no guard element is written and that every written value
    is finite.  Returns the whole buffers (output and guard)."""
    B, T, _ = dinp.x[0].shape
    n = B * T * e.cout
    bufs = [torch.empty(n + tc_rows(e.cout) * e.cout, dtype=torch.float32, device=dinp.x[0].device) for _ in range(e.nprob)]
    for b in bufs:
        b.view(torch.int32).fill_(SENTINEL)
    outs = [b[:n].view(B, T, e.cout) for b in bufs]
    l0 = eng.launch_count()
    eng.debug_conv_dispatch(mode, dinp.x, dinp.w, dinp.b, e.k, bns=dinp.bn, resids=dinp.resid, post_act=POST_ACT.get(e.epi, "none"),
                            len_t=lens_t, outs=outs)
    assert eng.launch_count() - l0 == (1 if mode == "fp32" else tc_launches(e)), mode
    assert eng.lib.vtts_get_precision(eng.h) == _ctx_mode(), mode
    valid = _valid(B, T, None if lens_t is None else lens_t.cpu().numpy(), bufs[0].device)
    for b, o in zip(bufs, outs):
        assert torch.isfinite(o[valid]).all(), mode
        assert (o.view(torch.int32)[~valid] == SENTINEL).all(), f"{mode}: a row at or past its length was written"
        assert (b[n:].view(torch.int32) == SENTINEL).all(), f"{mode}: the guard after the output was written"
    return bufs


def check(e, bufs, refs, B, T, lens, mode, what):
    """the per-element bound on every written element; returns the worst |err| / (|inv| (S + |b|))"""
    worst = 0.0
    valid = _valid(B, T, lens, bufs[0].device)
    for p, (b, (ref, a, ep)) in enumerate(zip(bufs, refs)):
        err = (b[: B * T * e.cout].view(B, T, e.cout).double() - ref).abs()[valid]
        a, ep = a[valid], ep[valid]
        bad = err > TOL[mode] * a + EPS * ep
        assert not bad.any(), (what, mode, p, float(err[bad].max()), int(bad.sum()))
        worst = max(worst, float((err / a).max()))
    return worst


def _bits_equal(xs, ys):
    return all(torch.equal(x.view(torch.int32), y.view(torch.int32)) for x, y in zip(xs, ys))


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(TABLE))
def test_entry_vs_float64(eng, name):
    """Every case of cases(name) in fp32 and bf16x3 against float64.  Also: fp16 gives the bits of bf16x3; each row of a
    ragged batch gives the bits of the same row run alone; the base and the wrapping case, repeated after calls of other
    sizes, give the same bits."""
    e = TABLE[name]
    dev = torch.device("cuda", 0)
    worst = {m: 0.0 for m in TOL}
    all_cases = cases(name)
    kept = {}
    for c, (B, T, lens, seed) in enumerate(all_cases):
        inp = make_inputs(e, B, T, seed, lens)
        dinp = _dev(inp, dev)
        lens_t = None if lens is None else torch.tensor(lens, dtype=torch.int32, device=dev)
        refs = reference(e, inp, lens, dev)
        for mode in TOL:
            bufs = run(eng, e, dinp, lens_t, mode)
            worst[mode] = max(worst[mode], check(e, bufs, refs, B, T, lens, mode, (name, B, T)))
            if mode == "bf16x3":
                assert _bits_equal(bufs, run(eng, e, dinp, lens_t, "fp16")), (name, B, T, "fp16 differs from bf16x3")
                if c in (0, len(all_cases) - 1):
                    kept[c] = (dinp, lens_t, bufs)
            if 1 < B <= 16:
                n = T * e.cout
                for r in range(B):
                    alone = run(eng, e, _row(dinp, r), lens_t[r : r + 1], mode)
                    assert _bits_equal([b[r * n : (r + 1) * n] for b in bufs], [b[:n] for b in alone]), \
                        (name, mode, T, r, lens[r], "row differs from the same row run alone")
        del inp, dinp, refs
    for c in sorted(kept):
        dinp, lens_t, bufs = kept[c]
        assert _bits_equal(bufs, run(eng, e, dinp, lens_t, "bf16x3")), (name, all_cases[c][:2], "repeated call differs")
    print(f"[conv_dispatch] {name}: worst |err| / (|inv| (S + |b|)): fp32 {worst['fp32']:.2e} bf16x3 {worst['bf16x3']:.2e}")


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(TABLE))
def test_value_edges(eng, name):
    """Inputs scaled by 1e-3 and 1e3 (the bound is relative), BatchNorm with var = 1e-4 (inv ~ 100x), tanh deep in
    saturation (scale 1e3 of the postnet layers)."""
    e = TABLE[name]
    dev = torch.device("cuda", 0)
    B, T, lens = (2, 300, [300, 129]) if e.ragged else (1, 300, None)
    variants = [dict(scale=1e-3), dict(scale=1e3)] + ([dict(tiny_var=True)] if e.epi in ("bn_relu", "bn_tanh") else [])
    for i, v in enumerate(variants):
        inp = make_inputs(e, B, T, base_seed(name) + 100 + i, lens, **v)
        refs = reference(e, inp, lens, dev)
        if e.epi == "bn_tanh" and v.get("scale") == 1e3:
            valid = _valid(B, T, lens, dev)
            assert (refs[0][0].abs()[valid] > 1 - 1e-6).double().mean() > 0.9    # deep saturation
        dinp = _dev(inp, dev)
        lens_t = None if lens is None else torch.tensor(lens, dtype=torch.int32, device=dev)
        for mode in TOL:
            nerr = check(e, run(eng, e, dinp, lens_t, mode), refs, B, T, lens, mode, (name, v))
            print(f"[conv_dispatch edges] {name} {v} {mode}: {nerr:.2e}")


@pytest.mark.gpu
def test_bad_arguments_fail_cleanly(eng):
    """Rejected calls raise, write nothing and leave the context's mode alone, also when the dispatcher itself rejects
    the call after the hook has switched modes (a halo beyond the kernels')."""
    from viettts_b200 import _lib
    dev = torch.device("cuda", 0)
    x = torch.zeros(1, 64, 256, device=dev)
    b = torch.zeros(256, device=dev)
    out = torch.full((1, 64, 256), 7.0, device=dev)
    good = dict(xs=[x], ws=[torch.zeros(3, 256, 256, device=dev)], biases=[b], k=3, outs=[out])
    bad = [dict(good, xs=[x] * 9, ws=good["ws"] * 9, biases=[b] * 9, outs=[out] * 9),   # more than 8 problems
           dict(good, xs=[torch.zeros(1, 64, 24, device=dev)], ws=[torch.zeros(3, 24, 256, device=dev)]),   # Cin % 16
           dict(good, ws=[torch.zeros(3, 256, 250, device=dev)], outs=[torch.zeros(1, 64, 250, device=dev)]),   # Cout % 4
           dict(good, ws=[torch.zeros(67, 256, 256, device=dev)], k=67)]   # halo (k - 1) * dil > 64
    for mode in ("fp32", "bf16x3", "fp16"):
        for kw in bad:
            with pytest.raises(_lib.VttsError):
                eng.debug_conv_dispatch(mode, **kw)
            assert eng.lib.vtts_get_precision(eng.h) == _ctx_mode()
    assert (out == 7.0).all()
    with pytest.raises(_lib.VttsError):
        eng.debug_conv_dispatch(3, **good)
    eng.debug_conv_dispatch("bf16x3", **good)
    assert (out == 0.0).all() and eng.lib.vtts_get_precision(eng.h) == _ctx_mode()
