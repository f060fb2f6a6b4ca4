"""The duration model (`vtts_duration_run`: `Engine.predict_duration`, `duration_forward` and the first half of every
`tts`) stage by stage against float64, and the text-to-speech plan (`vtts_tts_plan`) against the oracle's glue.  Each
stage starts from the GPU's own input to it, read through the `vtts_debug_read` taps, so each stage's error is measured
alone:
  enc         [B,L,512]  float64 TokenEncoder (`nat_oracle.token_encoder` with the duration checkpoint) of each row
                         alone at its own length; L-inf <= ENC_BOUND
  dur_hidden  [B,L,256]  float64 Linear(512->256) of the GPU `enc`; per element |err| <= HID_TOL * S,
                         S = |enc|.|W1| + |b1|, the conv dispatcher's tolerance (tests/test_gpu_conv_dispatch.py)
  durations   [B,L]      float64 gelu (tanh form) -> .w2 -> + b2 -> softplus of the GPU `dur_hidden`; per token
                         |err| <= HEAD_TOL units of 2^-24 (sigmoid(s) sum_i |gelu(y_i) w2_i| + softplus(s)), s the
                         pre-softplus value; exactly 0 past lengths[b]
Both taps are checked before lengths[b] only: past it the encoder scan runs on over the padding from unspecified
workspace rows, and the head never reads those positions.
HEAD_TOL is at least 4x the worst error of an fp32 emulation of duration_head_kernel and of the plain fp32 oracle on
every case here, and a wrong gelu form, a dropped b2 or w2 read one lane block off exceed it by far
(tests/test_duration_bounds.py).

Cases: ragged batches at every B where the encoder scan's row groups or register tiles change shape, B = 130 through
the host layer's 128-row chunks, every B*L around the head's 8-token CTA, a row longer than the acoustic model accepts,
padding filled with real token ids (0 and 3 among them), lengths = NULL, exact row independence and FP16 equal to
BF16X3.  The plan: `Engine.tts_plan` equals the oracle's adjust_durations / seconds_to_frames / trim_end_silence fed
the same raw durations, bit for bit, and a row built to sit on a frame-count boundary gets the same frame count from
every entry point."""
import functools
import math
import pickle

import numpy as np
import pytest
import torch

from oracle import nat_oracle as no
from viettts_b200 import config, synthetic

pytestmark = pytest.mark.gpu

F64 = torch.float64
ENC = no.DM + "token_encoder/~/"
HID_TOL = {"fp32": 2e-6, "bf16x3": 2e-5}          # the conv dispatcher's TOL (tests/test_gpu_conv_dispatch.py)
ENC_BOUND = {"fp32": 1e-5, "bf16x3": 1e-4}        # the acoustic encoder's bound (tests/test_gpu_acoustic_scans.py)
HEAD_TOL = 6.0                                    # units of 2^-24 (sigmoid(s) sum |gelu(y) w2| + softplus(s))
# end to end (tests/test_gpu_duration.py), in the same unit: the plain fp32 oracle's worst there is 2.6 units
# (tests/test_duration_bounds.py); BF16X3 runs the encoder convs and both GEMMs at the dispatcher's 10x larger TOL
E2E_UNITS = {"fp32": 16.0, "bf16x3": 160.0}

SIZES = [1, 8, 9, 31, 32, 33, 64, 65, 97, 127, 128]
EDGE_BL = [(1, 1), (1, 7), (1, 8), (3, 3), (3, 5), (2, 8), (1, 17)]   # B*L = 1, 7, 8, 9, 15, 16, 17
L_MAX = 37
LONG_L = 6001              # longer than the acoustic model's 5689 tokens (its upsample's shared-memory row)
VERY_LONG_L = 65537        # accepted too: the duration path's only limit is its workspace, 13.3 KB per token
PAD_IDS = np.array([0, 3, 77, 0, 3, 12, 3, 0], np.int32)
PROBE = (0, 1, 2, 31, 32, 63, 64, 96, 127)

# ------------------------------------------------------------------------------------------------ cases (CPU too)


@functools.lru_cache(maxsize=None)
def matrix_rows():
    """128 token rows: row 0 has L_MAX tokens, rows 1 and 2 one and two; the others 1..L_MAX, so that rows end at
    different tokens within each row group and register tile.  Silence (0) and word-end (3) ids occur anywhere."""
    rng = np.random.default_rng(4242)
    rows = []
    for b in range(128):
        n = L_MAX if b == 0 else 1 if b == 1 else 2 if b == 2 else 1 + (b * 11) % L_MAX
        tk = rng.integers(0, 90, n).astype(np.int32)
        tk[rng.random(n) < 0.15] = config.WORD_END_INDEX
        tk[0] = config.SIL_INDEX
        if b % 2:
            tk[-1] = config.SIL_INDEX
        rows.append(tk)
    return tuple(rows)


def pad(rows, L=None):
    """tokens [B,L] whose padding holds real token ids (0 and 3 among them), and lengths [B]"""
    L = L or max(len(r) for r in rows)
    tok = np.resize(PAD_IDS, (len(rows), L)).astype(np.int32)
    for b, r in enumerate(rows):
        tok[b, : len(r)] = r
    return tok, np.array([len(r) for r in rows], np.int32)


def edge_rows(B, L):
    rng = np.random.default_rng(100 * B + L)
    return [rng.integers(0, 90, L).astype(np.int32) for _ in range(B)]


def long_row(L):
    rng = np.random.default_rng(L)
    tk = rng.integers(4, config.ALPHABET_SIZE, L).astype(np.int32)
    tk[4::5] = config.WORD_END_INDEX
    tk[0] = tk[-1] = config.SIL_INDEX
    return tk


def cases():
    """(name, token rows) of every stage case with an encoder reference"""
    out = [(f"B={B}", list(matrix_rows()[:B])) for B in SIZES]
    out += [(f"B*L={B * L}", edge_rows(B, L)) for B, L in EDGE_BL]
    out.append((f"L={LONG_L}", [long_row(LONG_L)]))
    return out


# ------------------------------------------------------------------------------------------------ references

_enc_cache = {}


def enc_ref(ckpt, rows):
    """float64 TokenEncoder of each row alone at its own length ([L_b,512] per row); rows of one length run together"""
    P, S = ckpt["params"], ckpt["aux"]
    todo = {}
    for r in rows:
        key = (id(ckpt), r.tobytes())
        if key not in _enc_cache:
            todo.setdefault(len(r), {})[key] = r
    with torch.no_grad():
        for n, group in todo.items():
            tk = np.stack(list(group.values()))
            e = no.token_encoder(P, S, tk, np.full(len(tk), n), F64, T=ENC).numpy()
            for j, key in enumerate(group):
                _enc_cache[key] = e[j]
    return [_enc_cache[(id(ckpt), r.tobytes())] for r in rows]


def head_weights(ckpt):
    """(W1 [512,256], b1 [256], w2 [256], b2) in float64"""
    P = ckpt["params"]
    return (no._t(P[no.DM + "linear"]["w"], F64), no._t(P[no.DM + "linear"]["b"], F64),
            no._t(P[no.DM + "linear_1"]["w"], F64)[:, 0], float(P[no.DM + "linear_1"]["b"][0]))


def hidden_ref(ckpt, enc):
    """float64 first Linear of enc [...,512] (any float array), and the scale S = |enc|.|W1| + |b1| of each element"""
    w1, b1, _, _ = head_weights(ckpt)
    with torch.no_grad():
        x = torch.as_tensor(np.asarray(enc)).double()
        return (x @ w1 + b1).numpy(), (x.abs() @ w1.abs() + b1.abs()).numpy()


def head_ref(ckpt, y, gelu=no.gelu_tanh, softplus=no.softplus, w2_shift=0, bias=True):
    """float64 gelu -> .w2 -> + b2 -> softplus of y [...,256] (any float array): (durations, unit of each token), the
    unit 2^-24 (sigmoid(s) sum_i |gelu(y_i) w2_i| + softplus(s)) of the true head.  The keyword arguments give the
    wrong variants tests/test_duration_bounds.py checks the bound against (w2_shift: lane l reads lane l + shift/8)."""
    _, _, w2, b2 = head_weights(ckpt)
    with torch.no_grad():
        yt = torch.as_tensor(np.asarray(y)).double()
        g = no.gelu_tanh(yt)
        s = g @ w2 + b2
        unit = 2.0 ** -24 * (torch.sigmoid(s) * (g * w2).abs().sum(-1) + no.softplus(s))
        d = softplus(gelu(yt) @ torch.roll(w2, -w2_shift) + (b2 if bias else 0.0))
    return d.numpy(), unit.numpy()


def e2e_ref(ckpt, tokens, lengths):
    """float64 durations of tokens [B,L] (each row at lengths[b]; the reference's own batching) and each token's unit"""
    P, S = ckpt["params"], ckpt["aux"]
    with torch.no_grad():
        enc = no.token_encoder(P, S, tokens, lengths, F64, T=ENC)
    y, _ = hidden_ref(ckpt, enc.numpy())
    return head_ref(ckpt, y)


def f32_frame_count(frames):
    """the frame count as a float32 sum in numpy's pairwise order: what the Python entry points used to compute"""
    return int(np.sum(np.asarray(frames, np.float32), dtype=np.float32))


def silence_frames(raw, sd):
    """frames of an all-silence row with raw predictions `raw` [L] after the silence clip at sd"""
    d = no.adjust_durations(np.zeros(len(raw), np.int32), np.asarray(raw, np.float32)[None], sd)
    return no.seconds_to_frames(d)[0][0]


def boundary_silence_duration(raw, lo, hi):
    """A float32 silence_duration in [lo, hi] at which the all-silence row with raw predictions `raw` (all below lo)
    gets a different frame count from a float32 sum than from `frame_count`: bisect (over float32 bit patterns) to
    each integer the float64 sum crosses, then step by ulps around the crossing."""
    assert float(np.max(raw)) < lo, "the predictions must fall below the search range"
    val = lambda i: np.int32(i).view(np.float32)                                     # noqa: E731
    dsum = lambda i: float(np.sum(silence_frames(raw, val(i)), dtype=np.float64))    # noqa: E731
    a, b = int(np.float32(lo).view(np.int32)), int(np.float32(hi).view(np.int32))
    for k in range(math.floor(dsum(a)) + 1, math.floor(dsum(b)) + 1):
        x, y = a, b                                                                  # dsum(x) < k <= dsum(y)
        while y - x > 1:
            m = (x + y) // 2
            x, y = (m, y) if dsum(m) < k else (x, m)
        for i in range(y - 24, y + 24):
            fr = silence_frames(raw, val(i))
            if f32_frame_count(fr) != no.frame_count(fr):
                return val(i)
    raise AssertionError("no silence_duration in range separates the two frame counts")


# ------------------------------------------------------------------------------------------------ GPU


@pytest.fixture(scope="module")
def duration_ckpt():
    return synthetic.duration_ckpt(1234)


@pytest.fixture(scope="module", params=["fp32", "bf16x3"])
def eng(duration_ckpt, acoustic_ckpt, hifigan_params, request):
    from viettts_b200.engine import Engine
    e = Engine(0)
    e.load_duration(duration_ckpt)
    e.load_acoustic(acoustic_ckpt)
    e.load_hifigan(hifigan_params)
    e.set_precision(request.param)
    e.mode = request.param
    yield e
    e.close()


def read_taps(eng, B, L):
    return dict(enc=eng.debug_read("enc", (B, L, 512)), hid=eng.debug_read("dur_hidden", (B, L, 256)))


def run(eng, tok, lens):
    dur = eng.predict_duration(tok, lengths=lens)
    return dict(dur=dur, **read_taps(eng, *tok.shape))


def check(eng, ckpt, tok, lens, got, what, rows=None):
    """every stage of every row of one call (lens None: every row is L long); rows: the token rows, for the encoder
    stage (None: skip it).  Returns the worst error per stage (dur_hidden in units of S, durations in HEAD_TOL's)."""
    mode = eng.mode
    B, L = tok.shape
    lens = np.full(B, L) if lens is None else np.asarray(lens)
    worst = dict(enc=0.0, dur_hidden=0.0, durations=0.0)
    if rows is not None:
        for b, ref in enumerate(enc_ref(ckpt, rows)):
            n = int(lens[b])
            e = float(np.abs(got["enc"][b, :n] - ref).max())
            assert e <= ENC_BOUND[mode], (what, b, "enc", e)
            worst["enc"] = max(worst["enc"], e)
    valid = np.arange(L)[None, :] < lens[:, None]
    y, s = hidden_ref(ckpt, got["enc"][valid])
    r = np.abs(got["hid"][valid] - y) / s
    assert not (r > HID_TOL[mode]).any(), (what, "dur_hidden", np.argwhere(r > HID_TOL[mode])[:4], float(r.max()))
    worst["dur_hidden"] = float(r.max())
    d, unit = head_ref(ckpt, np.where(valid[..., None], got["hid"], 0.0))
    u = np.where(valid, np.abs(got["dur"] - d) / unit, 0.0)
    assert not (u > HEAD_TOL).any(), (what, "durations", np.argwhere(u > HEAD_TOL)[:4], float(u.max()))
    worst["durations"] = float(u.max())
    assert np.all(got["dur"][~valid] == 0), (what, "durations past the row")
    print(f"[duration] {what} {mode}: enc {worst['enc']:.2e}  dur_hidden {worst['dur_hidden']:.2e} S  "
          f"durations {worst['durations']:.2f} units")
    return worst


@pytest.mark.parametrize("B", SIZES)
def test_launch_and_tile_edges(eng, duration_ckpt, B):
    """Every row of a ragged batch of B rows (1..37 tokens, padding filled with real ids), every stage."""
    rows = list(matrix_rows()[:B])
    tok, lens = pad(rows)
    check(eng, duration_ckpt, tok, lens, run(eng, tok, lens), f"B={B}", rows)


@pytest.mark.parametrize("B,L", EDGE_BL, ids=[f"BL{B * L}" for B, L in EDGE_BL])
def test_head_cta_edges(eng, duration_ckpt, B, L):
    """B*L = 1, 7, 8, 9, 15, 16, 17: the head's last CTA of 8 tokens full, one token short and one token over."""
    rows = edge_rows(B, L)
    tok, lens = pad(rows)
    check(eng, duration_ckpt, tok, lens, run(eng, tok, lens), f"B={B} L={L}", rows)


def test_batch_of_130_through_chunks(eng, duration_ckpt):
    """B = 130: `predict_duration` runs 128 rows, then 2.  Each chunk gives the bits of its rows run as their own call;
    the last chunk's stages are checked (the taps hold the last call)."""
    rows = list(matrix_rows()) + [matrix_rows()[5], matrix_rows()[0]]
    tok, lens = pad(rows)
    got = dict(dur=eng.predict_duration(tok, lengths=lens))
    got.update(read_taps(eng, 2, tok.shape[1]))
    check(eng, duration_ckpt, tok[128:], lens[128:], dict(got, dur=got["dur"][128:]), "B=130 rows 128-129", rows[128:])
    assert np.array_equal(got["dur"][:128], eng.predict_duration(tok[:128], lengths=lens[:128]))
    assert np.array_equal(got["dur"][128:], eng.predict_duration(tok[128:], lengths=lens[128:]))
    assert np.array_equal(got["dur"][129], got["dur"][0])


def test_long_rows_past_the_acoustic_limit(eng, duration_ckpt):
    """L = 6001 (every stage against float64) and L = 65537 (the head's stages): the duration path has no token limit
    of its own; the acoustic model's 5689 comes from its upsample."""
    row = long_row(LONG_L)
    tok, lens = pad([row])
    check(eng, duration_ckpt, tok, lens, run(eng, tok, lens), f"L={LONG_L}", [row])
    tok = long_row(VERY_LONG_L)[None]
    got = run(eng, tok, None)
    assert np.all(np.isfinite(got["dur"])) and np.all(got["dur"] > 0)
    check(eng, duration_ckpt, tok, None, got, f"L={VERY_LONG_L}")


def test_lengths_null_on_the_device_entry(eng, duration_ckpt):
    """`duration_forward` with lengths = NULL: every position is a token; the same bits as the host call."""
    rows = edge_rows(5, 23)
    tok, _ = pad(rows)
    out = eng.duration_forward(torch.from_numpy(tok).cuda())
    torch.cuda.synchronize()
    got = dict(dur=out.cpu().numpy(), **read_taps(eng, *tok.shape))
    check(eng, duration_ckpt, tok, None, got, "lengths=NULL", rows)
    assert np.array_equal(got["dur"], eng.predict_duration(tok))


def test_rows_are_independent_bit_for_bit(eng):
    """B = 128: rows of every row group and tile have the bits of the same row run alone, and keep them when every other
    row changes its tokens, length and padding.  The encoder scan, the dispatcher's GEMM and the head treat every row
    alike and reduce only within a row."""
    rows = list(matrix_rows())
    tok, lens = pad(rows)
    got = run(eng, tok, lens)
    for b in PROBE:
        n = int(lens[b])
        alone = run(eng, rows[b][None], None)
        assert np.array_equal(got["dur"][b, :n], alone["dur"][0]), b
        assert np.array_equal(got["enc"][b, :n], alone["enc"][0]), b
        assert np.array_equal(got["hid"][b, :n], alone["hid"][0]), b
    rng = np.random.default_rng(8)
    other = [r if b in PROBE else rng.integers(0, 90, int(rng.integers(1, L_MAX + 1))).astype(np.int32)
             for b, r in enumerate(rows)]
    tok2, lens2 = pad(other, L_MAX)
    tok2[:, ::3] = np.where(np.isin(np.arange(128), PROBE)[:, None], tok2[:, ::3], 3)
    tok2[list(PROBE)] = tok[list(PROBE)]
    got2 = run(eng, tok2, lens2)
    for b in PROBE:
        for k in got:
            n = int(lens[b])
            assert np.array_equal(got[k][b, :n], got2[k][b, :n]), (b, k, "changed with the other rows")
        assert np.all(got2["dur"][b, lens[b]:] == 0)


def test_fp16_mode_is_bf16x3(eng):
    """FP16 is a generator mode: the duration model gives the bits of BF16X3 in every tap and output."""
    if eng.mode != "bf16x3":
        pytest.skip("compares FP16 with BF16X3 once, on the bf16x3 engine")
    tok, lens = pad(list(matrix_rows()[:33]))
    eng.set_precision("fp16")
    try:
        a = run(eng, tok, lens)
    finally:
        eng.set_precision("bf16x3")
    b = run(eng, tok, lens)
    for k in a:
        assert np.array_equal(a[k], b[k]), k


def test_dur_hidden_tap_lifetime(eng):
    """dur_hidden is set by a duration call only: an acoustic call leaves it unset, and a call that grows the workspace
    clears it.  Both are refused with VTTS_ERR_BAD_ARG before any copy."""
    from viettts_b200._lib import VttsError

    def refused():
        with pytest.raises(VttsError) as ei:
            eng.debug_read("dur_hidden", (2, 9, 256))
        assert ei.value.code == -1 and "tap dur_hidden is not set" in str(ei.value), str(ei.value)

    tok, lens = pad(edge_rows(2, 9))
    eng.predict_duration(tok, lengths=lens)
    eng.debug_read("dur_hidden", (2, 9, 256))
    frames = np.full((2, 9), 1.5, np.float32)
    eng.predict_mel(tok, frames, lengths=lens)
    refused()
    eng.predict_duration(tok, lengths=lens)
    eng.debug_read("dur_hidden", (2, 9, 256))
    eng.mel2wave(np.zeros((8, 2048, 80), np.float32))                   # a larger workspace
    refused()


# ------------------------------------------------------------------------------------------------ the plan


def plan_rows():
    """token rows for the plan: silence at both ends; ending in a word end; ending in a phoneme; only word ends before
    a trailing silence (nothing left after the trim); two phonemes before a silence; a short padded row"""
    rng = np.random.default_rng(55)
    body = lambda n: rng.integers(4, 90, n).astype(np.int32)            # noqa: E731
    r0 = np.concatenate([[0], body(6), [3], body(4), [3, 0, 3], body(3), [3, 0]])
    r1 = np.concatenate([[0], body(7), [3], body(5), [3]])
    r2 = np.concatenate([[3, 0], body(9), [0, 0], body(2)])
    r3 = np.array([3, 3, 3, 0], np.int32)
    r4 = np.array([17, 22, 0], np.int32)
    r5 = np.array([0, 44, 3, 21, 0], np.int32)
    return [r.astype(np.int32) for r in (r0, r1, r2, r3, r4, r5)]


def plan_ref(tokens, raw, sd):
    """the oracle's glue for one row: (adjusted seconds [L], frames [L], n_frames, n_emit)"""
    d = no.adjust_durations(tokens, np.asarray(raw, np.float32)[None], sd)
    fr, n = no.seconds_to_frames(d)
    kept = no.trim_end_silence([int(t) for t in tokens], d, np.zeros((1, n, 1), np.float32)).shape[1]
    return d[0], fr[0], n, kept


def test_plan_equals_the_oracle_glue(eng):
    """`Engine.tts_plan` against adjust_durations / seconds_to_frames / trim_end_silence fed the raw durations of
    `predict_duration` on the same rows: seconds and frames bit-equal, n_frames and n_emit equal, padding 0."""
    rows = plan_rows()
    tok, lens = pad(rows, 26)
    raw = eng.predict_duration(tok, lengths=lens)
    sil = np.concatenate([raw[b, : lens[b]][rows[b] == 0] for b in range(len(rows))])
    mid = float(np.float32(np.median(sil)))
    assert (sil < mid).any() and (sil > mid).any()
    for sd in (-1.0, mid, 0.5):
        sec, frames, nf, ne = eng.tts_plan(tok, lens, silence_duration=sd)
        for b, r in enumerate(rows):
            n = int(lens[b])
            d, fr, nfr, kept = plan_ref(r, raw[b, :n], sd)
            assert np.array_equal(sec[b, :n], d) and np.array_equal(frames[b, :n], fr), (sd, b)
            assert nf[b] == nfr and ne[b] == kept, (sd, b, nf[b], nfr, ne[b], kept)
            assert np.all(sec[b, n:] == 0) and np.all(frames[b, n:] == 0), (sd, b)
        assert ne[3] == 0                                                # only word ends before the trailing silence
        if sd == 0.5:
            assert ne[4] > 0 and frames[4, 2] > frames[4, :2].sum()      # a trailing silence longer than the rest


BOUNDARY_L = 111


def test_frame_count_boundary_row(eng, duration_ckpt, acoustic_ckpt, golden_dir, tmp_path, monkeypatch):
    """An all-silence row whose silence_duration puts the frame sum where a float32 sum and the float64 one truncate to
    different counts.  `tts_plan`, `tts`, `predict_mel`'s default n_frames, `synthesize_many` and the drop-in
    `predict_mel` / `text2mel` all give the count of `frame_count`."""
    from viettts_b200.engine import get_engine
    from viettts_b200.nat import text2mel as t2m
    tok = np.zeros((1, BOUNDARY_L), np.int32)
    raw = eng.predict_duration(tok)[0]
    sd = boundary_silence_duration(raw, 0.3, 0.32)
    d, fr, n, kept = plan_ref(tok[0], raw, sd)
    assert f32_frame_count(fr) != n, "the row must separate the two definitions"
    print(f"[boundary] silence_duration {float(sd)!r}: float64 {np.sum(fr, dtype=np.float64)!r} -> {n}, "
          f"float32 {np.sum(fr, dtype=np.float32)!r} -> {f32_frame_count(fr)}")
    _, frames, nf, ne = eng.tts_plan(tok, silence_duration=float(sd))
    assert np.array_equal(frames[0], fr) and nf[0] == n and ne[0] == kept
    waves, _ = eng.tts(tok, silence_duration=float(sd))
    assert waves[0].size == kept * config.HOP
    assert eng.predict_mel(tok, fr[None]).shape[1] == n
    assert eng.synthesize_many([(tok[0], fr)])[0].size == n * config.HOP
    for sub in ("assets/infore/nat", "assets/hifigan"):
        (tmp_path / sub).mkdir(parents=True)
    with open(tmp_path / config.ACOUSTIC_CKPT, "wb") as f:
        pickle.dump(acoustic_ckpt, f)
    with open(tmp_path / config.DURATION_CKPT, "wb") as f:
        pickle.dump(duration_ckpt, f)
    monkeypatch.chdir(tmp_path)
    get_engine(0).set_precision(eng.mode)
    assert t2m.predict_mel(tok[0].tolist(), d[None], dropout=False).shape[1] == n
    mel = t2m.text2mel(" ".join(["sil"] * (BOUNDARY_L - 2)), golden_dir / "lexicon_small.txt", silence_duration=float(sd),
                       dropout=False)
    assert mel.shape[1] == kept
