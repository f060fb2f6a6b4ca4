"""The acoustic model's recurrent scans, stage by stage against float64: the encoder BiLSTM (`enc_scan_kernel`), the
Gaussian upsampling (`upsample_kernel`), the autoregressive decoder scan (`decoder_scan_kernel`) and the teacher-forced
zoneout scan (`decoder_tf_scan_kernel`).

Each stage is compared with a float64 computation that starts from the GPU's own input to that stage, read through the
`vtts_debug_read` taps, so each stage's error is measured alone:
  enc      [B,L,512]  float64 TokenEncoder of the row alone, with its true length (ResetCore at the row's end);
  cond     [B,N,512]  float64 upsample of the GPU `enc` of the row and its durations; exactly 0 past n_frames[b];
  mel_pre  [B,N,80]   float64 decoder loop (prenet, both LSTMs, projection) on the GPU `cond`, same keep-masks; the model
                      is causal, so the first n_frames[b] frames of a padded row must match; exactly 0 past them;
  mel      [B,N,80]   the whole float64 chain from the tokens (end to end, L-inf <= 1e-3 as tests/test_gpu_nat.py).
The bounds (BOUND) are at least 4x the error of the plain fp32 oracle on the same utterances and masks
(tests/test_acoustic_scan_bounds.py) and were set from H100 measurements.

The row-group matrix runs ragged batches at every B where the decoder scan's row groups (32 rows) or register tiles
(8 rows) change shape -- a partial last tile, a last group of one row, the 128-row launch maximum -- in every dropout
mode, and checks every row."""
import numpy as np
import pytest
import torch

from helpers.threefry import prenet_keep_masks, zoneout_masks
from oracle import nat_oracle as no
from viettts_b200 import synthetic

pytestmark = pytest.mark.gpu

F64 = torch.float64
MEL_LINF = 1e-3                  # end to end, after the postnet
# per stage and arithmetic mode, L-inf.  Worst measured on an H100 80GB HBM3 (400 W power limit) over every case here:
#   fp32    enc 2.4e-6  cond 1.2e-5  mel_pre 6.1e-6
#   bf16x3  enc 4.1e-5  cond 1.2e-5  mel_pre 3.0e-5
# (cond's error is fp32's cumsum of the durations, largest at N ~ 937; bf16x3's extra error comes from the hoisted
# GEMMs and the convs, the scans are fp32 in both modes).  enc keeps the 1e-4 of tests/test_gpu_nat.py in bf16x3.
BOUND = {"fp32": {"enc": 1e-5, "cond": 5e-5, "mel_pre": 2.5e-5},
         "bf16x3": {"enc": 1e-4, "cond": 5e-5, "mel_pre": 1.2e-4}}
SIZES = [1, 8, 9, 31, 32, 33, 64, 65, 97, 127, 128]
DROPOUT = ["off", "mask", "seed"]
N_MAX = 24                       # frames of the longest row of every matrix batch (row 0)
MASK_SEED = 31
SEED = (0x5EED << 32) | 0xC0FFEE
GROUP_EDGES = (0, 31, 32, 63, 64, 95, 96, 127)

# ------------------------------------------------------------------------------------------------ cases (CPU too)


def _durations(rng, L, n):
    """float32 frame durations of L tokens whose float32 sum is n + 0.5 (int(sum) == n, as the engine computes it)"""
    d = rng.uniform(0.3, 1.7, L)
    d = (d * (n + 0.5) / d.sum()).astype(np.float32)
    assert int(np.sum(d, dtype=np.float32)) == n
    return d


def matrix_rows():
    """The 128 utterances whose first B rows form every matrix batch: (tokens int32 [L_b], durations f32 [L_b], n_b).
    Row 0 has N_MAX frames, row 1 one frame; the others end at frames spread over 1..N_MAX, so that within each row
    group (and each register tile) rows end at different frames.  3..14 tokens."""
    rng = np.random.default_rng(2024)
    rows = []
    for b in range(128):
        n = N_MAX if b == 0 else 1 if b == 1 else 1 + (b * 7) % N_MAX
        L = 3 + (b * 5) % 12
        tk = rng.integers(0, 90, L).astype(np.int32)
        rows.append((tk, _durations(rng, L, n), n))
    return rows


def pad(rows):
    B = len(rows)
    Lmax = max(len(r[0]) for r in rows)
    tokens = np.zeros((B, Lmax), np.int32)
    dur = np.zeros((B, Lmax), np.float32)
    for b, (tk, d, _) in enumerate(rows):
        tokens[b, : len(tk)] = tk
        dur[b, : len(tk)] = d
    lens = np.array([len(r[0]) for r in rows], np.int32)
    nfs = np.array([r[2] for r in rows], np.int32)
    return tokens, dur, lens, nfs


def keep_masks(dmode, B, N):
    """the keep-masks rows 0..B-1 of a call see over N frames: None (off), a fixed 128-row set (mask) or the device's
    documented SEED stream (seed); the masks of a row do not depend on B"""
    if dmode == "off":
        return None
    if dmode == "mask":
        return synthetic.dropout_masks(MASK_SEED, 128, N)[:B]
    return prenet_keep_masks(SEED, range(B), N)


def long_rows():
    """B = 128, L = 100, N = 312 (the config-3 shape)"""
    out = []
    for b in range(128):
        tokens, dur = synthetic.utterance(500 + b, 100, 5.0)
        d, n = no.seconds_to_frames(dur)
        out.append((np.asarray(tokens, np.int32), d[0], n))
    assert all(r[2] == 312 for r in out)
    return out


LONG_CHECKED = sorted(set(range(0, 128, 8)) | set(GROUP_EDGES))


def long_masks():
    return synthetic.dropout_masks(77, 128, 312)


def enc64(ckpt, tk, dtype=F64):
    """the TokenEncoder on one row alone, with its true length: [L,512]"""
    P, S = ckpt["params"], ckpt["aux"]
    with torch.no_grad():
        return no.token_encoder(P, S, tk[None], [len(tk)], dtype)[0]


def cond_of(enc, d, n, dtype=F64):
    """the upsample of one row's encoder output [L,512] (any float tensor) with its durations: [n,512]"""
    with torch.no_grad():
        return no.upsample(torch.as_tensor(enc).to(dtype)[None], torch.as_tensor(d).to(dtype)[None], n)[0][0]


def decode(ckpt, cond, masks, dtype=F64):
    """the decoder loop over a batch of cond [B,N,512]: pre-postnet mel [B,N,80]"""
    with torch.no_grad():
        return no.decode(ckpt["params"], torch.as_tensor(cond).to(dtype), masks, dtype)


def postnet_rows(ckpt, pre, nfs):
    """mel = pre + postnet(pre) of every row at its own length (the postnet's zero padding starts at n_frames[b])"""
    P, S = ckpt["params"], ckpt["aux"]
    out = []
    with torch.no_grad():
        for b, n in enumerate(nfs):
            x = pre[b : b + 1, :n]
            out.append((x + no.postnet(P, S, x, x.dtype))[0])
    return out


# ------------------------------------------------------------------------------------------------ GPU


@pytest.fixture(scope="module", params=["fp32", "bf16x3"])
def eng(acoustic_ckpt, request):
    from viettts_b200.engine import Engine
    e = Engine(0)
    e.load_acoustic(acoustic_ckpt)
    e.load_mel_filterbank()
    e.set_precision(request.param)
    e.mode = request.param
    yield e
    e.close()


_cache = {}


def _cached(key, fn):
    if key not in _cache:
        _cache[key] = fn()
    return _cache[key]


def _run(eng, rows, dmode, masks=None):
    """predict_mel of a ragged batch; returns (mel, enc, cond, mel_pre) as numpy"""
    tokens, dur, lens, nfs = pad(rows)
    B, L = tokens.shape
    N = int(nfs.max())
    kw = dict(masks=masks) if dmode == "mask" else dict(seed=SEED) if dmode == "seed" else {}
    mel = eng.predict_mel(tokens, dur, lengths=lens, n_frames=nfs, **kw)
    return mel, eng.debug_read("enc", (B, L, 512)), eng.debug_read("cond", (B, N, 512)), eng.debug_read("mel_pre", (B, N, 80))


def check_stages(eng, ckpt, rows, idx, masks, enc_ref, mel_ref, got, what):
    """every stage of the rows `idx` of a batch (rows[i] is batch row idx[i]); masks [len(idx),N,2,256] or None;
    enc_ref / mel_ref: float64 per row.  Returns the worst error per stage."""
    mel, enc, cond, pre = got
    bound = BOUND[eng.mode]
    worst = dict(enc=0.0, cond=0.0, mel_pre=0.0, mel=0.0)
    for i, b in enumerate(idx):
        tk, d, n = rows[i]
        e = float(np.abs(enc[b, : len(tk)] - enc_ref[i].numpy()).max())
        assert e <= bound["enc"], (what, b, "enc", e)
        worst["enc"] = max(worst["enc"], e)
        c = cond_of(enc[b, : len(tk)], d, n)
        e = float(np.abs(cond[b, :n] - c.numpy()).max())
        assert e <= bound["cond"], (what, b, "cond", e)
        assert np.all(cond[b, n:] == 0), (what, b, "cond past n_frames")
        worst["cond"] = max(worst["cond"], e)
    pre_ref = decode(ckpt, cond[list(idx)], masks).numpy()
    for i, b in enumerate(idx):
        n = rows[i][2]
        e = float(np.abs(pre[b, :n] - pre_ref[i, :n]).max())
        assert e <= bound["mel_pre"], (what, b, "mel_pre", e)
        assert np.all(pre[b, n:] == 0) and np.all(mel[b, n:] == 0), (what, b, "mel past n_frames")
        worst["mel_pre"] = max(worst["mel_pre"], e)
        e = float(np.abs(mel[b, :n] - mel_ref[i].numpy()).max())
        assert e < MEL_LINF, (what, b, "mel", e)
        worst["mel"] = max(worst["mel"], e)
    print(f"[acoustic_scans] {what} {eng.mode}: " + " ".join(f"{k} {v:.2e}" for k, v in worst.items()))
    return worst


def _matrix_refs(ckpt, dmode):
    """float64 encoder of every matrix row, and the float64 end-to-end mel of every row in this dropout mode"""
    rows = matrix_rows()
    encs = _cached("matrix_enc", lambda: [enc64(ckpt, tk) for tk, _, _ in rows])

    def e2e():
        conds = torch.zeros(128, N_MAX, 512, dtype=F64)
        for b, (tk, d, n) in enumerate(rows):
            conds[b, :n] = cond_of(encs[b], d, n)
        pre = decode(ckpt, conds, keep_masks(dmode, 128, N_MAX))
        return postnet_rows(ckpt, pre, [r[2] for r in rows])
    return rows, encs, _cached(("matrix_mel", dmode), e2e)


@pytest.mark.parametrize("dmode", DROPOUT)
@pytest.mark.parametrize("B", SIZES)
def test_row_group_matrix(eng, acoustic_ckpt, B, dmode):
    """Every row of a ragged batch of B rows, every stage, against float64 (see the module docstring)."""
    rows, encs, mels = _matrix_refs(acoustic_ckpt, dmode)
    rows = rows[:B]
    masks = keep_masks(dmode, B, N_MAX)
    got = _run(eng, rows, dmode, masks)
    assert got[2].shape[1] == N_MAX
    check_stages(eng, acoustic_ckpt, rows, range(B), masks, encs[:B], mels[:B], got, f"B={B} {dmode}")


@pytest.fixture(scope="module")
def long_refs(acoustic_ckpt):
    """float64 encoder and end-to-end mel of the checked rows of the long batch"""
    rows = long_rows()
    sel = [rows[b] for b in LONG_CHECKED]
    P, S = acoustic_ckpt["params"], acoustic_ckpt["aux"]
    with torch.no_grad():
        enc = no.token_encoder(P, S, np.stack([r[0] for r in sel]), [100] * len(sel), F64)
        d = torch.as_tensor(np.stack([r[1] for r in sel])).to(F64)
        cond, _ = no.upsample(enc, d, 312)
        pre = decode(acoustic_ckpt, cond, long_masks()[LONG_CHECKED])
    return rows, list(enc), postnet_rows(acoustic_ckpt, pre, [312] * len(sel))


def test_long_full_batch(eng, acoustic_ckpt, long_refs):
    """B = 128, L = 100, N = 312, MASK: all four stages of every 8th row and of the group-edge rows.  Two identical calls
    give the same bits."""
    rows, encs, mels = long_refs
    masks = long_masks()
    got = _run(eng, rows, "mask", masks)
    check_stages(eng, acoustic_ckpt, [rows[b] for b in LONG_CHECKED], LONG_CHECKED, masks[LONG_CHECKED], encs, mels, got,
                 "B=128 L=100 N=312")
    again = _run(eng, rows, "mask", masks)
    for name, x, y in zip(("mel", "enc", "cond", "mel_pre"), got, again):
        assert np.array_equal(x, y), (name, "a repeated call differs", float(np.abs(x - y).max()))


def l300_rows():
    """B = 8 ragged rows of 251..300 tokens and about 830..937 frames (the longest of the mixed-length workload)"""
    rows = []
    for b in range(8):
        tokens, dur = synthetic.utterance(900 + b, 300 - 7 * b, 15.0 - 0.4 * b)
        d, n = no.seconds_to_frames(dur)
        rows.append((np.asarray(tokens, np.int32), d[0], n))
    return rows


def l300_masks(N):
    return synthetic.dropout_masks(78, 8, N)


def test_long_utterance_300_phonemes_batch8(eng, acoustic_ckpt):
    """B = 8, L = 300, N ~ 937, MASK: every stage of every row (the longest encoder and decoder scans)."""
    rows = l300_rows()
    N = max(r[2] for r in rows)
    masks = l300_masks(N)
    got = _run(eng, rows, "mask", masks)

    def refs():
        encs = [enc64(acoustic_ckpt, r[0]) for r in rows]
        conds = torch.zeros(8, N, 512, dtype=F64)
        for b, (_, d, n) in enumerate(rows):
            conds[b, :n] = cond_of(encs[b], d, n)
        return encs, postnet_rows(acoustic_ckpt, decode(acoustic_ckpt, conds, masks), [r[2] for r in rows])
    encs, mels = _cached("l300", refs)
    check_stages(eng, acoustic_ckpt, rows, range(8), masks, encs, mels, got, f"B=8 L=300 N={N}")


# ------------------------------------------------------------------------------------------------ determinism


def test_rows_are_independent_bit_for_bit(eng):
    """MASK mode (in SEED mode a row's stream depends on its row index), B = 128, N = 312.  Row b of the batch has the
    bits of the same row run alone, for rows of every group, and keeps them when every OTHER row changes its tokens,
    length, frame count and masks.  This holds exactly because no kernel of the path reduces across rows and every
    per-row reduction runs in an order fixed by the layer's shape alone: the hoisted GEMMs and convs sum K in the same
    order wherever the row sits in a tile, and the scans' butterfly reductions treat every row of a register tile alike."""
    rows = long_rows()
    masks = long_masks()
    got = _run(eng, rows, "mask", masks)
    probe = (0, 31, 32, 63, 64, 96, 127)
    for b in probe:
        alone = _run(eng, [rows[b]], "mask", masks[b : b + 1])
        for name, x, y in zip(("mel", "enc", "cond", "mel_pre"), got, alone):
            assert np.array_equal(x[b], y[0]), (b, name, float(np.abs(x[b] - y[0]).max()))
    # the other rows: other utterances, other lengths and frame counts, other masks
    rng = np.random.default_rng(5)
    other = list(rows)
    for b in range(128):
        if b not in probe:
            L = int(rng.integers(5, 100))
            tokens, dur = synthetic.utterance(1000 + b, L, float(rng.uniform(0.2, 4.9)))
            d, n = no.seconds_to_frames(dur)
            other[b] = (np.asarray(tokens, np.int32), d[0], n)
    masks2 = synthetic.dropout_masks(99, 128, 312)
    masks2[list(probe)] = masks[list(probe)]
    got2 = _run(eng, other, "mask", masks2)
    for b in probe:
        for name, x, y in zip(("mel", "enc", "cond", "mel_pre"), got, got2):
            assert np.array_equal(x[b], y[b]), (b, name, "changed with the other rows", float(np.abs(x[b] - y[b]).max()))


# ------------------------------------------------------------------------------------------------ teacher forced


def _tf_rows(B):
    rng = np.random.default_rng(41)
    out = []
    for b in range(B):
        L = int(rng.integers(6, 18))
        tokens, dur = synthetic.utterance(700 + b, L, None)
        d, n = no.seconds_to_frames(dur)
        out.append((np.asarray(tokens, np.int32), d[0], max(n, 1)))
    return out


TF_ROWS = GROUP_EDGES


@pytest.mark.parametrize("dmode", DROPOUT)
def test_teacher_forced_four_zoneout_launches(eng, acoustic_ckpt, dmode):
    """B = 128 rows of the teacher-forced pass (four zoneout scan launches of 32 rows): mel1 and mel2 of the rows at the
    launch edges against float64, fed the same masks.  In SEED mode the masks are rebuilt from the documented stream:
    the prenet keep draw of `prenet_act_kernel` and the zoneout draw of `zone_keep`, both keyed by the row's index in
    the call, so rows 32+ test the zoneout launches' row offset."""
    B = 128
    rows = _tf_rows(B)
    tokens, dur, lens, nfs = pad(rows)
    N = int(nfs.max())
    mels_in = synthetic.mel_input(12, B, N)
    if dmode == "mask":
        rng = np.random.default_rng(13)
        keep = (rng.random((B, N, 2, 256)) < 0.5).astype(np.uint8)
        zone = (rng.random((B, N, 4, 512)) < 0.1).astype(np.uint8)
        m1, m2 = eng.teacher_forced(tokens, dur, mels_in, lengths=lens, n_frames=nfs, keep_masks=keep, zone_masks=zone)
    else:
        m1, m2 = eng.teacher_forced(tokens, dur, mels_in, lengths=lens, n_frames=nfs, seed=SEED if dmode == "seed" else None)
        if dmode == "seed":
            keep, zone = prenet_keep_masks(SEED, range(B), N), zoneout_masks(SEED, range(B), N)
            sel_k, sel_z = keep[list(TF_ROWS)], zone[list(TF_ROWS)]
            assert 0.48 < sel_k.mean() < 0.52 and 0.09 < sel_z.mean() < 0.11, (sel_k.mean(), sel_z.mean())
            assert not np.array_equal(zone[0], zone[32]) and not np.array_equal(keep[0], keep[32])
    worst = 0.0
    for b in TF_ROWS:
        tk, d, n = rows[b]
        km, zm = (None, None) if dmode == "off" else (keep[b : b + 1, :n], zone[b : b + 1, :n])
        r1, r2 = no.teacher_forced(acoustic_ckpt, tk[None], np.array([len(tk)]), d[None], mels_in[b : b + 1, :n], km, zm, dtype=F64)
        e1, e2 = float(np.abs(m1[b, :n] - r1[0]).max()), float(np.abs(m2[b, :n] - r2[0]).max())
        assert e1 < MEL_LINF and e2 < MEL_LINF, (dmode, b, e1, e2)
        assert np.all(m1[b, n:] == 0) and np.all(m2[b, n:] == 0)
        worst = max(worst, e1, e2)
    print(f"[acoustic_scans] teacher forced B=128 {dmode} {eng.mode}: mel1/mel2 {worst:.2e}")


def test_gta_seed_mode_ragged_wav_lengths(eng, acoustic_ckpt):
    """Engine.gta at B = 40 (two zoneout launches, the second of 8 rows) in SEED mode with ragged wav_lengths, against
    nat_oracle.gta_forward fed the restated masks.  A row cut at wav_lengths[b] // 256 = n frames runs the postnet on
    its first n frames alone, so its oracle is the teacher-forced pass over those frames of the same ground-truth mel."""
    B, L, N = 40, 14, 32
    S = 256 * N
    rng = np.random.default_rng(17)
    wav = (np.tanh(rng.standard_normal((B, S)) * 0.4) * 20000).astype(np.int16)
    tok = np.stack([np.asarray(synthetic.utterance(800 + b, L, None)[0], np.int32) for b in range(B)])
    dur_sec = np.stack([synthetic.utterance(800 + b, L, S / 16000)[1][0] for b in range(B)])
    wl = np.array([S if b % 3 == 0 else 256 * int(rng.integers(2, N)) + int(rng.integers(0, 256)) for b in range(B)], np.int32)
    wl[1] = 256                                   # one frame
    out, gt = eng.gta(wav, tok, dur_sec, lengths=np.full(B, L, np.int32), wav_lengths=wl, seed=SEED, return_gt=True)
    keep, zone = prenet_keep_masks(SEED, range(B), N), zoneout_masks(SEED, range(B), N)
    worst = 0.0
    for b in (0, 1, 2, 30, 31, 32, 33, 38, 39):
        n = int(wl[b]) // 256
        gt_ref, ref = no.gta_forward(acoustic_ckpt, wav[b : b + 1], tok[b : b + 1], np.array([L]), dur_sec[b : b + 1], keep[b : b + 1],
                                     zone[b : b + 1], dtype=F64)
        if n < N:
            inp = np.concatenate([np.zeros_like(gt_ref[:, :1]), gt_ref[:, : n - 1]], axis=1)
            frames = (dur_sec[b : b + 1] * np.float32(16000)) / np.float32(256)
            _, ref = no.teacher_forced(acoustic_ckpt, tok[b : b + 1], np.array([L]), frames, inp, keep[b : b + 1, :n], zone[b : b + 1, :n], F64)
        e_gt, e = float(np.abs(gt[b] - gt_ref[0]).max()), float(np.abs(out[b, :n] - ref[0, :n]).max())
        assert e_gt < 2e-3 and e < 2e-3, (b, n, e_gt, e)         # includes the fp32 STFT's error on the teacher-forcing input
        assert np.all(out[b, n:] == 0), b
        worst = max(worst, e)
    print(f"[acoustic_scans] gta B=40 seed {eng.mode}: mel2 {worst:.2e}")


# ------------------------------------------------------------------------------------------------ long token sequences


def test_upsample_beyond_48k_shared_memory(eng, acoustic_ckpt):
    """L = 1400 tokens with durations of about 0.2 frames (N ~ 280): the upsample kernel needs (L + 8 L) * 4 B > 48 KB of
    shared memory and takes the opt-in path; the encoder scans 1400 steps.  enc, cond and mel_pre of the row."""
    rng = np.random.default_rng(1400)
    L, n = 1400, 280
    rows = [(rng.integers(0, 90, L).astype(np.int32), _durations(rng, L, n), n)]
    masks = synthetic.dropout_masks(14, 1, n)
    got = _run(eng, rows, "mask", masks)
    enc = enc64(acoustic_ckpt, rows[0][0])
    pre = decode(acoustic_ckpt, cond_of(enc, rows[0][1], n)[None], masks)
    check_stages(eng, acoustic_ckpt, rows, [0], masks, [enc], postnet_rows(acoustic_ckpt, pre, [n]), got, f"B=1 L={L} N={n}")


def test_upsample_limit_fails_cleanly(eng, acoustic_ckpt):
    """L = 5700 needs more than the upsample kernel's 200 KB of shared memory: the call fails with VTTS_ERR_BAD_ARG,
    and the same engine then runs a normal call with the bits it gave before.  (`enc` is compared within each row's
    length: its padded positions come from workspace rows the encoder convs never write, which the failed call has
    overwritten; nothing reads them.)"""
    from viettts_b200._lib import VttsError
    rows = matrix_rows()[:9]
    masks = keep_masks("mask", 9, N_MAX)
    before = _run(eng, rows, "mask", masks)
    rng = np.random.default_rng(5700)
    L = 5700
    tk, d = rng.integers(0, 90, L).astype(np.int32), _durations(rng, L, 40)
    with pytest.raises(VttsError) as ei:
        eng.predict_mel(tk[None], d[None], n_frames=[40])
    assert ei.value.code == -1 and "too long for the upsample kernel" in str(ei.value), str(ei.value)
    after = _run(eng, rows, "mask", masks)
    for name, x, y in zip(("mel", "cond", "mel_pre"), before[:1] + before[2:], after[:1] + after[2:]):
        assert np.array_equal(x, y), name
    for b, (tk, _, _) in enumerate(rows):
        assert np.array_equal(before[1][b, : len(tk)], after[1][b, : len(tk)]), ("enc", b)
