"""The teacher-forced pass (`vtts_acoustic_teacher_run`: `Engine.teacher_forced`, `Engine.gta`), stage by stage against
float64.  Each stage starts from the GPU's own input to it, read through the `vtts_debug_read` taps, so each stage's
error is measured alone:
  cond     dec_in[..., :512]   float64 upsample of the GPU `enc` of the row and its durations; exactly 0 past n_frames[b]
  p2       dec_in[..., 512:]   float64 prenet (`tf_prenet`) of mels_in with the same keep masks, every frame; per element
                               |err| <= P2_TOL * S, S the conv-dispatch scale |x|.|W| carried through both layers and
                               the 1 / 0.5 keep scale (tests/test_gpu_conv_dispatch.py)
  dec_out  [B,N,1024]          float64 zoneout scan (`zoneout_decode`) of the GPU `dec_in` with the same zone masks,
                               frames < n_frames[b] (the scan is causal; it runs every row over all N frames); this
                               includes the hoisted input GEMMs (PK_TF_L0) and decoder_tf_scan_kernel
  mel_pre  [B,N,80] (= mel1)   float64 projection of the GPU `dec_out`; exactly 0 past n_frames[b]
  mel2     [B,N,80]            float64 postnet of the GPU mel1, each row at its own length; exactly 0 past n_frames[b]
BOUND is at least 4x the error of the plain fp32 oracle fed the float64 stage input on every case here
(tests/test_teacher_forced_bounds.py), and was set from H100 measurements.

Cases: ragged batches at every B where the zoneout launches (<= 32 rows) or their register tiles (8 rows) change shape,
in every dropout mode (OFF, MASK, SEED and REFERENCE, the latter drawn for the call's own B and N); N = 1, 2 and 3;
MASK runs with exactly one zoneout plane always on; two long batches; exact row independence; FP16 mode equal to
BF16X3; GTA with ragged wav lengths; and the taps' own lifetime."""
import functools

import numpy as np
import pytest
import torch

from helpers.threefry import prenet_keep_masks, zoneout_masks
from oracle import nat_oracle as no
from test_gpu_acoustic_scans import (BOUND as SCAN_BOUND, F64, LONG_CHECKED, N_MAX, SEED, _durations, cond_of,
                                     l300_masks, l300_rows, long_masks, long_rows, matrix_rows, pad, postnet_rows)
from viettts_b200 import jaxrng, synthetic

pytestmark = pytest.mark.gpu

P2_TOL = {"fp32": 2e-6, "bf16x3": 2e-5}          # the conv dispatcher's TOL (tests/test_gpu_conv_dispatch.py)
# per stage and arithmetic mode, L-inf.  Worst measured on an H100 80GB HBM3 (700 W power limit) over every case here:
#   fp32    dec_out 7.8e-7  mel_pre 5.9e-6  mel2 2.4e-6   (p2 2.4e-8 S)
#   bf16x3  dec_out 3.6e-5  mel_pre 3.1e-5  mel2 2.2e-5   (p2 4.3e-7 S)
# and of the plain fp32 oracle (tests/test_teacher_forced_bounds.py): dec_out 1.8e-6  mel_pre 2.7e-6  mel2 1.4e-6.
# bf16x3's extra error comes from the hoisted input GEMMs, the projection and the postnet; the scan is fp32 in both.
BOUND = {"fp32": {"dec_out": 1e-5, "mel_pre": 2.5e-5, "mel2": 1e-5},
         "bf16x3": {"dec_out": 1.5e-4, "mel_pre": 1.5e-4, "mel2": 1e-4}}
STAGES = ("cond", "p2", "dec_out", "mel_pre", "mel2")
SIZES = [1, 8, 9, 31, 32, 33, 40, 64, 65, 97, 127, 128]
DROPOUT = ["off", "mask", "seed", "reference"]
REF_RNG = (0x12345678, 0x9ABCDEF0)                # the checkpoint key of REFERENCE mode
PROBE = (0, 31, 32, 63, 64, 96, 127)

# ------------------------------------------------------------------------------------------------ cases (CPU too)


def zone_set(seed, B, N):
    """uint8 [B,N,4,512] Bernoulli(0.1) zoneout masks (1 = keep the previous state)"""
    rng = np.random.default_rng(seed)
    return (rng.random((B, N, 4, 512)) < 0.1).astype(np.uint8)


@functools.lru_cache(maxsize=None)
def tf_masks(dmode, B, N):
    """(keep [B,N,2,256], zone [B,N,4,512]) a call of B rows and N frames applies: None (off), the first B rows of a
    fixed 128-row set (mask), the device's documented SEED stream (seed) or the reference's whole-batch draws for this
    B and N (reference)"""
    if dmode == "off":
        return None, None
    if dmode == "mask":
        return synthetic.dropout_masks(31, 128, N)[:B], zone_set(32, 128, N)[:B]
    if dmode == "seed":                           # a row's SEED masks do not depend on B
        if B < 128:
            keep, zone = tf_masks("seed", 128, N)
            return keep[:B], zone[:B]
        return prenet_keep_masks(SEED, range(B), N), zoneout_masks(SEED, range(B), N)
    return jaxrng.teacher_forced_masks(np.array(REF_RNG, np.uint32), B, N)


def matrix_mels():
    return synthetic.mel_input(21, 128, N_MAX)


def short_rows(n):
    """40 rows of 3..14 tokens, every one n frames long"""
    rng = np.random.default_rng(100 + n)
    rows = []
    for b in range(40):
        L = 3 + (b * 5) % 12
        rows.append((rng.integers(0, 90, L).astype(np.int32), _durations(rng, L, n), n))
    return rows


def plane_masks(which):
    """MASK mode at B = 40, N_MAX: random keep masks, zoneout plane `which` (h0, c0, h1, c1) always on, the others off"""
    zone = np.zeros((40, N_MAX, 4, 512), np.uint8)
    zone[:, :, which] = 1
    return synthetic.dropout_masks(33, 40, N_MAX), zone


def long_tf():
    """B = 128, L = 100, N = 312, MASK: rows, mels_in, keep, zone"""
    return long_rows(), synthetic.mel_input(312, 128, 312), long_masks(), zone_set(78, 128, 312)


def l300_tf():
    """B = 8, L = 251..300, N ~ 937, MASK: rows, mels_in, keep, zone"""
    rows = l300_rows()
    N = max(r[2] for r in rows)
    return rows, synthetic.mel_input(300, 8, N), l300_masks(N), zone_set(79, 8, N)


GTA_B, GTA_L, GTA_N = 40, 14, 32


def gta_case():
    """Engine.gta at B = 40, L = 14, N = 32, SEED: (wav int16, tokens, durations in seconds, wav_lengths, n_frames)"""
    S = 256 * GTA_N
    rng = np.random.default_rng(17)
    wav = (np.tanh(rng.standard_normal((GTA_B, S)) * 0.4) * 20000).astype(np.int16)
    tok = np.stack([np.asarray(synthetic.utterance(800 + b, GTA_L, None)[0], np.int32) for b in range(GTA_B)])
    dur_sec = np.stack([synthetic.utterance(800 + b, GTA_L, S / 16000)[1][0] for b in range(GTA_B)])
    wl = np.array([S if b % 3 == 0 else 256 * int(rng.integers(2, GTA_N)) + int(rng.integers(0, 256)) for b in range(GTA_B)], np.int32)
    wl[1] = 256                                   # one frame
    return wav, tok, dur_sec, wl, np.clip(wl // 256, 1, GTA_N)


def gta_frames(dur_sec):
    """gta.py:37: durations in frames, float32 as the library computes them"""
    return (np.asarray(dur_sec, np.float32) * np.float32(16000)) / np.float32(256)


def _w(P, name):
    return no._t(P[no.A + name]["w"], F64)


def p2_scale(P, mels_in, keep):
    """S of every p2 element: |x|.|W1| through the first keep scale, then .|W2| through the second ([B,N,256])"""
    with torch.no_grad():
        a = torch.as_tensor(np.asarray(mels_in)).double().abs() @ _w(P, "linear_1").abs()
        k = None if keep is None else torch.as_tensor(np.asarray(keep)).double()
        if k is not None:
            a = k[:, :, 0] * a * 2
        a = a @ _w(P, "linear_2").abs()
        return a if k is None else k[:, :, 1] * a * 2


def stage_refs(ckpt, rows, got, mels_in, keep, zone):
    """float64 reference of every stage of rows `rows` ([(tokens, durations, n)]) from the GPU's own stage inputs `got`
    (dicts of numpy arrays with the same rows): (cond per row, p2, S of p2, dec_out, mel_pre, mel2 per row)"""
    P = ckpt["params"]
    conds = [cond_of(got["enc"][i, : len(tk)], d, n).numpy() for i, (tk, d, n) in enumerate(rows)]
    with torch.no_grad():
        p2 = no.tf_prenet(P, np.asarray(mels_in, np.float64), keep, F64).numpy()
        s = p2_scale(P, mels_in, keep).numpy()
        h = no.zoneout_decode(P, got["dec_in"].astype(np.float64), zone, F64).numpy()
        pre = no.project(P, got["dec_out"].astype(np.float64), F64).numpy()
    mel2 = [m.numpy() for m in postnet_rows(ckpt, torch.from_numpy(got["mel_pre"]).double(), [r[2] for r in rows])]
    return conds, p2, s, h, pre, mel2


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


def read_taps(eng, B, L, N):
    return dict(enc=eng.debug_read("enc", (B, L, 512)), dec_in=eng.debug_read("dec_in", (B, N, 768)),
                dec_out=eng.debug_read("dec_out", (B, N, 1024)), mel_pre=eng.debug_read("mel_pre", (B, N, 80)))


def run_tf(eng, rows, mels_in, dmode, keep=None, zone=None):
    """Engine.teacher_forced of a ragged batch: every tap and output as numpy (mel1, mel2, enc, dec_in, dec_out, mel_pre)"""
    tokens, dur, lens, nfs = pad(rows)
    B, L = tokens.shape
    N = mels_in.shape[1]
    kw = dict(keep_masks=keep, zone_masks=zone) if dmode == "mask" else dict(seed=SEED) if dmode == "seed" else \
        dict(rng=REF_RNG) if dmode == "reference" else {}
    m1, m2 = eng.teacher_forced(tokens, dur, mels_in, lengths=lens, n_frames=nfs, **kw)
    return dict(mel1=m1, mel2=m2, **read_taps(eng, B, L, N))


def check(eng, ckpt, rows, idx, got, mels_in, keep, zone, what):
    """every stage of the batch rows `idx` (rows[i] is batch row idx[i]; mels_in, keep and zone hold those rows) against
    float64.  Returns the worst error per stage (p2: the worst |err| / S)."""
    bound = BOUND[eng.mode]
    sel = list(idx)
    g = {k: v[sel] for k, v in got.items()}
    assert np.array_equal(g["mel1"], g["mel_pre"]), (what, "mel1 differs from the mel_pre tap")
    conds, p2, s, h, pre, mel2 = stage_refs(ckpt, rows, g, mels_in, keep, zone)
    worst = dict.fromkeys(STAGES, 0.0)
    err = np.abs(g["dec_in"][..., 512:] - p2)
    bad = err > P2_TOL[eng.mode] * s
    assert not bad.any(), (what, "p2", np.argwhere(bad)[:4], float(err[bad].max()))
    worst["p2"] = float((err / np.maximum(s, 1e-300)).max())
    for i, (tk, d, n) in enumerate(rows):
        e = dict(cond=np.abs(g["dec_in"][i, :n, :512] - conds[i]).max(), dec_out=np.abs(g["dec_out"][i, :n] - h[i, :n]).max(),
                 mel_pre=np.abs(g["mel_pre"][i, :n] - pre[i, :n]).max(), mel2=np.abs(g["mel2"][i, :n] - mel2[i]).max())
        for k, v in e.items():
            assert v <= (SCAN_BOUND[eng.mode]["cond"] if k == "cond" else bound[k]), (what, sel[i], k, float(v))
            worst[k] = max(worst[k], float(v))
        assert np.all(g["dec_in"][i, n:, :512] == 0), (what, sel[i], "cond past n_frames")
        assert np.all(g["mel_pre"][i, n:] == 0) and np.all(g["mel2"][i, n:] == 0), (what, sel[i], "mel past n_frames")
    print(f"[teacher_forced] {what} {eng.mode}: " + " ".join(f"{k} {v:.2e}" for k, v in worst.items()))
    return worst


@pytest.mark.parametrize("dmode", DROPOUT)
@pytest.mark.parametrize("B", SIZES)
def test_launch_and_tile_edges(eng, acoustic_ckpt, B, dmode):
    """Every row of a ragged batch of B rows (3..14 tokens; row 1 one frame, the others ending over 1..N_MAX), every
    stage, in every dropout mode."""
    rows = matrix_rows()[:B]
    mels = matrix_mels()[:B]
    keep, zone = tf_masks(dmode, B, N_MAX)
    got = run_tf(eng, rows, mels, dmode, keep, zone)
    check(eng, acoustic_ckpt, rows, range(B), got, mels, keep, zone, f"B={B} {dmode}")


@pytest.mark.parametrize("dmode", DROPOUT)
@pytest.mark.parametrize("n", [1, 2, 3])
def test_short_sequences(eng, acoustic_ckpt, n, dmode):
    """N = 1, 2, 3 at B = 40 with every row at full length: the skewed LSTM1 step of the last frame and the first h1
    fetch (frame 1) run at the sequence's end."""
    rows = short_rows(n)
    mels = synthetic.mel_input(50 + n, 40, n)
    keep, zone = tf_masks(dmode, 40, n)
    got = run_tf(eng, rows, mels, dmode, keep, zone)
    check(eng, acoustic_ckpt, rows, range(40), got, mels, keep, zone, f"N={n} {dmode}")


@pytest.mark.parametrize("which", range(4), ids=["h0", "c0", "h1", "c1"])
def test_single_zoneout_plane(eng, acoustic_ckpt, which):
    """MASK at B = 40 with exactly one zoneout plane on everywhere (that state stays at zero): a plane read from the
    wrong place, or applied to the wrong state, shows at once."""
    rows = matrix_rows()[:40]
    mels = matrix_mels()[:40]
    keep, zone = plane_masks(which)
    got = run_tf(eng, rows, mels, "mask", keep, zone)
    check(eng, acoustic_ckpt, rows, range(40), got, mels, keep, zone, f"plane {which}")


def test_long_utterance_300_phonemes_batch8(eng, acoustic_ckpt):
    """B = 8, L = 300, N ~ 937, MASK: every stage of every row."""
    rows, mels, keep, zone = l300_tf()
    got = run_tf(eng, rows, mels, "mask", keep, zone)
    check(eng, acoustic_ckpt, rows, range(8), got, mels, keep, zone, f"B=8 L=300 N={mels.shape[1]}")


def test_long_full_batch(eng, acoustic_ckpt):
    """B = 128, L = 100, N = 312, MASK: every 8th row and the launch-edge rows."""
    rows, mels, keep, zone = long_tf()
    got = run_tf(eng, rows, mels, "mask", keep, zone)
    idx = LONG_CHECKED
    check(eng, acoustic_ckpt, [rows[b] for b in idx], idx, got, mels[idx], keep[idx], zone[idx], "B=128 N=312")


NAMES = ("mel1", "mel2", "enc", "dec_in", "dec_out", "mel_pre")


def test_rows_are_independent_bit_for_bit(eng):
    """MASK, B = 128, N = 312: rows of every launch have the bits of the same row run alone (at its own N), and keep
    them when every other row changes its tokens, length, frame count, input mel and masks.  This holds exactly: no
    kernel of the pass reduces across rows, the hoisted GEMMs and the postnet convs sum K in an order fixed by the
    layer's shape, prenet_act_kernel is elementwise, and decoder_tf_scan_kernel's butterfly reductions treat every row
    of a register tile alike, with the row's masks indexed by its row in the call."""
    rows, mels, keep, zone = long_tf()
    got = run_tf(eng, rows, mels, "mask", keep, zone)
    for b in PROBE:
        alone = run_tf(eng, [rows[b]], mels[b : b + 1], "mask", keep[b : b + 1], zone[b : b + 1])
        for name in NAMES:
            assert np.array_equal(got[name][b], alone[name][0]), (b, name, float(np.abs(got[name][b] - alone[name][0]).max()))
    rng = np.random.default_rng(6)
    other = list(rows)
    for b in range(128):
        if b not in PROBE:
            L = int(rng.integers(5, 100))
            tokens, dur = synthetic.utterance(1100 + b, L, float(rng.uniform(0.2, 4.9)))
            d, n = no.seconds_to_frames(dur)
            other[b] = (np.asarray(tokens, np.int32), d[0], max(n, 1))
    p = list(PROBE)
    mels2, keep2, zone2 = synthetic.mel_input(99, 128, 312), synthetic.dropout_masks(98, 128, 312), zone_set(97, 128, 312)
    mels2[p], keep2[p], zone2[p] = mels[p], keep[p], zone[p]
    got2 = run_tf(eng, other, mels2, "mask", keep2, zone2)
    for b in PROBE:
        for name in NAMES:
            assert np.array_equal(got[name][b], got2[name][b]), (b, name, "changed with the other rows")


def test_fp16_mode_is_bf16x3(eng):
    """FP16 is a generator mode: the teacher-forced pass gives the bits of BF16X3 in every tap and output."""
    if eng.mode != "bf16x3":
        pytest.skip("compares FP16 with BF16X3 once, on the bf16x3 engine")
    rows = matrix_rows()[:40]
    mels = matrix_mels()[:40]
    eng.set_precision("fp16")
    try:
        a = run_tf(eng, rows, mels, "seed")
    finally:
        eng.set_precision("bf16x3")
    b = run_tf(eng, rows, mels, "seed")
    for name in NAMES:
        assert np.array_equal(a[name], b[name]), (name, float(np.abs(a[name] - b[name]).max()))


def test_gta_seed_mode_ragged_wav_lengths(eng, acoustic_ckpt):
    """Engine.gta at B = 40 (two zoneout launches, the second of 8 rows) in SEED mode with ragged wav_lengths.  p2 is
    checked against the prenet of the GPU's own ground-truth mel shifted by one frame, so the STFT's error stays out of
    the later stages."""
    wav, tok, dur_sec, wl, nfs = gta_case()
    out, gt = eng.gta(wav, tok, dur_sec, lengths=np.full(GTA_B, GTA_L, np.int32), wav_lengths=wl, seed=SEED, return_gt=True)
    got = dict(mel1=eng.debug_read("mel_pre", (GTA_B, GTA_N, 80)), mel2=out, **read_taps(eng, GTA_B, GTA_L, GTA_N))
    mels_in = np.concatenate([np.zeros_like(gt[:, :1]), gt[:, :-1]], axis=1)
    keep, zone = tf_masks("seed", GTA_B, GTA_N)
    frames = gta_frames(dur_sec)
    rows = [(tok[b], frames[b], int(nfs[b])) for b in range(GTA_B)]
    check(eng, acoustic_ckpt, rows, range(GTA_B), got, mels_in, keep, zone, "gta B=40 seed")


def test_taps_do_not_outlive_their_call(acoustic_ckpt, hifigan_params):
    """A tap is readable only for the call that set it: a call that grows the workspace frees what the taps pointed
    into, so they are cleared, and a call that does not produce a tap leaves it unset.  Both are refused with
    VTTS_ERR_BAD_ARG before any copy."""
    from viettts_b200._lib import VttsError
    from viettts_b200.engine import Engine
    e = Engine(0)
    try:
        e.load_acoustic(acoustic_ckpt)
        e.load_duration(synthetic.duration_ckpt(1234))
        e.load_hifigan(hifigan_params)

        def refused(name, shape):
            with pytest.raises(VttsError) as ei:
                e.debug_read(name, shape)
            assert ei.value.code == -1 and f"tap {name} is not set" in str(ei.value), str(ei.value)

        rows = matrix_rows()[:2]
        tokens, dur, lens, nfs = pad(rows)
        B, L = tokens.shape
        mel = e.predict_mel(tokens, dur, lengths=lens, n_frames=nfs)
        for name, shape in (("enc", (B, L, 512)), ("cond", (B, N_MAX, 512)), ("mel_pre", (B, N_MAX, 80)),
                            ("dec_out", (B, N_MAX, 1024))):
            e.debug_read(name, shape)
        refused("dec_in", (B, N_MAX, 768))
        e.mel2wave(np.tile(mel, (4, 20, 1)))                               # 8 rows of 480 frames: a larger workspace
        for name, shape in (("enc", (B, L, 512)), ("cond", (B, N_MAX, 512)), ("mel_pre", (B, N_MAX, 80)),
                            ("dec_out", (B, N_MAX, 1024))):
            refused(name, shape)
        got = run_tf(e, rows, matrix_mels()[:2], "off")
        assert np.array_equal(got["mel1"], got["mel_pre"])
        refused("cond", (B, N_MAX, 512))                                    # the teacher-forced cond is dec_in[..., :512]
        e.predict_duration(tokens, lengths=lens)
        e.debug_read("enc", (B, L, 512))
        for name, shape in (("cond", (B, N_MAX, 512)), ("mel_pre", (B, N_MAX, 80)), ("dec_in", (B, N_MAX, 768)),
                            ("dec_out", (B, N_MAX, 1024))):
            refused(name, shape)
    finally:
        e.close()
