"""GPU: the log-mel kernel (csrc/melspec.cu) against float64 MelFilter at every frame position, signal class, batch edge
and filterbank; the ground-truth half of Engine.gta; and the argument checks and filterbank bookkeeping of the Engine.

Every comparison is oracle/mel_oracle.py `mel_error` within TOL units, the tolerance test_melspec_cpu.py pins against
the kernel's fp32 arithmetic: |exp(got) - max(m64, 1e-5)| <= TOL scale, and bins clipped on both sides are log(1e-5)
bit for bit."""
import numpy as np
import pytest
import torch

from oracle import mel_oracle as mo
from test_melspec_cpu import SIGNALS, TOL, banks, error_units, signal, three_minutes
from viettts_b200 import synthetic

pytestmark = pytest.mark.gpu
WORST = {}           # signal class -> worst units seen on the device (printed by test_report_worst_per_class)


@pytest.fixture(scope="module")
def eng():
    from viettts_b200.engine import Engine
    e = Engine(0)
    e.load_mel_filterbank()
    yield e
    e.close()


@pytest.fixture(scope="module")
def acoustic_eng(acoustic_ckpt):
    from viettts_b200.engine import Engine
    e = Engine(0)
    e.load_acoustic(acoustic_ckpt)
    yield e
    e.close()


def _check(got, y, fb, what):
    e, bad = error_units(got, y, fb)
    WORST[what] = max(WORST.get(what, 0.0), e)
    assert bad == 0, what
    assert e <= TOL, (what, e)
    return e


# ---- frame positions x signal classes ----------------------------------------------------------------------------

@pytest.mark.parametrize("S", range(512, 4608 + 1, 256))
def test_every_frame_position(eng, S):
    """F = S / 256 = 2 .. 18: odd and even F (the lone last frame), frames on the reflect path at both ends and the
    first and last pairs on the interior path (256 fa >= 384 and 256 fa + 896 <= S)"""
    fb = banks()["default"]
    for name in SIGNALS:
        y = signal(name, 3, S, seed=7)
        got = eng.melspec(y)
        assert got.shape == (3, S // 256, 80)
        _check(got, y, fb, name)


def test_three_minute_row(eng):
    y = three_minutes(1)
    _check(eng.melspec(y), y, banks()["default"], "3 min")


def test_report_worst_per_class(eng):
    """runs after the tests above (file order): the worst device error per class over TOL, next to the emulation's"""
    fb = banks()["default"]
    for name, worst in WORST.items():
        if name not in SIGNALS:
            print(f"{name}: device {worst:.3f} units = {worst / TOL:.3f} TOL")
            continue
        emu = max(error_units(mo.emulate(y, fb), y, fb)[0] for y in (signal(name, 3, S, seed=7) for S in (512, 768, 4608)))
        print(f"{name}: device {worst:.3f} units = {worst / TOL:.3f} TOL; emulation {emu:.3f} units")


# ---- batch -----------------------------------------------------------------------------------------------------

def test_row_bits_do_not_depend_on_batch_position(eng):
    S = 2304
    rows = np.concatenate([signal(n, 3, S, seed=2) for n in ("noise", "chirp", "clicks")])       # 9 distinct rows
    alone = np.stack([eng.melspec(rows[b : b + 1])[0] for b in range(len(rows))])
    assert np.array_equal(eng.melspec(rows), alone)
    perm = np.random.default_rng(0).permutation(len(rows))
    assert np.array_equal(eng.melspec(rows[perm]), alone[perm])


def test_grid_y_limit(eng):
    """B = 65535 rows (the grid's y limit) run and match the same rows alone; B = 65536 fails with VTTS_ERR_BAD_ARG"""
    from viettts_b200._lib import VttsError
    B, S = 65535, 512
    y = np.random.default_rng(5).standard_normal((B, S), dtype=np.float32) * np.float32(0.1)
    got = eng.melspec(y)
    for b in (0, 1, 4096, 32767, 65533, 65534):
        assert np.array_equal(got[b], eng.melspec(y[b : b + 1])[0]), b
    _check(got[-3:], y[-3:], banks()["default"], "noise")
    with pytest.raises(VttsError) as ei:
        eng.melspec(np.zeros((B + 1, S), np.float32))
    assert ei.value.code == -1


# ---- filterbanks -----------------------------------------------------------------------------------------------

def test_other_filterbanks_and_back(eng):
    """each bank through load_mel_filterbank (so through mel_span_kernel's spans) against float64 with that bank; then
    the default bank again gives the bits it gave before"""
    default = banks()["default"]
    probe = {S: np.concatenate([signal(n, 2, S, seed=3) for n in ("noise", "chirp", "tones_half_bin", "tiny")]) for S in (1280, 4608)}
    before = {S: eng.melspec(y) for S, y in probe.items()}
    try:
        for name in ("fmin80_fmax7600", "sr22050", "holed"):
            fb = banks()[name]
            eng.load_mel_filterbank(fb)
            for S, y in probe.items():
                got = eng.melspec(y)
                _check(got, y, fb, f"bank {name}")
                assert np.abs(got - before[S]).max() > 1e-2, name     # the bank really changed
            if name == "holed":
                assert np.all(got[:, :, 7] == mo.LOG_CLIP)
    finally:
        eng.load_mel_filterbank()
    for S, y in probe.items():
        assert np.array_equal(eng.melspec(y), before[S])
        _check(before[S], y, default, "bank default")


# ---- the ground-truth half of gta ------------------------------------------------------------------------------

def _gta_batch(S):
    B, L = 3, 20
    n = np.arange(S)
    rng = np.random.default_rng(11)
    wav = np.stack([np.where((n // 40) % 2 == 0, 32767, -32768),
                    np.clip(rng.standard_normal(S) * 30000, -32768, 32767),
                    np.round(8000 * np.sin(2 * np.pi * 1000.0 / 16000 * n))]).astype(np.int16)
    wav[2, ::97] = -32768
    tok = np.stack([np.asarray(synthetic.utterance(30 + b, L, None)[0], np.int32) for b in range(B)])
    dur = np.stack([synthetic.utterance(30 + b, L, S / 16000)[1][0] for b in range(B)]).astype(np.float32)
    return wav, tok, dur


def test_gta_ground_truth_on_full_scale_int16(acoustic_eng):
    S = 256 * 37
    wav, tok, dur = _gta_batch(S)
    wl = np.array([S, 256 * 20 + 31, 256 * 3], np.int32)
    out, gt = acoustic_eng.gta(wav, tok, dur, wav_lengths=wl, return_gt=True)
    y = wav.astype(np.float32) / np.float32(32768)
    assert (wav == -32768).any() and (wav == 32767).any()
    _check(gt, y, banks()["default"], "gta int16")
    # the ground truth covers every frame of the padded row; wav_lengths cuts the model's output only
    out_full, gt_full = acoustic_eng.gta(wav, tok, dur, return_gt=True)
    assert np.array_equal(gt, gt_full)
    N = S // 256
    nf = np.clip(wl // 256, 1, N)
    for b in range(3):
        assert np.all(out[b, nf[b] :] == 0) and np.any(out[b, : nf[b]] != 0), b
    # and the model's input is the ground truth shifted by one frame behind a zero frame (gta.py:34-36)
    frames = (dur * np.float32(16000)) / np.float32(256)
    mels_in = np.concatenate([np.zeros_like(gt[:, :1]), gt[:, :-1]], axis=1)
    _, m2 = acoustic_eng.teacher_forced(tok, frames, mels_in, n_frames=nf)
    assert np.array_equal(out, m2)


# ---- the Engine's bookkeeping and argument checks ----------------------------------------------------------------

def test_gta_uses_the_default_bank_after_another_was_loaded(acoustic_ckpt, acoustic_eng):
    from viettts_b200.engine import Engine
    from viettts_b200.nat.dsp import MelFilter
    S = 256 * 24
    wav, tok, dur = _gta_batch(S)
    fresh = Engine(0)
    try:
        fresh.load_acoustic(acoustic_ckpt)
        ref_out, ref_gt = fresh.gta(wav, tok, dur, return_gt=True)
    finally:
        fresh.close()
    y = signal("chirp", 2, 2048)
    mf = MelFilter(16000, 1024, 80, fmin=80, fmax=7600, engine=acoustic_eng)
    m80 = mf(y)
    out, gt = acoustic_eng.gta(wav, tok, dur, return_gt=True)
    assert np.array_equal(gt, ref_gt) and np.array_equal(out, ref_out)
    # the bank MelFilter loaded is still the one melspec uses
    assert np.array_equal(acoustic_eng.melspec(y), m80)
    _check(m80, y, mf.melfb, "bank fmin80_fmax7600")


def test_melspec_forward_equals_melspec(eng):
    y = signal("noise", 3, 4352, seed=9)
    t = torch.from_numpy(y).cuda()
    got = eng.melspec_forward(t)
    torch.cuda.synchronize()
    assert np.array_equal(got.cpu().numpy(), eng.melspec(y))
    out = torch.full((3, 17, 80), float("nan"), device="cuda")
    assert eng.melspec_forward(t, out=out) is out
    torch.cuda.synchronize()
    assert np.array_equal(out.cpu().numpy(), eng.melspec(y))


def test_melspec_forward_rejects_bad_tensors_before_any_launch(eng):
    x = torch.zeros((2, 1024), device="cuda")
    good_out = torch.empty((2, 4, 80), device="cuda")
    bad = [dict(wav_t=x.double()), dict(wav_t=x.cpu()), dict(wav_t=torch.zeros((1024, 2), device="cuda").t()),
           dict(wav_t=x[0]), dict(wav_t=x, out=torch.empty((2, 5, 80), device="cuda")),
           dict(wav_t=x, out=torch.empty((2, 80, 4), device="cuda")), dict(wav_t=x, out=good_out.double()),
           dict(wav_t=x, out=torch.empty((2, 4, 80))), dict(wav_t=x, out=torch.empty((2, 80, 4), device="cuda").transpose(1, 2))]
    eng.melspec_forward(x, out=good_out)
    torch.cuda.synchronize()
    n = eng.launch_count()
    for kw in bad:
        with pytest.raises((AssertionError, ValueError)):
            eng.melspec_forward(**kw)
    assert eng.launch_count() == n
