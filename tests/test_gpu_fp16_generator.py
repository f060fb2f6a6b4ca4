"""GPU: the fast fp16 generator mode (Engine.set_precision("fp16"), VTTS_PRECISION_FP16).

Tolerance (tests/test_fast_precision_modes.py derives it from the CPU emulation of the mode on synthetic weights):
waveform L-inf <= 3e-3 and RMS <= 6e-4 against float64; one conv or fused ResBlock pair within a normalised L-inf
(max |err| / max |ref|) of 1e-3.  The mode covers the generator only: every other model must give the bits of
bf16x3."""
import numpy as np
import pytest
import torch

from oracle import hifigan_oracle as ho
from oracle import nat_oracle as no
from viettts_b200 import synthetic

pytestmark = pytest.mark.gpu
FAST_WAV_LINF, FAST_WAV_RMS = 3e-3, 6e-4
LAYER_NLINF = 1e-3
FP16_MAX = 65504.0


@pytest.fixture(scope="module")
def eng(hifigan_params):
    from viettts_b200.engine import Engine
    e = Engine(0)
    e.load_hifigan(hifigan_params)
    e.set_precision("fp16")
    yield e
    e.close()


@pytest.fixture(scope="module")
def oracle_wavs(hifigan_params):
    """float64 oracle waveforms of config 2 (one 400-frame mel) and of a 1000-frame mel"""
    out = {}
    for T, seed in ((400, 0), (1000, 4)):
        mel = synthetic.mel_input(seed, 1, T)
        out[T] = (mel, ho.mel2wave(hifigan_params, mel, torch.float64).reshape(1, -1))
    return out


def _check(wav, ref, what):
    err = np.abs(wav.astype(np.float64) - ref)
    linf, rms = float(err.max()), float(np.sqrt(np.mean(err ** 2)))
    print(f"[fp16 {what}] Linf={linf:.3e} rms={rms:.3e}")
    assert linf <= FAST_WAV_LINF and rms <= FAST_WAV_RMS, (what, linf, rms)


@pytest.mark.parametrize("fused", [True, False])
@pytest.mark.parametrize("tag", ["small", "t32"])
def test_generator_fp16_golden(eng, golden_dir, tag, fused):
    g = np.load(golden_dir / f"hifigan_ref_{tag}.npz")
    eng.set_fused_pairs(fused)
    try:
        _check(eng.mel2wave(g["mel"]), g["wav"], f"golden-{tag} fused={fused}")
    finally:
        eng.set_fused_pairs(True)


@pytest.mark.parametrize("fused", [True, False])
@pytest.mark.parametrize("T", [400, 1000])
def test_generator_fp16_vs_oracle(eng, oracle_wavs, T, fused):
    mel, ref = oracle_wavs[T]
    eng.set_fused_pairs(fused)
    try:
        _check(eng.mel2wave(mel), ref, f"T={T} fused={fused}")
    finally:
        eng.set_fused_pairs(True)


def test_fp16_really_runs(eng, golden_dir):
    g = np.load(golden_dir / "hifigan_ref_small.npz")
    fast = eng.mel2wave(g["mel"])
    eng.set_precision("bf16x3")
    try:
        split = eng.mel2wave(g["mel"])
    finally:
        eng.set_precision("fp16")
    d = float(np.abs(fast - split).max())
    print(f"max |fp16 - bf16x3| = {d:.3e}")
    assert d > 1e-5


def _ref_conv(x, w, b, k, dil, slope, resid):
    xt = torch.nn.functional.leaky_relu(torch.from_numpy(x).double(), slope)
    wt = torch.from_numpy(w).double().permute(2, 1, 0).contiguous()
    y = torch.nn.functional.conv1d(xt.transpose(1, 2), wt, torch.from_numpy(b).double(), padding=(k - 1) * dil // 2, dilation=dil)
    return (y.transpose(1, 2) + torch.from_numpy(resid).double()).numpy()


@pytest.mark.parametrize("C", [32, 64, 128, 256])
@pytest.mark.parametrize("k", [3, 7, 11])
@pytest.mark.parametrize("dil", [1, 3, 5])
def test_layer_fp16_vs_float64(eng, C, k, dil):
    rng = np.random.default_rng(C * 100 + k * 10 + dil)
    B, T = 2, 600
    x = rng.standard_normal((B, T, C)).astype(np.float32)
    w = (rng.standard_normal((k, C, C)) / np.sqrt(k * C)).astype(np.float32)
    b = (rng.standard_normal(C) * 0.1).astype(np.float32)
    res = rng.standard_normal((B, T, C)).astype(np.float32)
    lens = np.array([T, 257], np.int32)
    dev = torch.device("cuda", 0)
    t = lambda a: torch.from_numpy(a).to(dev)  # noqa: E731
    out = eng.debug_conv1d("fp16", t(x), t(w), t(b), k, dil, 0.1, t(res), t(lens)).cpu().numpy()
    split = eng.debug_conv1d("bf16x3", t(x), t(w), t(b), k, dil, 0.1, t(res), t(lens)).cpu().numpy()
    for bb in range(B):
        n = lens[bb]
        ref = _ref_conv(x[bb : bb + 1, :n], w, b, k, dil, 0.1, res[bb : bb + 1, :n])[0]
        e = np.abs(out[bb, :n] - ref).max() / np.abs(ref).max()
        assert e <= LAYER_NLINF, (C, k, dil, bb, e)
        assert np.abs(split[bb, :n] - ref).max() < 2e-4          # the bf16x3 hook is unchanged
    assert np.abs(out[0] - split[0]).max() > 1e-5                # the fp16 packing and kernel really ran


def _ref_pair(x, w1, b1, w2, b2, k, dil, slope):
    xt = torch.from_numpy(x).double()
    f = torch.nn.functional
    y = f.leaky_relu(xt, slope).transpose(1, 2)
    y = f.conv1d(y, torch.from_numpy(w1).double().permute(2, 1, 0).contiguous(), torch.from_numpy(b1).double(), padding=(k - 1) * dil // 2, dilation=dil)
    y = f.leaky_relu(y, slope)
    y = f.conv1d(y, torch.from_numpy(w2).double().permute(2, 1, 0).contiguous(), torch.from_numpy(b2).double(), padding=(k - 1) // 2)
    return (y.transpose(1, 2) + xt).numpy()


@pytest.mark.parametrize("C", [32, 64])
@pytest.mark.parametrize("k", [3, 7, 11])
@pytest.mark.parametrize("dil", [1, 3, 5])
def test_fused_pair_fp16_vs_float64(eng, C, k, dil):
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
        ref = _ref_pair(x[bb : bb + 1, :n], w1, b1, w2, b2, k, dil, 0.1)[0]
        e = np.abs(out[bb, :n] - ref).max() / np.abs(ref).max()
        assert e <= LAYER_NLINF, (C, k, dil, bb, e)


@pytest.mark.parametrize("fused", [True, False])
def test_fp16_ragged_rows_and_repeated_calls_bit_identical(eng, fused):
    eng.set_fused_pairs(fused)
    try:
        mel = synthetic.mel_input(3, 3, 40)
        nf = np.array([40, 23, 1], np.int32)
        wav = eng.mel2wave(mel, n_frames=nf)
        for b in range(3):
            alone = eng.mel2wave(mel[b : b + 1, : nf[b]])
            assert np.array_equal(alone[0], wav[b, : nf[b] * 256]), b
            assert np.all(wav[b, nf[b] * 256 :] == 0.0)
        calls = [(mel, nf), (synthetic.mel_input(2, 1, 9), np.array([9], np.int32)),
                 (synthetic.mel_input(5, 4, 64), np.array([64, 64, 64, 64], np.int32))]
        first = [eng.mel2wave(m, n_frames=n) for m, n in calls]
        for _ in range(2):
            for (m, n), w0 in zip(calls, first):
                assert np.array_equal(eng.mel2wave(m, n_frames=n), w0)
    finally:
        eng.set_fused_pairs(True)


def test_launches_per_generator_call_match_bf16x3(eng):
    mel = synthetic.mel_input(7, 2, 50)
    for fused in (True, False):
        eng.set_fused_pairs(fused)
        counts = {}
        for mode in ("bf16x3", "fp16"):
            eng.set_precision(mode)
            l0 = eng.launch_count()
            eng.mel2wave(mel)
            counts[mode] = eng.launch_count() - l0
        assert counts["bf16x3"] == counts["fp16"], (fused, counts)
    eng.set_fused_pairs(True)
    eng.set_precision("fp16")


@pytest.mark.parametrize("kind", ["tmem", "smem"])
def test_other_pair_forms_reject_fp16(eng, kind):
    from viettts_b200._lib import VttsError
    mel = synthetic.mel_input(8, 1, 20)
    C, k = 32, 3
    dev = torch.device("cuda", 0)
    x = torch.zeros((1, 100, C), device=dev)
    w = torch.zeros((k, C, C), device=dev)
    b = torch.zeros(C, device=dev)
    eng.set_fused_pairs(True, kind=kind)
    try:
        with pytest.raises(VttsError):
            eng.mel2wave(mel)
        with pytest.raises(VttsError):
            eng.debug_pair(x, w, b, w, b, k, 1)
    finally:
        eng.set_fused_pairs(True, kind="smem2")
    assert np.isfinite(eng.mel2wave(mel)).all()


def test_saturation_keeps_the_waveform_finite(hifigan_params):
    """conv_pre weights scaled by 2^16 drive the input of the first ConvTranspose past the fp16 range: the kernels must
    saturate instead of producing inf (and from it NaN)."""
    from viettts_b200.engine import Engine
    params = {k: dict(v) for k, v in hifigan_params.items()}
    p0 = params["generator/~/conv1_d"]
    p0["w"] = np.asarray(p0["w"], np.float32) * np.float32(2.0 ** 16)
    mel = synthetic.mel_input(0, 1, 24)
    taps = {}
    with torch.no_grad():
        ho.generator_forward(params, mel, torch.float64, taps=taps)
    big = float(torch.nn.functional.leaky_relu(taps["pre"], 0.1).abs().max())
    assert big > FP16_MAX, big          # an operand of the first ConvTranspose is outside the fp16 range
    e = Engine(0)
    try:
        e.load_hifigan(params)
        e.set_precision("fp16")
        for fused in (True, False):
            e.set_fused_pairs(fused)
            wav = e.mel2wave(mel)
            assert np.isfinite(wav).all() and np.abs(wav).max() <= 1.0, fused
    finally:
        e.close()


def _utt(seed, L, seconds):
    tokens, dur = synthetic.utterance(seed, L, seconds)
    d, n = no.seconds_to_frames(dur)
    return np.asarray(tokens, np.int32), d[0], n


def test_other_models_ignore_the_fp16_mode(hifigan_params, acoustic_ckpt):
    """Mode 2 runs the acoustic, duration, teacher-forced and GTA paths exactly like mode 1, also after the generator ran
    in fp16; a bf16x3 generator call after such a detour equals one from a fresh engine."""
    from viettts_b200.engine import Engine
    dk = synthetic.duration_ckpt(1234)
    B, L = 3, 30
    utts = [_utt(300 + b, L, 1.0) for b in range(B)]
    tok = np.stack([u[0] for u in utts])
    dur = np.stack([u[1] for u in utts]).astype(np.float32)
    nf = np.array([u[2] for u in utts], np.int32)
    N = int(nf.max())
    masks = synthetic.dropout_masks(11, B, N)
    rng = np.random.default_rng(12)
    keep = (rng.random((B, N, 2, 256)) < 0.5).astype(np.uint8)
    zone = (rng.random((B, N, 4, 512)) < 0.1).astype(np.uint8)
    mels_in = synthetic.mel_input(13, B, N)
    wav_i16 = (rng.standard_normal((B, N * 256)) * 3000).astype(np.int16)
    dur_sec = dur * np.float32(256 / 16000)
    gen_mel = synthetic.mel_input(14, 2, 37)

    def outputs(e):
        return dict(mel=e.predict_mel(tok, dur, n_frames=nf, masks=masks), dur=e.predict_duration(tok),
                    tf=e.teacher_forced(tok, dur, mels_in, n_frames=nf, keep_masks=keep, zone_masks=zone),
                    gta=e.gta(wav_i16, tok, dur_sec, keep_masks=keep, zone_masks=zone))

    def engine():
        e = Engine(0)
        e.load_hifigan(hifigan_params)
        e.load_acoustic(acoustic_ckpt)
        e.load_duration(dk)
        e.load_mel_filterbank()
        return e

    e = engine()
    try:
        ref = outputs(e)
        gen_ref = e.mel2wave(gen_mel)
        e.set_precision("fp16")
        assert e.lib.vtts_get_precision(e.h) == 2
        e.mel2wave(gen_mel)                      # the detour through the fp16 generator
        got = outputs(e)
        for key in ref:
            a, b = ref[key], got[key]
            for x, y in zip(a if isinstance(a, tuple) else (a,), b if isinstance(b, tuple) else (b,)):
                assert np.array_equal(x, y), key
        e.set_precision("bf16x3")
        assert np.array_equal(e.mel2wave(gen_mel), gen_ref)
    finally:
        e.close()
    fresh = engine()
    try:
        assert np.array_equal(fresh.mel2wave(gen_mel), gen_ref)
    finally:
        fresh.close()


def test_cli_precision_flag(hifigan_params, acoustic_ckpt, golden_dir, tmp_path, monkeypatch):
    """`python -m viettts_b200.synthesizer --precision fp16` puts the engine both input paths use into the fp16 mode."""
    import json
    import pickle
    from viettts_b200 import config, synthesizer
    from viettts_b200.engine import get_engine
    for d in ("assets/hifigan", "assets/infore/hifigan", "assets/infore/nat"):
        (tmp_path / d).mkdir(parents=True)
    (tmp_path / "assets/hifigan/config.json").write_text(json.dumps(config.HIFIGAN))
    for name, obj in (("hifigan/hk_hifi", hifigan_params), ("nat/acoustic_latest_ckpt", acoustic_ckpt),
                      ("nat/duration_latest_ckpt", synthetic.duration_ckpt(1234))):
        with open(tmp_path / f"assets/infore/{name}.pickle", "wb") as f:
            pickle.dump(obj, f)
    monkeypatch.chdir(tmp_path)
    lex = str(golden_dir / "lexicon_small.txt")
    eng = get_engine(0)
    try:
        (tmp_path / "lines.txt").write_text("Xin chào, tôi là trợ lý ảo.\n")
        for flag, mode in (("fp16", 2), ("bf16x3", 1)):
            for src in (["--text-file", "lines.txt"], ["--text", "Xin chào, tôi là trợ lý ảo."]):
                eng.set_precision("fp32")
                assert synthesizer.main([*src, "--output", f"{flag}.wav", "--lexicon-file", lex, "--precision", flag]) == 0
                assert eng.lib.vtts_get_precision(eng.h) == mode
            one, _ = synthesizer.read_wav(tmp_path / f"{flag}.wav")
            assert one.size > 256 and np.abs(one).max() <= 1.0
    finally:
        eng.set_precision("bf16x3")
