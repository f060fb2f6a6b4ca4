"""GPU parity: DurationModel + the text2mel glue (CUDA, through the C ABI) vs the CPU restatement
(SURVEY.md §8f row 1: the callers of predict_mel).

Oracle status: pinned to the reference's own source (tests/test_reference_goldens.py; the CUDA path is also compared
with the reference-produced durations directly in tests/test_gpu_reference_goldens.py).  Tolerance, per token:
|gpu - float64 oracle| <= E2E_UNITS[mode] units of 2^-24 (sigmoid(s) sum_i |gelu(y_i) w2_i| + softplus(s)), the unit of
the head's own bound (tests/test_gpu_duration_stages.py), at most 1.1e-5 s on these rows; tests/test_duration_bounds.py
derives it from the plain fp32 oracle.  The stages one by one are pinned in tests/test_gpu_duration_stages.py."""
import json
import pickle

import numpy as np
import pytest
import torch

from oracle import hifigan_oracle as ho
from oracle import nat_oracle as no
from test_gpu_duration_stages import E2E_UNITS, e2e_ref
from viettts_b200 import config, synthetic

pytestmark = pytest.mark.gpu


def within_bound(eng, ckpt, tokens, lengths, got):
    """|got - float64| <= E2E_UNITS units on every token < lengths[b] of tokens [B,L]; returns the worst in units"""
    ref, unit = e2e_ref(ckpt, tokens, np.asarray(lengths))
    valid = np.arange(tokens.shape[1])[None, :] < np.asarray(lengths)[:, None]
    u = np.where(valid, np.abs(got - ref) / unit, 0.0)
    assert (u <= E2E_UNITS[eng.mode]).all(), (np.argwhere(u > E2E_UNITS[eng.mode])[:4], float(u.max()))
    return float(u.max())


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


def _tokens(seed, L):
    tk, _ = synthetic.utterance(seed, L, None)
    return np.asarray(tk, np.int32)


def test_single_utterance_vs_oracle(eng, duration_ckpt):
    tk = _tokens(0, 100)
    got = eng.predict_duration(tk[None])
    ref64 = no.duration_model(duration_ckpt, tk[None], np.array([100]), dtype=torch.float64)
    ref32 = no.predict_duration(duration_ckpt, tk)
    enc = eng.debug_read("enc", (1, 100, 512))
    P, S = duration_ckpt["params"], duration_ckpt["aux"]
    enc_ref = no.token_encoder(P, S, tk[None], np.array([100]), torch.float64, T=no.DM + "token_encoder/~/").numpy()
    print(f"duration: gpu-vs-f64 {np.abs(got-ref64).max():.3e}  f32-vs-f64 {np.abs(ref32-ref64).max():.3e}  enc {np.abs(enc-enc_ref).max():.3e}")
    assert got.shape == (1, 100) and got.dtype == np.float32
    assert np.abs(enc - enc_ref).max() < 1e-4
    print(f"duration: gpu-vs-f64 {within_bound(eng, duration_ckpt, tk[None], [100], got):.2f} units")


def test_reference_shape_case(eng, duration_ckpt):
    """tests/test_nat_duration.py's input (all-zero tokens, B=2, L=10)."""
    tok = np.zeros((2, 10), np.int32)
    got = eng.predict_duration(tok)
    assert got.shape == (2, 10)
    within_bound(eng, duration_ckpt, tok, [10, 10], got)
    assert np.array_equal(got[0], got[1])


def test_ragged_batch_rows_equal_single_runs(eng, duration_ckpt):
    """Batch contract: row b == the reference run on row b alone with L = lengths[b]; padding never leaks."""
    lens = np.array([100, 57, 23, 1, 64, 2], np.int32)
    L = int(lens.max())
    tok = np.full((len(lens), L), 77, np.int32)          # poison the padding with a real phoneme id
    rows = []
    for b, n in enumerate(lens):
        rows.append(_tokens(10 + b, max(int(n), 5))[: int(n)])
        tok[b, :n] = rows[-1]
    got = eng.predict_duration(tok, lengths=lens)
    for b, n in enumerate(lens):
        assert np.all(got[b, n:] == 0.0)
        within_bound(eng, duration_ckpt, rows[b][None], [n], got[b : b + 1, :n])
        alone = eng.predict_duration(rows[b][None])
        assert np.abs(alone[0] - got[b, :n]).max() < 1e-6


def test_batch_larger_than_one_launch(eng, duration_ckpt):
    B = 130                                               # > MAX_ROWS=128: the host layer chunks
    tok = np.stack([_tokens(300 + b, 12) for b in range(B)])
    got = eng.predict_duration(tok)
    for b in (0, 127, 128, 129):
        within_bound(eng, duration_ckpt, tok[b : b + 1], [12], got[b : b + 1])


def test_device_pointer_entry_point(eng):
    tk = np.stack([_tokens(1, 40), _tokens(2, 40)])
    host = eng.predict_duration(tk, lengths=[40, 33])
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        t = torch.from_numpy(tk).cuda()
        ln = torch.tensor([40, 33], dtype=torch.int32, device="cuda")
        out = eng.duration_forward(t, ln)
    st.synchronize()
    assert np.array_equal(out.cpu().numpy(), host)
    assert eng.last_stage_ms(3) > 0


def test_bad_arguments_raise(eng):
    from viettts_b200._lib import VttsError
    with pytest.raises(ValueError):
        eng.predict_duration(np.zeros(5, np.int32))
    from viettts_b200.engine import Engine
    e2 = Engine(0)
    try:
        with pytest.raises(VttsError):
            e2.predict_duration(np.zeros((1, 5), np.int32))      # weights not loaded
        with pytest.raises(VttsError):
            e2.load_duration(np.zeros(10, np.float32))           # wrong blob size
    finally:
        e2.close()


def test_reload_other_checkpoints_then_originals(eng, duration_ckpt, acoustic_ckpt, hifigan_params):
    """Loading replaces a model's device weights in place: after a second checkpoint and the original again, the
    acoustic and duration outputs equal those of a fresh engine."""
    from viettts_b200.engine import Engine
    tk = np.stack([_tokens(60, 24), _tokens(61, 24)])
    lens = np.array([24, 17], np.int32)
    frames, _ = no.seconds_to_frames(eng.predict_duration(tk, lengths=lens))
    nfs = frames.sum(axis=1, dtype=np.float32).astype(np.int32)
    fresh = Engine(0)
    try:
        fresh.load_duration(duration_ckpt)
        fresh.load_acoustic(acoustic_ckpt)
        fresh.set_precision(eng.lib.vtts_get_precision(eng.h))
        want_dur = fresh.predict_duration(tk, lengths=lens)
        want_mel = fresh.predict_mel(tk, frames, lengths=lens, n_frames=nfs)
    finally:
        fresh.close()
    try:
        eng.load_duration(synthetic.duration_ckpt(99))
        eng.load_acoustic(synthetic.acoustic_ckpt(99))
        assert not np.array_equal(eng.predict_duration(tk, lengths=lens), want_dur)
    finally:
        eng.load_duration(duration_ckpt)
        eng.load_acoustic(acoustic_ckpt)
    assert np.array_equal(eng.predict_duration(tk, lengths=lens), want_dur)
    assert np.array_equal(eng.predict_mel(tk, frames, lengths=lens, n_frames=nfs), want_mel)


def _staged_pipeline(eng, tok_row, silence_duration):
    """text2mel.py:85-103 + mel2wave through the separate entry points (dropout off)."""
    tokens = [int(t) for t in tok_row]
    d = no.adjust_durations(tokens, eng.predict_duration(np.asarray(tokens, np.int32)[None]), silence_duration)
    frames, n = no.seconds_to_frames(d)
    mel = eng.predict_mel(np.asarray(tokens, np.int32)[None], frames, n_frames=[n])
    mel = no.trim_end_silence(tokens, d, mel)
    return eng.mel2wave(mel)[0], d, mel


@pytest.mark.parametrize("silence_duration", [-1.0, 0.12])
def test_tts_equals_staged_pipeline(eng, silence_duration):
    lens = np.array([30, 18, 25], np.int32)
    tok = np.zeros((3, 30), np.int32)
    for b, n in enumerate(lens):
        tok[b, :n] = _tokens(40 + b, int(n))
    waves, dur = eng.tts(tok, lens, silence_duration=silence_duration)
    for b, n in enumerate(lens):
        wav, d, _ = _staged_pipeline(eng, tok[b, :n], silence_duration)
        assert np.array_equal(dur[b, :n], d[0])
        assert waves[b].shape == wav.shape, (waves[b].shape, wav.shape)
        assert np.abs(waves[b] - wav).max() < 1e-5
    # a buffer that is too small is reported and retried by the wrapper
    again, _ = eng.tts(tok, lens, silence_duration=silence_duration, max_frames=3)
    assert all(np.array_equal(a, w) for a, w in zip(again, waves))


def test_tts_vs_oracle_end_to_end(eng, duration_ckpt, acoustic_ckpt, hifigan_params):
    """Whole chain against the CPU restatement for one short utterance (dropout off)."""
    tk = _tokens(7, 14)
    tokens = [int(t) for t in tk]
    raw64, unit = e2e_ref(duration_ckpt, tk[None], np.array([len(tk)]))
    d = no.adjust_durations(tokens, raw64, 0.05)
    mel_ref = no.predict_mel(acoustic_ckpt, tokens, d, None)[None]
    mel_ref = no.trim_end_silence(tokens, d, mel_ref)
    wav_ref = ho.mel2wave(hifigan_params, mel_ref)
    waves, dur = eng.tts(tk[None], silence_duration=0.05)
    assert (np.abs(dur[0] - d[0]) <= E2E_UNITS[eng.mode] * unit[0]).all()     # the clip and word-end zeroing add no error
    assert waves[0].shape == wav_ref.shape, (waves[0].shape, wav_ref.shape)
    err = waves[0] - wav_ref
    print(f"tts e2e: Linf {np.abs(err).max():.3e} rms {np.sqrt(np.mean(err**2)):.3e}")
    assert np.sqrt(np.mean(err ** 2)) < 1e-3 and np.abs(err).max() < 1e-2


def test_cli_and_dropins(eng, duration_ckpt, acoustic_ckpt, hifigan_params, golden_dir, tmp_path, monkeypatch):
    """`python -m viettts_b200.synthesizer` with checkpoints at the reference's cwd-relative paths."""
    from viettts_b200 import synthesizer
    from viettts_b200.engine import get_engine
    (tmp_path / "assets/hifigan").mkdir(parents=True)
    (tmp_path / "assets/infore/hifigan").mkdir(parents=True)
    (tmp_path / "assets/infore/nat").mkdir(parents=True)
    (tmp_path / "assets/hifigan/config.json").write_text(json.dumps(config.HIFIGAN))
    with open(tmp_path / "assets/infore/hifigan/hk_hifi.pickle", "wb") as f:
        pickle.dump(hifigan_params, f)
    with open(tmp_path / "assets/infore/nat/acoustic_latest_ckpt.pickle", "wb") as f:
        pickle.dump(acoustic_ckpt, f)
    with open(tmp_path / "assets/infore/nat/duration_latest_ckpt.pickle", "wb") as f:
        pickle.dump(duration_ckpt, f)
    monkeypatch.chdir(tmp_path)
    lex = str(golden_dir / "lexicon_small.txt")
    get_engine(0).set_precision(eng.lib.vtts_get_precision(eng.h))
    rc = synthesizer.main(["--text", "Xin chào, tôi là trợ lý ảo.", "--output", "one.wav", "--lexicon-file", lex, "--silence-duration", "0.1"])
    assert rc == 0
    one, sr = synthesizer.read_wav(tmp_path / "one.wav")
    assert sr == 16000 and one.size % 256 == 0 and one.size > 256 and np.abs(one).max() <= 1.0
    (tmp_path / "lines.txt").write_text("Xin chào, tôi là trợ lý ảo.\n\nhôm nay trời đẹp quá! bạn có khỏe không?\n")
    rc = synthesizer.main(["--text-file", "lines.txt", "--output", "out.wav", "--lexicon-file", lex, "--silence-duration", "0.1", "--seed", "5"])
    assert rc == 0
    a, _ = synthesizer.read_wav(tmp_path / "out_0000.wav")
    b, _ = synthesizer.read_wav(tmp_path / "out_0001.wav")
    assert a.size == one.size and b.size > 256       # same text -> same durations -> same length (dropout differs)
    # the batched path equals the library call on the same batch (rows sorted by token count, as the CLI builds it;
    # the dropout stream is keyed by the row index)
    from viettts_b200.nat import text2mel as t2m
    texts = ["Xin chào, tôi là trợ lý ảo.", "hôm nay trời đẹp quá! bạn có khỏe không?"]
    toks = [t2m.text2tokens(synthesizer.nat_normalize_text(t), lex) for t in texts]
    order = sorted(range(2), key=lambda i: len(toks[i]))
    tok = np.zeros((2, max(map(len, toks))), np.int32)
    for r, i in enumerate(order):
        tok[r, : len(toks[i])] = toks[i]
    w, _ = get_engine(0).tts(tok, [len(toks[i]) for i in order], silence_duration=0.1, seed=5)
    for r, i in enumerate(order):
        got = (a, b)[i]
        assert got.size == w[r].size
        assert np.abs(synthesizer.float_to_pcm16(w[r]).astype(np.float32) / 32767.0 - got).max() <= 1e-6
