"""GPU: the REFERENCE dropout mode (VTTS_DROPOUT_REFERENCE, `rng=`) draws the reference's own JAX/Haiku mask stream on
the device.

The masks themselves are compared with the host statement of the stream (`viettts_b200.jaxrng`, pinned to the masks
recorded from the reference's own source) through the `debug_dropout_masks` hook: comparing outputs alone would miss
a wrong keep bit on a unit that relu has already zeroed.  The outputs of every entry point are then compared bit for
bit with the MASK mode fed those host masks, which is the path the drop-ins took before."""
import functools
import json
import pickle
from pathlib import Path

import numpy as np
import pytest

from oracle import nat_oracle as no
from viettts_b200 import config, jaxrng, synthetic

pytestmark = pytest.mark.gpu
GOLDEN = Path(__file__).resolve().parent / "golden"
GOLDEN_RNG = tuple(int(x) for x in np.load(GOLDEN / "nat_ref_predict_mel.npz")["rng"].ravel())
KEYS = [(0, 42), (0, 0), (0xFFFFFFFF, 0xFFFFFFFF), (0x12345678, 0x9ABCDEF0), GOLDEN_RNG]
KEY_IDS = ["0_42", "0_0", "ones", "12345678_9abcdef0", "golden"]


@pytest.fixture(scope="module", params=["fp32", "bf16x3"])
def eng(acoustic_ckpt, hifigan_params, request):
    from viettts_b200.engine import Engine
    e = Engine(0)
    e.load_acoustic(acoustic_ckpt)
    e.load_duration(synthetic.duration_ckpt(1234))
    e.load_hifigan(hifigan_params)
    e.load_mel_filterbank()
    e.set_precision(request.param)
    yield e
    e.close()


@functools.lru_cache(maxsize=None)
def _inf_masks(key, N):
    return jaxrng.inference_keep_masks(np.array(key, np.uint32), 1, N)[0]


@functools.lru_cache(maxsize=None)
def _tf_masks(key, B, N):
    return jaxrng.teacher_forced_masks(np.array(key, np.uint32), B, N)


def _utt(seed, L, seconds):
    tokens, dur = synthetic.utterance(seed, L, seconds)
    d, n = no.seconds_to_frames(dur)
    return np.asarray(tokens, np.int32), d[0], n


def _ragged(B, seed0=0):
    """B rows of 6..40 tokens lasting 0.2..0.9 s, padded to the longest."""
    rs = np.random.default_rng(seed0)
    utts = [_utt(seed0 + b, int(rs.integers(6, 41)), float(rs.uniform(0.2, 0.9))) for b in range(B)]
    L = max(len(u[0]) for u in utts)
    tok = np.zeros((B, L), np.int32)
    dur = np.zeros((B, L), np.float32)
    lens = np.array([len(u[0]) for u in utts], np.int32)
    nfs = np.array([u[2] for u in utts], np.int32)
    for b, (tk, d, _) in enumerate(utts):
        tok[b, : len(tk)] = tk
        dur[b, : len(tk)] = d
    return tok, dur, lens, nfs


# ---- 1. the masks the device draws are the reference's -------------------------------------------------------------
@pytest.mark.parametrize("key", KEYS, ids=KEY_IDS)
def test_inference_masks_equal_jaxrng(eng, key):
    for N in (1, 2, 3, 312, 937, 5000):
        got = eng.debug_dropout_masks(0, key, 1, N)
        assert got.shape == (N, 2, 256)
        assert np.array_equal(got, _inf_masks(key, N)), N


@pytest.mark.parametrize("key", KEYS, ids=KEY_IDS)
def test_teacher_forced_masks_equal_jaxrng(eng, key):
    for B, N in ((1, 1), (3, 17), (33, 312), (128, 312)):
        keep, zone = eng.debug_dropout_masks(1, key, B, N)
        want_keep, want_zone = _tf_masks(key, B, N)
        assert np.array_equal(keep, want_keep), (B, N)
        assert np.array_equal(zone, want_zone), (B, N)


# ---- 2. autoregressive outputs -------------------------------------------------------------------------------------
@pytest.mark.parametrize("key", [KEYS[0], KEYS[3], GOLDEN_RNG], ids=["0_42", "12345678_9abcdef0", "golden"])
@pytest.mark.parametrize("B", [1, 9, 33, 128])
def test_inference_equals_mask_mode(eng, key, B):
    tok, dur, lens, nfs = _ragged(B, seed0=10 * B)
    N = int(nfs.max())
    masks = np.ascontiguousarray(np.broadcast_to(_inf_masks(key, N)[None], (B, N, 2, 256)))
    got = eng.predict_mel(tok, dur, lengths=lens, n_frames=nfs, rng=key)
    want = eng.predict_mel(tok, dur, lengths=lens, n_frames=nfs, masks=masks)
    assert np.array_equal(got, want)
    # a row is the row alone, and the row in a longer padded batch
    b = B // 2
    alone = eng.predict_mel(tok[b : b + 1, : lens[b]], dur[b : b + 1, : lens[b]], n_frames=nfs[b : b + 1], rng=key)
    assert np.array_equal(alone[0], got[b, : nfs[b]])
    pad = np.concatenate([tok[b : b + 1], np.full((1, 7), 77, np.int32)], axis=1)
    dpad = np.concatenate([dur[b : b + 1], np.full((1, 7), 9.0, np.float32)], axis=1)
    longer = eng.predict_mel(np.concatenate([pad, pad]), np.concatenate([dpad, dpad]), lengths=[lens[b], lens[b] + 7],
                             n_frames=[nfs[b], nfs[b] + 63], rng=key)
    assert np.array_equal(longer[0, : nfs[b]], got[b, : nfs[b]])


def test_rows_across_launch_chunks_share_the_stream(eng):
    """B = 200 spans two 128-row calls: identical inputs give identical rows in REFERENCE mode (SEED keys each
    chunk and row differently)."""
    tk, d, n = _utt(3, 20, 0.5)
    B = 200
    tok, dur = np.repeat(tk[None], B, axis=0), np.repeat(d[None], B, axis=0)
    mel = eng.predict_mel(tok, dur, n_frames=[n] * B, rng=GOLDEN_RNG)
    assert np.array_equal(mel[0], mel[150]) and np.array_equal(mel[0], mel[127])
    seeded = eng.predict_mel(tok[:151], dur[:151], n_frames=[n] * 151, seed=5)
    assert not np.array_equal(seeded[0], seeded[150])


def test_device_pointer_entry_point(eng):
    import torch
    tok, dur, lens, nfs = _ragged(5, seed0=3)
    N = int(nfs.max())
    host = eng.predict_mel(tok, dur, lengths=lens, n_frames=nfs, rng=KEYS[3])
    dev = torch.device("cuda", 0)
    out = eng.acoustic_forward(torch.from_numpy(tok).to(dev), torch.from_numpy(dur).to(dev), N,
                               lengths_t=torch.from_numpy(lens).to(dev), n_frames_t=torch.from_numpy(nfs).to(dev), rng=KEYS[3])
    torch.cuda.synchronize()
    assert np.array_equal(out.cpu().numpy(), host)


# ---- 3. teacher-forced / GTA ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,N", [(1, 40), (3, 37), (33, 52)])
def test_teacher_forced_equals_mask_mode(eng, B, N):
    tok, dur, lens, _ = _ragged(B, seed0=100 + B)
    mels_in = synthetic.mel_input(4, B, N)
    for key in (KEYS[2], GOLDEN_RNG):
        keep, zone = _tf_masks(key, B, N)
        g1, g2 = eng.teacher_forced(tok, dur, mels_in, lengths=lens, rng=key)
        w1, w2 = eng.teacher_forced(tok, dur, mels_in, lengths=lens, keep_masks=keep, zone_masks=zone)
        assert np.array_equal(g1, w1) and np.array_equal(g2, w2)


def test_gta_golden_equals_mask_mode(eng):
    z = np.load(GOLDEN / "nat_ref_gta.npz")
    bits = lambda n: np.unpackbits(z[n + "_bits"])[: int(np.prod(z[n + "_shape"]))].reshape(tuple(int(s) for s in z[n + "_shape"]))  # noqa: E731
    got = eng.gta(z["wav_i16"], z["tokens"], z["durations_sec"], lengths=z["lengths"], rng=z["rng"])
    want = eng.gta(z["wav_i16"], z["tokens"], z["durations_sec"], lengths=z["lengths"], keep_masks=bits("keep"), zone_masks=bits("zone"))
    assert np.array_equal(got, want)
    B, S = z["wav_i16"].shape
    wav = np.concatenate([z["wav_i16"], z["wav_i16"][:, :256]], axis=1)     # odd frame count
    keep, zone = _tf_masks(tuple(int(x) for x in z["rng"].ravel()), B, wav.shape[1] // 256)
    got = eng.gta(wav, z["tokens"], z["durations_sec"], lengths=z["lengths"], rng=z["rng"])
    want = eng.gta(wav, z["tokens"], z["durations_sec"], lengths=z["lengths"], keep_masks=keep, zone_masks=zone)
    assert np.array_equal(got, want)


# ---- 4. one-call TTS -----------------------------------------------------------------------------------------------
def _staged(eng, tokens, silence_duration, key):
    d = no.adjust_durations(tokens, eng.predict_duration(np.asarray(tokens, np.int32)[None]), silence_duration)
    frames, n = no.seconds_to_frames(d)
    mel = eng.predict_mel(np.asarray(tokens, np.int32)[None], frames, n_frames=[n], masks=_inf_masks(key, n)[None])
    mel = no.trim_end_silence(tokens, d, mel)
    return eng.mel2wave(mel)[0], d


def test_tts_equals_staged_pipeline_with_reference_masks(eng):
    key = GOLDEN_RNG
    lens = np.array([30, 18, 25], np.int32)
    tok = np.zeros((3, 30), np.int32)
    rows = [_utt(40 + b, int(n), None)[0] for b, n in enumerate(lens)]
    for b, r in enumerate(rows):
        tok[b, : len(r)] = r
    waves, dur = eng.tts(tok, lens, silence_duration=0.12, rng=key)
    for b, r in enumerate(rows):
        wav, d = _staged(eng, [int(t) for t in r], 0.12, key)
        assert np.array_equal(dur[b, : len(r)], d[0])
        assert waves[b].shape == wav.shape
        assert np.abs(waves[b] - wav).max() < 1e-5
    # the same token row in another batch, at another row index: the same waveform
    other = np.zeros((2, 30), np.int32)
    other[0, :25] = _utt(77, 25, None)[0]
    other[1, : lens[1]] = rows[1]
    w2, _ = eng.tts(other, [25, lens[1]], silence_duration=0.12, rng=key)
    assert np.array_equal(w2[1], waves[1])


def test_cli_text_file_reference_dropout_equals_text(eng, acoustic_ckpt, hifigan_params, tmp_path, monkeypatch):
    from viettts_b200 import synthesizer
    from viettts_b200.engine import get_engine
    (tmp_path / "assets/hifigan").mkdir(parents=True)
    (tmp_path / "assets/infore/hifigan").mkdir(parents=True)
    (tmp_path / "assets/infore/nat").mkdir(parents=True)
    (tmp_path / "assets/hifigan/config.json").write_text(json.dumps(config.HIFIGAN))
    for path, obj in (("assets/infore/hifigan/hk_hifi.pickle", hifigan_params), ("assets/infore/nat/acoustic_latest_ckpt.pickle", acoustic_ckpt),
                      ("assets/infore/nat/duration_latest_ckpt.pickle", synthetic.duration_ckpt(1234))):
        with open(tmp_path / path, "wb") as f:
            pickle.dump(obj, f)
    monkeypatch.chdir(tmp_path)
    lex = str(GOLDEN / "lexicon_small.txt")
    get_engine(0).set_precision(eng.lib.vtts_get_precision(eng.h))
    texts = ["hôm nay trời đẹp quá! bạn có khỏe không?", "Xin chào, tôi là trợ lý ảo."]
    (tmp_path / "lines.txt").write_text("\n".join(texts) + "\n")
    assert synthesizer.main(["--text-file", "lines.txt", "--output", "out.wav", "--lexicon-file", lex, "--silence-duration", "0.1",
                             "--reference-dropout"]) == 0
    for i, text in enumerate(texts):
        assert synthesizer.main(["--text", text, "--output", f"one{i}.wav", "--lexicon-file", lex, "--silence-duration", "0.1"]) == 0
        one, _ = synthesizer.read_wav(tmp_path / f"one{i}.wav")
        many, _ = synthesizer.read_wav(tmp_path / f"out_{i:04d}.wav")
        assert one.size == many.size
        assert np.abs(one - many).max() * 32767.0 <= 1.0 + 1e-3, i
    for bad in (["--text-file", "lines.txt", "--reference-dropout", "--seed", "3"], ["--text", "xin chào", "--reference-dropout"]):
        with pytest.raises(SystemExit):
            synthesizer.main(bad + ["--lexicon-file", lex])


# ---- 5. errors -----------------------------------------------------------------------------------------------------
def test_mode_out_of_range_is_rejected(eng):
    tk, d, n = _utt(1, 8, 0.2)
    tok, dur, nf = np.ascontiguousarray(tk[None]), np.ascontiguousarray(d[None]), np.array([n], np.int32)
    mel = np.empty((1, n, 80), np.float32)
    rc = eng.lib.vtts_predict_mel_host(eng.h, tok.ctypes.data, None, dur.ctypes.data, nf.ctypes.data, None, 4, 0, 1, tok.shape[1], n,
                                       mel.ctypes.data)
    assert rc == -1 and b"dropout_mode 4" in eng.lib.vtts_last_error(eng.h)


def test_teacher_forced_draw_counter_limit(eng):
    import torch
    dummy = torch.zeros(1024, dtype=torch.float32, device="cuda")
    p = dummy.data_ptr()
    # B * N * 512 == 2^32: rejected before any workspace is sized
    rc = eng.lib.vtts_acoustic_teacher_forward(eng.h, p, None, p, None, p, None, None, 3, 42, 128, 1, 65536, None, p, None)
    assert rc == -1 and b"2^32" in eng.lib.vtts_last_error(eng.h)
    buf = np.zeros(16, np.uint8)
    assert eng.lib.vtts_debug_dropout_masks(eng.h, 1, 42, 128, 65536, buf.ctypes.data) == -1
    assert not buf.any()
    # modes past REFERENCE stay rejected on the teacher-forced path too
    rc = eng.lib.vtts_acoustic_teacher_forward(eng.h, p, None, p, None, p, None, None, 4, 42, 1, 1, 1, None, p, None)
    assert rc == -1 and b"dropout_mode 4" in eng.lib.vtts_last_error(eng.h)


def test_rng_argument_errors(eng):
    tk, d, n = _utt(1, 8, 0.2)
    m = _inf_masks(KEYS[0], n)[None]
    with pytest.raises(ValueError):
        eng.predict_mel(tk[None], d[None], n_frames=[n], masks=m, rng=KEYS[0])
    with pytest.raises(ValueError):
        eng.predict_mel(tk[None], d[None], n_frames=[n], seed=1, rng=KEYS[0])
    with pytest.raises(ValueError):
        eng.synthesize(tk[None], d[None], n_frames=[n], seed=1, rng=KEYS[0])
    with pytest.raises(ValueError):
        eng.tts(tk[None], seed=1, rng=KEYS[0])
    for bad in ([1, 2, 3], [7], np.zeros((2, 2), np.uint32), [0.5, 1.0]):
        with pytest.raises(ValueError):
            eng.predict_mel(tk[None], d[None], n_frames=[n], rng=bad)
    keep, zone = _tf_masks(KEYS[0], 1, n)
    mels_in = synthetic.mel_input(1, 1, n)
    with pytest.raises(ValueError):
        eng.teacher_forced(tk[None], d[None], mels_in, keep_masks=keep, zone_masks=zone, rng=KEYS[0])
    with pytest.raises(ValueError):
        eng.teacher_forced(tk[None], d[None], mels_in, seed=3, rng=KEYS[0])
    with pytest.raises(ValueError):
        eng.gta(np.zeros((1, 2048), np.int16), tk[None], d[None] / 62.5, seed=3, rng=[1])
