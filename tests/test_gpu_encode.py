"""GPU: the wire encodings (Engine.encode / encode_forward / decode / decode_forward, vtts_encode*, vtts_decode*), the TTS
stream's `encoding=`, the CLI's --encoding and watermark detection on a mu-law file.

Every comparison is bit for bit against the integer definition (oracle/g711_oracle.py)."""
import json
import pickle

import numpy as np
import pytest
import torch

from oracle import g711_oracle as g
from test_encode_cpu import edge_values, speech_like
from viettts_b200 import config, synthetic

pytestmark = pytest.mark.gpu
ENCS = ("pcm16", "ulaw", "alaw")
KEY = 7


@pytest.fixture(scope="module")
def eng():
    from viettts_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


def same(a, b):
    return a.dtype == b.dtype and a.shape == b.shape and np.array_equal(a, b)


@pytest.mark.parametrize("enc", ENCS)
def test_edge_set_equals_the_oracle(eng, enc):
    x = edge_values()
    assert same(eng.encode(x, enc), g.encode(x, enc))
    S = 4097
    rows = np.resize(x, (x.size + S - 1) // S * S).reshape(-1, S)
    assert same(eng.encode(rows, enc), g.encode(rows, enc))
    sp = speech_like(8, 40001, 1) * np.float32([[0.1], [0.5], [1.0], [1.5], [3.0], [1e-3], [0.8], [2.0]])
    assert same(eng.encode(sp, enc), g.encode(sp, enc))
    y_t = eng.encode_forward(torch.from_numpy(sp).cuda(), enc)
    assert same(y_t.cpu().numpy(), g.encode(sp, enc))


def test_decode_every_code(eng):
    for enc in ("ulaw", "alaw"):
        c = np.arange(256, dtype=np.uint8)
        y = eng.decode(c, enc)
        assert np.array_equal(y.view(np.int32), g.decode(c, enc).view(np.int32)), enc
        f = eng.decode_forward(torch.from_numpy(np.tile(c, (3, 1))).cuda(), enc).cpu().numpy()
        assert np.array_equal(f.view(np.int32), np.tile(g.decode(c, enc), (3, 1)).view(np.int32)), enc
    v = np.arange(-32768, 32768, dtype=np.int64).astype(np.int16)
    y = eng.decode(v, "pcm16")
    assert np.array_equal(y.view(np.int32), g.decode(v, "pcm16").view(np.int32))
    assert np.array_equal(y, v.astype(np.float32) / 32767.0)      # the scale of synthesizer.read_wav
    assert same(eng.encode(y, "pcm16"), v)


@pytest.mark.parametrize("enc", ENCS)
def test_ragged_odd_and_unaligned_rows(eng, enc):
    lengths = [0, 1, 3, 4, 5, 1001, 4099]
    B, S = len(lengths), 4099
    x = speech_like(B, S, 2)
    ref = g.encode(x, enc, lengths)
    assert same(eng.encode(x, enc, lengths=lengths), ref)
    for b, n in enumerate(lengths):
        assert np.all(ref[b, n:] == g.SILENCE[enc])
    dref = g.decode(ref, enc, lengths)
    assert np.array_equal(eng.decode(ref, enc, lengths=lengths).view(np.int32), dref.view(np.int32))
    n_t = torch.tensor(lengths, dtype=torch.int32, device="cuda")
    dt = torch.int16 if enc == "pcm16" else torch.uint8
    xbuf = torch.zeros(B * S + 8, dtype=torch.float32, device="cuda")
    cbuf = torch.zeros(B * S + 8, dtype=dt, device="cuda")
    fbuf = torch.zeros(B * S + 8, dtype=torch.float32, device="cuda")
    for ox, oc in ((0, 0), (1, 1), (3, 3), (1, 0), (2, 5), (0, 3)):    # same and different alignment phases
        xv = xbuf[ox:ox + B * S].view(B, S)
        xv.copy_(torch.from_numpy(x))
        cv = cbuf[oc:oc + B * S].view(B, S)
        assert eng.encode_forward(xv, enc, lengths_t=n_t, out=cv) is cv
        assert same(cv.cpu().numpy(), ref), (ox, oc)
        fv = fbuf[ox:ox + B * S].view(B, S)
        eng.decode_forward(cv, enc, lengths_t=n_t, out=fv)
        assert np.array_equal(fv.cpu().numpy().view(np.int32), dref.view(np.int32)), (ox, oc)


def test_same_bits_in_every_mode_and_batch_position(eng):
    lengths = [9000, 301, 16000, 7]
    x = speech_like(4, 16000, 3) * 1.7
    base = {enc: eng.encode(x, enc, lengths=lengths) for enc in ENCS}
    try:
        for mode in ("fp32", "bf16x3", "fp16"):
            eng.set_precision(mode)
            for enc in ENCS:
                assert same(eng.encode(x, enc, lengths=lengths), base[enc]), (mode, enc)
                assert np.array_equal(eng.decode(base[enc], enc), g.decode(base[enc], enc)), (mode, enc)
    finally:
        eng.set_precision("bf16x3")
    for enc in ENCS:
        for b in range(4):
            assert same(eng.encode(x[b, :lengths[b]], enc), base[enc][b, :lengths[b]]), (enc, b)
            perm = np.roll(np.arange(4), b)
            assert same(eng.encode(x[perm], enc, lengths=np.array(lengths)[perm]), base[enc][perm]), (enc, b)


def test_one_launch_per_call_and_argument_errors(eng):
    from viettts_b200 import _lib
    x = speech_like(3, 5001, 4)
    x_t = torch.from_numpy(x).cuda()
    for enc in ENCS:
        for call in (lambda: eng.encode(x, enc), lambda: eng.encode_forward(x_t, enc),
                     lambda: eng.decode(g.encode(x, enc), enc), lambda: eng.decode_forward(torch.from_numpy(g.encode(x, enc)).cuda(), enc)):
            c0 = eng.launch_count()
            call()
            assert eng.launch_count() - c0 == 1, enc
    lib = eng.lib
    y = np.zeros((3, 5001), np.int16)
    f = np.zeros((3, 5001), np.float32)
    c0 = eng.launch_count()
    for enc_id in (-1, 3, 7):
        with pytest.raises(_lib.VttsError, match="encoding"):
            eng._ck(lib.vtts_encode_host(eng.h, x.ctypes.data, None, 3, 5001, enc_id, y.ctypes.data))
        with pytest.raises(_lib.VttsError, match="encoding"):
            eng._ck(lib.vtts_decode(eng.h, y.ctypes.data, None, 3, 5001, enc_id, f.ctypes.data, None))
    for B, S in ((0, 5001), (-1, 5001), (3, 0), (3, -5), (65536, 1)):
        with pytest.raises(_lib.VttsError):
            eng._ck(lib.vtts_encode_host(eng.h, x.ctypes.data, None, B, S, 0, y.ctypes.data))
        with pytest.raises(_lib.VttsError):
            eng._ck(lib.vtts_decode_host(eng.h, y.ctypes.data, None, B, S, 0, f.ctypes.data))
    with pytest.raises(_lib.VttsError, match="null"):
        eng._ck(lib.vtts_encode(eng.h, None, None, 3, 5001, 1, x_t.data_ptr(), None))
    with pytest.raises(_lib.VttsError, match="null"):
        eng._ck(lib.vtts_encode(eng.h, x_t.data_ptr(), None, 3, 5001, 1, None, None))
    with pytest.raises(_lib.VttsError, match="null"):
        eng._ck(lib.vtts_decode_host(eng.h, None, None, 3, 5001, 1, f.ctypes.data))
    with pytest.raises(_lib.VttsError, match="overlaps"):     # y aliasing x, or inside it
        eng._ck(lib.vtts_encode(eng.h, x_t.data_ptr(), None, 3, 5001, 1, x_t.data_ptr(), None))
    with pytest.raises(_lib.VttsError, match="overlaps"):
        eng._ck(lib.vtts_decode(eng.h, x_t.data_ptr() + 4 * 5001, None, 3, 5001, 0, x_t.data_ptr(), None))
    n = np.array([5, 5002, 1], np.int32)
    with pytest.raises(_lib.VttsError, match="outside"):
        eng._ck(lib.vtts_encode_host(eng.h, x.ctypes.data, n.ctypes.data, 3, 5001, 2, y.ctypes.data))
    assert eng.launch_count() == c0
    for bad in ("mp3", "PCM16", None):
        with pytest.raises(ValueError):
            eng.encode(x, bad)
    with pytest.raises(ValueError):
        eng.decode(np.zeros(4, np.uint8), "pcm16")
    with pytest.raises(ValueError):
        eng.encode_forward(x_t, "ulaw", out=torch.zeros((3, 5001), dtype=torch.int16, device="cuda"))
    assert eng.launch_count() == c0


# ---- the TTS stream, the CLI and the mark through the phone path ----
@pytest.fixture(scope="module")
def tts_eng(acoustic_ckpt, hifigan_params):
    from viettts_b200.engine import Engine
    e = Engine(0)
    e.load_acoustic(acoustic_ckpt)
    e.load_hifigan(hifigan_params)
    e.load_duration(synthetic.duration_ckpt(1234))
    yield e
    e.close()


def tts_tokens(seed, L):
    rng = np.random.default_rng(seed)
    t = rng.integers(4, 90, size=L).astype(np.int32)
    t[4::5] = 3
    t[0] = t[-1] = 0
    return t


@pytest.mark.parametrize("enc,rate,eq", [("ulaw", 8000, "telephone"), ("pcm16", None, None)])
def test_tts_stream_encoding(tts_eng, enc, rate, eq):
    from viettts_b200.engine import AudioChain
    eng = tts_eng
    eng.set_precision("bf16x3")
    eng.set_fused_pairs(False)
    try:
        toks = [tts_tokens(190 + b, n) for b, n in enumerate([25, 40, 12])]
        audio = {s: [] for s in range(3)}
        with eng.open_tts_stream(3, 16, 2000, 100, output_rate=rate, eq=eq, meter=True, encoding=enc) as ts:
            for s in range(3):
                ts.begin(s, toks[s], silence_duration=0.1)
            while ts.busy().any():
                for s, w in ts.step().items():
                    assert w.dtype == g.DTYPES[enc]
                    audio[s].append(w)
            chain = AudioChain(output_rate=rate, eq=eq)
            floats = [chain.run(eng, eng.tts(toks[s][None], silence_duration=0.1)[0][0]) for s in range(3)]
            for s in range(3):
                got = np.concatenate(audio[s])
                assert same(got, eng.encode(floats[s], enc)) and same(got, g.encode(floats[s], enc)), s
        with pytest.raises(ValueError, match="encoding"):
            eng.open_tts_stream(1, 16, 2000, 100, encoding="opus")
    finally:
        eng.set_fused_pairs(True)


def cli_assets(tmp_path, monkeypatch, acoustic_ckpt, hifigan_params):
    (tmp_path / "assets/hifigan").mkdir(parents=True)
    (tmp_path / "assets/infore/hifigan").mkdir(parents=True)
    (tmp_path / "assets/infore/nat").mkdir(parents=True)
    (tmp_path / "assets/hifigan/config.json").write_text(json.dumps(config.HIFIGAN))
    for path, obj in (("assets/infore/hifigan/hk_hifi.pickle", hifigan_params), ("assets/infore/nat/acoustic_latest_ckpt.pickle", acoustic_ckpt),
                      ("assets/infore/nat/duration_latest_ckpt.pickle", synthetic.duration_ckpt(1234))):
        with open(tmp_path / path, "wb") as f:
            pickle.dump(obj, f)
    monkeypatch.chdir(tmp_path)


def test_cli_encoding(tts_eng, acoustic_ckpt, hifigan_params, golden_dir, tmp_path, monkeypatch, capsys):
    from viettts_b200 import synthesizer
    from viettts_b200 import watermark as wm_cli
    from viettts_b200.engine import get_engine
    from viettts_b200.hifigan.mel2wave import mel2wave
    from viettts_b200.nat.text2mel import text2mel
    cli_assets(tmp_path, monkeypatch, acoustic_ckpt, hifigan_params)
    lex = str(golden_dir / "lexicon_small.txt")
    ge = get_engine(0)
    text = "Xin chào, tôi là trợ lý ảo."
    base = ["--text", text, "--lexicon-file", lex, "--silence-duration", "0.1"]
    assert synthesizer.main([*base, "--output", "plain.wav"]) == 0
    assert synthesizer.main([*base, "--output", "pcm16.wav", "--encoding", "pcm16"]) == 0
    assert (tmp_path / "plain.wav").read_bytes() == (tmp_path / "pcm16.wav").read_bytes()

    wave = np.ravel(mel2wave(text2mel(synthesizer.nat_normalize_text(text), lex, 0.1)))
    assert synthesizer.main([*base, "--output", "phone.wav", "--output-rate", "8000", "--eq", "telephone", "--encoding", "ulaw"]) == 0
    raw = (tmp_path / "phone.wav").read_bytes()
    assert raw[20:22] == b"\x07\x00"
    codes, rate, enc = synthesizer.read_wav_codes(tmp_path / "phone.wav")
    assert (rate, enc) == (8000, "ulaw")
    assert same(codes, g.encode(ge.equalize(ge.resample(wave, 8000), "telephone", 8000), "ulaw"))

    assert synthesizer.main([*base, "--output", "marked.wav", "--watermark", f"key={KEY},strength=0.3", "--encoding", "ulaw"]) == 0
    codes, rate, enc = synthesizer.read_wav_codes(tmp_path / "marked.wav")
    assert (rate, enc) == (16000, "ulaw")
    ref = ge.detect_watermark(g.decode(codes, "ulaw"), [KEY, 99], rate=rate, search=False)
    capsys.readouterr()
    rc = wm_cli.main(["detect", "--key", str(KEY), "--key", "99", "--aligned", str(tmp_path / "marked.wav")])
    lines = capsys.readouterr().out.strip().splitlines()
    print("mu-law CLI file, aligned z:", ref.z)
    assert len(lines) == 2 and f"z={ref.z[0]:.2f}" in lines[0] and f"z={ref.z[1]:.2f}" in lines[1]
    assert rc == 0 and "\tmarked" in lines[0] and "not marked" in lines[1]


def test_watermark_through_the_phone_path(eng):
    from test_watermark_cpu import speech
    keys = [KEY] + list(range(2000, 2063))
    y = eng.watermark(speech(20.0).astype(np.float32), KEY)
    phone = eng.equalize(eng.resample(y, 8000), "telephone", 8000)
    codes = eng.encode(phone, "ulaw")
    assert same(codes, g.encode(phone, "ulaw"))
    heard = eng.decode(codes, "ulaw")
    r = eng.detect_watermark(heard, keys, rate=8000, search=True)
    a = eng.detect_watermark(heard, keys, rate=8000, search=False)
    print(f"marked, 8 kHz, telephone, mu-law: search z {r.z[0]:.2f} (offset {r.offset[0]}), aligned z {a.z[0]:.2f}; "
          f"wrong keys search max {r.z[1:].max():.2f}")
    d = int(r.offset[0]) % 65536
    assert r.detected[0] and min(d, 65536 - d) <= 2 * 64, (r.z[0], r.offset[0])     # the search grid is 64
    assert not r.detected[1:].any()
