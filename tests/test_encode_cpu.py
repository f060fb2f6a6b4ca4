"""CPU: the wire encodings' definition (oracle/g711_oracle.py) against CPython's audioop and float_to_pcm16, the WAVE
layouts of write_wav / read_wav_codes, and the rejection of a bad encoding by AudioChain and the CLI."""
import struct
import warnings

import numpy as np
import pytest

from oracle import g711_oracle as g
from viettts_b200 import synthesizer

ALL_INT16 = np.arange(-32768, 32768, dtype=np.int64)


def edge_values() -> np.ndarray:
    """float32 samples around every rounding edge of the quantizer: for each int16 k the three floats on each side of
    (k +- 0.5) / 32767, plus signed zeros, denormals, +-1 and their neighbours, the clip edges, +-Inf, NaN and large
    values"""
    mids = ((np.arange(-32769, 32768, dtype=np.float64) + 0.5) / 32767.0).astype(np.float32)
    near = [mids]
    up, down = mids.copy(), mids.copy()
    for _ in range(3):
        up = np.nextafter(up, np.float32(np.inf))
        down = np.nextafter(down, np.float32(-np.inf))
        near += [up, down]
    tiny = np.float32(1.4e-45)
    special = np.array([0.0, -0.0, tiny, -tiny, 1e-40, -1e-40, 1.1754942e-38, -1.1754942e-38, 1.0, -1.0,
                        np.nextafter(np.float32(1), np.float32(2)), np.nextafter(np.float32(1), np.float32(0)),
                        np.nextafter(np.float32(-1), np.float32(-2)), np.nextafter(np.float32(-1), np.float32(0)),
                        32768 / 32767, -32768 / 32767, -32768.5 / 32767, 2.0, -2.0, 1e4, -1e4, 3.4028235e38, -3.4028235e38,
                        np.inf, -np.inf, np.nan], np.float32)
    return np.concatenate(near + [special]).astype(np.float32)


def speech_like(B, S, seed=0) -> np.ndarray:
    """seeded rows of voiced tones under a syllable envelope with noise, peaking near full scale"""
    rng = np.random.default_rng(seed)
    t = np.arange(S) / 16000.0
    x = np.zeros((B, S), np.float64)
    for b in range(B):
        f0 = rng.uniform(90, 250)
        v = sum(np.sin(2 * np.pi * f0 * h * t + rng.uniform(0, 6.3)) / h for h in range(1, 12))
        env = np.abs(np.sin(2 * np.pi * rng.uniform(2, 5) * t)) ** 2
        x[b] = 0.3 * v * env + 0.01 * rng.standard_normal(S)
    return x.astype(np.float32)


def audioop_or_skip():
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", DeprecationWarning)
        return pytest.importorskip("audioop")


def test_oracle_equals_audioop_both_ways():
    audioop = audioop_or_skip()
    pcm = ALL_INT16.astype("<i2").tobytes()
    codes = np.arange(256, dtype=np.uint8)
    assert np.array_equal(g.ulaw_of(ALL_INT16), np.frombuffer(audioop.lin2ulaw(pcm, 2), np.uint8))
    assert np.array_equal(g.alaw_of(ALL_INT16), np.frombuffer(audioop.lin2alaw(pcm, 2), np.uint8))
    assert np.array_equal(g.ulaw_to_int16(codes), np.frombuffer(audioop.ulaw2lin(codes.tobytes(), 2), "<i2"))
    assert np.array_equal(g.alaw_to_int16(codes), np.frombuffer(audioop.alaw2lin(codes.tobytes(), 2), "<i2"))


def test_oracle_fixed_points():
    assert g.ulaw_to_int16([0x00])[0] == -32124 and g.ulaw_to_int16([0xFF])[0] == 0
    for enc, code in g.SILENCE.items():
        assert g.encode(np.zeros(3, np.float32), enc).tolist() == [code] * 3
    assert g.encode(np.float32([np.nan, np.inf, -np.inf]), "pcm16").tolist() == [0, 32767, -32768]
    y = g.encode(np.ones((2, 5), np.float32), "alaw", lengths=[5, 2])
    assert y[0].tolist() == [g.alaw_of([32767])[0]] * 5 and y[1, 2:].tolist() == [0xD5] * 3
    # every code decodes to a value that encodes back to the same code (the G.711 expansion picks a segment's midpoint)
    for enc in ("ulaw", "alaw"):
        c = np.arange(256, dtype=np.uint8)
        back = g.encode(g.decode(c, enc), enc)
        same = back == c
        assert same.sum() >= 254, (enc, c[~same])     # only mu-law's two zeros (0x7F, 0xFF) may collapse


def test_oracle_pcm16_is_float_to_pcm16():
    x = np.concatenate([edge_values(), speech_like(4, 20000).ravel(), 1.5 * speech_like(2, 9000, 3).ravel()])
    x = x[np.isfinite(x)]
    assert np.array_equal(g.encode(x, "pcm16"), synthesizer.float_to_pcm16(x))


def test_edge_values_cross_every_rounding_edge():
    x = edge_values()
    v = g.to_int16(x[np.isfinite(x)])
    assert np.array_equal(np.unique(v), ALL_INT16)      # every int16 value is reached


def chunks(raw: bytes) -> dict:
    out, pos = {}, 12
    while pos + 8 <= len(raw):
        cid, size = raw[pos:pos + 4], struct.unpack("<I", raw[pos + 4:pos + 8])[0]
        out[cid] = raw[pos + 8:pos + 8 + size]
        pos += 8 + size + size % 2
    return out


@pytest.mark.parametrize("enc,tag", [("ulaw", 7), ("alaw", 6)])
@pytest.mark.parametrize("n", [0, 1, 1000, 1001])
def test_g711_wav_layout(tmp_path, enc, tag, n):
    codes = g.encode(speech_like(1, max(n, 1), n)[0, :n], enc)
    fn = tmp_path / "x.wav"
    synthesizer.write_wav(fn, codes, 8000, encoding=enc)
    raw = fn.read_bytes()
    assert raw[:4] == b"RIFF" and raw[8:12] == b"WAVE" and struct.unpack("<I", raw[4:8])[0] == len(raw) - 8
    assert len(raw) % 2 == 0 and raw[12:16] == b"fmt "
    c = chunks(raw)
    assert list(c) == [b"fmt ", b"fact", b"data"]
    assert struct.unpack("<HHIIHHH", c[b"fmt "]) == (tag, 1, 8000, 8000, 1, 8, 0)
    assert struct.unpack("<I", c[b"fact"]) == (n,)
    assert c[b"data"] == codes.tobytes()
    back, rate, got = synthesizer.read_wav_codes(fn)
    assert (rate, got) == (8000, enc) and back.dtype == np.uint8 and np.array_equal(back, codes)
    with pytest.raises(AssertionError):
        synthesizer.read_wav(fn)


def test_pcm16_wav_is_todays_file(tmp_path):
    x = speech_like(1, 3001, 5)[0]
    synthesizer.write_wav(tmp_path / "a.wav", x, 22050)
    synthesizer.write_wav(tmp_path / "b.wav", g.encode(x, "pcm16"), 22050, encoding="pcm16")
    a = (tmp_path / "a.wav").read_bytes()
    assert a == (tmp_path / "b.wav").read_bytes() and len(a) == 44 + 2 * x.size
    codes, rate, enc = synthesizer.read_wav_codes(tmp_path / "a.wav")
    assert (rate, enc) == (22050, "pcm16") and np.array_equal(codes, synthesizer.float_to_pcm16(x))
    wav, rate = synthesizer.read_wav(tmp_path / "a.wav")
    assert rate == 22050 and np.array_equal(wav, g.decode(codes, "pcm16"))


def test_write_wav_rejects_codes_of_the_wrong_type(tmp_path):
    with pytest.raises(ValueError):
        synthesizer.write_wav(tmp_path / "x.wav", np.zeros(4, np.float32), 8000, encoding="ulaw")
    with pytest.raises(ValueError):
        synthesizer.write_wav(tmp_path / "x.wav", np.zeros(4, np.uint8), 8000, encoding="pcm16")
    with pytest.raises(ValueError):
        synthesizer.write_wav(tmp_path / "x.wav", np.zeros(4, np.uint8), 8000, encoding="mp3")
    (tmp_path / "y.wav").write_bytes(b"RIFF\x04\x00\x00\x00WAVE")
    with pytest.raises(ValueError):
        synthesizer.read_wav_codes(tmp_path / "y.wav")


def test_audio_chain_encoding():
    from viettts_b200.engine import AudioChain, OptionError
    assert AudioChain().encoding is None
    ch = AudioChain(output_rate=8000, eq="telephone", encoding="ulaw", meter=True)
    assert ch.encoding == "ulaw" and [s[0] for s in ch._stages()] == ["rs", "eq", "mt"]
    for bad in ("mp3", "ULAW", "", 1):
        with pytest.raises(OptionError) as e:
            AudioChain(encoding=bad)
        assert e.value.option == "encoding" and "encoding" in str(e.value)


@pytest.mark.parametrize("argv", [["--encoding", "mp3"], ["--encoding", "g722"], ["--encoding", ""]])
def test_cli_rejects_bad_encoding(argv, capsys):
    with pytest.raises(SystemExit):
        synthesizer.main(["--text", "xin chào", *argv])
    assert "--encoding" in capsys.readouterr().err
