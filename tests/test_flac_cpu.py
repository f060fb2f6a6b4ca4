"""CPU: the FLAC definition (oracle/flac_oracle.py) round-trips every signal class, its decoder is strict and takes what
other encoders write, the speech fixture compresses, and the `flac` option parses (AudioChain, the CLI)."""
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest

from oracle import flac_oracle as fo
from oracle import g711_oracle as g
from oracle import resample_oracle as ro
from viettts_b200 import synthesizer

GOLDEN = Path(__file__).resolve().parent / "golden"
TABLE_RATES = sorted(fo.RATE_CODES)
# one rate of each non-table branch: 8-bit kHz, 16-bit Hz (11 025 Hz), 16-bit tens of Hz
BRANCH_RATES = [(12, 9000), (13, 11025), (14, 110250)]


def speech_pcm() -> np.ndarray:
    return np.load(GOLDEN / "watermark_speech_clip.npz")["pcm"].astype(np.int16)


def flac_signals(block: int = 4096) -> dict:
    """float32 rows of the signal classes the encoder must survive"""
    rng = np.random.default_rng(5)
    n = 3 * block + 77
    t = np.arange(n)
    sq = np.where((t // 37) % 2 == 0, 1.0, -1.0)
    alt = np.where(t % 2 == 0, 32767, -32768) / 32767.0
    click = np.zeros(n)
    click[n // 3] = 0.9
    return {name: np.asarray(v, np.float32) for name, v in {
        "silence": np.zeros(n),
        "dc": np.full(n, 0.25),
        "nyquist": 0.5 * np.where(t % 2 == 0, 1.0, -1.0),
        "square": sq,
        "alternating": alt,
        "click": click,
        "noise": rng.uniform(-1.0, 1.0, n),
        "tone": 0.6 * np.sin(2 * np.pi * 440.0 * t / 16000.0),
    }.items()}


def lengths_for(block: int):
    return [0, 1, 15, 16, block - 1, block, block + 1, 5 * block + 3]


def roundtrip(codes, rate, block):
    data = fo.encode(codes, rate, block)
    y, r, si = fo.decode(data)
    assert np.array_equal(y, codes) and r == rate
    assert si["total"] == codes.size and si["min_block"] == si["max_block"] == block
    assert si["channels"] == 1 and si["bps"] == 16 and si["md5"] == bytes(16)
    frames = fo.frames_of(data)
    sizes = [len(f) for f in frames]
    assert (si["min_frame"], si["max_frame"]) == ((min(sizes), max(sizes)) if sizes else (0, 0))
    assert len(frames) == -(-codes.size // block)
    return data, frames


def subframe_type(frame: bytes) -> int:
    """the 6-bit subframe type of a frame of ours (the header length from its own fields)"""
    b = fo._Bits(frame)
    b.u(16)
    bc, rc = b.u(4), b.u(4)
    b.u(8)
    fo._utf8(b, 6)
    if bc in (6, 7):
        b.u(8 if bc == 6 else 16)
    if rc in (12, 13, 14):
        b.u(8 if rc == 12 else 16)
    b.u(8)
    b.u(1)
    return b.u(6)


def test_speech_roundtrip_and_compression():
    pcm = speech_pcm()
    data, frames = roundtrip(pcm, 16000, 4096)
    assert len(data) < 2 * pcm.size
    for i, f in enumerate(frames):       # no frame is larger than its VERBATIM form
        n = min(4096, pcm.size - 4096 * i)
        assert len(f) <= len(fo.frame_header(n, i, 16000, 4096)) + 1 + 2 * n + 2
    x = pcm.astype(np.float64) / 32767.0
    for rate in (8000, 48000):
        r = g.to_int16(ro.resample(x, 16000, rate).astype(np.float32)).astype(np.int16)
        d, _ = roundtrip(r, rate, 4096)
        assert len(d) < 2 * r.size


@pytest.mark.parametrize("block", fo.BLOCKS)
def test_signal_classes_roundtrip(block):
    for name, x in flac_signals(block).items():
        c = g.to_int16(x).astype(np.int16)
        for n in lengths_for(block):
            data, frames = roundtrip(c[:n], 44100, block)
            if name == "silence" and n:
                assert all(subframe_type(f) == 0 for f in frames), (name, n)       # CONSTANT
            if name == "noise" and n > 16:
                assert subframe_type(frames[0]) == 1, (name, n)                    # VERBATIM


def test_every_rate_branch():
    c = g.to_int16(flac_signals(256)["tone"]).astype(np.int16)[:1000]
    for rate in TABLE_RATES:
        data, frames = roundtrip(c, rate, 256)
        assert frames[0][2] & 0xF == fo.RATE_CODES[rate]
    for code, rate in BRANCH_RATES:
        data, frames = roundtrip(c, rate, 256)
        assert frames[0][2] & 0xF == code, rate
    for bad in (0, -1, 65537, 655351, 1_000_000):
        with pytest.raises(ValueError):
            fo.encode(c, bad, 256)
    with pytest.raises(ValueError):
        fo.encode(c, 16000, 1000)


@pytest.mark.parametrize("number", [127, 128, 2047, 2048, 65535, 65536, 2**21 - 1, 2**21, 2**26 - 1, 2**26, 2**31 - 1])
def test_frame_numbers_roundtrip(number):
    x = g.to_int16(flac_signals(256)["tone"][:256]).astype(np.int64)
    frame = fo.encode_frame(x, number, 16000, 256)
    si = {"rate": 16000, "bps": 16}
    y, end, h = fo.decode_frame(frame, 0, si, expect=number)
    assert end == len(frame) and h["number"] == number and np.array_equal(y, x)
    assert len(fo.utf8_number(number)) == 1 + sum(number >= v for v in (0x80, 0x800, 0x10000, 0x200000, 0x4000000))


# ---- the decoder is strict, and takes more than the encoder writes ----------------------------------------------
def _stream(frames, n_total=0, block=4096, rate=16000):
    return fo.streaminfo(block, rate, n_total, 0, 0) + b"".join(frames)


def _frame(sub_vals, sub_bits, n, number=0, block=4096, rate=16000, variable=False):
    """a hand-built frame: header + the given subframe fields + padding + CRC-16"""
    h = fo.frame_header(n, number, rate, block, variable=variable)
    f = h + fo._pack(sub_vals, sub_bits)
    return f + fo.crc16(f).to_bytes(2, "big")


def test_decoder_rejects_damage():
    c = g.to_int16(flac_signals(4096)["tone"]).astype(np.int16)[:6000]
    data = fo.encode(c, 16000, 4096)
    flip = bytearray(data)
    flip[len(data) - 40] ^= 0x10                       # payload bit: CRC-16
    with pytest.raises(fo.FlacError, match="CRC-16"):
        fo.decode(bytes(flip))
    hdr = bytearray(data)
    hdr[42 + 2] ^= 0x01                                # the rate code of frame 0: CRC-8
    with pytest.raises(fo.FlacError, match="CRC-8"):
        fo.decode(bytes(hdr))
    sync = bytearray(data)
    sync[42 + 1] = 0xFA                                # reserved bit after the sync code
    with pytest.raises(fo.FlacError):
        fo.decode(bytes(sync))
    sync[42] = 0xFE
    with pytest.raises(fo.FlacError, match="sync"):
        fo.decode(bytes(sync))
    n = 64
    # LPC order 1 (warm-up 5, precision code, shift, coefficient 1, method 0, partition order 0, k = 0, 63 zero
    # residuals) with a negative shift, and with precision code 15
    for pc, shift, msg in ((4, -1 & 31, "negative"), (15, 0, "precision code 15")):
        vals = [0x20 << 1, 5, pc, shift, 1, 0, 0, 0] + [1] * (n - 1)
        bits = [8, 16, 4, 5, 5, 2, 4, 4] + [1] * (n - 1)
        with pytest.raises(fo.FlacError, match=msg):
            fo.decode(_stream([_frame(vals, bits, n, block=256)], block=256))
    n = 60                                             # FIXED 1 at partition order 3: 60 is not divisible by 2^3
    vals = [0x09 << 1, 0, 0, 3]
    bits = [8, 16, 2, 4]
    with pytest.raises(fo.FlacError, match="does not divide"):
        fo.decode(_stream([_frame(vals, bits, n, block=256)], block=256))


def test_decoder_takes_what_our_encoder_never_writes():
    rng = np.random.default_rng(1)
    n = 64
    # wasted bits: VERBATIM of x = 4 y with 2 wasted bits (flag 1, unary 1 -> k = 2), 14-bit samples
    y = rng.integers(-8000, 8000, n)
    vals = [(1 << 1) | 1, 1] + [int(v) & 0x3FFF for v in y]
    bits = [8, 2] + [14] * n
    out, _, _ = fo.decode(_stream([_frame(vals, bits, n, block=256)], n, block=256))
    assert np.array_equal(out, 4 * y)
    # FIXED 2 with method 1 (5-bit Rice parameters): one partition, k = 20, and one escaped partition at order 1
    x = rng.integers(-30000, 30000, n)
    r = x[2:] - 2 * x[1:-1] + x[:-2]
    u = fo.zigzag(r)
    k = 20
    vals = [(0x08 | 2) << 1, int(x[0]) & 0xFFFF, int(x[1]) & 0xFFFF, 1, 0, k]
    bits = [8, 16, 16, 2, 4, 5]
    for v in u:
        vals.append((1 << k) | (int(v) & ((1 << k) - 1)))
        bits.append(int(v >> k) + 1 + k)
    out, _, _ = fo.decode(_stream([_frame(vals, bits, n, block=256)], n, block=256))
    assert np.array_equal(out, x)
    # escape partitions: FIXED 1, partition order 1, partition 0 escaped at 18 bits, partition 1 Rice k = 15
    r = np.diff(x)
    vals = [(0x08 | 1) << 1, int(x[0]) & 0xFFFF, 0, 1, 15, 18] + [int(v) & 0x3FFFF for v in r[:31]]
    bits = [8, 16, 2, 4, 4, 5] + [18] * 31
    vals += [14]
    bits += [4]
    for v in fo.zigzag(r[31:]):
        vals.append((1 << 14) | (int(v) & 0x3FFF))
        bits.append(int(v >> 14) + 15)
    out, _, _ = fo.decode(_stream([_frame(vals, bits, n, block=256)], n, block=256))
    assert np.array_equal(out, x)
    # variable blocksize: frames of 100 and 28 samples numbered by their first sample, CONSTANT and VERBATIM
    f0 = _frame([0, 123], [8, 16], 100, number=0, block=256, variable=True)
    f1 = _frame([1 << 1] + [int(v) & 0xFFFF for v in x[:28]], [8] + [16] * 28, 28, number=100, block=256, variable=True)
    out, _, si = fo.decode(_stream([f0, f1], 128, block=256))
    assert np.array_equal(out, np.concatenate([np.full(100, 123), x[:28]]))


def _external_decoder():
    try:
        import soundfile
        if "FLAC" in soundfile.available_formats():
            return "soundfile"
    except Exception:
        pass
    return "flac" if shutil.which("flac") else None


def test_external_decoder_agrees(tmp_path):
    which = _external_decoder()
    if which is None:
        pytest.skip("neither soundfile with FLAC support nor a flac binary is installed")
    pcm = speech_pcm()[:50000]
    f = tmp_path / "a.flac"
    f.write_bytes(fo.encode(pcm, 16000, 4096))
    if which == "soundfile":
        import soundfile
        y, sr = soundfile.read(str(f), dtype="int16")
    else:
        out = tmp_path / "a.raw"
        subprocess.run(["flac", "-d", "-s", "--force-raw-format", "--endian=little", "--sign=signed", "-o", str(out), str(f)],
                       check=True)
        y, sr = np.frombuffer(out.read_bytes(), "<i2"), 16000
    assert sr == 16000 and np.array_equal(y, pcm)


# ---- the option --------------------------------------------------------------------------------------------------
def test_audio_chain_flac_option():
    from viettts_b200.engine import AudioChain, OptionError, flac_params
    assert AudioChain(encoding="flac").flac == {"block": 4096}
    assert AudioChain(encoding="flac,block=1024").flac == {"block": 1024}
    assert flac_params("flac,block=256") == {"block": 256}
    for bad in ("flac,block=1000", "FLAC", "flac,level=5", "flac,block=", "flacx"):
        with pytest.raises(OptionError) as e:
            AudioChain(encoding=bad)
        assert e.value.option == "encoding"
    with pytest.raises(OptionError) as e:                # 127 875 Hz: reachable by the resampler, not stated by FLAC
        AudioChain(encoding="flac", output_rate=127875)
    assert e.value.option == "encoding"
    for bad in ("mp3", "g722", "opus", "ULAW"):
        with pytest.raises(OptionError):
            AudioChain(encoding=bad)


def test_per_sample_encode_points_at_encode_flac():
    from viettts_b200.engine import encoding_name
    with pytest.raises(ValueError, match="encode_flac"):
        encoding_name("flac")


def test_flac_bound_matches_the_oracle():
    from viettts_b200.engine import flac_bound
    for S in (0, 1, 255, 256, 4097, 80000, 2**28):
        for block in fo.BLOCKS:
            assert flac_bound(S, block) == fo.bound(S, block)


def test_cli_parses_flac(capsys):
    with pytest.raises(SystemExit):
        synthesizer.main(["--encoding", "flac,block=512"])     # no text: the chain parsed, the text is missing
    assert "--text" in capsys.readouterr().err
    with pytest.raises(SystemExit):
        synthesizer.main(["--text", "xin chào", "--encoding", "flac,block=1000"])
    assert "--encoding" in capsys.readouterr().err


# ---- known answers: the tables and CRCs the encoder and decoder share, pinned to published values -------------------
def test_crc_known_answers():
    assert fo.crc8(b"123456789") == 0xF4          # CRC-8 (poly 0x07, init 0): the catalogue check value
    assert fo.crc16(b"123456789") == 0xFEE8       # CRC-16/BUYPASS (poly 0x8005, init 0, no reflection)
    assert fo.crc8(b"") == 0 and fo.crc16(b"") == 0


def test_rfc_code_tables():
    # RFC 9639 section 9.1.2 (sample rate bits) and 9.1.1 (block size bits), written out here
    assert fo.RATE_CODES == {88200: 0b0001, 176400: 0b0010, 192000: 0b0011, 8000: 0b0100, 16000: 0b0101, 22050: 0b0110,
                             24000: 0b0111, 32000: 0b1000, 44100: 0b1001, 48000: 0b1010, 96000: 0b1011}
    assert fo.BLOCK_CODES == {256: 0b1000, 512: 0b1001, 1024: 0b1010, 2048: 0b1011, 4096: 0b1100}
    assert fo._BS_TABLE[1] == 192 and [fo._BS_TABLE[c] for c in range(2, 6)] == [576, 1152, 2304, 4608]
    # the coded-number examples: 1..7 bytes at each boundary
    assert fo.utf8_number(0x7F) == b"\x7f" and fo.utf8_number(0x80) == b"\xc2\x80"
    assert fo.utf8_number(0x7FF) == b"\xdf\xbf" and fo.utf8_number(0x800) == b"\xe0\xa0\x80"
    assert fo.utf8_number(0xFFFF) == b"\xef\xbf\xbf" and fo.utf8_number(0x10000) == b"\xf0\x90\x80\x80"
    assert fo.utf8_number(2**31 - 1) == b"\xfd\xbf\xbf\xbf\xbf\xbf" and len(fo.utf8_number(2**36 - 1)) == 7
    assert list(fo.zigzag(np.array([0, -1, 1, -2, 2, 2**31 - 1, -2**31]))) == [0, 1, 2, 3, 4, 2**32 - 2, 2**32 - 1]


def test_library_rate_codes_match_the_oracle():
    from viettts_b200 import _lib
    lib = _lib.load()
    for rate in TABLE_RATES + [r for _, r in BRANCH_RATES] + [1, 7, 65535, 65540, 255000, 256000, 655350, 655351, 0, -5]:
        try:
            want = fo.rate_code(rate)[0]
        except ValueError:
            want = -1
        assert lib.vtts_flac_rate_code(rate) == want, rate


def test_stream_frame_count_formula():
    from viettts_b200.engine import flac_stream_frames
    assert [flac_stream_frames(p, 256) for p in (0, 255, 256, 257, 512)] == [0, 0, 1, 1, 2]
    assert [flac_stream_frames(p, 256, True) for p in (0, 1, 256, 257)] == [0, 1, 1, 2]
