"""GPU: the watermark (Engine.watermark / watermark_forward, vtts_watermark*), its stream (Engine.open_watermark_stream),
the batched detector (Engine.detect_watermark / detect_watermark_forward), the TTS stream's `watermark=` stage and the
CLI's --watermark with the `python -m viettts_b200.watermark detect` entry point.

Embedded audio is held to the float64 definition (oracle/watermark_oracle.py) within TOL_EMBED error units and z within
TOL_Z (tests/test_watermark_cpu.py); everything that streams, and every precision mode and batch position, is compared
bit for bit with the one-shot call.  Detection floors are measured on the speech fixture through the library's own
device stages."""
import ctypes
import json
import pickle

import numpy as np
import pytest
import torch

from helpers import slot_streams as ss
from oracle import watermark_oracle as wo
from test_watermark_cpu import KEY, SR, TOL_EMBED, TOL_Z, embed_scale, speech
from viettts_b200 import config, synthetic

pytestmark = pytest.mark.gpu
KEYS64 = [KEY] + list(range(2000, 2063))


@pytest.fixture(scope="module")
def eng():
    from viettts_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


def rows(lengths, seed=0):
    S = max(max(lengths), 1)
    x = np.zeros((len(lengths), S), np.float32)
    for b, n in enumerate(lengths):
        x[b, :n] = speech(n / SR + 0.01, 1.0 + 0.37 * ((b + seed) % 7))[:n]
    return x


LENGTHS = [0, 1, 512, 513, 1023, 1024, 5000, 70001]


@pytest.mark.parametrize("eps", [0.05, 0.1, 0.3])
def test_ragged_rows_against_float64(eng, eps):
    x = rows(LENGTHS)
    y = eng.watermark(x, f"key={KEY},strength={eps}", lengths=LENGTHS)
    for b, n in enumerate(LENGTHS):
        assert np.all(y[b, n:] == 0), b
        if n == 0:
            continue
        if n <= 512:
            assert np.array_equal(y[b, :n], x[b, :n]), b
            continue
        ref = wo.embed(x[b, :n], KEY, np.float32(eps))
        e = np.max(np.abs(y[b, :n] - ref) / embed_scale(x[b, :n], eps))
        assert e <= TOL_EMBED, (b, n, e)


def test_three_minute_row_and_edge_cases(eng):
    x = np.tile(speech(20.0), 9).astype(np.float32)
    y = eng.watermark(x, KEY)
    e = np.max(np.abs(y - wo.embed(x, KEY, np.float32(0.1))) / embed_scale(x, 0.1))
    assert e <= TOL_EMBED, e
    x = rows([20000, 7000])
    x[1, 5] = -0.0
    y = eng.watermark(x, f"key={KEY},strength=0", lengths=[20000, 7000])
    assert np.array_equal(y[0].view(np.int32), x[0].view(np.int32)) and np.array_equal(y[1, :7000].view(np.int32), x[1, :7000].view(np.int32))
    assert np.all(y[1, 7000:] == 0)
    assert np.all(eng.watermark(np.zeros((2, 9000), np.float32), KEY) == 0)


def test_same_bits_in_every_mode_and_batch_position(eng):
    lengths = [5000, 3000, 70000, 600]
    x = rows(lengths, 1)
    base = eng.watermark(x, KEY, lengths=lengths)
    zb = eng.detect_watermark(x, KEYS64[:5], lengths=lengths)
    try:
        for mode in ("fp32", "bf16x3", "fp16"):
            eng.set_precision(mode)
            assert np.array_equal(eng.watermark(x, KEY, lengths=lengths), base), mode
            zm = eng.detect_watermark(x, KEYS64[:5], lengths=lengths)
            assert np.array_equal(zm.z, zb.z) and np.array_equal(zm.offset, zb.offset), mode
    finally:
        eng.set_precision("bf16x3")
    for b in range(4):
        assert np.array_equal(eng.watermark(x[b, :lengths[b]], KEY), base[b, :lengths[b]]), b
        perm = np.roll(np.arange(4), b)
        assert np.array_equal(eng.watermark(x[perm], KEY, lengths=np.array(lengths)[perm]), base[perm]), b
        one = eng.detect_watermark(x[b, :lengths[b]], KEYS64[:5])
        assert np.array_equal(one.z, zb.z[b]) and np.array_equal(one.offset, zb.offset[b]), b


def test_forward_matches_host(eng):
    lengths = [40000, 9000]
    x = rows(lengths, 2)
    ref = eng.watermark(x, KEY, lengths=lengths)
    x_t = torch.from_numpy(x).cuda()
    n_t = torch.tensor(lengths, dtype=torch.int32, device="cuda")
    assert np.array_equal(eng.watermark_forward(x_t, KEY, lengths_t=n_t).cpu().numpy(), ref)
    d = eng.detect_watermark(ref, KEYS64, lengths=lengths)
    f = eng.detect_watermark_forward(torch.from_numpy(ref).cuda(), KEYS64, lengths_t=n_t)
    assert np.array_equal(f.z.cpu().numpy(), d.z) and np.array_equal(f.offset.cpu().numpy(), d.offset)
    assert np.array_equal(f.detected.cpu().numpy(), d.detected)


def check_z(got, x, keys, search):
    zz = wo.scores(x, keys, search)
    ref, off = wo.detect(x, keys, search)
    assert np.max(np.abs(got.z - ref)) <= TOL_Z, np.max(np.abs(got.z - ref))
    for c in range(len(keys)):
        top = np.sort(zz[c].ravel())[::-1]
        if top.size == 1 or top[0] - top[1] > TOL_Z:
            assert got.offset[c] == off[c], (c, got.offset[c], off[c])


@pytest.mark.parametrize("search", [False, True])
def test_detect_against_float64(eng, search):
    y = eng.watermark(speech(8.0).astype(np.float32), KEY)
    for x in (y, y[777 * 64 + 5:], speech(3.0, 11.0).astype(np.float32), np.zeros(9000, np.float32), y[:600]):
        check_z(eng.detect_watermark(x, KEYS64[:8], search=search), x.astype(np.float64), KEYS64[:8], search)


@pytest.mark.parametrize("S", [1, 3, 32])
@pytest.mark.parametrize("pattern,device", [("one", False), ("full", False), ("full", True), ("random", False), ("random", True)])
def test_stream_equals_one_shot(eng, S, pattern, device):
    """rows pushed in `pattern` chunks and held to the stream's contract on every push (tests/helpers/slot_streams.py)"""
    if pattern == "one" and S == 32:
        pytest.skip("one-sample pushes run at S = 1 and 3")
    lengths = [int(v) for v in np.random.default_rng(S).integers(1, 2500 if pattern == "one" else 30000, size=S)]
    if S == 3:
        lengths[:2] = [512, 1024] if pattern != "one" else lengths[:2]
    x = rows(lengths, S)
    rng = np.random.default_rng(7)
    for spec in (KEY, f"key={2**64 - 1},strength=0.3", f"key={KEY},strength=0"):
        for chunk in (300, 1500):
            stage = ss.stage(eng, "watermark", S, chunk, spec=spec)
            with stage.open() as st:
                assert st.lookahead == 1023 and st.out_pitch == chunk + 1023
            ss.run(stage, [[ss.pattern(pattern, n, chunk, rng)] for n in lengths], lambda s, u, n: x[s, :n], host=not device)
            if pattern == "one":
                break


def test_launch_counts(eng):
    x = rows([4000])
    with eng.open_watermark_stream(1, 500, KEY) as st:
        for i in range(8):
            c0 = eng.launch_count()
            st.push(x[:, 500 * i:500 * i + 500], [500], [i == 0], [i == 7])
            assert eng.launch_count() - c0 == 3
    for search, rate, n in ((True, 16000, 3), (False, 16000, 3), (True, 48000, 4)):
        c0 = eng.launch_count()
        eng.detect_watermark(np.zeros((2, 30000), np.float32), [1, 2, 3], rate=rate, search=search)
        assert eng.launch_count() - c0 == n
    c0 = eng.launch_count()
    eng.watermark(x, KEY)
    assert eng.launch_count() - c0 == 2


def test_argument_errors(eng):
    from viettts_b200 import _lib
    x = np.zeros((2, 100), np.float32)
    for spec in ("key=1,strength=0.31", "key=1,strength=nan", "key=-1", f"key={2**64}", "strength=0.1", "key=1.5", "key=1,depth=2"):
        with pytest.raises(ValueError):
            eng.watermark(x, spec)
    for keys in ([], [-1], [2 ** 64], list(range(4097))):
        with pytest.raises(ValueError):
            eng.detect_watermark(x, keys)
    with pytest.raises(ValueError):
        eng.detect_watermark(x, [1], rate=16001 * 7)
    lib = eng.lib
    y = np.zeros_like(x)
    c0 = eng.launch_count()
    for eps in (float("nan"), -0.1, 0.31):
        with pytest.raises(_lib.VttsError, match="strength"):
            eng._ck(lib.vtts_watermark_host(eng.h, x.ctypes.data, None, 2, 100, 1, eps, y.ctypes.data))
    n = np.array([5, 200], np.int32)
    with pytest.raises(_lib.VttsError, match="outside"):
        eng._ck(lib.vtts_watermark_host(eng.h, x.ctypes.data, n.ctypes.data, 2, 100, 1, 0.1, y.ctypes.data))
    keys = np.arange(5000, dtype=np.uint64)
    z, off = np.zeros(2 * 5000, np.float32), np.zeros(2 * 5000, np.int32)
    for rate, K in ((16000, 0), (16000, 4097), (7999, 1), (192001, 1), (16001, 1)):
        with pytest.raises(_lib.VttsError):
            eng._ck(lib.vtts_watermark_detect_host(eng.h, x.ctypes.data, None, 2, 100, rate, keys.ctypes.data, K, 1, z.ctypes.data,
                                                   off.ctypes.data))
    h, p = ctypes.c_void_p(), ctypes.c_int()
    with pytest.raises(_lib.VttsError, match="strength"):
        eng._ck(lib.vtts_watermark_stream_create(eng.h, 2, 64, 1, 0.5, ctypes.byref(h), ctypes.byref(p)))
    assert eng.launch_count() == c0


# ---- detection floors on real speech, through the library's own stages ----
def test_detection_floors_on_the_fixture(eng):
    x = speech(20.0).astype(np.float32)
    y = eng.watermark(x, KEY)
    pcm = lambda v: (np.clip(np.rint(v.astype(np.float64) * 32767), -32768, 32767) / 32767).astype(np.float32)
    chains = {
        "pcm16": (lambda: pcm(y), SR),
        "48 kHz": (lambda: eng.resample(y, 48000), 48000),
        "8 kHz": (lambda: eng.resample(y, 8000), 8000),
        "telephone": (lambda: eng.equalize(y, "telephone", SR), SR),
        "voice compressor": (lambda: eng.compress(y, "voice", SR)[0], SR),
        "de-esser": (lambda: eng.deess(y, "voice", SR)[0], SR),
        "limiter": (lambda: eng.limit(y * 4, -1.0, SR)[0], SR),
        "room": (lambda: eng.reverb(y, "room", SR), SR),
        "hall": (lambda: eng.reverb(y, "hall", SR), SR),
    }
    found = {}
    for name, (f, rate) in chains.items():
        r = eng.detect_watermark(f(), KEYS64, rate=rate, search=False)
        found[name] = float(r.z[0])
        assert np.all(r.z[1:] < wo.ALIGNED_THRESHOLD), (name, r.z[1:].max())
        if name == "room":
            assert r.z[0] >= 8, (name, r.z[0])
        elif name != "hall":
            assert r.z[0] >= 10, (name, r.z[0])
    print("aligned z on the fixture:", {k: round(v, 1) for k, v in found.items()})
    crop = 64 * 1357 + 17
    r = eng.detect_watermark(y[crop:crop + 5 * SR], KEYS64)
    d = (int(r.offset[0]) - crop) % 65536
    assert r.z[0] >= 6.5 and min(d, 65536 - d) <= 2 * 64, (r.z[0], r.offset[0], crop % 65536)   # the search grid is 64
    assert np.all(r.z[1:] < 6.5)
    r = eng.detect_watermark(x, KEYS64)
    assert np.all(r.z < 6.5) and not r.detected.any()
    print(f"5 s crop: z {r.z[0]:.1f}; unmarked search max {r.z.max():.2f}")


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


@pytest.mark.parametrize("rate,denoise", [(None, None), (48000, None), (48000, 0.1)])
def test_tts_stream_watermark(tts_eng, rate, denoise):
    from viettts_b200.engine import AudioChain
    eng = tts_eng
    eng.set_precision("bf16x3")
    eng.set_fused_pairs(False)
    try:
        toks = [tts_tokens(170 + b, n) for b, n in enumerate([25, 40])]
        audio = {0: [], 1: []}
        spec = f"key={KEY},strength=0.2"
        with eng.open_tts_stream(2, 16, 2000, 100, output_rate=rate, denoise=denoise, watermark=spec) as ts:
            assert ts.wm is not None and ts.wm.lookahead == 1023
            ts.begin(0, toks[0], silence_duration=0.1)
            ts.begin(1, toks[1], silence_duration=0.1)
            while ts.busy().any():
                for s, w in ts.step().items():
                    audio[s].append(w)
        chain = AudioChain(output_rate=rate, denoise=denoise, watermark=spec)
        assert [s[0] for s in chain._stages()] == ["dn"] * (denoise is not None) + ["wm"] + ["rs"] * (rate is not None)
        for s in (0, 1):
            w = chain.run(eng, eng.tts(toks[s][None], silence_duration=0.1)[0][0])
            assert np.array_equal(np.concatenate(audio[s]), w), s
        with pytest.raises(ValueError, match="watermark"):
            eng.open_tts_stream(1, 16, 2000, 100, watermark="key=1,strength=2")
    finally:
        eng.set_fused_pairs(True)


def test_cli_watermark_round_trip(tts_eng, acoustic_ckpt, hifigan_params, golden_dir, tmp_path, monkeypatch, capsys):
    from viettts_b200 import synthesizer
    from viettts_b200 import watermark as wm_cli
    from viettts_b200.engine import get_engine
    from viettts_b200.hifigan.mel2wave import mel2wave
    from viettts_b200.nat.text2mel import text2mel
    (tmp_path / "assets/hifigan").mkdir(parents=True)
    (tmp_path / "assets/infore/hifigan").mkdir(parents=True)
    (tmp_path / "assets/infore/nat").mkdir(parents=True)
    (tmp_path / "assets/hifigan/config.json").write_text(json.dumps(config.HIFIGAN))
    for path, obj in (("assets/infore/hifigan/hk_hifi.pickle", hifigan_params), ("assets/infore/nat/acoustic_latest_ckpt.pickle", acoustic_ckpt),
                      ("assets/infore/nat/duration_latest_ckpt.pickle", synthetic.duration_ckpt(1234))):
        with open(tmp_path / path, "wb") as f:
            pickle.dump(obj, f)
    monkeypatch.chdir(tmp_path)
    lex = str(golden_dir / "lexicon_small.txt")
    ge = get_engine(0)
    text = "Xin chào, tôi là trợ lý ảo."
    wave = np.ravel(mel2wave(text2mel(synthesizer.nat_normalize_text(text), lex, 0.1)))
    assert synthesizer.main(["--text", text, "--output", "one.wav", "--lexicon-file", lex, "--silence-duration", "0.1",
                             "--watermark", f"key={KEY},strength=0.3", "--output-rate", "48000"]) == 0
    expect = synthesizer.float_to_pcm16(ge.resample(ge.watermark(wave, f"key={KEY},strength=0.3"), 48000)).astype(np.int32)
    raw = np.frombuffer((tmp_path / "one.wav").read_bytes()[44:], "<i2").astype(np.int32)
    assert raw.shape == expect.shape and np.abs(raw - expect).max() <= 1
    w48, rate = synthesizer.read_wav(tmp_path / "one.wav")
    ref = ge.detect_watermark(w48, [KEY, 99], rate=rate, search=False)
    capsys.readouterr()
    rc = wm_cli.main(["detect", "--key", str(KEY), "--key", "99", "--aligned", str(tmp_path / "one.wav")])
    lines = capsys.readouterr().out.strip().splitlines()
    assert len(lines) == 2 and f"z={ref.z[0]:.2f}" in lines[0] and f"z={ref.z[1]:.2f}" in lines[1]
    assert rc == (0 if ref.detected.any() else 1)
    assert ("\tmarked" in lines[0]) == bool(ref.detected[0]) and "not marked" in lines[1]
    with pytest.raises(SystemExit):
        synthesizer.main(["--text", text, "--output", "bad.wav", "--lexicon-file", lex, "--watermark", "key=1,strength=0.9"])
