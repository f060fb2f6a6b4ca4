"""GPU: the background bed (Engine.mix_bed / mix_bed_forward / open_bed_stream) against float64 (oracle/bed_oracle.py)
within TOL (tests/test_bed_cpu.py), its bit identities across modes, batch positions, entry points and the stream, the
TTS stream's `bed=` stage against AudioChain.run, the CLI's --bed, and the watermark under the default bed."""
import ctypes
import json
import pickle

import numpy as np
import pytest
import torch

from helpers import slot_streams as ss
from oracle import bed_oracle as bo
from oracle import watermark_oracle as wo
from test_bed_cpu import TOL, cases, error_units
from test_watermark_cpu import KEY, SR, speech
from viettts_b200 import config, synthetic

pytestmark = pytest.mark.gpu

KEYS64 = [KEY] + list(range(2000, 2063))
# two short beds (they wrap several times in a 1 s row) under the GPU tests' fade, tail, crossfade and offset
BANK = ["pink,seed=1,length=0.6,fade_in=250,tail=300,xfade=50,offset=0.1",
        "pink,seed=2,length=0.55,level=-24,fade_in=250,tail=300,xfade=50,offset=0.1"]


@pytest.fixture(scope="module")
def eng():
    from viettts_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


def rows(rate, lengths, seed=0):
    S = max(max(lengths), 1)
    x = np.zeros((len(lengths), S), np.float32)
    for b, n in enumerate(lengths):
        if n:
            x[b, :n] = cases(rate, n)[(b + seed) % 3]
    return x


def beds(bank):
    """the prepared beds of a bank as host arrays"""
    a = bank.audio.cpu().numpy()
    return [a[o:o + n] for o, n in zip(bank.offsets, bank.lengths)]


def oracle(x, n, bed, bank, rate):
    p = bank.params[0]
    b = None if bed < 0 else beds(bank)[bed]
    return bo.mix(x[:n], b, rate, p["Fi"], p["Tt"], p["C"], p["o"], parts=True,
                  **{k: p[k] for k in ("duck", "threshold", "attack", "release")})


def check_rows(y, red, x, lengths, idx, bank, rate, what):
    Tt = bank.params[0]["Tt"]
    assert y.shape == (x.shape[0], x.shape[1] + Tt)
    for b, n in enumerate(lengths):
        ref, rr, P = oracle(x[b], n, idx[b], bank, rate)
        m = ref.size
        assert m == n + (Tt if idx[b] >= 0 else 0)
        if idx[b] < 0:
            assert np.array_equal(y[b, :n], x[b, :n]) and red[b] == 0.0, (what, b)
        else:
            assert error_units(y[b, :m], ref, P) <= TOL, (what, b, n, error_units(y[b, :m], ref, P))
            assert abs(red[b] - rr) <= 1e-3 * max(1.0, abs(rr)), (what, b, red[b], rr)
        assert not y[b, m:].any(), (what, b)


LENGTHS = [0, 1, 255, 256, 257, 1023, 1024, 1025]


@pytest.mark.parametrize("rate", [16000, 44100, 48000])
def test_ragged_rows_against_float64(eng, rate):
    lengths = LENGTHS + [rate // 2, rate]
    x = rows(rate, lengths, rate)
    idx = np.array([(b % 3) - 1 for b in range(len(lengths))], np.int32)     # -1, 0, 1 in turn
    bank = eng.prepare_beds(BANK, rate)
    assert max(bank.lengths) < rate
    y, red = eng.mix_bed(x, bank, rate, lengths=lengths, index=idx)
    check_rows(y, red, x, lengths, idx, bank, rate, rate)


def test_three_minute_row(eng):
    rate = 48000
    n = 180 * rate
    x = rows(rate, [n], 1)
    bank = eng.prepare_beds("pink,length=7", rate)
    y, red = eng.mix_bed(x, bank, rate)
    check_rows(y, red, x, [n], [0], bank, rate, "3 min")


def test_same_bits_in_every_mode_batch_position_and_entry_point(eng):
    rate = 16000
    lengths = [3000, 17, 12000, 0, 8000]
    x = rows(rate, lengths, 5)
    idx = np.array([0, 1, -1, 0, 1], np.int32)
    bank = eng.prepare_beds(BANK, rate)
    ref, rr = eng.mix_bed(x, bank, rate, lengths=lengths, index=idx)
    try:
        for mode in ("fp32", "bf16x3", "fp16"):
            eng.set_precision(mode)
            y, red = eng.mix_bed(x, bank, rate, lengths=lengths, index=idx)
            assert np.array_equal(y, ref) and np.array_equal(red, rr), mode
    finally:
        eng.set_precision("bf16x3")
    for b in range(len(lengths)):
        y, red = eng.mix_bed(x[b, :lengths[b]], bank, rate, index=idx[b])
        m = lengths[b] + (bank.params[0]["Tt"] if idx[b] >= 0 else 0)
        assert y.shape == (m,) and np.array_equal(y, ref[b, :m]) and red == rr[b], b
    perm = [3, 0, 4, 2, 1]
    y, red = eng.mix_bed(x[perm], bank, rate, lengths=[lengths[p] for p in perm], index=idx[perm])
    assert np.array_equal(y, ref[perm]) and np.array_equal(red, rr[perm])
    n_t = torch.tensor(lengths, dtype=torch.int32, device="cuda")
    y_t, red_t = eng.mix_bed_forward(torch.from_numpy(x).cuda(), bank, rate, lengths_t=n_t, index=idx)
    assert np.array_equal(y_t.cpu().numpy(), ref) and np.array_equal(red_t.cpu().numpy(), rr)
    y_t, _ = eng.mix_bed_forward(torch.from_numpy(x).cuda(), BANK, rate, lengths_t=n_t, index=idx)    # a cached string bank
    assert np.array_equal(y_t.cpu().numpy(), ref)
    assert np.array_equal(eng.mix_bed(x, BANK[0], rate, lengths=lengths)[0][0], ref[0])             # bank entry 0 alone


@pytest.mark.parametrize("S", [1, 3, 32])
@pytest.mark.parametrize("pattern,device", [("full", False), ("random", False), ("random", True)])
def test_stream_equals_one_shot(eng, S, pattern, device):
    """rows go to the slots in turn (a slot takes its next row with BEGIN in the push after its last row's END), each
    with its own bank entry, pushed in `pattern` chunks and held to the stream's contract on every push
    (tests/helpers/slot_streams.py)"""
    rate = 48000
    bank = eng.prepare_beds(BANK, rate)
    Tt = bank.params[0]["Tt"]
    R = 2 * S
    rng = np.random.default_rng(S)
    lengths = [int(v) for v in rng.integers(0, 30000, size=R)]
    lengths[0] = 0                                       # BEGIN and END in one push, with nothing in it
    if R > 2:
        lengths[1] = 300                                 # BEGIN and END in one push
    idx = [(r % 3) - 1 for r in range(R)]
    x = rows(rate, lengths, S)
    rng = np.random.default_rng(11)
    for chunk in (700, 4096):
        stage = ss.stage(eng, "bed", S, chunk, rate, bed=bank)
        with stage.open() as st:
            assert st.lookahead == 0 and st.out_pitch == chunk + Tt and st.tail == Tt
        plans = [[ss.pattern(pattern, lengths[r], chunk, rng) for r in range(s, R, S)] for s in range(S)]
        ss.run(stage, plans, lambda s, u, n: x[s + u * S, :n], [idx[s::S] for s in range(S)], host=not device)


def test_launch_counts(eng):
    rate = 16000
    x = rows(rate, [4000], 0)
    eng.mix_bed(x, BANK, rate)                           # the bank is prepared once, before the counted calls
    with eng.open_bed_stream(1, 500, BANK, rate) as st:
        for i in range(8):
            c0 = eng.launch_count()
            st.push(x[:, 500 * i:500 * i + 500], [500], [i == 0], [i == 7], bed=1)
            assert eng.launch_count() - c0 == 7
    for shape in ((3, 50000), (1, 10)):
        c0 = eng.launch_count()
        eng.mix_bed(np.zeros(shape, np.float32), BANK, rate)
        assert eng.launch_count() - c0 == 7


def test_argument_errors(eng):
    from viettts_b200 import _lib
    rate = 16000
    bank = eng.prepare_beds(BANK, rate)
    x = np.zeros((2, 100), np.float32)
    with pytest.raises(ValueError, match="bed index"):
        eng.mix_bed(x, bank, rate, index=2)
    with pytest.raises(ValueError, match="prepared at"):
        eng.mix_bed(x, bank, 48000)
    lib = eng.lib
    y = np.zeros((2, 100 + 4800), np.float32)
    red = np.zeros(2, np.float32)
    A, off, ln = bank.audio.data_ptr(), bank.offsets, bank.lengths
    good = dict(K=2, duck=12.0, thr=-40.0, att=10.0, rel=500.0, Fi=4000, Tt=4800, C=800, o=0)
    bed = np.array([0, 1], np.int32)

    def call(B=2, S=100, rate=rate, idx=bed, lengths=ln, **kw):
        p = dict(good, **kw)
        return lib.vtts_bed_mix_host(eng.h, x.ctypes.data, None, B, S, rate, A, off.ctypes.data, lengths.ctypes.data, p["K"],
                                     idx.ctypes.data, p["duck"], p["thr"], p["att"], p["rel"], p["Fi"], p["Tt"], p["C"], p["o"],
                                     y.ctypes.data, red.ctypes.data)
    eng._ck(call())
    c0 = eng.launch_count()
    for kw in (dict(duck=41.0), dict(duck=float("nan")), dict(thr=1.0), dict(att=0.1), dict(rel=6000.0), dict(Fi=-1),
               dict(Fi=5 * rate + 1), dict(Tt=10 * rate + 1), dict(C=rate + 1), dict(C=5000), dict(o=int(ln.min())), dict(o=-1),
               dict(K=0), dict(K=9), dict(rate=7999), dict(B=0), dict(S=0), dict(idx=np.array([0, 2], np.int32)),
               dict(idx=np.array([-2, 0], np.int32)), dict(lengths=np.array([100, 8000], np.int32))):
        with pytest.raises(_lib.VttsError):
            eng._ck(call(**kw))
    h, p = ctypes.c_void_p(), ctypes.c_int()
    with pytest.raises(_lib.VttsError, match="max_streams"):
        eng._ck(lib.vtts_bed_stream_create(eng.h, 0, 64, rate, A, off.ctypes.data, ln.ctypes.data, 2, 12.0, -40.0, 10.0, 500.0, 0, 0, 0, 0,
                                           ctypes.byref(h), ctypes.byref(p)))
    assert eng.launch_count() == c0
    with eng.open_bed_stream(2, 64, bank, rate) as st:
        c0 = eng.launch_count()
        with pytest.raises(_lib.VttsError, match="not open"):
            st.push(np.zeros((2, 64), np.float32), [64, 0], None, None)
        st.push(np.zeros((2, 64), np.float32), [64, 0], [True, False], None, bed=1)
        c0 = eng.launch_count()
        with pytest.raises(ValueError, match="bed index"):
            st.push(np.zeros((2, 64), np.float32), [64, 0], [False, True], None, bed=5)
        xs, n_new, flags, bed = np.zeros((2, 64), np.float32), np.array([1, 0], np.int32), np.zeros(2, np.uint8), np.array([0, -1], np.int32)
        ys, n_out, red = np.zeros((2, st.out_pitch), np.float32), np.zeros(2, np.int32), np.zeros(2, np.float32)
        with pytest.raises(_lib.VttsError, match="changes"):
            eng._ck(lib.vtts_bed_stream_push_host(eng.h, st.h, xs.ctypes.data, n_new.ctypes.data, flags.ctypes.data, bed.ctypes.data,
                                                  ys.ctypes.data, n_out.ctypes.data, red.ctypes.data))
        assert eng.launch_count() == c0


# ---- the TTS stream and the CLI ----

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


@pytest.mark.parametrize("rate,reverb,limit", [(None, None, None), (48000, "room", -1.0)])
def test_tts_stream_bed(tts_eng, rate, reverb, limit):
    from viettts_b200.engine import AudioChain
    eng = tts_eng
    eng.set_precision("bf16x3")
    eng.set_fused_pairs(False)
    specs = ["pink,seed=5,tail=400", "pink,seed=6,level=-22,tail=400"]
    try:
        toks = [tts_tokens(190 + b, n) for b, n in enumerate([25, 40, 30])]
        choice = [1, -1, None]                 # entry 1, no bed, the default entry 0
        audio = {0: [], 1: [], 2: []}
        with eng.open_tts_stream(3, 16, 2000, 100, output_rate=rate, reverb=reverb, bed=specs, limit=limit, meter=True) as ts:
            assert ts.bd is not None and ts.bd.tail == (int(0.4 * (rate or 16000)))
            for s in range(3):
                ts.begin(s, toks[s], silence_duration=0.1, bed=choice[s])
            while ts.busy().any():
                for s, w in ts.step().items():
                    audio[s].append(w)
        for s in range(3):
            spec = None if choice[s] == -1 else specs[choice[s] or 0]
            chain = AudioChain(output_rate=rate, reverb=reverb, bed=spec, limit=limit)
            w = chain.run(eng, eng.tts(toks[s][None], silence_duration=0.1)[0][0])
            assert np.array_equal(np.concatenate(audio[s]), w), s
        with pytest.raises(ValueError, match="bed"):
            eng.open_tts_stream(1, 16, 2000, 100, bed="pink,duck=99")
        with eng.open_tts_stream(1, 16, 2000, 100) as ts:
            with pytest.raises(ValueError, match="bed="):
                ts.begin(0, toks[0], bed=0)
    finally:
        eng.set_fused_pairs(True)


def test_cli_bed(tts_eng, acoustic_ckpt, hifigan_params, golden_dir, tmp_path, monkeypatch):
    from viettts_b200 import synthesizer
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
                             "--bed", "pink,seed=4,duck=18"]) == 0
    expect = synthesizer.float_to_pcm16(ge.mix_bed(wave, "pink,seed=4,duck=18", 16000)[0]).astype(np.int32)
    raw = np.frombuffer((tmp_path / "one.wav").read_bytes()[44:], "<i2").astype(np.int32)
    assert raw.shape == expect.shape and np.abs(raw - expect).max() <= 1
    # a stereo 22.05 kHz file, resampled to the 48 kHz output and downmixed
    rng = np.random.default_rng(3)
    lr = (rng.standard_normal((30000, 2)) * 3000).clip(-32768, 32767).astype("<i2")
    synthesizer.write_wav(tmp_path / "stereo_src.wav", np.zeros(1, np.float32), 22050)
    raw_hdr = bytearray((tmp_path / "stereo_src.wav").read_bytes()[:44])
    raw_hdr[22:24] = (2).to_bytes(2, "little")
    raw_hdr[28:32] = (22050 * 4).to_bytes(4, "little")
    raw_hdr[32:34] = (4).to_bytes(2, "little")
    data = lr.tobytes()
    raw_hdr[40:44] = len(data).to_bytes(4, "little")
    raw_hdr[4:8] = (36 + len(data)).to_bytes(4, "little")
    (tmp_path / "bed.wav").write_bytes(bytes(raw_hdr) + data)
    assert synthesizer.main(["--text", text, "--output", "two.wav", "--lexicon-file", lex, "--silence-duration", "0.1",
                             "--output-rate", "48000", "--bed", "bed.wav,level=-26", "--limiter"]) == 0
    audio, r = synthesizer.read_bed_wav(tmp_path / "bed.wav")
    assert r == 22050
    spec = {"audio": audio, "audio_rate": 22050, "level": -26}
    expect = synthesizer.float_to_pcm16(ge.limit(ge.mix_bed(ge.resample(wave, 48000), spec, 48000)[0], -1.0, 48000)[0]).astype(np.int32)
    raw = np.frombuffer((tmp_path / "two.wav").read_bytes()[44:], "<i2").astype(np.int32)
    assert raw.shape == expect.shape and np.abs(raw - expect).max() <= 1


# ---- the watermark under a bed ----

def test_watermark_under_the_bed(eng):
    """The default pink bed (-30 LUFS, 12 dB duck) brings the aligned score on the fixture to about the threshold (4.8
    measured on an H100, below 5: it defeats aligned detection there); 10 dB lower the mark is found.  Wrong keys never
    reach the threshold under either."""
    x = speech(20.0).astype(np.float32)
    y = eng.watermark(x, KEY)
    found = {}
    for spec, rate in (("pink", SR), ("pink,level=-40", SR), ("pink,level=-40", 48000)):
        w = eng.mix_bed(y if rate == SR else eng.resample(y, rate), spec, rate)[0]
        r = eng.detect_watermark(w, KEYS64, rate=rate, search=False)
        found[f"{spec} at {rate}"] = (round(float(r.z[0]), 1), round(float(r.z[1:].max()), 1))
        assert np.all(r.z[1:] < wo.ALIGNED_THRESHOLD), (spec, rate, r.z[1:].max())
        if "level=-40" in spec:
            assert r.z[0] >= wo.ALIGNED_THRESHOLD, (spec, rate, r.z[0])
    print("aligned z (right key, largest wrong key):", found)
