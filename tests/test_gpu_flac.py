"""GPU: FLAC on the device (Engine.encode_flac / encode_flac_forward, vtts_flac_encode*, AudioChain and the CLI's
--encoding flac).  Every stream is compared byte for byte against the definition (oracle/flac_oracle.py)."""
import numpy as np
import pytest
import torch

from oracle import flac_oracle as fo
from oracle import g711_oracle as g
from test_flac_cpu import BRANCH_RATES, TABLE_RATES, flac_signals, lengths_for, speech_pcm

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    from viettts_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


def oracle_rows(x, lengths, rate, block):
    return [fo.encode(g.to_int16(x[b, :n]).astype(np.int16), rate, block) for b, n in enumerate(lengths)]


def signal_rows(block):
    sig = flac_signals(block)
    S = max(lengths_for(block))
    rows, lens = [], []
    for v in sig.values():
        for n in lengths_for(block):
            rows.append(np.resize(v, S).astype(np.float32))
            lens.append(n)
    return np.stack(rows), lens


def test_speech_equals_the_oracle(eng):
    x = (speech_pcm().astype(np.float32) / np.float32(32767.0))
    for rate, block in ((16000, 4096), (16000, 256), (48000, 1024)):
        got = eng.encode_flac(x, rate, block=block)
        assert got == fo.encode(g.to_int16(x).astype(np.int16), rate, block)
    y, _, _ = fo.decode(eng.encode_flac(x))
    assert np.array_equal(y, eng.encode(x, "pcm16"))


@pytest.mark.parametrize("block", fo.BLOCKS)
def test_signal_set_equals_the_oracle(eng, block):
    x, lens = signal_rows(block)
    got = eng.encode_flac(x, 44100, lengths=lens, block=block)
    assert got == oracle_rows(x, lens, 44100, block)


@pytest.mark.parametrize("B", [1, 3, 32, 65])
def test_batches_and_batch_positions(eng, B):
    rng = np.random.default_rng(B)
    S = 9000
    sig = list(flac_signals(1024).values())
    x = np.stack([np.resize(sig[b % len(sig)] * rng.uniform(0.2, 1.0), S) for b in range(B)]).astype(np.float32)
    lens = rng.integers(0, S + 1, B)
    lens[0] = S
    got = eng.encode_flac(x, 16000, lengths=lens, block=1024)
    ref = oracle_rows(x, lens, 16000, 1024)
    assert got == ref
    for b in (0, B // 2, B - 1):       # a row alone gives the bytes it gives in the batch
        assert eng.encode_flac(x[b, : lens[b]], 16000, block=1024) == ref[b]


def test_every_rate_branch(eng):
    x = flac_signals(256)["tone"][:3000]
    for rate in TABLE_RATES + [r for _, r in BRANCH_RATES]:
        assert eng.encode_flac(x, rate, block=256) == fo.encode(g.to_int16(x).astype(np.int16), rate, 256), rate


@pytest.mark.parametrize("mode", ["fp32", "bf16x3", "fp16"])
def test_precision_modes(eng, mode):
    x, lens = signal_rows(512)
    old = eng.get_precision()
    eng.set_precision(mode)
    try:
        assert eng.encode_flac(x, 16000, lengths=lens, block=512) == oracle_rows(x, lens, 16000, 512)
    finally:
        eng.set_precision(old)


def test_forward_agrees_and_writes_nothing_past_nbytes(eng):
    from viettts_b200.engine import flac_bound
    x, lens = signal_rows(2048)
    B, S = x.shape
    ref = oracle_rows(x, lens, 24000, 2048)
    bound = flac_bound(S, 2048)
    n_t = torch.tensor(lens, dtype=torch.int32, device="cuda")
    xbuf = torch.zeros(B * S + 8, dtype=torch.float32, device="cuda")
    for ox in (0, 1, 3):               # offset, unaligned views of the input
        xv = xbuf[ox:ox + B * S].view(B, S)
        xv.copy_(torch.from_numpy(x))
        out = torch.full((B, bound + 37), 0xA5, dtype=torch.uint8, device="cuda")
        y, nb = eng.encode_flac_forward(xv, 24000, lengths_t=n_t, block=2048, out=out)
        assert y is out
        yh, nbh = y.cpu().numpy(), nb.cpu().numpy()
        for b in range(B):
            assert nbh[b] == len(ref[b]) and yh[b, : nbh[b]].tobytes() == ref[b]
            assert np.all(yh[b, nbh[b]:] == 0xA5)
    assert eng.encode_flac(x, 24000, lengths=lens, block=2048) == ref


def test_empty_rows_and_lists(eng):
    assert eng.encode_flac(np.zeros(0, np.float32)) == fo.encode(np.zeros(0, np.int16), 16000, 4096)
    x = np.zeros((2, 5), np.float32)
    assert eng.encode_flac(x, lengths=[0, 5]) == [fo.encode(np.zeros(0, np.int16), 16000, 4096),
                                                  fo.encode(np.zeros(5, np.int16), 16000, 4096)]


def test_argument_rejections(eng):
    from viettts_b200 import _lib
    from viettts_b200.engine import flac_bound
    x = torch.zeros((2, 1000), dtype=torch.float32, device="cuda")
    with pytest.raises(ValueError):
        eng.encode_flac_forward(x, block=1000)
    with pytest.raises(ValueError):
        eng.encode_flac_forward(x, rate=65537)
    bound = flac_bound(1000, 4096)
    out = torch.zeros((2, bound), dtype=torch.uint8, device="cuda")
    nb = torch.zeros(2, dtype=torch.int32, device="cuda")
    lib, st = eng.lib, torch.cuda.current_stream().cuda_stream
    p = lambda t: t.data_ptr()
    for args in ((2, 1000, 16000, 1000, p(out), bound, p(nb)),          # block
                 (2, 1000, 65537, 4096, p(out), bound, p(nb)),         # rate
                 (2, 1000, 16000, 4096, p(out), bound - 1, p(nb)),     # pitch below the bound
                 (2, 1000, 16000, 4096, p(x) + 16, bound, p(nb)),      # output over the input
                 (2, 1000, 16000, 4096, p(out), bound, p(out) + 8)):   # nbytes inside the output
        assert lib.vtts_flac_encode(eng.h, p(x), None, *args, st) != 0
    with pytest.raises(_lib.VttsError):
        eng.encode_flac(np.zeros((2, 10), np.float32), lengths=[3, 11])
    assert lib.vtts_flac_bound(1000, 1000) == -1 and lib.vtts_flac_bound(1000, 4096) == bound


def test_audio_chain(eng):
    from viettts_b200.engine import AudioChain
    x = (speech_pcm()[:40000].astype(np.float32) / np.float32(32767.0))
    ch = AudioChain(output_rate=48000, encoding="flac,block=1024")
    got = ch.run(eng, x)
    wav = eng.resample(x, 48000)
    assert got == fo.encode(g.to_int16(wav).astype(np.int16), 48000, 1024)
    y, rate, _ = fo.decode(got)
    assert rate == 48000 and np.array_equal(y, eng.encode(wav, "pcm16"))


# ---- the per-slot stream ---------------------------------------------------------------------------------------------
def _slot_pushes(plans):
    from helpers.slot_streams import _pushes
    return [_pushes(p) for p in plans]


def drive_stream(eng, fs, plans, signal, host):
    """Pushes `plans` (one per slot, push sizes as tests/helpers/slot_streams.py plans them) through FlacStream fs;
    every push is held to the definition: a slot's bytes are the stream header with BEGIN and exactly the frames its
    samples complete (flac_stream_frames), each equal to the oracle's frame of that number; an idle slot gets nothing.
    Returns {(slot, utterance): bytes}."""
    from viettts_b200.engine import STREAM_BEGIN, STREAM_END, flac_stream_frames
    S, F, blk = fs.max_streams, fs.max_chunk_samples, fs.block
    pushes = _slot_pushes(plans)
    utt = {}
    for s, plan in enumerate(plans):
        for u, sizes in enumerate(plan):
            if all(q is None for q in sizes):              # pushes the slot sits out: no utterance
                continue
            n = sum(q for q in sizes if q is not None)
            x = signal(s, u, n)
            data = fo.encode(g.to_int16(x).astype(np.int16), fs.rate, blk)
            utt[s, u] = (x, fo.unknown_totals(data[:42]), fo.frames_of(data))
    got = {k: b"" for k in utt}
    pos = {k: 0 for k in utt}
    steps = max(len(p) for p in pushes)
    x_t = torch.zeros((S, F), dtype=torch.float32, device="cuda")
    out_t = torch.zeros(fs.out_bytes, dtype=torch.uint8, device="cuda")
    tbl_t = torch.zeros((S, 2), dtype=torch.int32, device="cuda")
    for i in range(steps):
        xh = np.zeros((S, F), np.float32)
        n_new, flags, cur = np.zeros(S, np.int32), np.zeros(S, np.uint8), {}
        for s in range(S):
            e = pushes[s][i] if i < len(pushes[s]) else None
            if e is None:
                continue
            n, fl, u = e
            p0 = pos[s, u]
            xh[s, :n] = utt[s, u][0][p0:p0 + n]
            n_new[s], flags[s], cur[s] = n, fl, (u, p0, p0 + n, fl)
            pos[s, u] = p0 + n
        if host:
            out = fs.push(xh, n_new, begin=flags & STREAM_BEGIN, end=flags & STREAM_END)
        else:
            x_t.copy_(torch.from_numpy(xh))
            fs.push_device(x_t, n_new, flags, out_t, tbl_t)
            tbl = tbl_t.cpu().numpy()
            buf = out_t.cpu().numpy().tobytes()
            out = [buf[o:o + c] for o, c in tbl]
        for s in range(S):
            if s not in cur:
                assert out[s] == b"", (i, s)                       # an idle slot's output stays empty
                continue
            u, p0, p1, fl = cur[s]
            _, head, frames = utt[s, u]
            end = bool(fl & STREAM_END)
            e0, e1 = flac_stream_frames(p0, blk), flac_stream_frames(p1, blk, end)
            want = (head if fl & STREAM_BEGIN else b"") + b"".join(frames[e0:e1])
            assert out[s] == want, (i, s, u, p0, p1, e0, e1)
            got[s, u] += out[s]
    return got, utt


@pytest.mark.parametrize("host", [False, True])
@pytest.mark.parametrize("block", [256, 4096])
def test_stream_push_plans(eng, host, block):
    from helpers.slot_streams import KINDS, push_plan
    F = 1024
    rng = np.random.default_rng(block + host)
    kinds = KINDS * 2
    plans = [push_plan(k, F, rng) for k in kinds]
    pcm = speech_pcm().astype(np.float32) / np.float32(32767.0)
    sil = flac_signals(256)

    def signal(s, u, n):
        if s % 5 == 4:                                     # silence and edge classes in some slots
            return np.resize(list(sil.values())[(s + u) % len(sil)], n).astype(np.float32)
        o = (7919 * (s + 3 * u)) % (pcm.size - n) if n < pcm.size else 0
        return np.resize(pcm[o:], n)

    with eng.open_flac_stream(len(plans), F, 16000, block) as fs:
        got, utt = drive_stream(eng, fs, plans, signal, host)
    for k, (x, head, frames) in utt.items():
        assert got[k] == head + b"".join(frames), k
        y, rate, si = fo.decode(got[k])
        assert np.array_equal(y, g.to_int16(x).astype(np.int16)) and si["total"] == 0 and si["max_frame"] == 0


def test_stream_rejections(eng):
    from viettts_b200 import _lib
    from viettts_b200.engine import Engine, FlacStream
    with pytest.raises(ValueError):
        eng.open_flac_stream(2, 100, 16000, 1000)
    with pytest.raises(ValueError):
        eng.open_flac_stream(2, 100, 65537, 4096)
    other = Engine(0)
    try:
        fs = FlacStream(other, 2, 100)
        x = np.zeros((2, 100), np.float32)
        y = np.zeros(fs.out_bytes, np.uint8)
        tbl = np.zeros((2, 2), np.int32)
        import ctypes as C
        p = lambda a: a.ctypes.data_as(C.c_void_p)
        rc = eng.lib.vtts_flac_stream_push_host(eng.h, fs.h, p(x), p(np.ones(2, np.int32)), p(np.ones(2, np.uint8)), p(y), p(tbl))
        assert rc != 0 and b"another context" in eng.lib.vtts_last_error(eng.h)
        with pytest.raises(_lib.VttsError, match="not open"):
            fs.push(x, [1, 0])                               # no BEGIN
        fs.close()
    finally:
        other.close()


def test_long_slot_past_2_31_samples(eng):
    """digital silence past 2^31 samples at block 256 (pushed from one device buffer in large pushes), then speech:
    the last frames carry 5-byte frame numbers and equal the oracle's frames of those numbers"""
    from viettts_b200.engine import STREAM_BEGIN, STREAM_END
    F, blk = 1 << 22, 256
    pcm = speech_pcm()[:5000]
    with eng.open_flac_stream(1, F, 16000, blk) as fs:
        x_t = torch.zeros((1, F), dtype=torch.float32, device="cuda")
        out_t = torch.empty(fs.out_bytes, dtype=torch.uint8, device="cuda")
        tbl_t = torch.zeros((1, 2), dtype=torch.int32, device="cuda")
        pushes = (1 << 31) // F + 3
        for i in range(pushes):
            fs.push_device(x_t, [F], [STREAM_BEGIN if i == 0 else 0], out_t, tbl_t)
        o, c = tbl_t.cpu().numpy()[0]                      # the last silence push: F / 256 CONSTANT frames
        f1 = (pushes - 1) * F // blk
        want = b"".join(fo.encode_frame(np.zeros(blk, np.int64), f1 + j, 16000, blk) for j in (0, F // blk - 1))
        last = out_t[o:o + c].cpu().numpy().tobytes()
        assert last.startswith(want[: len(want) // 2]) and last.endswith(want[len(want) // 2:])
        P = pushes * F
        assert P > 2**31
        x = np.zeros((1, F), np.float32)
        x[0, :pcm.size] = pcm / np.float32(32767.0)
        x_t.copy_(torch.from_numpy(x))
        fs.push_device(x_t, [pcm.size], [STREAM_END], out_t, tbl_t)
        o, c = tbl_t.cpu().numpy()[0]
        got = out_t[o:o + c].cpu().numpy().tobytes()
    f0 = P // blk
    assert len(fo.utf8_number(f0)) == 5
    want = b"".join(fo.encode_frame(pcm[i:i + blk].astype(np.int64), f0 + i // blk, 16000, blk) for i in range(0, pcm.size, blk))
    assert got == want


# ---- the TTS stream and the CLI ----------------------------------------------------------------------------------------
from test_gpu_encode import tts_eng, tts_tokens  # noqa: E402,F401


def run_flac_tts(eng, toks, **opts):
    audio = {s: b"" for s in range(len(toks))}
    with eng.open_tts_stream(len(toks), 16, 2000, 100, **opts) as ts:
        for s, t in enumerate(toks):
            ts.begin(s, t, silence_duration=0.1)
        while ts.busy().any():
            for s, w in ts.step().items():
                assert isinstance(w, bytes)
                audio[s] += w
    return audio


@pytest.mark.parametrize("opts", [dict(), dict(output_rate=48000, denoise=0.5, semitones=3.0, tempo=0.8, watermark="key=1",
                                             eq="hs:6000:3", compress="voice", deess="voice", reverb="room", limit=-1.0,
                                             meter=True)], ids=["alone", "all_stages"])
def test_tts_stream_flac(tts_eng, opts):
    from viettts_b200.engine import AudioChain
    eng = tts_eng
    eng.set_precision("bf16x3")
    eng.set_fused_pairs(False)
    try:
        toks = [tts_tokens(290 + b, n) for b, n in enumerate([25, 40, 12])]
        got = run_flac_tts(eng, toks, encoding="flac,block=1024", **opts)
        floats = run_flac_tts_floats(eng, toks, opts)
        rate = opts.get("output_rate") or 16000
        for s in range(3):
            y, r, si = fo.decode(got[s])
            codes = eng.encode(floats[s], "pcm16")
            assert r == rate and si["total"] == 0 and np.array_equal(y, codes), s
            assert got[s] == fo.unknown_totals(fo.encode(codes, rate, 1024)), s
            if "watermark" in opts:                       # the mark reads the same from the FLAC as from PCM-16
                z_flac = eng.detect_watermark(y.astype(np.float32) / np.float32(32767.0), 1, rate).z
                z_pcm = eng.detect_watermark(eng.decode(codes, "pcm16"), 1, rate).z
                assert np.array_equal(z_flac, z_pcm), (s, z_flac, z_pcm)
        chain = AudioChain(encoding="flac")
        assert chain.flac == {"block": 4096}
    finally:
        eng.set_fused_pairs(True)


def run_flac_tts_floats(eng, toks, opts):
    out = {s: [] for s in range(len(toks))}
    with eng.open_tts_stream(len(toks), 16, 2000, 100, **opts) as ts:
        for s, t in enumerate(toks):
            ts.begin(s, t, silence_duration=0.1)
        while ts.busy().any():
            for s, w in ts.step().items():
                out[s].append(w)
    return {s: np.concatenate(v) for s, v in out.items()}


def test_cli_writes_flac(tmp_path, monkeypatch, acoustic_ckpt, hifigan_params, golden_dir):
    """--encoding flac through main(): the file starts with fLaC, the oracle decodes it to the pcm16 codes of the
    audio, and --text-file outputs without a suffix get .flac"""
    import json
    import pickle
    from viettts_b200 import config, synthesizer, synthetic
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
    lex = str(golden_dir / "lexicon_small.txt")
    ge = get_engine(0)
    lines = ["Xin chào, tôi là trợ lý ảo.", "hôm nay trời đẹp quá!"]
    (tmp_path / "lines.txt").write_text("\n".join(lines) + "\n")
    assert synthesizer.main(["--text-file", "lines.txt", "--output", "out", "--lexicon-file", lex, "--silence-duration", "0.1",
                             "--seed", "5", "--encoding", "flac,block=1024"]) == 0
    waves = synthesizer.synthesize_lines(lines, lex, 0.1, seed=5)
    for i, w in enumerate(waves):
        data = (tmp_path / f"out_{i:04d}.flac").read_bytes()
        assert data[:4] == b"fLaC"
        y, rate, si = fo.decode(data)
        assert rate == 16000 and si["min_block"] == 1024 and np.array_equal(y, ge.encode(w, "pcm16")), i
