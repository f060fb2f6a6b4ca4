"""GPU: joined utterances.

A. `Engine.tts_joined` equals `mel2wave` of the host-joined `predict_mel` rows of the same sentences bit for bit: the
   rows padded as the call pads them, each cut to its `tts_plan` n_emit, concatenated per text and vocoded as one
   [G, n_max] batch with the joined counts.  Groups of 1, 3 and 7 sentences, a zero-frame sentence mid-group and a text
   of zero-frame sentences only; dropout OFF, SEED and REFERENCE; bf16x3, fp16 and fp32; more than 128 sentences in one
   call.  Sentence starts, a one-sentence text against `tts`, the retry protocol and every bad argument.
B. A TTS stream slot continued by `append` / `finish`, every stage on with the meter and pcm16: each joined utterance's
   codes, float audio and meter reading equal `AudioChain.run` of `tts_joined` of its sentences bit for bit.
C. The CLI's --split-sentences for --text and --text-file."""
import ctypes as C
import json
import pickle

import numpy as np
import pytest

from test_gpu_audio_chain import BANK, EMPTY, KEY, OPENED_WITH, SD, STREAM_OPTS, tts_eng, tts_tokens  # noqa: F401
from viettts_b200 import config

pytestmark = pytest.mark.gpu
HOP = config.HOP


def sentence(seed):
    return tts_tokens(seed, 6 + seed % 23)


GROUPS = [[sentence(1)], [sentence(2), EMPTY, sentence(3)], [sentence(10 + i) for i in range(7)], [EMPTY, EMPTY]]


def padded(texts):
    rows = [np.asarray(r, np.int32) for t in texts for r in t]
    tok = np.zeros((len(rows), max(r.size for r in rows)), np.int32)
    for b, r in enumerate(rows):
        tok[b, : r.size] = r
    return tok, np.array([r.size for r in rows], np.int32)


def host_joined(eng, texts, kw):
    """mel2wave of the concatenated predict_mel rows, and each text's sentence starts in samples"""
    tok, lens = padded(texts)
    _, frames, nf, ne = eng.tts_plan(tok, lens, silence_duration=SD)
    mel = eng.predict_mel(tok, frames, lengths=lens, n_frames=nf, **kw)
    bounds = np.cumsum([0] + [len(t) for t in texts])
    counts = [int(ne[a:b].sum()) for a, b in zip(bounds, bounds[1:])]
    joined = np.zeros((len(texts), max(counts), config.MEL_DIM), np.float32)
    for g, (a, b) in enumerate(zip(bounds, bounds[1:])):
        joined[g, : counts[g]] = np.concatenate([mel[r, : ne[r]] for r in range(a, b)])
    wav = eng.mel2wave(joined, n_frames=np.array(counts, np.int32))
    starts = [HOP * np.concatenate([[0], np.cumsum(ne[a:b])[:-1]]) for a, b in zip(bounds, bounds[1:])]
    return [wav[g, : counts[g] * HOP] for g in range(len(texts))], starts


DROPOUT = {"off": {}, "seed": {"seed": 77}, "reference": {"rng": KEY}}


@pytest.mark.parametrize("kind", list(DROPOUT))
@pytest.mark.parametrize("mode", ["bf16x3", "fp16", "fp32"])
def test_one_shot_equals_host_joined_mel(tts_eng, mode, kind):
    eng = tts_eng
    eng.set_precision(mode)
    try:
        assert eng.tts_plan(EMPTY[None], silence_duration=SD)[3][0] == 0
        waves, starts = eng.tts_joined(GROUPS, silence_duration=SD, **DROPOUT[kind])
        want, want_starts = host_joined(eng, GROUPS, DROPOUT[kind])
        assert waves[3].size == 0 and waves[0].size > 0
        for g in range(len(GROUPS)):
            assert waves[g].dtype == np.float32 and np.array_equal(waves[g], want[g]), g
            assert np.array_equal(starts[g], want_starts[g]), g
        # a text of one sentence is `tts` of that sentence
        one = eng.tts(GROUPS[0][0][None], silence_duration=SD, **DROPOUT[kind])[0][0]
        assert np.array_equal(eng.tts_joined(GROUPS[:1], silence_duration=SD, **DROPOUT[kind])[0][0], one)
    finally:
        eng.set_precision("bf16x3")


def test_more_than_128_sentences(tts_eng):
    """130 sentences in three texts: the acoustic model runs 128 rows and then 2, and in SEED mode row r draws as row r
    of predict_mel(seed=) on the same rows"""
    eng = tts_eng
    rows = [sentence(100 + i) for i in range(130)]
    texts = [rows[:60], rows[60:129], rows[129:]]
    for kw in ({"seed": 5}, {}):
        waves, starts = eng.tts_joined(texts, silence_duration=SD, **kw)
        want, want_starts = host_joined(eng, texts, kw)
        for g in range(3):
            assert np.array_equal(waves[g], want[g]) and np.array_equal(starts[g], want_starts[g]), (kw, g)


def test_retry_and_bad_arguments(tts_eng):
    eng = tts_eng
    lib, h = eng.lib, eng.h
    tok, lens = padded(GROUPS)
    B, L = tok.shape
    gs = np.array([0, 1, 4, 11, 13], np.int32)
    G = 4
    dur = np.empty((B, L), np.float32)
    starts = np.zeros(B, np.int32)
    nf = np.zeros(G, np.int32)
    nmax = C.c_int32(0)
    wav = np.full(G * 8 * HOP, 7.0, np.float32)

    def call(tok=tok, lens=lens, B=B, L=L, gs=gs, G=G, mode=0, cap=8, wav=wav, starts=starts):
        p = lambda a: None if a is None else a.ctypes.data
        return lib.vtts_tts_joined_host(h, p(tok), p(lens), B, L, p(gs), G, SD, mode, 0, cap, p(dur), p(starts), p(nf),
                                        C.byref(nmax), p(wav))

    n0 = eng.launch_count()
    assert call() != 0                                          # 8 frames are too few: sizes set, nothing vocoded
    _, _, _, ne = eng.tts_plan(tok, lens, silence_duration=SD)
    counts = [int(ne[a:b].sum()) for a, b in zip(gs, gs[1:])]
    assert nf.tolist() == counts and nmax.value == max(counts) and (wav == 7.0).all()
    assert starts.tolist() == [int(s) for a, b in zip(gs, gs[1:]) for s in np.concatenate([[0], np.cumsum(ne[a:b])[:-1]])]
    assert "retry" in lib.vtts_last_error(h).decode()
    n1 = eng.launch_count()
    bad = [dict(gs=np.array([1, 1, 4, 11, 13], np.int32)), dict(gs=np.array([0, 4, 4, 11, 13], np.int32)),
           dict(gs=np.array([0, 1, 4, 11, 12], np.int32)), dict(G=0), dict(B=0), dict(L=0), dict(mode=1), dict(mode=9),
           dict(cap=0), dict(tok=None), dict(gs=None), dict(wav=None), dict(starts=None)]
    for kw in bad:
        assert call(**kw) != 0, kw
        assert eng.launch_count() == n1, kw                      # failed before any launch
    long = np.zeros((1, 6000), np.int32)
    assert call(tok=long, lens=None, B=1, L=6000, gs=np.array([0, 1], np.int32), G=1) != 0
    assert eng.launch_count() == n1
    # Engine.tts_joined retries with the reported size
    got, _ = eng.tts_joined(GROUPS, silence_duration=SD, max_frames=8)
    want, _ = eng.tts_joined(GROUPS, silence_duration=SD)
    assert all(np.array_equal(a, b) for a, b in zip(got, want))


# ---- B. a continued TTS stream slot --------------------------------------------------------------------------------------

def joined_schedule():
    """per utterance: (first step it may begin in, slot, sentences, overrides, steps after begin at which each next
    sentence is appended, step after begin of `finish` or None)"""
    from viettts_b200.engine import MIN_TEMPO
    return [
        (0, 0, [sentence(200), sentence(201), sentence(202)], {}, [1, 2], None),          # appends while the first scans
        (0, 1, [sentence(203), sentence(204)], dict(tempo=MIN_TEMPO, bed=1, semitones=-4.0), [60], None),   # long wait
        (1, 2, [EMPTY, sentence(205), EMPTY, sentence(206)], dict(gain_db=3.0), [1, 2, 3], None),   # zero-frame first, mid
        (0, 3, [sentence(207), sentence(208)], dict(bed=-1), [2], 40),                   # finish with nothing queued
        (0, 4, [sentence(209)], dict(semitones=2.0), [], None),                          # a plain begin ...
        (0, 4, [sentence(210), sentence(211)], {}, [3], None),                           # ... its slot reused at once
        (2, 5, [EMPTY, EMPTY], {}, [1], 4),                                              # nothing to vocode at all
    ]


def run_joined_stream(eng, sched, S, max_frames, max_joined, opts, kw):
    pending = [[] for _ in range(S)]
    for u, e in enumerate(sched):
        pending[e[1]].append(u)
    pieces = {u: [] for u in range(len(sched))}
    meter, frames, ended, begun, waits = {}, {}, {}, {}, {u: 0 for u in range(len(sched))}
    owner = [None] * S
    with eng.open_tts_stream(S, 16, max_frames, 100, **opts, **kw, max_joined_frames=max_joined) as ts:
        step = 0
        while any(pending) or ts.busy().any():
            busy = ts.busy()
            for s in range(S):
                if not busy[s] and pending[s] and sched[pending[s][0]][0] <= step:
                    u = pending[s].pop(0)
                    _, _, sents, ov, at, fin = sched[u]
                    ov = {k: v for k, v in ov.items() if opts.get(OPENED_WITH[k]) is not None}
                    frames[u] = ts.begin(s, sents[0], silence_duration=SD, more=len(sents) > 1 or fin is not None, **ov)
                    owner[s], begun[u] = u, step
            for s in range(S):
                u = owner[s]
                if u is None or u in ended:
                    continue
                _, _, sents, _, at, fin = sched[u]
                for i, off in enumerate(at):
                    if step == begun[u] + off:
                        frames[u] += ts.append(s, sents[i + 1], more=i + 2 < len(sents) or fin is not None)
                if fin is not None and step == begun[u] + fin:
                    ts.finish(s)
            waiting = {s for s in range(S) if owner[s] is not None and ts.busy()[s] and not ts.ac.open[s] and not ts._queue[s]}
            out = ts.step()
            m = ts.meter() if ts.mt is not None else {}
            busy = ts.busy()
            for s, w in out.items():
                u = owner[s]
                pieces[u].append(w)
                if s in waiting and busy[s]:
                    assert w.size == 0, (u, step)
                    waits[u] += 1
                if s in m:
                    meter[u] = m[s]
                if not busy[s]:
                    ended[u] = step
            step += 1
            assert step < 3000
    for s in range(S):                                     # a slot's next utterance began in the step after its END
        us = [u for u in range(len(sched)) if sched[u][1] == s]
        for a, b in zip(us, us[1:]):
            assert begun[b] == ended[a] + 1, (s, a, b)
    return {u: (np.concatenate(pieces[u]) if pieces[u] else None, meter.get(u), frames[u], waits[u]) for u in range(len(sched))}


def joined_one_shot(eng, opts, sents, ov, kw, encoding):
    from viettts_b200.engine import AudioChain
    o = dict(opts)
    for k, v in ov.items():
        if opts.get(OPENED_WITH[k]) is not None and k != "bed":
            o[k] = v
    if o.get("bed") is not None:
        bank = o["bed"] if isinstance(o["bed"], list) else [o["bed"]]
        v = ov.get("bed", 0)
        o["bed"] = None if v == -1 else bank[v]
    wav = eng.tts_joined([sents], silence_duration=SD, **kw)[0][0]
    return AudioChain(**o, encoding=encoding).run(eng, wav)


def check_joined_stream(eng, sched, S, max_frames, max_joined, opts, kw):
    coded = run_joined_stream(eng, sched, S, max_frames, max_joined, dict(opts, encoding="pcm16"), kw)
    flt = run_joined_stream(eng, sched, S, max_frames, max_joined, opts, kw)
    for u, (_, _, sents, ov, _, _) in enumerate(sched):
        codes, reading, frames, _ = coded[u]
        if frames == 0:
            assert codes is not None and codes.size == 0 and codes.dtype == np.int16 and reading is None, u
            assert flt[u][0].size == 0 and flt[u][0].dtype == np.float32, u
            continue
        want = joined_one_shot(eng, opts, sents, ov, kw, "pcm16")
        assert codes.shape == want.shape and np.array_equal(codes, want), ("codes", u)
        audio = joined_one_shot(eng, opts, sents, ov, kw, None)
        assert np.array_equal(flt[u][0], audio), ("float audio", u)
        if opts.get("meter"):
            ref = np.array(eng.loudness(audio, opts.get("output_rate") or config.SAMPLE_RATE), np.float32)
            assert np.array_equal(np.array(reading, np.float32), ref), ("meter", u, reading, ref)
            assert np.array_equal(np.array(flt[u][1], np.float32), ref), ("meter, float run", u)
    return coded


@pytest.mark.parametrize("kind", ["off", "reference"])
@pytest.mark.parametrize("mode", ["bf16x3", "fp16"])
def test_continued_stream_equals_one_shot_chain(tts_eng, mode, kind):
    eng = tts_eng
    eng.set_precision(mode)
    eng.set_fused_pairs(False)
    try:
        kw = {"off": {}, "reference": {"rng": KEY}}[kind]
        coded = check_joined_stream(eng, joined_schedule(), 6, 2000, 6000, STREAM_OPTS, kw)
        assert coded[1][3] >= 5                                 # the long wait stepped out empty arrays
    finally:
        eng.set_fused_pairs(True)
        eng.set_precision("bf16x3")


def test_continued_stream_at_max_joined_frames(tts_eng):
    """a joined utterance of exactly max_joined_frames at MIN_TEMPO under a bed with a 10 s tail; an append past it is
    refused and leaves the slot as it was"""
    from viettts_b200.engine import MIN_TEMPO
    eng = tts_eng
    eng.set_precision("bf16x3")
    eng.set_fused_pairs(False)
    try:
        a, b = sentence(300), sentence(301)
        _, _, nf, ne = eng.tts_plan(np.stack([np.pad(a, (0, 40 - a.size)), np.pad(b, (0, 40 - b.size))]), [a.size, b.size],
                                    silence_duration=SD)
        cap = int(ne.sum())
        opts = dict(STREAM_OPTS, tempo=MIN_TEMPO, bed="pink,tail=10000")
        with eng.open_tts_stream(2, 16, int(nf.max()), 100, max_joined_frames=cap, **opts) as ts:
            ts.begin(0, a, silence_duration=SD, more=True)
            with pytest.raises(ValueError, match="max_joined_frames"):
                ts.append(0, b, more=True) and ts.append(0, a)
            assert ts._joined[0] == cap and ts._more[0]
            ts.finish(0)
            while ts.busy().any():
                ts.step()
        check_joined_stream(eng, [(0, 1, [a, b], {}, [3], None)], 2, int(nf.max()), cap, opts, {})
    finally:
        eng.set_fused_pairs(True)


# ---- C. the CLI ---------------------------------------------------------------------------------------------------------

def test_cli_split_sentences(acoustic_ckpt, hifigan_params, golden_dir, tmp_path, monkeypatch):
    from viettts_b200 import synthetic, synthesizer
    from viettts_b200.engine import AudioChain, get_engine
    from viettts_b200.nat import text2mel as t2m
    (tmp_path / "assets/hifigan").mkdir(parents=True)
    (tmp_path / "assets/infore/hifigan").mkdir(parents=True)
    (tmp_path / "assets/infore/nat").mkdir(parents=True)
    (tmp_path / "assets/hifigan/config.json").write_text(json.dumps(config.HIFIGAN))
    with open(tmp_path / "assets/infore/hifigan/hk_hifi.pickle", "wb") as f:
        pickle.dump(hifigan_params, f)
    with open(tmp_path / "assets/infore/nat/acoustic_latest_ckpt.pickle", "wb") as f:
        pickle.dump(acoustic_ckpt, f)
    with open(tmp_path / "assets/infore/nat/duration_latest_ckpt.pickle", "wb") as f:
        pickle.dump(synthetic.duration_ckpt(1234), f)
    monkeypatch.chdir(tmp_path)
    lex = str(golden_dir / "lexicon_small.txt")
    get_engine(0).set_precision("bf16x3")
    chain = AudioChain(eq="hs:6000:3", limit=-1.0)
    text = "Xin chào, tôi là trợ lý ảo. Hôm nay trời đẹp quá! Giá là 3.5 triệu…"
    rc = synthesizer.main(["--text", text, "--split-sentences", "--output", "one.wav", "--lexicon-file", lex,
                           "--silence-duration", "0.1", "--eq", "hs:6000:3", "--limiter"])
    assert rc == 0
    eng = get_engine(0)

    def toks(t):
        return [t2m.text2tokens(synthesizer.nat_normalize_text(s), lex) for s in synthesizer.split_sentences(t)]

    assert len(toks(text)) == 3
    w = eng.tts_joined([toks(text)], silence_duration=0.1, rng=t2m.checkpoint_rng())[0][0]
    synthesizer.write_wav(tmp_path / "want.wav", chain.run(eng, w))
    assert (tmp_path / "one.wav").read_bytes() == (tmp_path / "want.wav").read_bytes()

    lines = ["Xin chào. Tôi là trợ lý ảo, rất vui!", "hôm nay trời đẹp quá! bạn có khỏe không?"]
    (tmp_path / "lines.txt").write_text("\n".join(lines) + "\n")
    rc = synthesizer.main(["--text-file", "lines.txt", "--split-sentences", "--output", "out.wav", "--lexicon-file", lex,
                           "--silence-duration", "0.1", "--seed", "5"])
    assert rc == 0
    whole = [t2m.text2tokens(synthesizer.nat_normalize_text(t), lex) for t in lines]
    order = sorted(range(2), key=lambda i: len(whole[i]))
    waves, _ = eng.tts_joined([toks(lines[i]) for i in order], silence_duration=0.1, seed=5)
    for r, i in enumerate(order):
        synthesizer.write_wav(tmp_path / f"want_{i}.wav", waves[r])
        assert (tmp_path / f"out_{i:04d}.wav").read_bytes() == (tmp_path / f"want_{i}.wav").read_bytes(), i
