"""GPU: the streaming acoustic model (Engine.open_acoustic_stream, vtts_acoustic_stream_*) and the text-to-speech stream
(Engine.open_tts_stream).

Every comparison is bit-exact (np.array_equal) against `predict_mel` of the utterance alone, or `Engine.tts` of the same
tokens with the fused ResBlock-pair kernel off, unless stated otherwise."""
import numpy as np
import pytest
import torch

from viettts_b200 import synthetic
from viettts_b200.engine import acoustic_stream_schedule

pytestmark = pytest.mark.gpu
D_A = 10
NF_MAX = 1000
KEY = np.array([7, 1234567], np.uint32)
LENGTHS = [1, 9, 10, 11, 150, 937]


@pytest.fixture(scope="module")
def eng(acoustic_ckpt, hifigan_params):
    from viettts_b200.engine import Engine
    e = Engine(0)
    e.load_acoustic(acoustic_ckpt)
    e.load_hifigan(hifigan_params)
    e.load_duration(synthetic.duration_ckpt(1234))
    yield e
    e.set_precision("bf16x3")
    e.close()


def utt(seed, n):
    """tokens [L] and durations in frames [L] of an utterance of exactly n frames (n_frames is passed explicitly)"""
    rng = np.random.default_rng(seed)
    L = max(3, min(120, n // 6))
    tok = rng.integers(4, 90, size=L).astype(np.int32)
    d = rng.uniform(0.5, 1.5, size=L)
    d = (d * (n + 0.5) / d.sum()).astype(np.float32)
    return tok, d


DROP = ["off", "seed", "mask", "reference"]


def ref_mel(eng, kind, tok, d, n, slot, masks=None):
    """predict_mel of the utterance alone; SEED: as row `slot` of a call with the same seed"""
    if kind == "seed":
        B = slot + 1
        mel = eng.predict_mel(np.repeat(tok[None], B, 0), np.repeat(d[None], B, 0), n_frames=[n] * B, seed=11)
        return mel[slot]
    kw = {"off": {}, "mask": {"masks": masks}, "reference": {"rng": KEY}}[kind]
    return eng.predict_mel(tok[None], d[None], n_frames=[n], **kw)[0]


def open_stream(eng, kind, S, F):
    kw = {"off": {}, "seed": {"seed": 11}, "mask": {"masks": True}, "reference": {"rng": KEY}}[kind]
    return eng.open_acoustic_stream(S, F, NF_MAX, 200, **kw)


def run_until_done(st, on_push=None):
    """push until every slot has closed; returns {slot: [arrays per push]}"""
    outs = {s: [] for s in range(st.max_streams)}
    k = 0
    while st.open.any():
        was = st.open.copy()
        got = st.push()
        for s in np.flatnonzero(was):
            outs[int(s)].append(got[s])
        for s in np.flatnonzero(~was):
            assert got[s].shape[0] == 0
        k += 1
        if on_push:
            on_push(k)
    return outs


@pytest.mark.parametrize("precision", ["fp32", "bf16x3"])
@pytest.mark.parametrize("kind", DROP)
@pytest.mark.parametrize("F", [1, 5, 16, 64])
def test_stream_equals_predict_mel(eng, precision, kind, F):
    """Six lengths (shorter than the lookahead, at it, past it, long), each with and without n_emit, in 12 slots of one
    stream: every slot's frames equal predict_mel of its utterance alone, and n_out follows the host schedule."""
    eng.set_precision(precision)
    S = 2 * len(LENGTHS)
    cases = []
    with open_stream(eng, kind, S, F) as st:
        for i, n in enumerate(LENGTHS):
            for j in range(2):
                slot = 2 * i + j
                tok, d = utt(100 + i, n)
                ne = None if j == 0 else max(1, n - 4)
                m = synthetic.dropout_masks(300 + i, 1, n) if kind == "mask" else None
                st.begin([slot], tok[None], d[None], n_frames=[n], n_emit=None if ne is None else [ne], masks=m)
                cases.append((slot, tok, d, n, ne, m))
        outs = run_until_done(st)
    for slot, tok, d, n, ne, m in cases:
        ref = ref_mel(eng, kind, tok, d, n, slot, m)
        got = np.concatenate(outs[slot])
        want = ref[: n if ne is None else ne]
        assert [o.shape[0] for o in outs[slot]] == acoustic_stream_schedule(n, ne, F, D_A), (slot, n, ne)
        assert got.shape == want.shape and np.array_equal(got, want), (precision, kind, F, n, ne, float(np.abs(got - want).max()))


def test_continuous_batching(eng):
    """40 utterances of mixed lengths through 8 slots; a slot begins its next utterance in the push after its previous
    one closed, so the slots sit at different frames in every push."""
    eng.set_precision("bf16x3")
    rng = np.random.default_rng(9)
    lens = [int(x) for x in rng.integers(1, 320, size=40)]
    queue = list(range(40))
    where, outs = {}, {i: [] for i in range(40)}
    F, S = 16, 8
    with open_stream(eng, "reference", S, F) as st:
        frames_seen = set()
        while queue or st.open.any():
            for s in np.flatnonzero(~st.open):
                if queue:
                    i = queue.pop(0)
                    tok, d = utt(500 + i, lens[i])
                    st.begin([int(s)], tok[None], d[None], n_frames=[lens[i]])
                    where[int(s)] = i
            P = tuple(sorted(int(x) for x in st._left[st.open]))
            frames_seen.add(P)
            was = st.open.copy()
            got = st.push()
            for s in np.flatnonzero(was):
                outs[where[int(s)]].append(got[s])
    assert len(frames_seen) > 10
    for i in range(40):
        tok, d = utt(500 + i, lens[i])
        ref = eng.predict_mel(tok[None], d[None], n_frames=[lens[i]], rng=KEY)[0]
        assert np.array_equal(np.concatenate(outs[i]), ref), i


def test_all_128_slots_in_one_push(eng):
    eng.set_precision("bf16x3")
    S, F = 128, 32
    lens = np.random.default_rng(4).integers(20, 70, size=S)
    toks, durs = zip(*[utt(700 + s, int(lens[s])) for s in range(S)])
    L = max(len(t) for t in toks)
    tok = np.zeros((S, L), np.int32)
    dur = np.zeros((S, L), np.float32)
    ll = np.array([len(t) for t in toks], np.int32)
    for s in range(S):
        tok[s, : ll[s]] = toks[s]
        dur[s, : ll[s]] = durs[s]
    ref = eng.predict_mel(tok, dur, lengths=ll, n_frames=lens)     # OFF: row s equals the utterance alone
    with open_stream(eng, "off", S, F) as st:
        st.begin(np.arange(S), tok, dur, lengths=ll, n_frames=lens)
        outs = run_until_done(st)
    for s in range(S):
        assert np.array_equal(np.concatenate(outs[s]), ref[s, : lens[s]]), s


def test_resumed_state_matches_one_shot_mel_pre(eng):
    """After k pushes the projection outputs so far equal the one-shot mel_pre tap bit for bit."""
    eng.set_precision("bf16x3")
    n, F = 150, 16
    tok, d = utt(31, n)
    eng.predict_mel(tok[None], d[None], n_frames=[n], seed=11)
    pre = eng.debug_read("mel_pre", (1, n, 80))[0]
    with open_stream(eng, "seed", 1, F) as st:
        st.begin([0], tok[None], d[None], n_frames=[n])
        for k in range(1, 6):
            st.push()
            got = eng.debug_read("mel_pre", (1, NF_MAX, 80))[0]
            assert np.array_equal(got[: k * F], pre[: k * F]), k


def test_idle_slot_untouched_and_device_push(eng):
    """A closed slot gets n_out 0 and its rows of the output buffer are left as they were; push_device equals push."""
    eng.set_precision("bf16x3")
    F = 8
    tok, d = utt(3, 40)
    dev = torch.device("cuda", 0)
    with open_stream(eng, "off", 2, F) as a, open_stream(eng, "off", 2, F) as b:
        a.begin([0], tok[None], d[None], n_frames=[40])
        b.begin([0], tok[None], d[None], n_frames=[40])
        out = torch.full((2, F + D_A, 80), 7.0, device=dev)
        while a.open.any():
            host = a.push()
            n_out = b.push_device(out)
            got = out.cpu().numpy()
            assert n_out[1] == 0 and np.all(got[1] == 7.0)
            assert np.array_equal(got[0, : n_out[0]], host[0])


def test_bad_arguments(eng):
    from viettts_b200._lib import VttsError
    eng.set_precision("bf16x3")
    with pytest.raises(VttsError, match="max_streams"):
        eng.open_acoustic_stream(129, 8, 100, 50)
    with pytest.raises(VttsError, match="max_tokens"):
        eng.open_acoustic_stream(1, 8, 100, 100000)
    tok, d = utt(1, 30)
    with eng.open_acoustic_stream(2, 8, 100, 50) as st:
        with pytest.raises(VttsError, match="max_frames"):
            st.begin([0], tok[None], d[None], n_frames=[101])
        st.begin([0], tok[None], d[None], n_frames=[30])
        with pytest.raises(VttsError, match="still open"):
            st.begin([0], tok[None], d[None], n_frames=[30])
        with pytest.raises(VttsError, match="n_emit"):
            st.begin([1], tok[None], d[None], n_frames=[30], n_emit=[31])
        # the failed calls left the stream usable: slot 0 still equals predict_mel
        out = np.concatenate(run_until_done(st)[0])
        assert np.array_equal(out, eng.predict_mel(tok[None], d[None], n_frames=[30])[0])


# ---- text-to-speech stream ------------------------------------------------------------------------------------

def tts_tokens(seed, L):
    rng = np.random.default_rng(seed)
    t = rng.integers(4, 90, size=L).astype(np.int32)
    t[4::5] = 3
    t[0] = t[-1] = 0
    return t


def run_tts(ts, slots_tokens, silence):
    """begin every (slot, tokens), step until done; returns {slot: audio}, {slot: [samples per step]}, frames planned"""
    planned = {s: ts.begin(s, t, silence_duration=silence) for s, t in slots_tokens}
    pieces = {s: [] for s, _ in slots_tokens}
    while ts.busy().any():
        for s, w in ts.step().items():
            pieces[s].append(w)
    return {s: np.concatenate(p) for s, p in pieces.items()}, pieces, planned


@pytest.mark.parametrize("kind", ["off", "reference", "seed"])
@pytest.mark.parametrize("silence", [-1.0, 0.12])
def test_tts_stream_equals_tts(eng, kind, silence):
    eng.set_precision("bf16x3")
    eng.set_fused_pairs(False)
    try:
        lens = [30, 7, 55]
        tok = np.zeros((3, max(lens)), np.int32)
        for b, n in enumerate(lens):
            tok[b, :n] = tts_tokens(60 + b, n)
        kw = {"off": {}, "reference": {"rng": KEY}, "seed": {"seed": 5}}[kind]
        waves, _ = eng.tts(tok, lens, silence_duration=silence, **kw)
        with eng.open_tts_stream(4, 16, 2000, 100, **kw) as ts:
            audio, pieces, planned = run_tts(ts, [(b, tok[b, : lens[b]]) for b in range(3)], silence)
        for b in range(3):
            assert planned[b] * 256 == waves[b].size
            assert audio[b].shape == waves[b].shape and np.array_equal(audio[b], waves[b]), (kind, b)
            # first audio: at the first push after which the slot has scanned >= D_a + 13 + 1 frames, or its last push
            counts = [p.size for p in pieces[b]]
            first = next((i for i, c in enumerate(counts) if c > 0), None)
            if waves[b].size:
                assert first == min(len(counts) - 1, -(-(D_A + 14) // 16) - 1), (counts, b)
    finally:
        eng.set_fused_pairs(True)


def test_tts_stream_vs_fused_default(eng):
    """With the default fused ResBlock-pair kernel in Engine.tts the stream (two convs per pair) is held to 1e-5."""
    eng.set_precision("bf16x3")
    tok = tts_tokens(77, 60)
    waves, _ = eng.tts(tok[None], silence_duration=0.1)
    with eng.open_tts_stream(1, 16, 2000, 100) as ts:
        audio, _, _ = run_tts(ts, [(0, tok)], 0.1)
    err = float(np.abs(audio[0] - waves[0]).max())
    print(f"[tts stream vs fused tts] max |diff| = {err:.3e}")
    assert audio[0].shape == waves[0].shape and err <= 1e-5


def test_tts_stream_rejects_fp32(eng):
    eng.set_precision("fp32")
    try:
        with pytest.raises(ValueError, match="fp32"):
            eng.open_tts_stream(1, 16, 100)
    finally:
        eng.set_precision("bf16x3")
