"""GPU: the streaming generator (Engine.open_vocoder_stream, vtts_vocoder_stream_*).

Every comparison is bit-exact (np.array_equal) against `mel2wave` of the same whole mel in the same precision mode with
the fused ResBlock-pair kernel off, unless stated otherwise."""
import numpy as np
import pytest
import torch

from viettts_b200 import synthetic

pytestmark = pytest.mark.gpu
HOP = 256
F = 64                       # max_chunk_frames of the stream objects below
LAUNCHES_PER_PUSH = 31       # prep, conv_pre, 4 x (ConvTranspose + 3 pairs x 2 convs), conv_post


@pytest.fixture(scope="module")
def eng(hifigan_params):
    from viettts_b200.engine import Engine
    e = Engine(0)
    e.load_hifigan(hifigan_params)
    yield e
    e.close()


@pytest.fixture(params=["bf16x3", "fp16"])
def mode(request, eng):
    eng.set_precision(request.param)
    eng.set_fused_pairs(False)
    yield request.param
    eng.set_fused_pairs(True)
    eng.set_precision("bf16x3")


def one_shot(eng, mel):
    return eng.mel2wave(mel[None])[0]


def stream_chunks(vs, mel, chunks, slot=0):
    """push `mel` [T,80] into `slot` in pieces of the given sizes (BEGIN with the first, END with the last); returns the
    concatenated audio and the frames emitted per push"""
    S, T = vs.max_streams, mel.shape[0]
    out, counts, t = [], [], 0
    for i, c in enumerate(chunks):
        buf = np.zeros((S, vs.max_chunk_frames, 80), np.float32)
        buf[slot, :c] = mel[t: t + c]
        n = np.zeros(S, np.int32)
        n[slot] = c
        beg = np.zeros(S, bool)
        end = np.zeros(S, bool)
        beg[slot] = i == 0
        end[slot] = i == len(chunks) - 1
        got = vs.push(buf, n, beg, end)
        assert all(g.size == 0 for s, g in enumerate(got) if s != slot)
        out.append(got[slot])
        counts.append(got[slot].size // HOP)
        t += c
    assert t == T
    return np.concatenate(out), counts


def split(T, chunk):
    return [min(chunk, T - t) for t in range(0, T, chunk)]


def expected_counts(chunks, D):
    P, e, res = 0, 0, []
    for i, c in enumerate(chunks):
        P += c
        e_new = P if i == len(chunks) - 1 else max(e, P - D)
        res.append(e_new - e)
        e = e_new
    return res


@pytest.mark.parametrize("chunk", [1, 7, 16, 47, F])
def test_chunks_equal_one_shot(eng, mode, chunk):
    mel = synthetic.mel_input(21, 1, 150)[0]
    ref = one_shot(eng, mel)
    with eng.open_vocoder_stream(1, F) as vs:
        assert vs.lookahead == 13
        chunks = split(150, chunk)
        got, counts = stream_chunks(vs, mel, chunks)
        assert counts == expected_counts(chunks, vs.lookahead)
    assert got.shape == ref.shape and np.array_equal(got, ref), (mode, chunk, float(np.abs(got - ref).max()))


def test_long_utterance(eng, mode):
    mel = synthetic.mel_input(99, 1, 1000)[0]
    ref = one_shot(eng, mel)
    with eng.open_vocoder_stream(1, F) as vs:
        got, _ = stream_chunks(vs, mel, split(1000, 37))
    assert np.array_equal(got, ref)


@pytest.mark.parametrize("T", [1, 2, 5])
def test_shorter_than_lookahead(eng, mode, T):
    mel = synthetic.mel_input(30 + T, 1, T)[0]
    ref = one_shot(eng, mel)
    with eng.open_vocoder_stream(2, F) as vs:
        got, counts = stream_chunks(vs, mel, [T], slot=1)            # BEGIN|END in one push
        assert counts == [T] and np.array_equal(got, ref)
        got, counts = stream_chunks(vs, mel, split(T, 2), slot=0)   # everything arrives before END: all of it with END
        assert counts[-1] == T and np.array_equal(got, ref)


def test_begin_end_in_one_push_equals_mel2wave(eng, mode):
    mel = synthetic.mel_input(5, 1, F)[0]
    with eng.open_vocoder_stream(1, F) as vs:
        got, counts = stream_chunks(vs, mel, [F])
    assert counts == [F] and np.array_equal(got, one_shot(eng, mel))


def test_end_with_no_new_frames(eng, mode):
    mel = synthetic.mel_input(6, 1, 40)[0]
    with eng.open_vocoder_stream(1, F) as vs:
        got, counts = stream_chunks(vs, mel, [16, 24, 0])
    assert counts == expected_counts([16, 24, 0], 13) and counts[-1] == 13
    assert np.array_equal(got, one_shot(eng, mel))


def test_many_slots_ragged(eng, mode):
    """8 slots: ragged chunk sequences, staggered BEGINs, idle pushes, slots ending while others go on, a slot reused
    after END.  Every utterance equals its one-shot waveform and the same stream run alone in a 1-slot object."""
    S, rng = 8, np.random.default_rng(3)
    # per slot a queue of utterances (slot 2 runs two in a row); start push per slot
    utts = {s: [synthetic.mel_input(100 + s, 1, int(rng.integers(3, 130)))[0]] for s in range(S)}
    utts[2].append(synthetic.mel_input(200, 1, 61)[0])
    start = {s: int(rng.integers(0, 6)) for s in range(S)}
    plans = {s: [] for s in range(S)}   # list of (utterance index, chunk sizes)
    for s in range(S):
        for u, mel in enumerate(utts[s]):
            sizes, t = [], 0
            while t < mel.shape[0]:
                c = int(min(rng.integers(1, F + 1), mel.shape[0] - t))
                sizes.append(c)
                t += c
            plans[s].append(sizes)
    state = {s: [0, 0, 0] for s in range(S)}        # utterance, chunk index, frames pushed
    outs = {s: [[] for _ in utts[s]] for s in range(S)}
    chunk_log = {s: [[] for _ in utts[s]] for s in range(S)}
    with eng.open_vocoder_stream(S, F) as vs:
        step = 0
        while any(state[s][0] < len(utts[s]) for s in range(S)):
            buf = np.zeros((S, F, 80), np.float32)
            n = np.zeros(S, np.int32)
            beg, end = np.zeros(S, bool), np.zeros(S, bool)
            touched = []
            for s in range(S):
                u, ci, t = state[s]
                if u >= len(utts[s]) or step < start[s] or rng.random() < 0.25:   # not started, done, or idle this push
                    continue
                c = plans[s][u][ci]
                buf[s, :c] = utts[s][u][t: t + c]
                n[s] = c
                beg[s] = ci == 0
                end[s] = ci == len(plans[s][u]) - 1
                touched.append((s, u, c, end[s]))
            got = vs.push(buf, n, beg, end)
            for s in range(S):
                if all(s != x[0] for x in touched):
                    assert got[s].size == 0
            for s, u, c, e in touched:
                outs[s][u].append(got[s])
                chunk_log[s][u].append(c)
                state[s][1] += 1
                state[s][2] += c
                if e:
                    state[s] = [u + 1, 0, 0]
            step += 1
    with eng.open_vocoder_stream(1, F) as alone:
        for s in range(S):
            for u, mel in enumerate(utts[s]):
                got = np.concatenate(outs[s][u])
                ref = one_shot(eng, mel)
                assert np.array_equal(got, ref), (mode, s, u)
                solo, _ = stream_chunks(alone, mel, chunk_log[s][u])
                assert np.array_equal(solo, got)


def test_against_default_fused_one_shot(eng, mode):
    """The default one-shot path fuses the C <= 64 ResBlock pairs; the stream runs them as two convs.  Held to the 1e-6
    of test_streaming_chunks_equal_full_utterance.  Measured on an H100: 0 in both modes (the fused kernel rounds its
    on-chip intermediate exactly as the converter of the second conv does, and sums in the same order)."""
    mel = synthetic.mel_input(21, 1, 150)[0]
    with eng.open_vocoder_stream(1, F) as vs:
        got, _ = stream_chunks(vs, mel, split(150, 16))
    eng.set_fused_pairs(True)
    try:
        fused = one_shot(eng, mel)
    finally:
        eng.set_fused_pairs(False)
    err = float(np.abs(got - fused).max())
    print(f"[stream vs fused one-shot, {mode}] max |diff| = {err:.3e}")
    assert err <= 1e-6


def test_device_push_matches_host_push(eng, mode):
    S, T, chunk = 3, 90, 30
    mels = synthetic.mel_input(8, S, T)
    dev = torch.device("cuda", 0)
    with eng.open_vocoder_stream(S, chunk) as a, eng.open_vocoder_stream(S, chunk) as b:
        out_t = torch.empty((S, b.wav_ld), dtype=torch.float32, device=dev)
        for i in range(T // chunk):
            buf = np.ascontiguousarray(mels[:, i * chunk:(i + 1) * chunk])
            n = np.full(S, chunk, np.int32)
            flags = np.full(S, (1 if i == 0 else 0) | (2 if i == T // chunk - 1 else 0), np.uint8)
            host = a.push(buf, n, flags & 1, flags & 2)
            n_out = b.push_device(torch.from_numpy(buf).to(dev), n, flags, out_t)
            wav = out_t.cpu().numpy()
            for s in range(S):
                assert np.array_equal(wav[s, : n_out[s] * HOP], host[s])


@pytest.mark.parametrize("S,chunk", [(1, 1), (1, 40), (6, 5), (6, 64)])
def test_launch_count_fixed(eng, mode, S, chunk):
    mel = synthetic.mel_input(4, S, chunk)
    with eng.open_vocoder_stream(S, F) as vs:
        for flags in ((True, False), (False, False), (False, True)):
            n0 = eng.launch_count()
            vs.push(mel, np.full(S, chunk, np.int32), np.full(S, flags[0]), np.full(S, flags[1]))
            assert eng.launch_count() - n0 == LAUNCHES_PER_PUSH


def test_bad_arguments(eng, hifigan_params):
    from viettts_b200._lib import VttsError
    from viettts_b200.engine import Engine
    eng.set_precision("bf16x3")
    mel = np.zeros((2, 8, 80), np.float32)
    with eng.open_vocoder_stream(2, 8) as vs:
        with pytest.raises(VttsError, match="outside"):
            vs.push(np.zeros((2, 8, 80), np.float32), np.array([9, 0], np.int32))
        with pytest.raises(VttsError, match="not open"):            # never begun
            vs.push(mel, np.array([3, 0], np.int32))
        vs.push(mel, np.array([3, 0], np.int32), begin=[True, False], end=[True, False])
        with pytest.raises(VttsError, match="not open"):            # after END without BEGIN
            vs.push(mel, np.array([3, 0], np.int32))
        with pytest.raises(VttsError, match="flags"):
            vs.push_device(torch.zeros((2, 8, 80), device="cuda"), np.array([1, 0], np.int32), np.array([4, 0], np.uint8),
                           torch.zeros((2, vs.wav_ld), device="cuda"))
        eng.set_precision("fp32")
        try:
            with pytest.raises(VttsError, match="fp32"):
                vs.push(mel, np.array([3, 0], np.int32), begin=[True, False])
        finally:
            eng.set_precision("bf16x3")
        # the failed calls left the slots as they were: a fresh utterance still equals the one-shot waveform
        m = synthetic.mel_input(2, 1, 8)
        eng.set_fused_pairs(False)
        try:
            got = vs.push(np.concatenate([m, m]), np.array([8, 0], np.int32), begin=[True, False], end=[True, False])[0]
            assert np.array_equal(got, eng.mel2wave(m)[0])
        finally:
            eng.set_fused_pairs(True)
    bare = Engine(0)
    try:
        with pytest.raises(VttsError, match="not loaded"):
            bare.open_vocoder_stream(1, 8)
    finally:
        bare.close()
