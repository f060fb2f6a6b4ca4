"""CPU: joined utterances without a GPU.  `split_sentences` over a table of texts; with the recording fake lib of
test_stream_handles_cpu.py, what `Engine.tts_joined` hands to vtts_tts_joined_host, and the flags, frames and errors of
a TTS stream slot continued by `append` / `finish`."""
import ctypes as C

import numpy as np
import pytest
import torch

from test_stream_handles_cpu import FakeLib, eng  # noqa: F401  (the fixture)
from viettts_b200 import engine as E
from viettts_b200.synthesizer import nat_normalize_text, split_sentences


@pytest.mark.parametrize("text, want", [
    ("Xin chào. Tôi là ai?", ["Xin chào", " Tôi là ai"]),
    ("Một!!! Hai?! Ba...", ["Một", " Hai", " Ba"]),
    ("Chờ đã… rồi đi", ["Chờ đã", " rồi đi"]),
    ("Giá là 3.5 triệu. Rẻ", ["Giá là 3.5 triệu", " Rẻ"]),
    ("dòng một\ndòng hai", ["dòng một", "dòng hai"]),
    ("không có dấu câu", ["không có dấu câu"]),
    ("... ! ?\n\n. Một câu.", [" Một câu"]),
    ("", []),
    ("Năm 2024. Được", ["Năm 2024", " Được"]),
    ("a.b.c. d", ["a.b.c", " d"]),
    ("Đường phố Hà Nội! Ồ.", ["Đường phố Hà Nội", " Ồ"]),
])
def test_split_sentences(text, want):
    assert split_sentences(text) == want


def test_split_sentences_keep_one_silence_between():
    """each piece normalizes to words alone: the only silence between two joined sentences is the next one's leading sil"""
    for piece in split_sentences("Xin chào, bạn. Hôm nay trời đẹp! Đi chơi nhé?"):
        words = nat_normalize_text(piece).split()
        assert words and words[-1] != "sil" and words[0] != "sil", piece


def test_tts_joined_marshalling(eng):
    calls = []

    def joined(h, tok, lens, B, L, gs, G, sil, mode, seed, cap, dur, starts, nf, nmax, wav):
        calls.append(dict(tok=eng.lib.arrays[tok].copy(), lens=eng.lib.arrays[lens].copy(), B=B, L=L, gs=eng.lib.arrays[gs].copy(),
                          G=G, sil=sil, mode=mode, seed=seed, cap=cap))
        eng.lib.arrays[starts][...] = [0, 5, 0, 4][:B]   # text 1 ends in a zero-frame sentence
        eng.lib.arrays[nf][...] = [9, 4][:G]
        nmax._obj.value = 9
        return 0 if cap >= 9 else 1

    eng.lib.vtts_tts_joined_host = joined
    eng.lib.vtts_last_error = lambda h: b"retry"
    texts = [[[0, 5, 6, 0], [0, 7, 0]], [np.array([0, 9, 9, 9, 9, 0], np.int64), [0, 1, 2]]]
    waves, starts = eng.tts_joined(texts, silence_duration=0.2, seed=11, max_frames=4)
    assert len(calls) == 2 and calls[0]["cap"] == 4 and calls[1]["cap"] == 9        # the retry with the reported size
    c = calls[1]
    assert (c["B"], c["L"], c["G"], c["mode"], c["seed"]) == (4, 6, 2, E.DROPOUT_SEED, 11) and c["sil"] == pytest.approx(0.2)
    assert c["tok"].dtype == np.int32 and c["tok"].tolist() == [[0, 5, 6, 0, 0, 0], [0, 7, 0, 0, 0, 0], [0, 9, 9, 9, 9, 0],
                                                                 [0, 1, 2, 0, 0, 0]]
    assert c["lens"].tolist() == [4, 3, 6, 3] and c["gs"].dtype == np.int32 and c["gs"].tolist() == [0, 2, 4]
    assert [w.size for w in waves] == [9 * 256, 4 * 256]
    assert [s.tolist() for s in starts] == [[0, 5 * 256], [0, 4 * 256]] and starts[0].dtype == np.int64
    eng.tts_joined([[[0, 3, 0]]], rng=np.array([1, 2], np.uint32), max_frames=9)
    assert calls[-1]["mode"] == E.DROPOUT_REFERENCE and calls[-1]["seed"] == (1 << 32) | 2
    eng.tts_joined([[[0, 3, 0]]], max_frames=9)
    assert calls[-1]["mode"] == E.DROPOUT_OFF
    n = len(calls)
    for bad in ([], [[]], [[[]]], [[[[0, 1]]]], [[[0.5, 1.0]]]):
        with pytest.raises(ValueError):
            eng.tts_joined(bad)
    assert len(calls) == n


# ---- a TTS stream slot continued by append -----------------------------------------------------------------------------
S, F, NF = 3, 4, 10            # slots, chunk frames, acoustic frames of every sentence

PLANS = {1: (NF, 8), 2: (NF, 0), 3: (NF, 6)}   # a sentence's first token -> (n_frames, n_emit) of its plan


@pytest.fixture
def ts(eng, monkeypatch):
    """a TtsStream on the fake lib (tensors on the host), its tts_plan from PLANS, with a meter; the acoustic push emits
    2 frames per open slot"""
    monkeypatch.setattr(torch, "device", lambda *a: "cpu")
    monkeypatch.setattr(torch.Tensor, "pin_memory", lambda self: self)
    monkeypatch.setattr(torch.cuda, "current_stream", lambda *a: type("St", (), {"cuda_stream": 0})())
    eng.get_precision = lambda: E.PRECISION_BF16X3

    def plan(tok, silence_duration=-1.0):
        nf, ne = PLANS[int(np.asarray(tok).ravel()[0])]
        return None, np.ones((1, tok.shape[1]), np.float32), np.array([nf], np.int32), np.array([ne], np.int32)

    eng.tts_plan = plan
    t = E.TtsStream(eng, S, F, 2 * NF, 16, meter=True, max_joined_frames=22)
    real = eng.lib.__getattr__("vtts_acoustic_stream_push")

    def ac_push(h, hs, out, n_out, st):
        eng.lib.arrays[n_out][...] = np.where(t.ac.open, 2, 0)
        return real(h, hs, out, n_out, st)

    eng.lib.vtts_acoustic_stream_push = ac_push
    return t


def voc_pushes(eng):
    return [(r[3]["data"].tolist(), r[4]["data"].tolist()) for r in eng.lib.named("vtts_vocoder_stream_push")]


def test_continued_slot_flags(ts, eng):
    """BEGIN with the slot's first frames only, no flags between sentences, END with the last sentence's last push; a
    waiting slot is pushed with n_new 0 and no flags, and steps out an empty array"""
    sched = E.acoustic_stream_schedule(NF, 8, F, 3)           # pushes of one sentence on the fake (lookahead 3)
    assert ts.begin(0, [1, 0], more=True) == 8
    ts.begin(1, [3, 0])                                        # a plain utterance alongside
    outs = [ts.step() for _ in range(len(sched))]
    assert ts.busy().tolist() == [True, False, False]          # slot 0 waits
    for _ in range(3):
        outs.append(ts.step())
    assert all(o[0].size == 0 for o in outs[-3:]) and all(set(o) == {0} for o in outs[-3:])
    assert ts.append(0, [3, 0], more=True) == 6
    assert ts.append(0, [2, 0]) == 0                           # zero frames, last: END once the acoustic side closes
    while ts.busy().any():
        outs.append(ts.step())
    pushes = voc_pushes(eng)
    flags0 = [f[0] for _, f in pushes]
    assert flags0[0] == E.STREAM_BEGIN and flags0.count(E.STREAM_BEGIN) == 1
    assert flags0[-1] == E.STREAM_END and flags0.count(E.STREAM_END) == 1
    assert all(f == 0 for f in flags0[1:-1])
    assert pushes[-1][0][0] == 0                               # END alone: the last sentence planned no frames
    assert pushes[0][1][1] == E.STREAM_BEGIN and [f[1] for _, f in pushes].count(E.STREAM_END) == 1


def test_waiting_slot_pushed_idle(ts, eng):
    """while another slot runs, a waiting slot is in the vocoder push with n_new 0 and flags 0"""
    ts.begin(0, [1, 0], more=True)
    while ts.ac.open[0]:
        ts.step()
    ts.begin(1, [1, 0])
    before = len(voc_pushes(eng))
    out = ts.step()
    p = voc_pushes(eng)[before:]
    assert len(p) == 1 and p[0][0][0] == 0 and p[0][1][0] == 0 and p[0][1][1] == E.STREAM_BEGIN
    assert out[0].size == 0 and ts.busy()[0]
    ts.finish(0)
    ts.step()
    assert voc_pushes(eng)[-1][1][0] == E.STREAM_END and not ts.busy()[0]


def test_all_zero_sentences_report_one_empty_output(ts, eng):
    assert ts.begin(2, [2, 0], more=True) == 0
    assert ts.busy()[2]
    out = ts.step()
    assert set(out) == {2} and out[2].size == 0 and ts.busy()[2]     # waiting
    ts.append(2, [2, 0])
    out = ts.step()
    assert set(out) == {2} and out[2].size == 0 and not ts.busy()[2]
    assert all(f[2] == 0 for _, f in voc_pushes(eng))          # nothing was ever pushed for it


def test_continued_slot_errors(ts, eng):
    ts.begin(0, [1, 0], more=True)
    with pytest.raises(ValueError, match="still open"):
        ts.begin(0, [1, 0])                                     # begin on an open / waiting slot
    with pytest.raises(ValueError, match="no more"):
        ts.append(1, [1, 0])                                    # never begun with more=True
    ts.begin(1, [1, 0])
    with pytest.raises(ValueError, match="no more"):
        ts.append(1, [1, 0])                                    # begun without more
    with pytest.raises(ValueError, match="no more"):
        ts.finish(1)
    with pytest.raises(ValueError, match="max_joined_frames"):
        ts.append(0, [1, 0], more=True)                         # 8 + 8 fits, 8 + 8 + 8 does not ...
        ts.append(0, [1, 0])
    assert ts._joined[0] == 16 and len(ts._queue[0]) == 1 and ts._more[0]   # ... and the refused one left no trace
    with pytest.raises(ValueError, match="max_tokens"):
        ts.append(0, [1] + [0] * 16)
    ts.append(0, [3, 0])
    assert ts._joined[0] == 16 + 6
    with pytest.raises(ValueError, match="no more"):
        ts.append(0, [1, 0])                                    # after more=False
    with pytest.raises(ValueError, match="no more"):
        ts.finish(0)
    ts.begin(2, [3, 0], more=True)
    ts.finish(2)
    with pytest.raises(ValueError, match="no more"):
        ts.append(2, [3, 0])                                    # after finish


def test_meter_sized_by_max_joined_frames(eng, monkeypatch):
    monkeypatch.setattr(torch, "device", lambda *a: "cpu")
    monkeypatch.setattr(torch.Tensor, "pin_memory", lambda self: self)
    eng.get_precision = lambda: E.PRECISION_BF16X3
    seconds = {}
    for mj in (None, 40000):
        eng.lib.calls.clear()
        E.TtsStream(eng, S, F, 100, 16, meter=True, max_joined_frames=mj).close()
        (rec,) = eng.lib.named("vtts_loudness_stream_create")
        seconds[mj] = rec[4]
    assert seconds[None] == -(-100 * 256 // 16000) + 1
    assert seconds[40000] == -(-40000 * 256 // 16000) + 1
    with pytest.raises(ValueError, match="max_joined_frames"):
        E.TtsStream(eng, S, F, 100, 16, max_joined_frames=0)
