"""Joined utterances (Engine.tts_joined, TtsStream.append) against one long row and separate utterances.

    python scripts/bench_joined.py [--out FILE.json]

  * wall time, ending in a synchronise, of one ~90 s text of ~20 sentences: `tts` of the whole text as one row against
    `tts_joined` of its sentences, alternated in one process, with the acoustic sub-stage times of each (the last
    acoustic launch of the call);
  * 8 texts of ~20 s each: `tts` of the 8 rows against `tts_joined` of 8 groups;
  * one stream slot fed 10 sentences by `append` (each appended as soon as the previous one is planned) against 10
    separate `begin`s (each begun the step after the previous one ends): steps, and steps with nothing out while text
    was queued;
  * that `tts_joined` equals `mel2wave` of the host-joined `predict_mel` rows at the timed sizes.

Synthetic weights and a synthetic duration checkpoint, bf16x3.  The card name and power limit are read (nvidia-smi,
read-only) in the same run.  Prints one JSON object; `--out` also writes it."""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from viettts_b200 import config as C  # noqa: E402
from viettts_b200 import synthetic  # noqa: E402
from viettts_b200.engine import Engine  # noqa: E402

HOP = 256


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                           text=True, timeout=30)
        name, power = [x.strip() for x in r.stdout.strip().split(",")]
        return {"name": name, "power_limit": power}
    except Exception as e:  # noqa: BLE001
        return {"error": str(e)}


def sentence(seed, L):
    t = np.asarray(synthetic.utterance(seed, L, None)[0], np.int32)
    t[0] = t[-1] = C.SIL_INDEX
    return t


def text_of(eng, seconds, n_sent, seed):
    """n_sent sentences (token rows) whose planned frames add up to about `seconds`"""
    L = 40
    for _ in range(3):
        sents = [sentence(seed + i, L) for i in range(n_sent)]
        tok = np.zeros((n_sent, L), np.int32)
        for i, s in enumerate(sents):
            tok[i] = s
        frames = int(eng.tts_plan(tok)[3].sum())
        L = int(np.clip(round(L * seconds * C.SAMPLE_RATE / HOP / max(frames, 1)), 6, 2000))
    return [sentence(seed + i, L) for i in range(n_sent)]


def whole(sents):
    """the text as one row: the sentences back to back, one silence token between them"""
    return np.concatenate([sents[0]] + [s[1:] for s in sents[1:]]).astype(np.int32)


def pad(rows):
    tok = np.zeros((len(rows), max(r.size for r in rows)), np.int32)
    for i, r in enumerate(rows):
        tok[i, : r.size] = r
    return tok, np.array([r.size for r in rows], np.int32)


def timed(fn, reps):
    ts = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append((time.perf_counter() - t0) * 1e3)
    return ts


def substages(eng, fn):
    eng.substages(True)
    fn()
    d = eng.substages(False)
    return {k: float(d.get(k, 0.0)) for k in d}


def one_vs_joined(eng, texts, reps):
    rows = [whole(t) for t in texts]
    tok, lens = pad(rows)
    eng.tts(tok, lens)
    eng.tts_joined(texts)                               # warm-up of both shapes
    a, b = [], []
    for _ in range(reps):                               # alternated
        a += timed(lambda: eng.tts(tok, lens), 1)
        b += timed(lambda: eng.tts_joined(texts), 1)
    frames_one = [int(x) for x in eng.tts_plan(tok, lens)[3]]
    frames_joined = [int(w.size // HOP) for w in eng.tts_joined(texts)[0]]
    return {"texts": len(texts), "sentences": sum(len(t) for t in texts), "tokens_one_row": [int(r.size) for r in rows],
            "frames_one_row": frames_one, "frames_joined": frames_joined,
            "tts_one_row_ms": {"median": float(np.median(a)), "min": float(np.min(a)), "max": float(np.max(a))},
            "tts_joined_ms": {"median": float(np.median(b)), "min": float(np.min(b)), "max": float(np.max(b))},
            "speedup_median": float(np.median(a) / np.median(b)),
            "substages_one_row_ms": substages(eng, lambda: eng.tts(tok, lens)),
            "substages_joined_last_launch_ms": substages(eng, lambda: eng.tts_joined(texts))}


def equality(eng, texts):
    """tts_joined == mel2wave of the host-joined predict_mel rows"""
    rows = [r for t in texts for r in t]
    tok, lens = pad(rows)
    _, frames, nf, ne = eng.tts_plan(tok, lens)
    mel = eng.predict_mel(tok, frames, lengths=lens, n_frames=nf)
    bounds = np.cumsum([0] + [len(t) for t in texts])
    counts = [int(ne[a:b].sum()) for a, b in zip(bounds, bounds[1:])]
    joined = np.zeros((len(texts), max(counts), C.MEL_DIM), np.float32)
    for g, (a, b) in enumerate(zip(bounds, bounds[1:])):
        joined[g, : counts[g]] = np.concatenate([mel[r, : ne[r]] for r in range(a, b)])
    want = eng.mel2wave(joined, n_frames=np.array(counts, np.int32))
    got = eng.tts_joined(texts)[0]
    return all(np.array_equal(got[g], want[g, : counts[g] * HOP]) for g in range(len(texts)))


def stream(eng, sents):
    """one slot: every sentence appended at once against one begin per sentence"""
    res = {}
    n_max = max(int(eng.tts_plan(s[None])[2][0]) for s in sents)
    total = sum(int(eng.tts_plan(s[None])[3][0]) for s in sents)
    with eng.open_tts_stream(1, 16, n_max + 16, 1024, max_joined_frames=total + 16) as ts:
        for kind in ("append", "begin"):
            steps = idle = 0
            queue = list(sents)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            if kind == "append":
                ts.begin(0, queue.pop(0), more=True)
                for i, s in enumerate(queue):
                    ts.append(0, s, more=i + 1 < len(queue))
                queue = []
            else:
                ts.begin(0, queue.pop(0))
            samples = 0
            while ts.busy().any() or queue:
                if not ts.busy()[0] and queue:
                    ts.begin(0, queue.pop(0))
                w = ts.step()[0]
                steps += 1
                samples += w.size
                idle += int(w.size == 0 and (bool(queue) or bool(ts._queue[0])))
            torch.cuda.synchronize()
            res[kind] = {"steps": steps, "steps_with_nothing_out_while_text_queued": idle, "samples": int(samples),
                         "wall_ms": (time.perf_counter() - t0) * 1e3}
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", type=Path)
    ap.add_argument("--reps", type=int, default=7)
    args = ap.parse_args()
    eng = Engine(0)
    eng.load_hifigan(synthetic.hifigan_params(1))
    eng.load_acoustic(synthetic.acoustic_ckpt(2))
    eng.load_duration(synthetic.duration_ckpt(1234))
    eng.set_precision("bf16x3")
    res = {"card": card(), "precision": "bf16x3", "weights": "synthetic (hifigan 1, acoustic 2, duration 1234)"}
    long_text = text_of(eng, 90.0, 20, 1000)
    res["one_90s_text_of_20_sentences"] = one_vs_joined(eng, [long_text], args.reps)
    eight = [text_of(eng, 20.0, 5, 2000 + 50 * i) for i in range(8)]
    res["eight_20s_texts"] = one_vs_joined(eng, eight, args.reps)
    res["equal_to_host_joined_mel"] = {"90s": equality(eng, [long_text]), "8x20s": equality(eng, eight)}
    eng.set_fused_pairs(False)
    res["stream_10_sentences"] = stream(eng, [sentence(3000 + i, 30) for i in range(10)])
    eng.set_fused_pairs(True)
    print(json.dumps(res))
    if args.out:
        args.out.parent.mkdir(parents=True, exist_ok=True)
        args.out.write_text(json.dumps(res, indent=1) + "\n")


if __name__ == "__main__":
    main()
