"""Streaming text to speech (Engine.open_tts_stream / open_acoustic_stream) against the one-call paths.

    python scripts/bench_tts_stream.py [--out FILE.json]

  * time to first and to last audio (wall clock from the call / begin) for one ~5 s and one ~30 s utterance: TTS stream
    (F = 16) against Engine.tts;
  * acoustic push device time (CUDA events around push_device, steady state, every slot open) for S in {1, 32, 128} x
    F in {8, 16, 32}, per decoder frame, beside the one-shot scan's per-frame time at B = S (sub-stage events of
    predict_mel);
  * the C5 workload (256 utterances, 50-300 phonemes) through S = 128 slots refilled as they close, acoustic stream
    feeding a vocoder stream: samples/s and p50 / p99 latency of first audio and of completion per utterance (all
    utterances queued at t = 0), against Engine.synthesize_many;
  * the slowest push of that run against the F x 16 ms of audio one push produces.

Synthetic weights, bf16x3.  The card name and power limit are read (nvidia-smi, read-only) in the same run.  Prints one
JSON object; `--out` also writes it."""
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
from viettts_b200.engine import STREAM_BEGIN, STREAM_END, Engine  # noqa: E402

HOP = 256


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                           timeout=30)
        name, power = [x.strip() for x in r.stdout.strip().split(",")]
        return {"name": name, "power_limit": power}
    except Exception as e:  # noqa: BLE001
        return {"error": str(e)}


def tokens_for_frames(eng, target, seed):
    """token row whose planned frame count is close to `target` (synthetic duration weights)"""
    L = 100
    for _ in range(3):
        tk = np.asarray(synthetic.utterance(seed, L, None)[0], np.int32)
        n = int(eng.tts_plan(tk[None])[2][0])
        L = int(np.clip(round(L * target / max(n, 1)), 8, 1000))
    tk = np.asarray(synthetic.utterance(seed, L, None)[0], np.int32)
    return tk, int(eng.tts_plan(tk[None])[2][0])


def latency(eng, seconds, seed):
    tk, n = tokens_for_frames(eng, int(seconds * C.SAMPLE_RATE / HOP), seed)
    res = {"target_s": seconds, "frames": n, "tokens": int(tk.size)}
    eng.tts(tk[None])                                   # warm-up
    t0 = time.perf_counter()
    eng.tts(tk[None])
    res["tts_ms"] = (time.perf_counter() - t0) * 1e3
    with eng.open_tts_stream(1, 16, n + 64, 1024) as ts:
        for rep in range(2):                            # the first run warms up
            t0 = time.perf_counter()
            ts.begin(0, tk)
            first, steps, slow = None, 0, 0.0
            while ts.busy().any():
                s0 = time.perf_counter()
                w = ts.step()[0]
                slow = max(slow, time.perf_counter() - s0)
                steps += 1
                if first is None and w.size:
                    first = time.perf_counter() - t0
            last = time.perf_counter() - t0
        res.update(stream_first_audio_ms=first * 1e3, stream_last_audio_ms=last * 1e3, stream_steps=steps, slowest_step_ms=slow * 1e3,
                   audio_per_step_ms=16 * HOP / C.SAMPLE_RATE * 1e3)
    return res


def push_times(eng, S, F):
    dev = torch.device("cuda", 0)
    n = 600
    tok, dur = zip(*[synthetic.utterance(900 + s, 120, n / 62.5) for s in range(S)])
    tok = np.asarray(tok, np.int32)
    dur = (np.concatenate(dur) * np.float32(C.SAMPLE_RATE)) / np.float32(HOP)
    res = {"S": S, "F": F}
    with eng.open_acoustic_stream(S, F, n, 128, seed=3) as st:
        st.begin(np.arange(S), tok, dur, n_frames=[n] * S)
        out = torch.empty((S, F + st.lookahead, C.MEL_DIM), device=dev)
        for _ in range(2):
            st.push_device(out)
        k = min(10, (n - 3 * F) // F)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(k):
            st.push_device(out)
        b.record()
        b.synchronize()
        res["push_ms"] = a.elapsed_time(b) / k
    res["push_us_per_frame"] = res["push_ms"] * 1e3 / F
    eng.substages(True)
    eng.predict_mel(tok, dur, n_frames=[n] * S, seed=3)
    sub = eng.substages(False)
    res["one_shot_scan_us_per_frame"] = sub.get("acoustic.decoder_scan", float("nan")) * 1e3 / n
    return res


def c5(eng, S=128, F=16):
    rng = np.random.default_rng(77)
    utts = []
    for i in range(256):
        L = int(rng.integers(50, 301))
        tk, d = synthetic.utterance(5000 + i, L, None)
        d = (np.asarray(d, np.float32) * np.float32(C.SAMPLE_RATE)) / np.float32(HOP)
        utts.append((np.asarray(tk, np.int32), d[0], int(np.sum(d, dtype=np.float32))))
    total = sum(u[2] for u in utts) * HOP
    eng.synthesize_many([(t, d) for t, d, _ in utts[:8]])          # warm-up
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    eng.synthesize_many([(t, d) for t, d, _ in utts])
    base_s = time.perf_counter() - t0
    dev = torch.device("cuda", 0)
    nmax = max(u[2] for u in utts)
    with eng.open_acoustic_stream(S, F, nmax, 320) as ac, eng.open_vocoder_stream(S, F + ac.lookahead) as voc:
        mel = torch.zeros((S, F + ac.lookahead, C.MEL_DIM), device=dev)
        wav = torch.zeros((S, voc.wav_ld), device=dev)
        queue, owner = list(range(256)), {}
        first, done, got = {}, {}, 0
        fresh = np.zeros(S, bool)
        slow = 0.0
        t0 = time.perf_counter()
        while queue or ac.open.any():
            free = [int(s) for s in np.flatnonzero(~ac.open)][: len(queue)]
            if free:
                ids = [queue.pop(0) for _ in free]
                L = max(utts[i][0].size for i in ids)
                tk = np.zeros((len(ids), L), np.int32)
                du = np.zeros((len(ids), L), np.float32)
                for r, i in enumerate(ids):
                    tk[r, : utts[i][0].size] = utts[i][0]
                    du[r, : utts[i][0].size] = utts[i][1]
                ac.begin(free, tk, du, lengths=[utts[i][0].size for i in ids], n_frames=[utts[i][2] for i in ids])
                for s, i in zip(free, ids):
                    owner[s] = i
                    fresh[s] = True
            s0 = time.perf_counter()
            active = ac.open.copy()
            n_out = ac.push_device(mel)
            flags = (fresh & active).astype(np.uint8) * STREAM_BEGIN | (active & ~ac.open).astype(np.uint8) * STREAM_END
            n_wav = voc.push_device(mel, n_out, flags, wav)
            w = wav.cpu()
            now = time.perf_counter()
            slow = max(slow, now - s0)
            fresh &= ~active
            for s in np.flatnonzero(active):
                i = owner[int(s)]
                got += int(n_wav[s]) * HOP
                if n_wav[s] and i not in first:
                    first[i] = now - t0
                if not ac.open[s]:
                    done[i] = now - t0
        stream_s = time.perf_counter() - t0
        del w
    assert got == total, (got, total)
    f = np.array([first[i] for i in range(256)]) * 1e3
    d = np.array([done[i] for i in range(256)]) * 1e3
    return {"utterances": 256, "samples": total, "S": S, "F": F,
            "synthesize_many_s": base_s, "synthesize_many_samples_per_s": total / base_s,
            "stream_s": stream_s, "stream_samples_per_s": total / stream_s,
            "first_audio_ms_p50": float(np.percentile(f, 50)), "first_audio_ms_p99": float(np.percentile(f, 99)),
            "completion_ms_p50": float(np.percentile(d, 50)), "completion_ms_p99": float(np.percentile(d, 99)),
            "slowest_push_ms": slow * 1e3, "audio_per_push_ms": F * HOP / C.SAMPLE_RATE * 1e3}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    eng = Engine(0)
    eng.load_acoustic(synthetic.acoustic_ckpt(1234))
    eng.load_hifigan(synthetic.hifigan_params(1234))
    eng.load_duration(synthetic.duration_ckpt(1234))
    eng.set_precision("bf16x3")
    res = {"card": card(), "precision": "bf16x3"}
    res["latency"] = [latency(eng, 5.0, 11), latency(eng, 30.0, 12)]
    res["push"] = [push_times(eng, S, F) for S in (1, 32, 128) for F in (8, 16, 32)]
    res["c5"] = c5(eng)
    s = json.dumps(res, indent=1)
    print(s)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(s + "\n")
    eng.close()


if __name__ == "__main__":
    main()
