"""Streaming generator (Engine.open_vocoder_stream) against the existing ways to vocode the same audio.

    python scripts/bench_stream.py [--precision bf16x3] [--out FILE.json]

  * S = 1 slot, F in {4, 8, 16, 32} frames per push: device time per steady-state push (CUDA events around
    push_device) and time to first audio (wall clock from BEGIN until a push returns samples, host API), against
    Engine.mel2wave_stream at the same chunk size (per-chunk wall time and its first chunk).
  * S in {8, 32, 128} slots x 16-frame pushes in steady state: samples/s against one-shot mel2wave of the same audio
    as one batch (hifigan_forward, B = S).

Synthetic weights.  The card name and power limit are read (nvidia-smi, read-only) in the same run.  Prints one JSON
object; `--out` also writes it."""
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
from viettts_b200 import synthetic  # noqa: E402
from viettts_b200.engine import Engine  # noqa: E402

HOP = 256


def card():
    q = "name,power.limit"
    try:
        r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30)
        name, power = [x.strip() for x in r.stdout.strip().split(",")]
        return {"name": name, "power_limit": power}
    except Exception as e:  # noqa: BLE001
        return {"error": str(e)}


def device_ms(fn, n):
    st = torch.cuda.current_stream()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(st)
    for _ in range(n):
        fn()
    b.record(st)
    b.synchronize()
    return a.elapsed_time(b) / n


def single_slot(eng, F, pushes=40):
    dev = torch.device("cuda", 0)
    T = F * pushes
    mel = synthetic.mel_input(1, 1, T)
    res = {"F": F}
    with eng.open_vocoder_stream(1, F) as vs:
        # time to first audio, host API: BEGIN, then pushes until samples come back
        t0 = time.perf_counter()
        for i in range(pushes):
            got = vs.push(mel[:, i * F:(i + 1) * F], np.array([F], np.int32), begin=[i == 0])
            if got[0].size:
                break
        res["stream_first_audio_ms"] = (time.perf_counter() - t0) * 1e3
        res["stream_first_audio_pushes"] = i + 1
        # steady-state device time per push
        mel_t = torch.from_numpy(mel[:, :F].copy()).to(dev)
        out_t = torch.empty((1, vs.wav_ld), dtype=torch.float32, device=dev)
        n, fl = np.array([F], np.int32), np.zeros(1, np.uint8)
        vs.push_device(mel_t, n, np.ones(1, np.uint8), out_t)
        for _ in range(20):
            vs.push_device(mel_t, n, fl, out_t)
        res["stream_push_device_ms"] = device_ms(lambda: vs.push_device(mel_t, n, fl, out_t), 50)
        t1 = time.perf_counter()
        for _ in range(20):
            vs.push(mel[:, :F], n)
        res["stream_push_host_ms"] = (time.perf_counter() - t1) * 1e3 / 20
    # recomputed-halo chunking at the same chunk size
    gen = eng.mel2wave_stream(mel[0], chunk_frames=F)
    t0 = time.perf_counter()
    next(gen)
    res["mel2wave_stream_first_audio_ms"] = (time.perf_counter() - t0) * 1e3
    t1 = time.perf_counter()
    k = sum(1 for _ in gen)
    res["mel2wave_stream_chunk_ms"] = (time.perf_counter() - t1) * 1e3 / max(k, 1)
    res["stream_speedup_per_chunk"] = res["mel2wave_stream_chunk_ms"] / res["stream_push_host_ms"]
    return res


def many_slots(eng, S, F=16, pushes=20):
    dev = torch.device("cuda", 0)
    res = {"S": S, "F": F}
    mel = synthetic.mel_input(2, S, F)
    with eng.open_vocoder_stream(S, F) as vs:
        mel_t = torch.from_numpy(mel).to(dev)
        out_t = torch.empty((S, vs.wav_ld), dtype=torch.float32, device=dev)
        n, fl = np.full(S, F, np.int32), np.zeros(S, np.uint8)
        vs.push_device(mel_t, n, np.ones(S, np.uint8), out_t)
        for _ in range(5):
            vs.push_device(mel_t, n, fl, out_t)
        ms = device_ms(lambda: vs.push_device(mel_t, n, fl, out_t), pushes)
    res["stream_push_ms"] = ms
    res["stream_samples_per_s"] = S * F * HOP / (ms * 1e-3)
    T = F * pushes
    mel_b = torch.from_numpy(synthetic.mel_input(3, S, T)).to(dev)
    out = torch.empty((S, T * HOP), dtype=torch.float32, device=dev)
    eng.hifigan_forward(mel_b, out=out)
    ms1 = device_ms(lambda: eng.hifigan_forward(mel_b, out=out), 3)
    res["one_shot_T"] = T
    res["one_shot_ms"] = ms1
    res["one_shot_samples_per_s"] = S * T * HOP / (ms1 * 1e-3)
    res["stream_over_one_shot"] = res["stream_samples_per_s"] / res["one_shot_samples_per_s"]
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--precision", default="bf16x3")
    ap.add_argument("--out", type=Path, default=None)
    a = ap.parse_args()
    eng = Engine(0)
    eng.load_hifigan(synthetic.hifigan_params(1234))
    eng.set_precision(a.precision)
    res = {"card": card(), "precision": a.precision, "lookahead_frames": int(eng.lib.vtts_vocoder_stream_lookahead()),
           "single_slot": [single_slot(eng, F) for F in (4, 8, 16, 32)],
           "many_slots": [many_slots(eng, S) for S in (8, 32, 128)]}
    eng.close()
    text = json.dumps(res, indent=1)
    print(text)
    if a.out:
        a.out.parent.mkdir(parents=True, exist_ok=True)
        a.out.write_text(text + "\n")


if __name__ == "__main__":
    main()
