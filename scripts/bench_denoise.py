"""Bias denoiser (Engine.denoise_forward, Engine.open_tts_stream(denoise=)) against the generator.

    python scripts/bench_denoise.py [--out FILE.json]

  * device time (CUDA events, 20 calls after a warm-up) of denoising the 32 x 5 s batch (B = 32, 313 frames = 80128
    samples at 16 kHz), beside the generator's time for that batch in the same process;
  * TTS stream step time (host clock around step(), which ends in the step's one synchronisation) at S in {1, 32},
    F = 16, with and without denoise=0.1, the two streams stepped alternately in one process;
  * decoder frames scanned until a slot's first audio, with and without denoising (S = 1, F = 16).

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
from viettts_b200 import synthetic  # noqa: E402
from viettts_b200.engine import Engine  # noqa: E402

HOP = 256
STRENGTH = 0.1


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                           timeout=30)
        name, power = [x.strip() for x in r.stdout.strip().split(",")]
        return {"name": name, "power_limit": power}
    except Exception as e:  # noqa: BLE001
        return {"error": str(e)}


def device_ms(fn, reps=20):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def batch(eng, B=32, T=313):
    dev = torch.device("cuda", 0)
    mel = torch.from_numpy(synthetic.mel_input(7, B, T)).to(dev)
    wav = torch.empty((B, T * HOP), device=dev)
    res = {"B": B, "frames": T, "samples_16k": T * HOP, "generator_ms": device_ms(lambda: eng.hifigan_forward(mel, out=wav), reps=5)}
    eng.hifigan_forward(mel, out=wav)
    bias = torch.from_numpy(eng.denoiser_bias()).to(dev)
    out = torch.empty_like(wav)
    ms = device_ms(lambda: eng.denoise_forward(wav, STRENGTH, bias_t=bias, out=out))
    frames = B * (T * HOP // HOP + 1)
    res["denoise"] = {"strength": STRENGTH, "ms": ms, "stft_frames": frames, "us_per_frame": ms * 1e3 / frames,
                      "share_of_generator_time": ms / res["generator_ms"]}
    return res


def tts_steps(eng, S, F=16, reps=2):
    tok = [np.asarray(synthetic.utterance(300 + s, 120, None)[0], np.int32) for s in range(S)]
    res = {"S": S, "F": F}
    times = {"plain": [], "denoise": []}
    with eng.open_tts_stream(S, F, 4000, 1024) as a, eng.open_tts_stream(S, F, 4000, 1024, denoise=STRENGTH) as b:
        for rep in range(reps + 1):            # the first run warms up
            for s in range(S):
                a.begin(s, tok[s])
                b.begin(s, tok[s])
            while a.busy().any() or b.busy().any():
                for key, ts in (("plain", a), ("denoise", b)):
                    if ts.busy().any():
                        t0 = time.perf_counter()
                        ts.step()
                        if rep:
                            times[key].append(time.perf_counter() - t0)
    for key, t in times.items():
        t = np.array(t) * 1e3
        res[f"step_ms_{key}"] = {"steps": int(t.size), "mean": float(t.mean()), "p50": float(np.percentile(t, 50)),
                                 "p90": float(np.percentile(t, 90))}
    res["mean_step_overhead_ms"] = res["step_ms_denoise"]["mean"] - res["step_ms_plain"]["mean"]
    return res


def first_audio(eng, F=16):
    """decoder frames scanned (F per step) up to and including the step that returns a slot's first samples"""
    tok = np.asarray(synthetic.utterance(300, 120, None)[0], np.int32)
    res = {"F": F}
    for key, kw in (("plain", {}), ("denoise", {"denoise": STRENGTH})):
        with eng.open_tts_stream(1, F, 4000, 1024, **kw) as ts:
            n_emit = ts.begin(0, tok)
            steps = 0
            while ts.busy().any():
                steps += 1
                if ts.step()[0].size:
                    break
            res[key] = {"steps": steps, "frames_scanned": min(steps * F, n_emit + 10), "utterance_frames": n_emit}
            while ts.busy().any():
                ts.step()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    eng = Engine(0)
    eng.load_acoustic(synthetic.acoustic_ckpt(1234))
    eng.load_hifigan(synthetic.hifigan_params(1234))
    eng.load_duration(synthetic.duration_ckpt(1234))
    eng.set_precision("bf16x3")
    res = {"card": card(), "precision": "bf16x3", "batch": batch(eng), "tts_stream": [tts_steps(eng, S) for S in (1, 32)],
           "first_audio": first_audio(eng)}
    s = json.dumps(res, indent=1)
    print(s)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(s + "\n")
    eng.close()


if __name__ == "__main__":
    main()
