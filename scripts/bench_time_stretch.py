"""Time stretcher (Engine.time_stretch_forward, Engine.open_tts_stream(tempo=)) against the generator.

    python scripts/bench_time_stretch.py [--out FILE.json]

  * device time (CUDA events, 20 calls after a warm-up) of stretching the 32 x 5 s batch (B = 32, 313 frames = 80128
    samples at 16 kHz) at tempo 0.75, 1.25 and 2, beside the generator's time for that batch in the same process;
  * each kernel's share of that time (torch.profiler with CUDA activities, 5 calls, in a pass of its own);
  * one 3-minute row (2 880 000 samples) at tempo 1.25, where the sequential phase kernel dominates;
  * TTS stream step time (host clock around step(), which ends in the step's one synchronisation) at S in {1, 32},
    F = 16, with and without tempo=1.25, the two streams stepped alternately in one process.

Synthetic weights, bf16x3.  The card name and power limit are read (nvidia-smi, read-only) in the same run.  Prints one
JSON object; `--out` also writes it."""
from __future__ import annotations

import argparse
import json
import sys
import time
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
sys.path.insert(0, str(Path(__file__).resolve().parent))
from bench_denoise import HOP, card, device_ms  # noqa: E402
from bench_pitch import kernel_split  # noqa: E402
from viettts_b200 import synthetic  # noqa: E402
from viettts_b200.engine import Engine  # noqa: E402

TEMPOS = (0.75, 1.25, 2.0)
STREAM_TEMPO = 1.25


def stretch(eng, x, tempo):
    out = torch.empty((x.shape[0], eng.time_stretch_length(x.shape[1], tempo)), device=x.device)
    fn = lambda: eng.time_stretch_forward(x, tempo, out=out)   # noqa: E731
    ms = device_ms(fn)
    split = kernel_split(fn)
    frames = x.shape[0] * (out.shape[1] // HOP + 1)
    return {"tempo": tempo, "ms": ms, "synthesis_frames": frames, "us_per_frame": ms * 1e3 / frames, "kernel_ms": split,
            "phase_share": split.get("pitch_phase_kernel", 0.0) / max(sum(split.values()), 1e-9)}


def batch(eng, B=32, T=313):
    dev = torch.device("cuda", 0)
    mel = torch.from_numpy(synthetic.mel_input(7, B, T)).to(dev)
    wav = torch.empty((B, T * HOP), device=dev)
    res = {"B": B, "frames": T, "samples_16k": T * HOP, "generator_ms": device_ms(lambda: eng.hifigan_forward(mel, out=wav), reps=5)}
    eng.hifigan_forward(mel, out=wav)
    res["time_stretch"] = []
    for a in TEMPOS:
        r = stretch(eng, wav, a)
        r["share_of_generator_time"] = r["ms"] / res["generator_ms"]
        res["time_stretch"].append(r)
    return res


def long_row(eng, n=3 * 60 * 16000):
    rng = np.random.default_rng(11)
    t = np.arange(n) / 16000
    x = torch.from_numpy((0.3 * np.sin(2 * np.pi * 180 * t) + 0.02 * rng.standard_normal(n)).astype(np.float32)[None]).cuda()
    return {"samples": n, **stretch(eng, x, STREAM_TEMPO)}


def tts_steps(eng, S, F=16, reps=2):
    tok = [np.asarray(synthetic.utterance(300 + s, 120, None)[0], np.int32) for s in range(S)]
    res = {"S": S, "F": F, "tempo": STREAM_TEMPO}
    times = {"plain": [], "tempo": []}
    with eng.open_tts_stream(S, F, 4000, 1024) as a, eng.open_tts_stream(S, F, 4000, 1024, tempo=STREAM_TEMPO) as b:
        for rep in range(reps + 1):            # the first run warms up
            for s in range(S):
                a.begin(s, tok[s])
                b.begin(s, tok[s])
            while a.busy().any() or b.busy().any():
                for key, ts in (("plain", a), ("tempo", b)):
                    if ts.busy().any():
                        t0 = time.perf_counter()
                        ts.step()
                        if rep:
                            times[key].append(time.perf_counter() - t0)
    for key, t in times.items():
        t = np.array(t) * 1e3
        res[f"step_ms_{key}"] = {"steps": int(t.size), "mean": float(t.mean()), "p50": float(np.percentile(t, 50)),
                                 "p90": float(np.percentile(t, 90))}
    res["mean_step_overhead_ms"] = res["step_ms_tempo"]["mean"] - res["step_ms_plain"]["mean"]
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
    res = {"card": card(), "precision": "bf16x3", "batch": batch(eng), "three_minute_row": long_row(eng),
           "tts_stream": [tts_steps(eng, S) for S in (1, 32)]}
    s = json.dumps(res, indent=1)
    print(s)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(s + "\n")
    eng.close()


if __name__ == "__main__":
    main()
