#!/usr/bin/env python
"""Speed and waveform difference of the fast fp16 generator mode against bf16x3, in one process on one GPU.

    python scripts/bench_fp16.py [--rounds 2] [--steps 10] [--warmup 3] [--out FILE.json]

The workload is bench.py's: synthetic 100-phoneme / 5 s utterances (312 mel frames) through the acoustic model and the
generator, batches of 1, 8, 32 and 128, inputs resident on the device, CUDA-event timing (bench.time_jobs).  For every
batch the two modes run alternately, `--rounds` times each, so that drifting clocks and other tenants of the host hit
both.  The acoustic model runs bf16x3 in both modes (the fp16 mode covers the generator only), so the step difference is
the generator's.  At B = 32 the waveforms of the two modes are compared (same inputs, same dropout stream).  The card's
name and power limit are read (nvidia-smi, read-only) in the same run.  Prints one JSON object; `--out` also writes it.
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

REPO = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(REPO))

from bench import Job, make_batch, time_jobs  # noqa: E402
from viettts_b200 import synthetic  # noqa: E402

BATCHES = (1, 8, 32, 128)
MODES = ("bf16x3", "fp16")


def card():
    q = "name,power.limit,clocks.max.sm,driver_version"
    try:
        r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30)
        vals = [v.strip() for v in r.stdout.strip().split(",")]
        return dict(zip(q.split(","), vals)) if r.returncode == 0 and len(vals) == 4 else dict(error=r.stderr.strip())
    except Exception as e:          # noqa: BLE001
        return dict(error=str(e))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", type=Path, default=None)
    args = ap.parse_args()

    import torch
    from viettts_b200.engine import Engine
    if not torch.cuda.is_available():
        raise SystemExit("bench_fp16: no CUDA device")
    dev = torch.device("cuda", 0)
    eng = Engine(0)
    eng.load_hifigan(synthetic.hifigan_params(1234))
    eng.load_acoustic(synthetic.acoustic_ckpt(1234))
    jobs = {}
    for B in BATCHES:
        tokens, durs, nfs = make_batch(B, 100, 5.0, 0)
        jobs[B] = Job(eng, dev, tokens, durs, nfs, 0xC0FFEE)

    gpu = card()
    runs = {str(B): {m: [] for m in MODES} for B in BATCHES}
    t0 = time.perf_counter()
    for rnd in range(args.rounds):
        for B in BATCHES:
            for m in MODES:
                eng.set_precision(m)
                ms, ac, hg = time_jobs([jobs[B]], args.steps, args.warmup, lambda: None)
                runs[str(B)][m].append(dict(round=rnd, ms_per_step=ms, acoustic_ms=ac, generator_ms=hg,
                                            samples_per_s=jobs[B].samples / (ms / 1e3)))
    wall = time.perf_counter() - t0

    summary = {}
    for B in BATCHES:
        r = runs[str(B)]
        s = {m: dict(ms_per_step=[x["ms_per_step"] for x in r[m]], generator_ms=[x["generator_ms"] for x in r[m]],
                     samples_per_s=[x["samples_per_s"] for x in r[m]]) for m in MODES}
        g16, g3 = s["fp16"]["generator_ms"], s["bf16x3"]["generator_ms"]
        spread = max(max(g16) - min(g16), max(g3) - min(g3))
        s["generator_speedup"] = float(np.mean(g3) / np.mean(g16))
        s["generator_ms_saved"] = float(np.mean(g3) - np.mean(g16))
        s["generator_round_spread_ms"] = float(spread)
        s["faster_than_spread"] = bool(max(g16) < min(g3) and np.mean(g3) - np.mean(g16) > spread)
        s["step_speedup"] = float(np.mean(s["bf16x3"]["ms_per_step"]) / np.mean(s["fp16"]["ms_per_step"]))
        summary[str(B)] = s

    # waveform difference of the two modes at B = 32 (same mel: the acoustic model is bf16x3 in both)
    j = jobs[32]
    out = {}
    for m in MODES:
        eng.set_precision(m)
        j.step()
        torch.cuda.synchronize()
        out[m] = (j.mel_t.cpu().numpy().copy(), j.wav_t.cpu().numpy().astype(np.float64))
    d = out["fp16"][1] - out["bf16x3"][1]
    valid = np.zeros_like(d, dtype=bool)
    for b, n in enumerate(j.nfs):
        valid[b, : int(n) * 256] = True
    sig_rms = float(np.sqrt(np.mean(out["bf16x3"][1][valid] ** 2)))
    diff = dict(batch=32, linf=float(np.abs(d).max()), rms=float(np.sqrt(np.mean(d[valid] ** 2))), signal_rms=sig_rms,
                mel_bit_identical=bool(np.array_equal(out["fp16"][0], out["bf16x3"][0])),
                note="fp16 minus bf16x3 waveform over the valid samples; bf16x3 is within 1e-4 of float64, so this is the fp16 "
                     "mode's own error to that accuracy")
    eng.close()

    res = dict(what="fast fp16 generator mode vs bf16x3 (default), alternating in one process",
               gpu=gpu, torch_device=torch.cuda.get_device_name(0),
               workload="bench.py workload: synthetic 100-phoneme / 5 s utterances (312 mel frames, 79 872 samples), acoustic model + "
                        "generator per step, device-resident inputs, CUDA events; the acoustic model runs bf16x3 in both modes",
               rounds=args.rounds, steps=args.steps, warmup=args.warmup, wall_s=wall,
               weights="synthetic (seed 1234)", runs=runs, summary=summary, waveform_fp16_vs_bf16x3=diff)
    text = json.dumps(res, indent=1)
    print(text)
    if args.out is not None:
        args.out.parent.mkdir(parents=True, exist_ok=True)
        args.out.write_text(text + "\n")


if __name__ == "__main__":
    main()
