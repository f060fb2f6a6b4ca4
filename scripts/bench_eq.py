"""Equalizer (Engine.equalize_forward, open_tts_stream(eq=)) against the generator.

    python scripts/bench_eq.py [--out FILE.json]

  * device time (CUDA events, 20 calls after a warm-up) of equalizing the 32 x 5 s batch (B = 32, 313 frames = 80128
    samples at 16 kHz, and the same batch resampled to 48 kHz) through the 5-section voice EQ, beside the generator's
    time for that batch in the same process; the telephone preset on the batch resampled to 8 kHz; the 8-section worst
    case at 48 kHz;
  * one 3-minute row at 16 kHz through the voice EQ, where the per-row block chain dominates;
  * TTS stream step time (host clock around step(), which ends in the step's one synchronisation) at S in {1, 32},
    F = 16, with and without eq=VOICE, the two streams stepped alternately in one process.

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
from bench_denoise import card, device_ms  # noqa: E402
from viettts_b200 import synthetic  # noqa: E402
from viettts_b200.engine import Engine, eq_sections  # noqa: E402

HOP = 256
VOICE = "hp:80:4,ls:200:-2,pk:3000:1:3,hs:6000:2"
WORST = "hp:60:8,lp:7000:8"


def batch(eng, B=32, T=313):
    dev = torch.device("cuda", 0)
    mel = torch.from_numpy(synthetic.mel_input(7, B, T)).to(dev)
    wav = torch.empty((B, T * HOP), device=dev)
    res = {"B": B, "frames": T, "samples_16k": T * HOP, "generator_ms": device_ms(lambda: eng.hifigan_forward(mel, out=wav), reps=5)}
    eng.hifigan_forward(mel, out=wav)
    for name, spec, rate in (("voice_16k", VOICE, 16000), ("voice_48k", VOICE, 48000), ("telephone_8k", "telephone", 8000),
                             ("worst_48k", WORST, 48000)):
        x = wav if rate == 16000 else eng.resample_forward(wav, rate)
        sos = eq_sections(spec, rate)
        y = torch.empty_like(x)
        ms = device_ms(lambda: eng.equalize_forward(x, sos, rate, out=y))
        res[name] = {"spec": spec, "rate": rate, "sections": int(sos.shape[0]), "samples": int(x.shape[1]), "eq_ms": ms,
                     "share_of_generator_time": ms / res["generator_ms"], "input_GB_per_s": x.numel() * 4 / (ms * 1e-3) / 1e9,
                     "section_samples_per_ns": x.numel() * sos.shape[0] / (ms * 1e6)}
    return res


def long_row(eng, seconds=180, rate=16000):
    dev = torch.device("cuda", 0)
    x = (0.3 * torch.randn((1, seconds * rate), generator=torch.Generator().manual_seed(3))).to(dev)
    y = torch.empty_like(x)
    sos = eq_sections(VOICE, rate)
    return {"seconds": seconds, "rate": rate, "spec": VOICE, "eq_ms": device_ms(lambda: eng.equalize_forward(x, sos, rate, out=y), reps=10)}


def tts_steps(eng, S, F=16, reps=2):
    tok = [np.asarray(synthetic.utterance(300 + s, 120, None)[0], np.int32) for s in range(S)]
    res = {"S": S, "F": F}
    times = {"plain": [], "eq": []}
    with eng.open_tts_stream(S, F, 4000, 1024) as a, eng.open_tts_stream(S, F, 4000, 1024, eq=VOICE) as b:
        for rep in range(reps + 1):            # the first run warms up
            for s in range(S):
                a.begin(s, tok[s])
                b.begin(s, tok[s])
            while a.busy().any() or b.busy().any():
                for key, ts in (("plain", a), ("eq", b)):
                    if ts.busy().any():
                        t0 = time.perf_counter()
                        ts.step()
                        if rep:
                            times[key].append(time.perf_counter() - t0)
    for key, t in times.items():
        t = np.array(t) * 1e3
        res[f"step_ms_{key}"] = {"steps": int(t.size), "mean": float(t.mean()), "p50": float(np.percentile(t, 50)),
                                 "p90": float(np.percentile(t, 90))}
    res["mean_step_overhead_ms"] = res["step_ms_eq"]["mean"] - res["step_ms_plain"]["mean"]
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
    res = {"card": card(), "precision": "bf16x3", "batch": batch(eng), "long_row": long_row(eng),
           "tts_stream": [tts_steps(eng, S) for S in (1, 32)]}
    s = json.dumps(res, indent=1)
    print(s)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(s + "\n")
    eng.close()


if __name__ == "__main__":
    main()
