"""Pitch shifter (Engine.pitch_shift_forward, Engine.open_tts_stream(semitones=)) against the generator.

    python scripts/bench_pitch.py [--formant PHI] [--out FILE.json]

  * device time (CUDA events, 20 calls after a warm-up) of shifting the 32 x 5 s batch (B = 32, 313 frames = 80128
    samples at 16 kHz) by +3 semitones, beside the generator's time for that batch in the same process;
  * each kernel's share of that time (torch.profiler with CUDA activities, 5 calls, in a pass of its own);
  * one 3-minute row (2 880 000 samples, 11 251 frames), where the sequential phase kernel dominates;
  * TTS stream step time (host clock around step(), which ends in the step's one synchronisation) at S in {1, 32},
    F = 16, with and without semitones=3, the two streams stepped alternately in one process.

`--formant PHI` adds the voice shift (formant=PHI, the cepstral-envelope kernels) to each case, measured beside the
pitch shift in the same process (a third TTS stream with semitones=3, formant=PHI).  Synthetic weights, bf16x3.  The card name and power limit are read (nvidia-smi, read-only) in the same run.  Prints one
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
from viettts_b200 import synthetic  # noqa: E402
from viettts_b200.engine import Engine  # noqa: E402

SEMITONES = 3.0
FORMANT = None     # --formant


def kernel_split(fn, reps=5):
    """device time per kernel name (ms per call) of `fn` under torch.profiler"""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    out = {}
    for ev in prof.key_averages():
        for name in ("pitch_analysis_kernel", "pitch_phase_kernel", "pitch_synth_kernel", "denoise_ola_kernel"):
            if name in ev.key:
                t = getattr(ev, "device_time_total", None)
                if t is None:
                    t = ev.cuda_time_total
                out[name] = out.get(name, 0.0) + t / 1e3 / reps
    return out


def shift_ms(eng, B, n, reps=20):
    dev = torch.device("cuda", 0)
    rng = np.random.default_rng(11)
    t = np.arange(n) / 16000
    x = torch.from_numpy(np.stack([0.3 * np.sin(2 * np.pi * 180 * (1 + 0.1 * b) * t) + 0.02 * rng.standard_normal(n)
                                   for b in range(B)]).astype(np.float32)).to(dev)
    out = torch.empty_like(x)
    fn = lambda: eng.pitch_shift_forward(x, SEMITONES, out=out)   # noqa: E731
    ms = device_ms(fn, reps=reps)
    split = kernel_split(fn)
    frames = B * (n // HOP + 1)
    res = {"B": B, "samples": n, "stft_frames": frames, "ms": ms, "us_per_frame": ms * 1e3 / frames, "kernel_ms": split,
           "phase_share": split.get("pitch_phase_kernel", 0.0) / max(sum(split.values()), 1e-9)}
    if FORMANT is not None:
        fv = lambda: eng.pitch_shift_forward(x, SEMITONES, out=out, formant=FORMANT)   # noqa: E731
        vms = device_ms(fv, reps=reps)
        res["voice_shift"] = {"formant": FORMANT, "ms": vms, "us_per_frame": vms * 1e3 / frames, "over_pitch_shift": vms / ms,
                              "kernel_ms": kernel_split(fv)}
    return res


def batch(eng, B=32, T=313):
    dev = torch.device("cuda", 0)
    mel = torch.from_numpy(synthetic.mel_input(7, B, T)).to(dev)
    wav = torch.empty((B, T * HOP), device=dev)
    res = {"B": B, "frames": T, "samples_16k": T * HOP, "generator_ms": device_ms(lambda: eng.hifigan_forward(mel, out=wav), reps=5)}
    eng.hifigan_forward(mel, out=wav)
    out = torch.empty_like(wav)
    fn = lambda: eng.pitch_shift_forward(wav, SEMITONES, out=out)   # noqa: E731
    ms = device_ms(fn)
    split = kernel_split(fn)
    frames = B * (T * HOP // HOP + 1)
    res["pitch_shift"] = {"semitones": SEMITONES, "ms": ms, "stft_frames": frames, "us_per_frame": ms * 1e3 / frames,
                          "share_of_generator_time": ms / res["generator_ms"], "kernel_ms": split,
                          "phase_share": split.get("pitch_phase_kernel", 0.0) / max(sum(split.values()), 1e-9)}
    if FORMANT is not None:
        fv = lambda: eng.pitch_shift_forward(wav, SEMITONES, out=out, formant=FORMANT)   # noqa: E731
        vms = device_ms(fv)
        res["voice_shift"] = {"semitones": SEMITONES, "formant": FORMANT, "ms": vms, "us_per_frame": vms * 1e3 / frames,
                              "share_of_generator_time": vms / res["generator_ms"], "over_pitch_shift": vms / ms,
                              "kernel_ms": kernel_split(fv)}
    return res


def tts_steps(eng, S, F=16, reps=2):
    tok = [np.asarray(synthetic.utterance(300 + s, 120, None)[0], np.int32) for s in range(S)]
    res = {"S": S, "F": F}
    times = {"plain": [], "pitch": []}
    if FORMANT is not None:
        times["voice"] = []
    with eng.open_tts_stream(S, F, 4000, 1024) as a, eng.open_tts_stream(S, F, 4000, 1024, semitones=SEMITONES) as b, \
            eng.open_tts_stream(S, F, 4000, 1024, semitones=SEMITONES, formant=0.0 if FORMANT is None else FORMANT) as c:
        streams = [("plain", a), ("pitch", b)] + ([("voice", c)] if FORMANT is not None else [])
        for rep in range(reps + 1):            # the first run warms up
            for s in range(S):
                for _, ts in streams:
                    ts.begin(s, tok[s])
            while any(ts.busy().any() for _, ts in streams):
                for key, ts in streams:
                    if ts.busy().any():
                        t0 = time.perf_counter()
                        ts.step()
                        if rep:
                            times[key].append(time.perf_counter() - t0)
    for key, t in times.items():
        t = np.array(t) * 1e3
        res[f"step_ms_{key}"] = {"steps": int(t.size), "mean": float(t.mean()), "p50": float(np.percentile(t, 50)),
                                 "p90": float(np.percentile(t, 90))}
    res["mean_step_overhead_ms"] = res["step_ms_pitch"]["mean"] - res["step_ms_plain"]["mean"]
    if FORMANT is not None:
        res["mean_step_overhead_ms_voice"] = res["step_ms_voice"]["mean"] - res["step_ms_plain"]["mean"]
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--formant", default=None, type=float)
    args = ap.parse_args()
    global FORMANT
    FORMANT = args.formant
    eng = Engine(0)
    eng.load_acoustic(synthetic.acoustic_ckpt(1234))
    eng.load_hifigan(synthetic.hifigan_params(1234))
    eng.load_duration(synthetic.duration_ckpt(1234))
    eng.set_precision("bf16x3")
    res = {"card": card(), "precision": "bf16x3", "formant": FORMANT, "batch": batch(eng), "three_minute_row": shift_ms(eng, 1, 3 * 60 * 16000, reps=5),
           "tts_stream": [tts_steps(eng, S) for S in (1, 32)]}
    s = json.dumps(res, indent=1)
    print(s)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(s + "\n")
    eng.close()


if __name__ == "__main__":
    main()
