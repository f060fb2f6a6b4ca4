"""Convolution reverb (Engine.reverb_forward, open_tts_stream(reverb=)) against the generator.

    python scripts/bench_reverb.py [--out FILE.json]

  * device time (CUDA events, 20 calls after a warm-up) of the reverb on the 32 x 5 s batch (B = 32, 313 frames = 80128
    samples at 16 kHz, and the same batch resampled to 48 kHz) with the `room` and `hall` presets and a 4 s IR, beside
    the generator's time for that batch in the same process; the MAC kernel's FP32 work is 8 B nb 513 K FLOPs
    (nb = ceil(n / 512) blocks, K = ceil(L / 512) partitions), reported over the call time and over the 67 TFLOP/s
    FP32 data-sheet peak of the H100 SXM;
  * per-kernel device times of the hall call at 48 kHz from torch.profiler (a separate run after the timed ones);
  * one 3-minute row at 16 kHz with `hall`;
  * TTS stream step time (host clock around step(), which ends in the step's one synchronisation) at S in {1, 32},
    F = 16, with and without reverb='hall', the two streams stepped alternately in one process.

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
from viettts_b200.engine import Engine, reverb_params  # noqa: E402

HOP = 256
BLK = 512
FP32_PEAK = 67e12


def mac_flops(B, n, L):
    return 8 * B * -(-n // BLK) * 513 * -(-L // BLK)


def four_second_ir(rate):
    return {"ir": reverb_params("rt60=4,predelay=0", rate)["ir"][:4 * rate], "mix": 0.25}


def batch(eng, B=32, T=313):
    dev = torch.device("cuda", 0)
    mel = torch.from_numpy(synthetic.mel_input(7, B, T)).to(dev)
    wav = torch.empty((B, T * HOP), device=dev)
    res = {"B": B, "frames": T, "samples_16k": T * HOP, "generator_ms": device_ms(lambda: eng.hifigan_forward(mel, out=wav), reps=5)}
    eng.hifigan_forward(mel, out=wav)
    for rate in (16000, 48000):
        x = wav if rate == 16000 else eng.resample_forward(wav, rate)
        y = torch.empty_like(x)
        r = {"samples": int(x.shape[1])}
        for name, spec in (("room", "room"), ("hall", "hall"), ("ir_4s", four_second_ir(rate))):
            L = reverb_params(spec, rate)["ir"].size
            ms = device_ms(lambda: eng.reverb_forward(x, spec, rate, out=y))
            fl = mac_flops(B, x.shape[1], L)
            r[name] = {"taps": L, "partitions": -(-L // BLK), "reverb_ms": ms, "share_of_generator_time": ms / res["generator_ms"],
                       "mac_gflop": fl / 1e9, "mac_tflops_over_call_time": fl / (ms * 1e-3) / 1e12,
                       "share_of_fp32_peak_over_call_time": fl / (ms * 1e-3) / FP32_PEAK}
        res[f"rate_{rate}"] = r
    return res, wav


def kernel_times(eng, wav, rate=48000, reps=10):
    """device time per kernel of the hall call at 48 kHz (torch.profiler, CUDA activities)"""
    from torch.profiler import ProfilerActivity, profile
    x = eng.resample_forward(wav, rate)
    y = torch.empty_like(x)
    eng.reverb_forward(x, "hall", rate, out=y)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            eng.reverb_forward(x, "hall", rate, out=y)
        torch.cuda.synchronize()
    out = {}
    for ev in prof.key_averages():
        if "reverb" in ev.key:
            name = next(k for k in ("ir_kernel", "frame_kernel", "mac_kernel", "out_kernel") if k in ev.key)
            t = getattr(ev, "device_time_total", None)
            t = ev.cuda_time_total if t is None else t
            out[name] = t / 1e3 / reps
    L = reverb_params("hall", rate)["ir"].size
    if "mac_kernel" in out:
        fl = mac_flops(x.shape[0], x.shape[1], L)
        out["mac_tflops"] = fl / (out["mac_kernel"] * 1e-3) / 1e12
        out["mac_share_of_fp32_peak"] = out["mac_tflops"] * 1e12 / FP32_PEAK
    return {k: out[k] for k in sorted(out)}


def long_row(eng, seconds=180, rate=16000):
    dev = torch.device("cuda", 0)
    x = (0.5 * torch.randn((1, seconds * rate), generator=torch.Generator().manual_seed(3))).to(dev)
    y = torch.empty_like(x)
    return {"seconds": seconds, "rate": rate, "spec": "hall",
            "reverb_ms": device_ms(lambda: eng.reverb_forward(x, "hall", rate, out=y), reps=10)}


def tts_steps(eng, S, F=16, reps=2):
    tok = [np.asarray(synthetic.utterance(300 + s, 120, None)[0], np.int32) for s in range(S)]
    res = {"S": S, "F": F, "spec": "hall"}
    times = {"plain": [], "reverb": []}
    with eng.open_tts_stream(S, F, 4000, 1024) as a, eng.open_tts_stream(S, F, 4000, 1024, reverb="hall") as b:
        for rep in range(reps + 1):            # the first run warms up
            for s in range(S):
                a.begin(s, tok[s])
                b.begin(s, tok[s])
            while a.busy().any() or b.busy().any():
                for key, ts in (("plain", a), ("reverb", b)):
                    if ts.busy().any():
                        t0 = time.perf_counter()
                        ts.step()
                        if rep:
                            times[key].append(time.perf_counter() - t0)
    for key, t in times.items():
        t = np.array(t) * 1e3
        res[f"step_ms_{key}"] = {"steps": int(t.size), "mean": float(t.mean()), "p50": float(np.percentile(t, 50)),
                                 "p90": float(np.percentile(t, 90))}
    res["mean_step_overhead_ms"] = res["step_ms_reverb"]["mean"] - res["step_ms_plain"]["mean"]
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
    b, wav = batch(eng)
    res = {"card": card(), "precision": "bf16x3", "batch": b, "long_row": long_row(eng),
           "tts_stream": [tts_steps(eng, S) for S in (1, 32)], "kernels_hall_48k": kernel_times(eng, wav)}
    s = json.dumps(res, indent=1)
    print(s)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(s + "\n")
    eng.close()


if __name__ == "__main__":
    main()
