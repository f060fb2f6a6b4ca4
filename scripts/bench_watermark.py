"""Watermark (Engine.watermark_forward, detect_watermark_forward, open_tts_stream(watermark=)) against the generator.

    python scripts/bench_watermark.py [--out FILE.json]

  * device time (CUDA events, 20 calls after a warm-up) of the embed and of search-mode and aligned detection with 16
    keys on the 32 x 5 s batch (B = 32, 313 frames = 80128 samples at 16 kHz), beside the generator's time for that
    batch in the same process; detection also from the batch resampled to 48 kHz;
  * per-kernel device times of the embed and the search from torch.profiler (a separate run after the timed ones);
  * one 3-minute row at 16 kHz: embed, and search with 16 keys;
  * TTS stream step time (host clock around step(), which ends in the step's one synchronisation) at S in {1, 32},
    F = 16, with and without a watermark, the two streams stepped alternately in one process.

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
from viettts_b200.engine import Engine  # noqa: E402

HOP = 256
SPEC = "key=7,strength=0.1"
KEYS = list(range(7, 23))      # 16 keys


def batch(eng, B=32, T=313):
    dev = torch.device("cuda", 0)
    mel = torch.from_numpy(synthetic.mel_input(7, B, T)).to(dev)
    wav = torch.empty((B, T * HOP), device=dev)
    res = {"B": B, "frames": T, "samples_16k": T * HOP, "keys": len(KEYS),
           "generator_ms": device_ms(lambda: eng.hifigan_forward(mel, out=wav), reps=5)}
    eng.hifigan_forward(mel, out=wav)
    y = torch.empty_like(wav)
    keys = torch.tensor(KEYS, dtype=torch.uint64, device=dev)
    res["embed_ms"] = device_ms(lambda: eng.watermark_forward(wav, SPEC, out=y))
    res["detect_search_ms"] = device_ms(lambda: eng.detect_watermark_forward(y, keys))
    res["detect_aligned_ms"] = device_ms(lambda: eng.detect_watermark_forward(y, keys, search=False))
    y48 = eng.resample_forward(y, 48000)
    res["detect_search_48k_ms"] = device_ms(lambda: eng.detect_watermark_forward(y48, keys, rate=48000))
    for k in ("embed_ms", "detect_search_ms", "detect_aligned_ms", "detect_search_48k_ms"):
        res[k.replace("_ms", "_share_of_generator_time")] = res[k] / res["generator_ms"]
    d = eng.detect_watermark_forward(y, keys)
    res["batch_min_z_right_key"] = float(d.z[:, 0].min())
    res["batch_max_z_wrong_keys"] = float(d.z[:, 1:].max())
    return res, wav, y, keys


def kernel_times(eng, wav, y, keys, reps=10):
    """device time per kernel of the embed and the search on the batch (torch.profiler, CUDA activities)"""
    from torch.profiler import ProfilerActivity, profile
    out_t = torch.empty_like(wav)
    eng.watermark_forward(wav, SPEC, out=out_t)
    eng.detect_watermark_forward(y, keys)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            eng.watermark_forward(wav, SPEC, out=out_t)
            eng.detect_watermark_forward(y, keys)
        torch.cuda.synchronize()
    out = {}
    for ev in prof.key_averages():
        for name in ("gain_frame_kernel", "denoise_ola_kernel", "wm_spec_kernel", "wm_fold_kernel", "wm_corr_kernel"):
            if name in ev.key:
                t = getattr(ev, "device_time_total", None)
                t = ev.cuda_time_total if t is None else t
                out[name] = out.get(name, 0.0) + t / 1e3 / reps
    return {k: out[k] for k in sorted(out)}


def long_row(eng, seconds=180, rate=16000):
    dev = torch.device("cuda", 0)
    x = (0.3 * torch.randn((1, seconds * rate), generator=torch.Generator().manual_seed(3))).to(dev)
    y = torch.empty_like(x)
    keys = torch.tensor(KEYS, dtype=torch.uint64, device=dev)
    return {"seconds": seconds, "rate": rate, "embed_ms": device_ms(lambda: eng.watermark_forward(x, SPEC, out=y), reps=10),
            "detect_search_ms": device_ms(lambda: eng.detect_watermark_forward(y, keys), reps=10)}


def tts_steps(eng, S, F=16, reps=2):
    tok = [np.asarray(synthetic.utterance(300 + s, 120, None)[0], np.int32) for s in range(S)]
    res = {"S": S, "F": F, "spec": SPEC}
    times = {"plain": [], "watermark": []}
    with eng.open_tts_stream(S, F, 4000, 1024) as a, eng.open_tts_stream(S, F, 4000, 1024, watermark=SPEC) as b:
        for rep in range(reps + 1):            # the first run warms up
            for s in range(S):
                a.begin(s, tok[s])
                b.begin(s, tok[s])
            while a.busy().any() or b.busy().any():
                for key, ts in (("plain", a), ("watermark", b)):
                    if ts.busy().any():
                        t0 = time.perf_counter()
                        ts.step()
                        if rep:
                            times[key].append(time.perf_counter() - t0)
    for key, t in times.items():
        t = np.array(t) * 1e3
        res[f"step_ms_{key}"] = {"steps": int(t.size), "mean": float(t.mean()), "p50": float(np.percentile(t, 50)),
                                 "p90": float(np.percentile(t, 90))}
    res["mean_step_overhead_ms"] = res["step_ms_watermark"]["mean"] - res["step_ms_plain"]["mean"]
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
    b, wav, y, keys = batch(eng)
    res = {"card": card(), "precision": "bf16x3", "spec": SPEC, "batch": b, "long_row": long_row(eng),
           "tts_stream": [tts_steps(eng, S) for S in (1, 32)], "kernels": kernel_times(eng, wav, y, keys)}
    s = json.dumps(res, indent=1)
    print(s)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(s + "\n")
    eng.close()


if __name__ == "__main__":
    main()
