"""Split-band de-esser (Engine.deess_forward, open_tts_stream(deess=)) against the generator.

    python scripts/bench_deesser.py [--out FILE.json]

  * device time (CUDA events, 20 calls after a warm-up) of de-essing the 32 x 5 s batch (B = 32, 313 frames = 80128
    samples at 16 kHz, and the same batch resampled to 48 kHz) with the `voice` preset, beside the generator's time for
    that batch and the times of its two parts run on their own (the crossover high-pass through Engine.equalize_forward
    and the compressor with the preset's detector settings through compress_forward) in the same process;
  * one 3-minute row at 16 kHz, which the detector's sequential chains dominate;
  * TTS stream step time (host clock around step(), which ends in the step's one synchronisation) at S in {1, 32},
    F = 16, with and without deess='voice', the two streams stepped alternately in one process.

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
from viettts_b200.engine import Engine, deesser_params  # noqa: E402

HOP = 256
SPEC = "voice"


def batch(eng, B=32, T=313):
    dev = torch.device("cuda", 0)
    mel = torch.from_numpy(synthetic.mel_input(7, B, T)).to(dev)
    wav = torch.empty((B, T * HOP), device=dev)
    res = {"B": B, "frames": T, "samples_16k": T * HOP, "generator_ms": device_ms(lambda: eng.hifigan_forward(mel, out=wav), reps=5)}
    eng.hifigan_forward(mel, out=wav)
    for rate in (16000, 48000):
        x = wav if rate == 16000 else eng.resample_forward(wav, rate)
        y, r = torch.empty_like(x), torch.empty(B, device=dev)
        ms = device_ms(lambda: eng.deess_forward(x, SPEC, rate, out=y, reduction_db=r))
        red = float(-r.min())
        hp = f"hp:{deesser_params(SPEC, rate)['freq']}:2"
        eq_ms = device_ms(lambda: eng.equalize_forward(x, hp, rate, out=y))
        detector = {k: v for k, v in deesser_params(SPEC, rate).items() if k not in ("freq", "range")}
        cp_ms = device_ms(lambda: eng.compress_forward(x, detector, rate, out=y, reduction_db=r))
        res[f"rate_{rate}"] = {"samples": int(x.shape[1]), "deess_ms": ms, "share_of_generator_time": ms / res["generator_ms"],
                               "highpass_alone_ms": eq_ms, "compress_alone_ms": cp_ms,
                               "input_GB_per_s": x.numel() * 4 / (ms * 1e-3) / 1e9, "max_reduction_db": red}
    return res


def long_row(eng, seconds=180, rate=16000):
    dev = torch.device("cuda", 0)
    x = (0.5 * torch.randn((1, seconds * rate), generator=torch.Generator().manual_seed(3))).to(dev)
    y, r = torch.empty_like(x), torch.empty(1, device=dev)
    return {"seconds": seconds, "rate": rate, "deess_ms": device_ms(lambda: eng.deess_forward(x, SPEC, rate, out=y, reduction_db=r),
                                                                    reps=10)}


def tts_steps(eng, S, F=16, reps=2):
    tok = [np.asarray(synthetic.utterance(300 + s, 120, None)[0], np.int32) for s in range(S)]
    res = {"S": S, "F": F}
    times = {"plain": [], "deess": []}
    with eng.open_tts_stream(S, F, 4000, 1024) as a, eng.open_tts_stream(S, F, 4000, 1024, deess=SPEC) as b:
        for rep in range(reps + 1):            # the first run warms up
            for s in range(S):
                a.begin(s, tok[s])
                b.begin(s, tok[s])
            while a.busy().any() or b.busy().any():
                for key, ts in (("plain", a), ("deess", b)):
                    if ts.busy().any():
                        t0 = time.perf_counter()
                        ts.step()
                        if rep:
                            times[key].append(time.perf_counter() - t0)
    for key, t in times.items():
        t = np.array(t) * 1e3
        res[f"step_ms_{key}"] = {"steps": int(t.size), "mean": float(t.mean()), "p50": float(np.percentile(t, 50)),
                                 "p90": float(np.percentile(t, 90))}
    res["mean_step_overhead_ms"] = res["step_ms_deess"]["mean"] - res["step_ms_plain"]["mean"]
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
    res = {"card": card(), "precision": "bf16x3", "spec": deesser_params(SPEC, 16000), "batch": batch(eng), "long_row": long_row(eng),
           "tts_stream": [tts_steps(eng, S) for S in (1, 32)]}
    s = json.dumps(res, indent=1)
    print(s)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(s + "\n")
    eng.close()


if __name__ == "__main__":
    main()
