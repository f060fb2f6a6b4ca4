"""Background bed (Engine.mix_bed_forward, open_bed_stream) against the generator.

    python scripts/bench_bed.py [--out FILE.json]

  * device time (CUDA events, 20 calls after a warm-up) of mixing the default `pink` bed under the 32 x 5 s batch
    (B = 32, 313 frames = 80128 samples at 16 kHz, and the same batch resampled to 48 kHz), beside the generator's time
    for that batch and the compressor's time on the same rows with the bed's detector settings (compress_forward) in the
    same process; the bank is prepared once before the timed calls;
  * one 3-minute row at 16 kHz, which the detector's sequential chains dominate;
  * one push of a 128-slot bed stream at 16 kHz, 4096 samples per slot (device time from CUDA events, and the host
    clock around push_device plus a synchronisation), every slot open and none ending, so no tail is released.

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
from viettts_b200.engine import Engine, bed_params  # noqa: E402

HOP = 256
SPEC = "pink"


def detector(rate):
    p = bed_params(SPEC, rate)
    return dict(threshold=p["threshold"], ratio=20.0, knee=6.0, attack=p["attack"], release=p["release"], makeup=0.0)


def batch(eng, B=32, T=313):
    dev = torch.device("cuda", 0)
    mel = torch.from_numpy(synthetic.mel_input(7, B, T)).to(dev)
    wav = torch.empty((B, T * HOP), device=dev)
    res = {"B": B, "frames": T, "samples_16k": T * HOP, "generator_ms": device_ms(lambda: eng.hifigan_forward(mel, out=wav), reps=5)}
    eng.hifigan_forward(mel, out=wav)
    for rate in (16000, 48000):
        x = wav if rate == 16000 else eng.resample_forward(wav, rate)
        bank = eng.prepare_beds(SPEC, rate)
        tail = bank.params[0]["Tt"]
        y, r = torch.empty((B, x.shape[1] + tail), device=dev), torch.empty(B, device=dev)
        ms = device_ms(lambda: eng.mix_bed_forward(x, bank, rate, out=y, reduction_db=r))
        red = float(-r.min())
        yc, det = torch.empty_like(x), detector(rate)
        cp_ms = device_ms(lambda: eng.compress_forward(x, det, rate, out=yc, reduction_db=r))
        res[f"rate_{rate}"] = {"samples": int(x.shape[1]), "tail": tail, "bed_ms": ms, "share_of_generator_time": ms / res["generator_ms"],
                               "compress_alone_ms": cp_ms, "output_GB_per_s": y.numel() * 4 / (ms * 1e-3) / 1e9,
                               "max_duck_db": red}
    return res


def long_row(eng, seconds=180, rate=16000):
    dev = torch.device("cuda", 0)
    x = (0.5 * torch.randn((1, seconds * rate), generator=torch.Generator().manual_seed(3))).to(dev)
    bank = eng.prepare_beds(SPEC, rate)
    y, r = torch.empty((1, x.shape[1] + bank.params[0]["Tt"]), device=dev), torch.empty(1, device=dev)
    return {"seconds": seconds, "rate": rate, "bed_ms": device_ms(lambda: eng.mix_bed_forward(x, bank, rate, out=y, reduction_db=r),
                                                                  reps=10)}


def stream_step(eng, S=128, chunk=4096, rate=16000, reps=50):
    dev = torch.device("cuda", 0)
    x = (0.3 * torch.randn((S, chunk), generator=torch.Generator().manual_seed(5))).to(dev)
    n = np.full(S, chunk, np.int32)
    with eng.open_bed_stream(S, chunk, SPEC, rate) as st:
        y, r = torch.empty((S, st.out_pitch), device=dev), torch.empty(S, device=dev)
        st.push_device(x, n, np.full(S, 1, np.uint8), y, r)         # BEGIN every slot
        cont = np.zeros(S, np.uint8)
        ms = device_ms(lambda: st.push_device(x, n, cont, y, r), reps=reps)
        torch.cuda.synchronize()
        t = []
        for _ in range(reps):
            t0 = time.perf_counter()
            st.push_device(x, n, cont, y, r)
            torch.cuda.synchronize()
            t.append(time.perf_counter() - t0)
    t = np.array(t) * 1e3
    return {"S": S, "chunk": chunk, "rate": rate, "device_ms": ms, "host_ms_with_sync": {"mean": float(t.mean()),
                                                                                          "p50": float(np.percentile(t, 50))}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    eng = Engine(0)
    eng.load_hifigan(synthetic.hifigan_params(1234))
    eng.set_precision("bf16x3")
    p = {k: v for k, v in bed_params(SPEC, 16000).items() if k != "audio"}
    res = {"card": card(), "precision": "bf16x3", "spec": p, "batch": batch(eng), "long_row": long_row(eng), "stream_step": stream_step(eng)}
    s = json.dumps(res, indent=1)
    print(s)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(s + "\n")
    eng.close()


if __name__ == "__main__":
    main()
