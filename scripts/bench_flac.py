"""FLAC on the device (Engine.encode_flac_forward / encode_flac) against the generator.

    python scripts/bench_flac.py [--out FILE.json]

  * the 32 x 5 s batch (B = 32, 313 frames = 80128 samples at 16 kHz, and the same batch resampled to 48 kHz) at every
    block size: the kernels alone (200 calls captured in one CUDA graph and replayed, CUDA events around the replay) and
    the call from Python (CUDA events over 200 calls after a warm-up), beside the generator's time for that batch in
    the same process;
  * one 3-minute row at 16 kHz (2 880 000 samples), both ways;
  * a 128-slot stream push (FlacStream.push_device, 4096 new samples per slot, block 4096, every slot open): device time
    per push (CUDA events over 50 pushes) and bytes per push;
  * a 32-slot TTS stream step with encoding 'flac' against 'pcm16', the two streams stepped alternately in one process:
    host clock around step() and the bytes each step copies to the host;
  * the compression ratio (FLAC bytes over PCM-16 bytes) of the 20 s speech fixture at 16 and 48 kHz and of the
    synthesized batch.  The synthetic weights make noise-like audio, so its ratio is a lower bound of what real speech
    gets, not an estimate of it.

Synthetic weights, bf16x3.  The card name and power limit are read (nvidia-smi, read-only) in the same run.  Prints one
JSON object; `--out` also writes it."""
from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
sys.path.insert(0, str(Path(__file__).resolve().parent))
from bench_denoise import card, device_ms  # noqa: E402
from bench_encode import graph_ms  # noqa: E402
from viettts_b200 import synthetic  # noqa: E402
from viettts_b200.engine import FLAC_BLOCKS, Engine, flac_bound  # noqa: E402

HOP = 256
REPS = 200
REPO = Path(__file__).resolve().parents[1]


def timed(eng, x, rate, block, reps=REPS):
    B, S = x.shape
    out = torch.empty((B, flac_bound(S, block)), dtype=torch.uint8, device=x.device)
    fn = lambda: eng.encode_flac_forward(x, rate, block=block, out=out)   # noqa: E731
    _, nb = fn()
    total = int(nb.sum())
    return {"kernel_ms": graph_ms(fn, reps), "call_ms": device_ms(fn, reps=reps), "bytes": total,
            "ratio_to_pcm16": total / (2 * x.numel())}


def batch(eng, B=32, T=313):
    dev = torch.device("cuda", 0)
    mel = torch.from_numpy(synthetic.mel_input(7, B, T)).to(dev)
    wav = torch.empty((B, T * HOP), device=dev)
    res = {"B": B, "frames": T, "samples_16k": T * HOP, "generator_ms": device_ms(lambda: eng.hifigan_forward(mel, out=wav), reps=5)}
    eng.hifigan_forward(mel, out=wav)
    for rate in (16000, 48000):
        x = wav if rate == 16000 else eng.resample_forward(wav, rate)
        for block in FLAC_BLOCKS:
            r = timed(eng, x, rate, block)
            r["kernel_share_of_generator_time"] = r["kernel_ms"] / res["generator_ms"]
            res[f"{rate // 1000}k_block{block}"] = r
    return res


def long_row(eng):
    pcm = np.load(REPO / "tests" / "golden" / "watermark_speech_clip.npz")["pcm"]
    x = torch.from_numpy(np.resize(pcm.astype(np.float32) / np.float32(32767.0), 180 * 16000)[None]).cuda()
    return {"samples": int(x.shape[1]), "block4096": timed(eng, x, 16000, 4096, reps=20)}


def stream_push(eng, S=128, F=4096, reps=50):
    from viettts_b200.engine import STREAM_BEGIN
    pcm = np.load(REPO / "tests" / "golden" / "watermark_speech_clip.npz")["pcm"].astype(np.float32) / np.float32(32767.0)
    x = torch.from_numpy(np.stack([np.resize(pcm[997 * s:], F) for s in range(S)])).cuda()
    with eng.open_flac_stream(S, F, 16000, 4096) as fs:
        out = torch.empty(fs.out_bytes, dtype=torch.uint8, device="cuda")
        tbl = torch.zeros((S, 2), dtype=torch.int32, device="cuda")
        n = np.full(S, F, np.int32)
        fs.push_device(x, n, np.full(S, STREAM_BEGIN, np.uint8), out, tbl)
        zero = np.zeros(S, np.uint8)
        ms = device_ms(lambda: fs.push_device(x, n, zero, out, tbl), reps=reps)
        nbytes = int(tbl[:, 1].sum())
    return {"S": S, "new_samples_per_slot": F, "block": 4096, "push_ms": ms, "bytes_per_push": nbytes,
            "pcm16_bytes_per_push": 2 * S * F}


def tts_steps(eng, S=32, F=16, reps=3):
    import time
    tok = [np.asarray(synthetic.utterance(300 + s, 120, None)[0], np.int32) for s in range(S)]
    times = {"pcm16": [], "flac": []}
    copied = {"pcm16": [], "flac": []}
    with eng.open_tts_stream(S, F, 4000, 1024, encoding="pcm16") as a, eng.open_tts_stream(S, F, 4000, 1024, encoding="flac") as b:
        for rep in range(reps + 1):            # the first run warms up
            for s in range(S):
                a.begin(s, tok[s])
                b.begin(s, tok[s])
            while a.busy().any() or b.busy().any():
                for key, ts in (("pcm16", a), ("flac", b)):
                    if ts.busy().any():
                        t0 = time.perf_counter()
                        out = ts.step()
                        dt = time.perf_counter() - t0
                        if rep:
                            times[key].append(dt)
                            copied[key].append(ts._codes.numel() * 2 if key == "pcm16" else
                                               S * 8 + sum(len(v) for v in out.values()))
    res = {"S": S, "F": F, "block": 4096}
    for key in times:
        t = np.array(times[key]) * 1e3
        res[key] = {"steps": int(t.size), "mean_step_ms": float(t.mean()), "p50_step_ms": float(np.percentile(t, 50)),
                    "mean_bytes_copied_per_step": float(np.mean(copied[key]))}
    return res


def speech_ratio(eng):
    pcm = np.load(REPO / "tests" / "golden" / "watermark_speech_clip.npz")["pcm"]
    x = pcm.astype(np.float32) / np.float32(32767.0)
    out = {}
    for rate in (16000, 48000):
        y = x if rate == 16000 else eng.resample(x, rate)
        for block in FLAC_BLOCKS:
            out[f"{rate // 1000}k_block{block}"] = len(eng.encode_flac(y, rate, block=block)) / (2 * y.size)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    eng = Engine(0)
    eng.load_hifigan(synthetic.hifigan_params(1234))
    eng.load_acoustic(synthetic.acoustic_ckpt(1234))
    eng.load_duration(synthetic.duration_ckpt(1234))
    eng.set_precision("bf16x3")
    res = {"card": card(), "precision": "bf16x3", "batch": batch(eng), "three_minute_row": long_row(eng),
           "stream_push_128": stream_push(eng), "tts_stream": tts_steps(eng),
           "speech_fixture_ratio_to_pcm16": speech_ratio(eng)}
    s = json.dumps(res, indent=1)
    print(s)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(s + "\n")
    eng.close()


if __name__ == "__main__":
    main()
