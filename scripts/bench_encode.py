"""Wire encodings (Engine.encode_forward / decode_forward, open_tts_stream(encoding=)) against the generator.

    python scripts/bench_encode.py [--out FILE.json]

  * time per call (CUDA events over 200 calls from Python after a warm-up) of encoding the 32 x 5 s batch (B = 32, 313
    frames = 80128 samples at 16 kHz, and the same batch resampled to 8 kHz) into each encoding, and of decoding it
    back, beside the generator's time for that batch in the same process.  A call's host side (argument checks, ctypes)
    takes longer than its kernel, so this is the rate a Python caller gets;
  * the kernel alone: the same 200 calls captured in one CUDA graph and replayed (CUDA events around the replay), with
    bytes moved over that time as GB/s and as a share of the H100 SXM data sheet's 3.35 TB/s.  The batch is 13 MB or
    less, so it may be served from the 50 MB L2 between calls;
  * TTS stream step time (host clock around step(), which ends in the step's one synchronisation) and the bytes each
    step copies to the host, for a 32-slot stream at 8 kHz with the telephone EQ, float32 output against ulaw, the two
    streams stepped alternately in one process.

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
from viettts_b200.engine import ENCODING_DTYPES, Engine  # noqa: E402

HOP = 256
HBM_TB_S = 3.35
REPS = 200


def graph_ms(fn, reps=REPS):
    """device time per call of `reps` calls of fn captured in one CUDA graph, replayed after a warm-up replay"""
    fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(reps):
            fn()
    g.replay()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    g.replay()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def batch(eng, B=32, T=313):
    dev = torch.device("cuda", 0)
    mel = torch.from_numpy(synthetic.mel_input(7, B, T)).to(dev)
    wav = torch.empty((B, T * HOP), device=dev)
    res = {"B": B, "frames": T, "samples_16k": T * HOP, "generator_ms": device_ms(lambda: eng.hifigan_forward(mel, out=wav), reps=5)}
    eng.hifigan_forward(mel, out=wav)
    for rate in (16000, 8000):
        x = wav if rate == 16000 else eng.resample_forward(wav, rate)
        for enc, dt in ENCODING_DTYPES.items():
            codes = eng.encode_forward(x, enc)
            back = torch.empty_like(x)
            e_ms = device_ms(lambda: eng.encode_forward(x, enc, out=codes), reps=REPS)
            d_ms = device_ms(lambda: eng.decode_forward(codes, enc, out=back), reps=REPS)
            ek_ms = graph_ms(lambda: eng.encode_forward(x, enc, out=codes))
            dk_ms = graph_ms(lambda: eng.decode_forward(codes, enc, out=back))
            nbytes = x.numel() * (4 + np.dtype(dt).itemsize)
            res[f"{enc}_{rate // 1000}k"] = {
                "rate": rate, "samples": int(x.numel()), "bytes_moved": int(nbytes),
                "encode_ms": e_ms, "decode_ms": d_ms, "encode_share_of_generator_time": e_ms / res["generator_ms"],
                "encode_kernel_ms": ek_ms, "decode_kernel_ms": dk_ms,
                "encode_kernel_GB_per_s": nbytes / (ek_ms * 1e-3) / 1e9, "decode_kernel_GB_per_s": nbytes / (dk_ms * 1e-3) / 1e9,
                "encode_kernel_share_of_hbm_peak": nbytes / (ek_ms * 1e-3) / (HBM_TB_S * 1e12),
                "decode_kernel_share_of_hbm_peak": nbytes / (dk_ms * 1e-3) / (HBM_TB_S * 1e12)}
    return res


def tts_steps(eng, S=32, F=16, reps=4):
    tok = [np.asarray(synthetic.utterance(300 + s, 120, None)[0], np.int32) for s in range(S)]
    res = {"S": S, "F": F, "output_rate": 8000, "eq": "telephone"}
    times = {"float32": [], "ulaw": []}
    copied = {}
    with eng.open_tts_stream(S, F, 4000, 1024, output_rate=8000, eq="telephone") as a, \
            eng.open_tts_stream(S, F, 4000, 1024, output_rate=8000, eq="telephone", encoding="ulaw") as b:
        copied["float32"] = a._stages[-1][1].numel() * 4
        copied["ulaw"] = b._codes.numel() * b._codes.element_size()
        for rep in range(reps + 1):            # the first run warms up
            for s in range(S):
                a.begin(s, tok[s])
                b.begin(s, tok[s])
            while a.busy().any() or b.busy().any():
                for key, ts in (("float32", a), ("ulaw", b)):
                    if ts.busy().any():
                        t0 = time.perf_counter()
                        ts.step()
                        if rep:
                            times[key].append(time.perf_counter() - t0)
    for key, t in times.items():
        t = np.array(t) * 1e3
        res[f"step_ms_{key}"] = {"steps": int(t.size), "mean": float(t.mean()), "p50": float(np.percentile(t, 50)),
                                 "p90": float(np.percentile(t, 90)), "bytes_copied_to_host_per_step": int(copied[key])}
    res["mean_step_difference_ms"] = res["step_ms_ulaw"]["mean"] - res["step_ms_float32"]["mean"]
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
    res = {"card": card(), "precision": "bf16x3", "batch": batch(eng), "tts_stream": tts_steps(eng)}
    s = json.dumps(res, indent=1)
    print(s)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(s + "\n")
    eng.close()


if __name__ == "__main__":
    main()
