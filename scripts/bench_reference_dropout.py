"""Cost of the reference's dropout stream: host masks (MASK mode fed by viettts_b200.jaxrng) against the device draws
of the REFERENCE mode (`rng=`), and REFERENCE against the SEED and MASK modes on the device.

    python scripts/bench_reference_dropout.py [--rounds 3] [--out profiles/h100_reference_dropout.json]

Synthetic checkpoints (seed 1234), written as pickles for the drop-ins.  Each old/new pair alternates inside one
process for `--rounds` rounds, so both see the same machine state.  Records:

  * drop-in `text2mel.predict_mel` wall time per call at N = 312 and 937 frames: explicit `masks=jaxrng...` (the
    mask generation is part of the call, as it was in the drop-in) against the default, which now draws on the device;
  * `gta.forward_fn` wall time per call at B = 32, N = 937, the same two ways;
  * device time of ref_subkey_chain_kernel at N = 312, 937 and 5000 (torch.profiler, CUDA activity, B = 1);
  * acoustic-stage device time (CUDA events, Engine.last_stage_ms(1)) at B = 1 and 32, N = 312, in the REFERENCE,
    SEED and MASK modes.

Old and new outputs are compared bit for bit at every timed size.  The card name and power limit are read (nvidia-smi,
read-only) in the same run.  Prints one JSON object; `--out` also writes it."""
from __future__ import annotations

import argparse
import json
import pickle
import subprocess
import sys
import tempfile
import time
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from viettts_b200 import config as C  # noqa: E402
from viettts_b200 import jaxrng, synthetic  # noqa: E402


def card():
    q = "name,power.limit"
    try:
        r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30)
        name, power = [x.strip() for x in r.stdout.strip().split(",")]
        return {"name": name, "power_limit": power}
    except Exception as e:  # noqa: BLE001
        return {"error": str(e)}


def stats(xs):
    xs = np.asarray(xs, np.float64)
    return {"median": float(np.median(xs)), "min": float(xs.min()), "max": float(xs.max()), "n": int(xs.size)}


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


def alternate(pairs, rounds, calls):
    """pairs: {name: fn}; every round runs each fn `calls` times, in turn.  Returns {name: stats of s/call}, last outputs."""
    times = {k: [] for k in pairs}
    outs = {}
    for k, fn in pairs.items():       # warm-up
        outs[k] = fn()
    for _ in range(rounds):
        for k, fn in pairs.items():
            for _ in range(calls):
                dt, outs[k] = timed(fn)
                times[k].append(dt)
    return {k: stats(v) for k, v in times.items()}, outs


def dropin_predict_mel(rng, rounds):
    from viettts_b200.nat import text2mel as t2m
    res = []
    for phonemes, seconds in ((100, 5.0), (300, 15.0)):
        tk, dur = synthetic.utterance(0, phonemes, seconds)
        n = t2m.seconds_to_frames(dur)[1]
        pairs = {"old_host_masks": lambda: t2m.predict_mel(tk, dur, masks=jaxrng.inference_keep_masks(rng, 1, n)),
                 "new_device_draws": lambda: t2m.predict_mel(tk, dur)}
        st, outs = alternate(pairs, rounds, 3)
        res.append({"frames": n, "s_per_call": st, "identical": bool(np.array_equal(outs["old_host_masks"], outs["new_device_draws"]))})
    return res


def gta_forward(rng, rounds, B=32, N=937):
    from viettts_b200.nat import gta
    rs = np.random.default_rng(5)
    wavs = (rs.standard_normal((B, N * C.HOP)) * 3000).astype(np.int16)
    L = 300
    toks, durs = [], []
    for b in range(B):
        tk, d = synthetic.utterance(b, L, N / 62.5 - 0.2)
        toks.append(tk)
        durs.append(d[0])
    tok, dur, lens = np.asarray(toks, np.int32), np.asarray(durs, np.float32), np.full(B, L, np.int32)

    def old():
        keep, zone = jaxrng.teacher_forced_masks(rng, B, N)
        return gta.forward_fn(wavs, tok, lens, dur, keep_masks=keep, zone_masks=zone)

    pairs = {"old_host_masks": old, "new_device_draws": lambda: gta.forward_fn(wavs, tok, lens, dur)}
    st, outs = alternate(pairs, rounds, 1)
    return {"B": B, "frames": N, "s_per_call": st, "identical": bool(np.array_equal(outs["old_host_masks"], outs["new_device_draws"]))}


def device_batch(B, phonemes, seconds):
    dev = torch.device("cuda", 0)
    toks, durs, nfs = [], [], []
    for b in range(B):
        tk, d = synthetic.utterance(b, phonemes, seconds)
        d = (np.asarray(d, np.float32) * np.float32(C.SAMPLE_RATE)) / np.float32(C.HOP)
        toks.append(np.asarray(tk, np.int32))
        durs.append(d[0])
        nfs.append(int(np.sum(d, dtype=np.float32)))
    nfs = np.asarray(nfs, np.int32)
    tok_t, dur_t, nf_t = (torch.from_numpy(np.ascontiguousarray(a)).to(dev) for a in (np.stack(toks), np.stack(durs).astype(np.float32), nfs))
    return tok_t, dur_t, nf_t, int(nfs.max())


def chain_kernel_us(eng, rng, frames=(312, 937, 5000)):
    from torch.profiler import ProfilerActivity, profile
    out = {}
    for n in frames:
        tok_t, dur_t, nf_t, N = device_batch(1, max(8, n // 3), n / 62.5)     # synthetic.utterance: int(n + 0.3) = n frames
        for _ in range(2):
            eng.acoustic_forward(tok_t, dur_t, N, n_frames_t=nf_t, rng=rng)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(5):
                eng.acoustic_forward(tok_t, dur_t, N, n_frames_t=nf_t, rng=rng)
            torch.cuda.synchronize()
        ev = [e for e in prof.key_averages() if "ref_subkey_chain_kernel" in e.key]
        scan = [e for e in prof.key_averages() if "decoder_scan_kernel" in e.key and "tf" not in e.key]
        out[str(N)] = {"chain_us": ev[0].device_time_total / ev[0].count if ev else None,
                       "decoder_scan_us": scan[0].device_time_total / scan[0].count if scan else None}
    return out


def acoustic_modes(eng, rng, rounds, batches=(1, 32)):
    seed = (int(rng[0]) << 32) | int(rng[1])
    res = []
    for B in batches:
        tok_t, dur_t, nf_t, N = device_batch(B, 100, 5.0)
        masks = np.ascontiguousarray(np.broadcast_to(jaxrng.inference_keep_masks(rng, 1, N), (B, N, 2, 256)))
        masks_t = torch.from_numpy(masks).to(tok_t.device)
        out = torch.empty((B, N, C.MEL_DIM), dtype=torch.float32, device=tok_t.device)
        fns = {"REFERENCE": lambda: eng.acoustic_forward(tok_t, dur_t, N, n_frames_t=nf_t, rng=rng, out=out),
               "SEED": lambda: eng.acoustic_forward(tok_t, dur_t, N, n_frames_t=nf_t, seed=seed, out=out),
               "MASK": lambda: eng.acoustic_forward(tok_t, dur_t, N, n_frames_t=nf_t, masks_t=masks_t, out=out)}
        ms = {k: [] for k in fns}
        mels = {}
        for k, fn in fns.items():
            for _ in range(3):
                fn()
        for _ in range(rounds):
            for k, fn in fns.items():
                for _ in range(5):
                    fn()
                    ms[k].append(eng.last_stage_ms(1))
                mels[k] = out.cpu().numpy()
        res.append({"B": B, "frames": N, "acoustic_ms": {k: stats(v) for k, v in ms.items()},
                    "reference_equals_mask": bool(np.array_equal(mels["REFERENCE"], mels["MASK"]))})
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", type=Path, default=None)
    a = ap.parse_args()
    from viettts_b200.engine import get_engine
    from viettts_b200.nat import text2mel as t2m
    ck = synthetic.acoustic_ckpt(1234)
    rng = jaxrng.rng_key(ck["rng"])
    with tempfile.TemporaryDirectory() as tmp:
        t2m.CKPT_FILE = Path(tmp) / "acoustic_latest_ckpt.pickle"
        with open(t2m.CKPT_FILE, "wb") as f:
            pickle.dump(ck, f)
        eng = get_engine(0)
        eng.set_precision("bf16x3")
        eng.load_mel_filterbank()
        res = {"card": card(), "precision": "bf16x3", "rounds": a.rounds, "rng": [int(x) for x in rng],
               "dropin_predict_mel": dropin_predict_mel(rng, a.rounds),
               "gta_forward_fn": gta_forward(rng, max(2, a.rounds - 1)),
               "chain_kernel": chain_kernel_us(eng, rng),
               "acoustic_stage": acoustic_modes(eng, rng, a.rounds)}
    text = json.dumps(res, indent=1)
    print(text)
    if a.out:
        a.out.parent.mkdir(parents=True, exist_ok=True)
        a.out.write_text(text + "\n")


if __name__ == "__main__":
    main()
