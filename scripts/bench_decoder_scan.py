"""Autoregressive decoder scan (decoder_scan_kernel): time per frame and where it goes, per batch size.

    python scripts/bench_decoder_scan.py [--batches 1,8,32,128] [--calls 10] [--out FILE.json]

For each batch B (synthetic acoustic checkpoint, 100-phoneme / 5 s utterances = 312 frames, on-device seed dropout):

  * scan time: the `acoustic.decoder_scan` sub-stage (CUDA events around the scan launches, Engine.substages),
    warmed up and averaged over `--calls` forward calls;
  * per-phase breakdown: decoder_scan_kernel adds the clock64 cycles between its phase marks (DEC_MARK) into the
    profiling buffer that Engine.tc_stats switches on and reads.  Each phase's share of a CTA's cycles is scaled by the
    event-measured scan time, so no clock rate is assumed.  The counters are read from a forward call in the 'fp32'
    precision mode, whose projection and postnet convs do not write that buffer (the scan itself is the same kernel
    in every mode).

The kernel's grid size tells the two kernel forms apart: 132 CTAs (128 LSTM + 4 prenet CTAs) or 128 CTAs (prenet
columns inside the LSTM CTAs).  The card name and power limit are read (nvidia-smi, read-only) in the same run.
Prints one JSON object; `--out` also writes it."""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from viettts_b200 import config as C  # noqa: E402
from viettts_b200 import synthetic  # noqa: E402
from viettts_b200.engine import Engine  # noqa: E402

# phase marks of decoder_scan_kernel: slot -> what the CTA did since the previous mark
PHASES = {
    132: {
        "lstm": {0: "EA: zp0/zp1 pre-accumulation", 3: "wait grid.sync 1 (p2 ready)", 4: "C: LSTM0", 5: "wait grid.sync 2 (h0 ready)",
                 6: "D: LSTM1", 7: "wait grid.sync 3 (h1 ready)"},
        "prenet": {0: "EA: p1, h1 half (8 pre_gemm8 passes)", 1: "wait prenet barrier (p1 ready)", 2: "B: p2 (8 pre_gemm8 passes)",
                   3: "wait grid.sync 1", 5: "wait grid.sync 2", 6: "D window: h0 half of next p1 (8 passes)",
                   7: "wait grid.sync 3"},
    },
    128: {
        "lstm": {0: "A: p1 columns (K = 1024)", 1: "A: zp1 = h1.W1h1, zc prefetch, wait (p1 ready)", 2: "B: p2 columns",
                 3: "wait (p2 ready)", 4: "C: LSTM0", 5: "wait (h0 ready)", 6: "D: LSTM1",
                 7: "D: zp0 = h0.W0h, wait (h1 ready)"},
    },
}


def card():
    q = "name,power.limit"
    try:
        r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30)
        name, power = [x.strip() for x in r.stdout.strip().split(",")]
        return {"name": name, "power_limit": power}
    except Exception as e:  # noqa: BLE001
        return {"error": str(e)}


def make_batch(batch, phonemes=100, seconds=5.0, seed0=0):
    toks, durs, nfs = [], [], []
    for b in range(batch):
        tk, d = synthetic.utterance(seed0 + b, phonemes, seconds)
        d = (np.asarray(d, np.float32) * np.float32(C.SAMPLE_RATE)) / np.float32(C.HOP)
        toks.append(np.asarray(tk, np.int32))
        durs.append(d[0])
        nfs.append(int(np.sum(d, dtype=np.float32)))
    return np.stack(toks), np.stack(durs).astype(np.float32), np.asarray(nfs, np.int32)


def phase_table(cnt, scan_us, N):
    """cnt [grid][8] cycles per CTA -> {role: {phase: us per frame}} (mean over the CTAs of the role)."""
    grid = int(np.count_nonzero(cnt.any(axis=1)))
    labels = PHASES.get(grid)
    if labels is None:
        return grid, {"error": f"unknown grid size {grid}"}
    roles = {"lstm": cnt[:128]}
    if "prenet" in labels:
        roles["prenet"] = cnt[128:grid]
    out = {}
    for role, c in roles.items():
        c = c.astype(np.float64)
        total = c.sum(axis=1).mean()
        per = {labels[role].get(i, f"slot {i}"): float(c[:, i].mean() / total * scan_us / N) for i in range(8) if c[:, i].any()}
        out[role] = per
    return grid, out


def one_batch(eng, B, calls, seed=7):
    dev = torch.device("cuda", 0)
    tok, dur, nfs = make_batch(B)
    N = int(nfs.max())
    tok_t, dur_t, nf_t = (torch.from_numpy(a).to(dev) for a in (tok, dur, nfs))
    mel_t = torch.empty((B, N, C.MEL_DIM), dtype=torch.float32, device=dev)
    fwd = lambda: eng.acoustic_forward(tok_t, dur_t, N, n_frames_t=nf_t, seed=seed, out=mel_t)  # noqa: E731
    for _ in range(3):
        fwd()
    torch.cuda.synchronize()
    scans, acoustic = [], []
    for _ in range(calls):
        eng.substages(True)
        fwd()
        ms = eng.substages(False)
        scans.append(ms["acoustic.decoder_scan"])
        acoustic.append(sum(v for k, v in ms.items() if k.startswith("acoustic.")))
    scan_ms = float(np.mean(scans))
    eng.set_precision("fp32")
    fwd()
    eng.tc_stats(True)
    fwd()
    cnt = eng.tc_stats(False)[:, :8]
    eng.set_precision("bf16x3")
    launches = (B + 127) // 128
    grid, phases = phase_table(cnt, 1e3 * scan_ms / launches, N)
    return {"B": B, "frames": N, "scan_ms": scan_ms, "scan_ms_min": float(np.min(scans)), "scan_ms_max": float(np.max(scans)),
            "us_per_frame": 1e3 * scan_ms / (N * launches), "acoustic_ms": float(np.mean(acoustic)), "grid_ctas": grid,
            "phase_us_per_frame": phases}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="1,8,32,128")
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--out", type=Path, default=None)
    a = ap.parse_args()
    eng = Engine(0)
    eng.load_acoustic(synthetic.acoustic_ckpt(1234))
    eng.set_precision("bf16x3")
    res = {"card": card(), "calls": a.calls, "batches": [one_batch(eng, int(b), a.calls) for b in a.batches.split(",")]}
    eng.close()
    text = json.dumps(res, indent=1)
    print(text)
    if a.out:
        a.out.parent.mkdir(parents=True, exist_ok=True)
        a.out.write_text(text + "\n")


if __name__ == "__main__":
    main()
