"""Where the generator's ResBlock conv time goes: MMA waits and the epilogue, per up-sampling stage.

    python scripts/bench_generator_epilogue.py [--batch 32] [--calls 5] [--out FILE.json]

At the flagship shape (B = 32 synthetic 100-phoneme / 5 s utterances, 312 mel frames, bf16x3):

  * counters: every ResBlock step of stages 0-3 runs once through Engine.debug_hifigan_layer with the profiling
    counters on (Engine.tc_stats).  The counters are those of the step's last launch: conv2 of the unfused pair
    (tc_conv_kernel, stages 0 and 1) or the fused pair (tc_pair_kernel, stages 2 and 3).  Per launch, the mean over
    the CTAs of: the consumer warpgroups' cycles, their waits for activations and weights, and (tc_conv_kernel only)
    the cycles from a tile's last retired wgmma until its outputs are stored.  Cycles become ms through the median SM
    clock sampled while the launches ran.
  * stage times: the hifigan.stage0..3 sub-stages (CUDA events, Engine.substages) of whole generator calls at the
    same shape, warmed up and averaged over `--calls` calls.

The card name, power limit and SM clock are read (nvidia-smi, read-only) in the same run.  Prints one JSON object;
`--out` also writes it."""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
import threading
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from viettts_b200 import config as C  # noqa: E402
from viettts_b200 import synthetic  # noqa: E402
from viettts_b200.engine import Engine  # noqa: E402

SCALE = [8, 64, 128, 256]   # generator rows per mel frame after the ConvTranspose of stage i


def card():
    q = "name,power.limit"
    try:
        r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30)
        name, power = [x.strip() for x in r.stdout.strip().split(",")]
        return {"name": name, "power_limit": power}
    except Exception as e:  # noqa: BLE001
        return {"error": str(e)}


class SmClock:
    """nvidia-smi SM clock samples taken beside the profiled launches (median MHz)."""

    def __enter__(self):
        self.rows = []
        self.proc = subprocess.Popen(["nvidia-smi", "--query-gpu=clocks.sm", "--format=csv,noheader,nounits", "-lms", "100", "-i", "0"],
                                     stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
        self.t = threading.Thread(target=lambda: self.rows.extend(self.proc.stdout), daemon=True)
        self.t.start()
        return self

    def __exit__(self, *exc):
        self.proc.terminate()
        self.proc.wait(timeout=5)
        self.t.join(timeout=5)
        mhz = [float(r) for r in self.rows if r.strip().replace(".", "", 1).isdigit()]
        self.mhz = float(np.median(mhz)) if mhz else None
        self.samples = len(mhz)


def n_frames(batch, phonemes=100, seconds=5.0):
    nfs = []
    for b in range(batch):
        _, d = synthetic.utterance(b, phonemes, seconds)
        d = (np.asarray(d, np.float32) * np.float32(C.SAMPLE_RATE)) / np.float32(C.HOP)
        nfs.append(int(np.sum(d[0], dtype=np.float32)))
    return np.asarray(nfs, np.int32)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--calls", type=int, default=5)
    ap.add_argument("--out", type=Path, default=None)
    a = ap.parse_args()
    dev = torch.device("cuda", 0)
    eng = Engine(0)
    eng.load_hifigan(synthetic.hifigan_params(1234))
    eng.set_precision("bf16x3")
    nfs = n_frames(a.batch)
    T = int(nfs.max())
    nf_t = torch.from_numpy(nfs).to(dev)
    gen = torch.Generator(device=dev).manual_seed(0)

    # stage times of whole generator calls
    mel = (np.random.default_rng(0).standard_normal((a.batch, T, C.MEL_DIM)) * 2 - 4).astype(np.float32)
    wav = np.empty((a.batch, T * C.HOP), np.float32)
    for _ in range(3):
        eng.mel2wave(mel, nfs, out=wav)
    stage_ms = {i: [] for i in range(4)}
    for _ in range(a.calls):
        eng.substages(True)
        eng.mel2wave(mel, nfs, out=wav)
        ms = eng.substages(False)
        for i in range(4):
            stage_ms[i].append(ms[f"hifigan.stage{i}"])

    # counters of each ResBlock step's last launch
    counters = {}
    with SmClock() as clk:
        for i in range(4):
            Cc = C.HIFIGAN["upsample_initial_channel"] >> (i + 1)
            xs = [torch.randn((a.batch, T * SCALE[i], Cc), device=dev, generator=gen) for _ in range(3)]
            outs = [torch.empty_like(x) for x in xs]
            rows = []
            for m in range(3):
                layer = 5 + 3 * i + m
                eng.debug_hifigan_layer(layer, xs, outs, nf_t, T)   # warm-up
                eng.tc_stats(True)
                eng.debug_hifigan_layer(layer, xs, outs, nf_t, T)
                cnt = eng.tc_stats(False).astype(np.float64)
                cnt = cnt[cnt[:, 0] > 0]
                rows.append({"layer": layer, "ctas": int(cnt.shape[0]), "consumer": cnt[:, 0].mean(), "epilogue": cnt[:, 1].mean(),
                             "a_wait": cnt[:, 2].mean(), "w_wait": cnt[:, 3].mean()})
            counters[i] = rows
            del xs, outs
    eng.close()

    cyc_ms = 1.0 / (clk.mhz * 1e3) if clk.mhz else None
    stages = {}
    for i in range(4):
        rows = counters[i]
        tot = {k: float(sum(r[k] for r in rows)) for k in ("consumer", "epilogue", "a_wait", "w_wait")}
        st = {"kernel": "tc_conv_kernel (conv2 of the unfused pair)" if i < 2 else "tc_pair_kernel (fused pair)",
              "stage_ms": float(np.mean(stage_ms[i])), "stage_ms_min": float(np.min(stage_ms[i])), "stage_ms_max": float(np.max(stage_ms[i])),
              "cycles_per_step": tot, "layers": [{k: (float(v) if isinstance(v, np.floating) else v) for k, v in r.items()} for r in rows]}
        if cyc_ms:
            st["ms_per_step"] = {k: v * cyc_ms for k, v in tot.items()}
        if i >= 2:
            st["note"] = "tc_pair_kernel has no epilogue counter: its epilogue already batches its residual loads"
        stages[f"stage{i}"] = st
    res = {"card": card(), "sm_clock_mhz": clk.mhz, "sm_clock_samples": clk.samples, "batch": a.batch, "mel_frames": T,
           "precision": "bf16x3", "calls": a.calls, "stages": stages}
    text = json.dumps(res, indent=1)
    print(text)
    if a.out:
        a.out.parent.mkdir(parents=True, exist_ok=True)
        a.out.write_text(text + "\n")


if __name__ == "__main__":
    main()
