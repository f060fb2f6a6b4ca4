"""Device time of every launch of one generator call, and of each stage, at the flagship shape.

    python scripts/bench_upsample.py [--batch 32] [--calls 5] [--precision bf16x3] [--out FILE.json]

The workload is bench.py's generator half: B = 32 synthetic 100-phoneme / 5 s utterances (312 mel frames), their
n_frames, a seeded mel, inputs resident on the device.

  * stages: the hifigan.conv_pre / stage0..3 / conv_post sub-stages (CUDA events, Engine.substages) of whole
    generator calls, warmed up, over `--calls` calls, with the profiler off.
  * launches: `--calls` further calls under torch.profiler (CUDA activities), after the timed ones.  The generator's
    kernels are identified by launch order: conv_pre, then per stage the ConvTranspose (`ups`) and its ResBlock steps
    (two tc_conv_kernel launches per step for C > 64, one fused tc_pair_kernel launch for C <= 64), then conv_post.
    Per launch: the median device time over the calls.  For the ConvTranspose launches also the DRAM bytes (three
    chain inputs read once, the output written once) and the FLOP of the layer, and the time they take at the H100 SXM
    data-sheet rates (3.35 TB/s, 989 TFLOP/s dense BF16): a bound, not a measurement.

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

RATES = [8, 8, 2, 2]
C0 = 512
KERNELS = ("tc_conv_kernel", "tc_pair_kernel", "conv_post_kernel")


def card():
    q = "name,power.limit,clocks.max.sm"
    try:
        r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30)
        vals = [v.strip() for v in r.stdout.strip().split(",")]
        return dict(zip(q.split(","), vals)) if r.returncode == 0 and len(vals) == 3 else dict(error=r.stderr.strip())
    except Exception as e:  # noqa: BLE001
        return dict(error=str(e))


class SmClock:
    """nvidia-smi SM clock samples taken beside the profiled calls (median MHz)."""

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


def launch_labels():
    """The generator's launches in issue order (vtts_hifigan_run with fused pairs on)."""
    labels = ["conv_pre"]
    for i in range(4):
        labels.append(f"stage{i}.ups")
        co = C0 >> (i + 1)
        for m in range(3):
            labels += [f"stage{i}.rb{m}"] if co <= 64 else [f"stage{i}.rb{m}.conv1", f"stage{i}.rb{m}.conv2"]
    labels.append("conv_post")
    return labels


def ups_work(i, B, T):
    """DRAM bytes and FLOP of the ConvTranspose of stage i over B rows of T mel frames."""
    scale = int(np.prod(RATES[:i])) if i else 1
    rows_in, c = T * scale, C0 >> i
    n_in = 1 if i == 0 else 3
    by = 4 * B * rows_in * c * n_in + 4 * B * rows_in * RATES[i] * (c // 2)
    fl = 2.0 * B * rows_in * RATES[i] * (c // 2) * c * 2   # two taps per output row
    return by, fl


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--calls", type=int, default=5)
    ap.add_argument("--precision", default="bf16x3", choices=("bf16x3", "fp16"))
    ap.add_argument("--out", type=Path, default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_upsample: no CUDA device")
    dev = torch.device("cuda", 0)
    gpu = card()
    eng = Engine(0)
    eng.load_hifigan(synthetic.hifigan_params(1234))
    eng.set_precision(a.precision)
    nfs = n_frames(a.batch)
    T = int(nfs.max())
    nf_t = torch.from_numpy(nfs).to(dev)
    mel = (torch.randn((a.batch, T, C.MEL_DIM), device=dev, generator=torch.Generator(device=dev).manual_seed(0)) * 2 - 4).contiguous()
    wav = torch.empty((a.batch, T * C.HOP), device=dev)

    # stage times of whole calls (profiler off)
    for _ in range(3):
        eng.hifigan_forward(mel, nf_t, out=wav)
    torch.cuda.synchronize()
    names = ["hifigan.conv_pre"] + [f"hifigan.stage{i}" for i in range(4)] + ["hifigan.conv_post"]
    stage_ms = {n: [] for n in names}
    call_ms = []
    for _ in range(a.calls):
        eng.substages(True)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        eng.hifigan_forward(mel, nf_t, out=wav)
        e1.record()
        torch.cuda.synchronize()
        ms = eng.substages(False)
        call_ms.append(e0.elapsed_time(e1))
        for n in names:
            stage_ms[n].append(ms[n])

    # per-launch device times under the profiler, in a pass of their own
    labels = launch_labels()
    per_call = []
    with SmClock() as clk:
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(a.calls):
                eng.hifigan_forward(mel, nf_t, out=wav)
                torch.cuda.synchronize()
    kern = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and any(k in e.name for k in KERNELS)]
    kern.sort(key=lambda e: e.time_range.start)
    n = len(labels)
    if len(kern) != n * a.calls:
        raise SystemExit(f"bench_upsample: {len(kern)} generator kernels traced, expected {n} x {a.calls}")
    for c in range(a.calls):
        per_call.append([(e.name, e.time_range.elapsed_us() / 1e3) for e in kern[c * n:(c + 1) * n]])
    eng.close()

    launches = []
    for li, lab in enumerate(labels):
        t = [per_call[c][li][1] for c in range(a.calls)]
        row = {"launch": li, "label": lab, "kernel": per_call[0][li][0], "ms": float(np.median(t)), "ms_min": float(np.min(t)),
               "ms_max": float(np.max(t))}
        if lab.endswith(".ups"):
            i = int(lab[5])
            by, fl = ups_work(i, a.batch, T)
            row.update(dram_bytes=by, flop=fl, bound_ms=max(by / 3.35e12, fl / 989e12) * 1e3)
        launches.append(row)
    ups13 = sum(r["ms"] for r in launches if r["label"] in ("stage1.ups", "stage2.ups", "stage3.ups"))
    res = {"card": gpu, "sm_clock_mhz": clk.mhz, "sm_clock_samples": clk.samples, "torch_device": torch.cuda.get_device_name(0),
           "batch": a.batch, "mel_frames": T, "precision": a.precision, "calls": a.calls,
           "call_ms": {"mean": float(np.mean(call_ms)), "min": float(np.min(call_ms)), "max": float(np.max(call_ms))},
           "stages": {n: {"mean": float(np.mean(v)), "min": float(np.min(v)), "max": float(np.max(v))} for n, v in stage_ms.items()},
           "launches": launches, "ups_stage1_3_ms": ups13,
           "ups_all_ms": sum(r["ms"] for r in launches if r["label"].endswith(".ups"))}
    text = json.dumps(res, indent=1)
    print(text)
    if a.out:
        a.out.parent.mkdir(parents=True, exist_ok=True)
        a.out.write_text(text + "\n")


if __name__ == "__main__":
    main()
