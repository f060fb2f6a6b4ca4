"""Does the ConvTranspose (`ups`) launch of each generator stage wait on re-reads of its three chain inputs?

    python scripts/bench_ups_l2.py [--batch 32] [--rounds 5] [--reps 20] [--precision bf16x3] [--out FILE.json]

Each stage's ConvTranspose runs alone through Engine.debug_hifigan_layer (layer 1 + i, the code the forward runs) at
the flagship shape: B = 32 rows of 312 mel frames (bench.py's synthetic utterances, their n_frames), seeded inputs.
Stages 1..3 read the 3-way mean of the previous stage's ResBlock chains; they are timed two ways:

  (a) three distinct input tensors, as in the forward;
  (b) one tensor passed three times: the same instructions and FLOP, a third of the input bytes and of the L2
      working set, the same output writes.

Stage 0 reads conv_pre's output alone and is timed in (a) only.  (a) and (b) alternate, `--rounds` times, each round
`--reps` launches after a warm-up, under torch.profiler (CUDA activities): the kernel's device time, without the hook's
host synchronisation.  Per variant the median over all launches is reported.  A launch
bound by DRAM traffic that L2 should have absorbed runs markedly faster in (b); one bound elsewhere times alike.

Per stage and variant also the per-role stall counters of one launch (Engine.tc_stats, SM clocks averaged over the
CTAs): the consumer warpgroup's whole run, its epilogue, its waits for activations and for weights, the weight
producer's and the converters' waits for free ring stages.

Per stage also the algorithmic bytes (each input read once, the output written once) and their rate at the median of
(a).  The card name, power limit and SM clock are read (nvidia-smi, read-only) in the same run.  Prints one JSON
object; `--out` also writes it."""
from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
sys.path.insert(0, str(Path(__file__).resolve().parent))
from bench_upsample import C0, RATES, SmClock, card, n_frames  # noqa: E402
from viettts_b200 import synthetic  # noqa: E402
from viettts_b200.engine import Engine  # noqa: E402


def ups_bytes(i, B, T):
    """DRAM bytes of the ConvTranspose of stage i with every input read once and the output written once."""
    scale = int(np.prod(RATES[:i])) if i else 1
    rows_in, c = T * scale, C0 >> i
    n_in = 1 if i == 0 else 3
    return 4 * B * rows_in * c * n_in + 4 * B * rows_in * RATES[i] * (c // 2)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--precision", default="bf16x3", choices=("bf16x3", "fp16"))
    ap.add_argument("--out", type=Path, default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_ups_l2: no CUDA device")
    dev = torch.device("cuda", 0)
    gpu = card()
    eng = Engine(0)
    eng.load_hifigan(synthetic.hifigan_params(1234))
    eng.set_precision(a.precision)
    nfs = n_frames(a.batch)
    T = int(nfs.max())
    nf_t = torch.from_numpy(nfs).to(dev)
    gen = torch.Generator(device=dev).manual_seed(0)

    def time_ms(layer, xs, out):
        """device ms of each of `reps` launches of the layer's tc_conv_kernel"""
        for _ in range(2):
            eng.debug_hifigan_layer(layer, xs, [out], nf_t, T)
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(a.reps):
                eng.debug_hifigan_layer(layer, xs, [out], nf_t, T)
        kern = [e.time_range.elapsed_us() / 1e3 for e in prof.events()
                if e.device_type == torch.autograd.DeviceType.CUDA and "tc_conv_kernel" in e.name]
        if len(kern) != a.reps:
            raise SystemExit(f"bench_ups_l2: {len(kern)} tc_conv_kernel launches traced, expected {a.reps}")
        return kern

    def counters(layer, xs, out):
        eng.tc_stats(True)
        eng.debug_hifigan_layer(layer, xs, [out], nf_t, T)
        cnt = eng.tc_stats(False).astype(np.float64)
        cnt = cnt[cnt[:, 0] > 0]
        names = ("consumer", "epilogue", "a_wait", "w_wait", "producer_wait", "converter_wait")
        return {"ctas": int(cnt.shape[0]), **{n: float(cnt[:, c].mean()) for c, n in enumerate(names)}}

    stages = []
    with SmClock() as clk:
        for i in range(4):
            scale = int(np.prod(RATES[:i])) if i else 1
            c = C0 >> i
            xs = [torch.randn((a.batch, T * scale, c), device=dev, generator=gen) for _ in range(1 if i == 0 else 3)]
            out = torch.empty((a.batch, T * scale * RATES[i], c // 2), device=dev)
            variants = {"a_distinct": xs} if i == 0 else {"a_distinct": xs, "b_same": [xs[0]] * 3}
            ms = {k: [] for k in variants}
            for _ in range(a.rounds):
                for k, v in variants.items():
                    ms[k] += time_ms(1 + i, v, out)
            by = ups_bytes(i, a.batch, T)
            row = {"stage": i, "layer": 1 + i, "cin": c, "rows_in": T * scale, "algorithmic_bytes": by}
            for k, v in ms.items():
                row[k] = {"ms_median": float(np.median(v)), "ms_min": float(np.min(v)), "ms_max": float(np.max(v)), "launches": len(v),
                          "counters_clk": counters(1 + i, variants[k], out)}
            row["a_tb_per_s"] = by / (row["a_distinct"]["ms_median"] * 1e-3) / 1e12
            if i > 0:
                row["a_over_b"] = row["a_distinct"]["ms_median"] / row["b_same"]["ms_median"]
            stages.append(row)
            del xs, out
    eng.close()
    res = {"card": gpu, "sm_clock_mhz": clk.mhz, "sm_clock_samples": clk.samples, "torch_device": torch.cuda.get_device_name(0),
           "batch": a.batch, "mel_frames": T, "precision": a.precision, "rounds": a.rounds, "reps": a.reps, "stages": stages,
           "ups_all_ms_a": sum(s["a_distinct"]["ms_median"] for s in stages)}
    text = json.dumps(res, indent=1)
    print(text)
    if a.out:
        a.out.parent.mkdir(parents=True, exist_ok=True)
        a.out.write_text(text + "\n")


if __name__ == "__main__":
    main()
