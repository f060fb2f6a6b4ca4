"""Build recipe for libviettts_b200.so (sm_90a only, built in-tree so that the
.so travels to the GPU box with the repo snapshot)."""
from __future__ import annotations

import os
import subprocess
import sys
from pathlib import Path

PKG = Path(__file__).resolve().parent
CSRC = PKG / "csrc"
LIB = PKG / "libviettts_b200.so"
SOURCES = ["api.cu", "conv1d.cu", "tc_conv.cu", "hifigan.cu", "vocoder_stream.cu", "acoustic_stream.cu", "nat.cu", "melspec.cu",
           "resample.cu", "denoise.cu", "loudness.cu", "pitch.cu"]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC",
    "--expt-relaxed-constexpr",
]


def nvcc() -> str:
    cand = os.environ.get("NVCC") or "/usr/local/cuda/bin/nvcc"
    return cand if Path(cand).exists() else "nvcc"


def needs_build() -> bool:
    if not LIB.exists():
        return True
    t = LIB.stat().st_mtime
    deps = list(CSRC.glob("*.cu")) + list(CSRC.glob("*.cuh")) + [PKG.parent / "include" / "viettts_b200.h", Path(__file__)]
    return any(d.stat().st_mtime > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> Path:
    if not force and not needs_build():
        return LIB
    objs = []
    obj_dir = PKG / "build"
    obj_dir.mkdir(exist_ok=True)
    procs = []
    for s in SOURCES:
        o = obj_dir / (s[:-3] + ".o")
        cmd = [nvcc(), *NVCC_FLAGS, "-c", str(CSRC / s), "-o", str(o)]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
        procs.append((s, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(str(o))
    failed = False
    for s, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0 or verbose:
            sys.stderr.write(f"--- nvcc {s} ---\n{out}\n")
        failed |= p.returncode != 0
    if failed:
        raise RuntimeError("nvcc failed (see stderr)")
    cmd = [nvcc(), "-shared", "-o", str(LIB), *objs, "-gencode", "arch=compute_90a,code=sm_90a", "-lcudart", "-ldl"]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout)
        raise RuntimeError("link failed")
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
