"""Generate golden vectors for the HiFiGAN path from the REFERENCE ITSELF.

Run where a checkout of NTT123/vietTTS is available (VIETTTS_REFERENCE=<path>):

    python tests/golden/make_golden.py

What it does
  1. draws the seeded synthetic Haiku-layout parameters (viettts_b200.synthetic),
  2. maps them back to the torch layout (inverse of the reference converter),
     loads them into the reference's own `vietTTS.hifigan.torch_model.Generator`
     (torch_model.py:156-218, the model the Haiku weights are converted FROM),
  3. runs the reference's own `convert_to_haiku`
     (convert_torch_model_to_haiku.py:27-62) on that torch checkpoint and asserts
     that the pickle it writes equals the parameters of step 1 bit for bit
     (pins the layout contract: swapaxes(0,2) for Conv1d, rot90 for ConvTranspose1d),
  4. runs the reference torch forward on seeded mels and stores input + output
     (+ a few intermediate activations) in tests/golden/hifigan_ref_*.npz.

The reference's JAX/Haiku Generator (hifigan/model.py) cannot be imported here
(jax / dm-haiku absent); torch_model.py is the reference's own second
implementation of the same network and IS importable.
"""
from __future__ import annotations

import json
import os
import pickle
import sys
import tempfile
import types
from pathlib import Path

import numpy as np
import torch

REPO = Path(__file__).resolve().parents[2]
REF = Path(os.environ.get("VIETTTS_REFERENCE", "vietTTS-reference"))   # a checkout of NTT123/vietTTS
sys.path.insert(0, str(REPO))

from viettts_b200 import synthetic  # noqa: E402


def _import_reference():
    """Import vietTTS.hifigan.{torch_model,convert_torch_model_to_haiku} without
    triggering vietTTS/__init__ side effects."""
    import importlib.util

    pkg = types.ModuleType("vietTTS")
    pkg.__path__ = [str(REF / "vietTTS")]
    sys.modules["vietTTS"] = pkg
    sub = types.ModuleType("vietTTS.hifigan")
    sub.__path__ = [str(REF / "vietTTS" / "hifigan")]
    sys.modules["vietTTS.hifigan"] = sub
    mods = {}
    for name in ("config", "torch_model", "convert_torch_model_to_haiku"):
        spec = importlib.util.spec_from_file_location(
            f"vietTTS.hifigan.{name}", REF / "vietTTS" / "hifigan" / f"{name}.py"
        )
        m = importlib.util.module_from_spec(spec)
        sys.modules[f"vietTTS.hifigan.{name}"] = m
        spec.loader.exec_module(m)
        mods[name] = m
    return mods


def haiku_to_torch_state(hk: dict) -> dict:
    """Inverse of convert_to_haiku's mapping, for a weight-norm-free Generator."""
    sd = {}

    def conv(w):  # [K,Cin,Cout] -> [Cout,Cin,K]
        return torch.from_numpy(np.ascontiguousarray(np.swapaxes(w, 0, 2)))

    def convT(w):  # [K,Cout,Cin] -> [Cin,Cout,K]  (inverse of rot90(k=1, axes=(0,2)))
        return torch.from_numpy(np.ascontiguousarray(np.rot90(w, k=-1, axes=(0, 2))))

    for name, d in hk.items():
        short = name.split("generator/~/")[1]
        if short == "conv1_d":
            key, f = "conv_pre", conv
        elif short == "conv1_d_1":
            key, f = "conv_post", conv
        elif short.startswith("ups_"):
            key, f = f"ups.{short[4:]}", convT
        else:
            rb, cv = short.split("/~/")
            n = rb.split("_")[-1]
            y, z = cv.split("_")
            key, f = f"resblocks.{n}.{y}.{z}", conv
        sd[key + ".weight"] = f(d["w"])
        sd[key + ".bias"] = torch.from_numpy(d["b"].copy())
    return sd


def main():
    mods = _import_reference()
    tm, cv = mods["torch_model"], mods["convert_torch_model_to_haiku"]
    h = cv.AttrDict(json.loads((REF / "assets/hifigan/config.json").read_text()))
    hk = synthetic.hifigan_params(1234)
    assert synthetic.n_params(hk) == 13_926_017

    torch.manual_seed(0)
    gen = tm.Generator(h)
    gen.eval()
    gen.remove_weight_norm()
    missing = gen.load_state_dict(haiku_to_torch_state(hk), strict=True)
    print("loaded synthetic weights into reference torch Generator:", missing)

    # --- step 3: run the reference's own converter on a weight-normed checkpoint ---
    # convert_to_haiku builds Generator(h) WITH weight norm and loads state_dict["generator"],
    # so store weight_g/weight_v such that g*v/|v| == w exactly (g=|v|, v=w).
    gen_wn = tm.Generator(h)
    sd_plain = haiku_to_torch_state(hk)
    sd_wn = {}
    for k, v in gen_wn.state_dict().items():
        if k.endswith("weight_v"):
            sd_wn[k] = sd_plain[k[: -len("_v")]]
        elif k.endswith("weight_g"):
            w = sd_plain[k[: -len("_g")]]
            sd_wn[k] = w.reshape(w.shape[0], -1).norm(dim=1).reshape(v.shape)
        else:
            sd_wn[k] = sd_plain[k]
    with tempfile.TemporaryDirectory() as td:
        ck = os.path.join(td, "g_synth")
        torch.save({"generator": sd_wn}, ck)
        cwd = os.getcwd()
        os.chdir(td)
        try:
            a = types.SimpleNamespace(checkpoint_file=ck)
            cv.convert_to_haiku(a, h, torch.device("cpu"))
            with open(Path(td) / "assets/infore/hifigan/hk_hifi.pickle", "rb") as f:
                hk_ref = pickle.load(f)
        finally:
            os.chdir(cwd)
    assert set(hk_ref) == set(hk), (sorted(set(hk_ref) ^ set(hk))[:5])
    worst = 0.0
    for k in hk:
        for kk in ("w", "b"):
            assert hk_ref[k][kk].shape == hk[k][kk].shape, (k, kk)
            worst = max(worst, float(np.max(np.abs(hk_ref[k][kk] - hk[k][kk]) / (np.abs(hk[k][kk]) + 1e-6))))
    # weight norm g*v/|v| re-multiplication costs ~1 ulp; layout must be exact
    print("converter round trip: max relative deviation (weight-norm ulp noise) =", worst)
    assert worst < 1e-5

    out_dir = Path(__file__).resolve().parent
    # --- step 3b: converter fixture with a NON-trivial weight norm (random g), a few small tensors only ---
    rng = np.random.default_rng(11)
    sd_wn2 = {k: (v * torch.from_numpy(rng.uniform(0.5, 1.5, size=tuple(v.shape)).astype(np.float32)) if k.endswith("weight_g") else v)
              for k, v in sd_wn.items()}
    with tempfile.TemporaryDirectory() as td:
        ck = os.path.join(td, "g_synth2")
        torch.save({"generator": sd_wn2}, ck)
        cwd = os.getcwd()
        os.chdir(td)
        try:
            cv.convert_to_haiku(types.SimpleNamespace(checkpoint_file=ck), h, torch.device("cpu"))
            with open(Path(td) / "assets/infore/hifigan/hk_hifi.pickle", "rb") as f:
                hk_ref2 = pickle.load(f)
        finally:
            os.chdir(cwd)
    fx = {}
    for tname, hname in (("ups.3", "generator/~/ups_3"), ("ups.2", "generator/~/ups_2"),
                         ("resblocks.9.convs1.0", "generator/~/res_block1_9/~/convs1_0"),
                         ("resblocks.11.convs2.2", "generator/~/res_block1_11/~/convs2_2"),
                         ("conv_post", "generator/~/conv1_d_1")):
        for suffix in ("weight_g", "weight_v", "bias"):
            fx[f"torch/{tname}.{suffix}"] = sd_wn2[f"{tname}.{suffix}"].numpy()
        fx[f"haiku/{hname}/w"] = np.ascontiguousarray(hk_ref2[hname]["w"])
        fx[f"haiku/{hname}/b"] = hk_ref2[hname]["b"]
    np.savez_compressed(out_dir / "hifigan_converter_ref.npz", **fx)
    print("converter fixture:", len(fx), "arrays")

    for tag, (B, T, seed) in {"small": (2, 12, 7), "t32": (1, 32, 0)}.items():
        mel = synthetic.mel_input(seed, B, T)
        acts = {}
        with torch.no_grad():
            x = torch.from_numpy(mel).transpose(1, 2)  # NCW for the torch reference
            # replicate Generator.forward (torch_model.py:194-209) while tapping activations
            y = gen.conv_pre(x)
            acts["pre"] = y.transpose(1, 2).numpy().copy()
            import torch.nn.functional as F
            for i in range(gen.num_upsamples):
                y = F.leaky_relu(y, tm.LRELU_SLOPE)
                y = gen.ups[i](y)
                if i == 0:
                    acts["ups_0"] = y.transpose(1, 2).numpy().copy()
                xs = None
                for j in range(gen.num_kernels):
                    r = gen.resblocks[i * gen.num_kernels + j](y)
                    xs = r if xs is None else xs + r
                y = xs / gen.num_kernels
                if i == 0:
                    acts["stage_0"] = y.transpose(1, 2).numpy().copy()
            y = torch.tanh(gen.conv_post(F.leaky_relu(y)))
            wav_tapped = y.squeeze(1).numpy()
            wav = gen(x).squeeze(1).numpy()  # the reference's own forward
        assert np.array_equal(wav, wav_tapped)
        rms = {k: float(np.sqrt(np.mean(v**2))) for k, v in acts.items()}
        print(tag, "wav rms", float(np.sqrt(np.mean(wav**2))), "max", float(np.abs(wav).max()), rms)
        np.savez_compressed(
            out_dir / f"hifigan_ref_{tag}.npz",
            mel=mel,
            wav=wav.astype(np.float32),
            pre=acts["pre"].astype(np.float32) if tag == "small" else np.zeros(0, np.float32),
            ups_0=acts["ups_0"].astype(np.float32) if tag == "small" else np.zeros(0, np.float32),
            stage_0=acts["stage_0"].astype(np.float32) if tag == "small" else np.zeros(0, np.float32),
            weight_seed=np.array(1234),
            weight_checksum=np.array(weight_checksum(hk)),
        )
    print("wrote fixtures to", out_dir)


def weight_checksum(hk: dict) -> float:
    """Order-independent float64 checksum, so tests can assert they regenerated
    the same synthetic weights the fixture was made with."""
    s = 0.0
    for k in sorted(hk):
        for kk in sorted(hk[k]):
            a = hk[k][kk].astype(np.float64).ravel()
            s += float(np.dot(a, np.cos(np.arange(a.size) * 1e-3)))
    return s


if __name__ == "__main__":
    main()
