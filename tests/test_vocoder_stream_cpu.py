"""CPU: the streaming generator's lookahead D, pinned independently of the library's layer table.

D is the generator's right receptive field in whole mel frames: after P frames, the first 256 * (P - D) samples of the
one-shot waveform no longer depend on any later frame, and D - 1 would be too few.  Checked on the float64 oracle with
synthetic weights, then against vtts_vocoder_stream_lookahead() (needs the built library, not a device)."""
import numpy as np
import pytest
import torch

from oracle import hifigan_oracle as ho
from viettts_b200 import synthetic

T, P = 40, 26


@pytest.fixture(scope="module")
def oracle_d(hifigan_params):
    mel = synthetic.mel_input(7, 1, T)
    pert = mel.copy()
    pert[:, P:] = synthetic.mel_input(8, 1, T - P)[:, :]
    a = ho.mel2wave(hifigan_params, mel, torch.float64).reshape(-1)
    b = ho.mel2wave(hifigan_params, pert, torch.float64).reshape(-1)
    diff = np.abs(a - b)
    first = int(np.argmax(diff > 0))          # first sample that sees a frame >= P
    assert diff.max() > 1e-3 and first > 0
    D = P - first // 256
    print(f"lookahead D = {D} frames: first sample seeing frame {P} is {first} = 256 * {P} - {256 * P - first}")
    return D, first, diff


def test_lookahead_is_the_receptive_field(oracle_d):
    D, first, diff = oracle_d
    # frames >= P leave wav[: 256 (P - D)] unchanged ...
    assert np.all(diff[: 256 * (P - D)] == 0)
    # ... and D - 1 is not enough: frame P - D + 1 already has samples that see frame P (at the edge of the receptive
    # field the influence is small, ~1e-11, but in float64 a sample outside it is exactly unchanged)
    assert np.any(diff[256 * (P - D): 256 * (P - D + 1)] > 0)
    assert first < 256 * (P - D + 1)


def test_library_lookahead_matches_oracle(oracle_d):
    from viettts_b200 import _lib, build
    build.build()
    assert _lib.load().vtts_vocoder_stream_lookahead() == oracle_d[0]
