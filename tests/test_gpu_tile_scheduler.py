"""GPU: the run-time tile scheduler of the tensor-core conv and fused-pair kernels.

Tiles go to CTAs in whatever order the CTAs ask for them, and each launch resets the ticket counters for the next one.
A tile's arithmetic does not depend on the CTA that runs it, so repeated calls of any shape must give identical bits,
also when calls of other shapes (other tile counts, skipped tiles of ragged rows) run in between."""
import numpy as np
import pytest

from viettts_b200 import synthetic

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng(hifigan_params):
    from viettts_b200.engine import Engine
    e = Engine(0)
    e.load_hifigan(hifigan_params)
    yield e
    e.set_fused_pairs(True)
    e.close()


@pytest.mark.parametrize("fused", [True, False])
def test_repeated_calls_are_bit_identical(eng, fused):
    eng.set_fused_pairs(fused)
    calls = [(synthetic.mel_input(1, 3, 40), np.array([40, 23, 1], np.int32)),
             (synthetic.mel_input(2, 1, 9), np.array([9], np.int32)),
             (synthetic.mel_input(3, 4, 64), np.array([64, 64, 64, 64], np.int32))]
    first = [eng.mel2wave(mel, n_frames=nf) for mel, nf in calls]
    for _ in range(2):
        for (mel, nf), w0 in zip(calls, first):
            assert np.array_equal(eng.mel2wave(mel, n_frames=nf), w0)

