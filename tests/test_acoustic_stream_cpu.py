"""CPU: the streaming acoustic model's lookahead D_a and its emission schedule.

D_a is the postnet's right receptive field: after P decoder frames, postnet frames < P - D_a no longer depend on any
later frame, and D_a - 1 would be too few.  Checked on the float64 oracle with synthetic weights, then against
vtts_acoustic_stream_lookahead() (needs the built library, not a device)."""
import numpy as np
import pytest
import torch

from oracle import nat_oracle as no
from viettts_b200.engine import acoustic_stream_schedule

T, P = 60, 37


@pytest.fixture(scope="module")
def oracle_da(acoustic_ckpt):
    rng = np.random.default_rng(5)
    pre = rng.standard_normal((1, T, 80))
    pert = pre.copy()
    pert[:, P:] = rng.standard_normal((1, T - P, 80))
    Pp, Ss = acoustic_ckpt["params"], acoustic_ckpt["aux"]
    with torch.no_grad():
        a = (torch.as_tensor(pre) + no.postnet(Pp, Ss, torch.as_tensor(pre), torch.float64)).numpy()[0]
        b = (torch.as_tensor(pert) + no.postnet(Pp, Ss, torch.as_tensor(pert), torch.float64)).numpy()[0]
    diff = np.abs(a - b).max(axis=1)
    first = int(np.argmax(diff > 0))          # first frame that sees a frame >= P
    assert diff.max() > 1e-3 and first > 0
    return P - first, diff


def test_lookahead_is_the_postnet_receptive_field(oracle_da):
    D, diff = oracle_da
    assert D == 10
    assert np.all(diff[: P - D] == 0)         # frames >= P leave frames < P - D unchanged ...
    assert diff[P - D] > 0                    # ... and D - 1 is not enough


def test_library_lookahead_matches_oracle(oracle_da):
    from viettts_b200 import _lib, build
    build.build()
    assert _lib.load().vtts_acoustic_stream_lookahead() == oracle_da[0]


@pytest.mark.parametrize("n_frames,n_emit,F,expected", [
    (1, None, 5, [1]),                                 # shorter than the lookahead: all at the last push
    (9, None, 5, [0, 9]),
    (10, None, 1, [0] * 9 + [10]),
    (11, None, 1, [0] * 10 + [11]),                    # one frame past the lookahead: the last push emits everything ...
    (12, None, 1, [0] * 10 + [1, 11]),                 # ... frame 0 is final once 11 frames are scanned
    (11, None, 16, [11]),                              # one push does it all
    (150, None, 16, [6] + [16] * 8 + [16]),
    (150, 120, 16, [6] + [16] * 7 + [2]),              # trimmed: the scan stops at n_emit + D_a = 130 frames
    (150, 145, 64, [54, 64, 27]),                      # n_emit + D_a past the end: scan everything
    (937, None, 64, [54] + [64] * 13 + [51]),
])
def test_emission_schedule(n_frames, n_emit, F, expected):
    got = acoustic_stream_schedule(n_frames, n_emit, F, 10)
    assert got == expected
    assert sum(got) == (n_frames if n_emit is None else n_emit)


@pytest.mark.parametrize("n_frames", [1, 9, 10, 11, 24, 150, 937])
@pytest.mark.parametrize("F", [1, 5, 16, 64])
def test_schedule_properties(n_frames, F):
    """After P frames scanned a slot has emitted min(n_emit, max(0, P - 10)), and the last push emits the rest."""
    for n_emit in sorted({1, max(1, n_frames // 2), n_frames}):
        counts = acoustic_stream_schedule(n_frames, n_emit, F, 10)
        end = min(n_frames, n_emit + 10)
        assert len(counts) == -(-end // F)
        assert sum(counts) == n_emit and all(c >= 0 for c in counts)
        for k in range(len(counts) - 1):
            assert sum(counts[: k + 1]) == min(n_emit, max(0, (k + 1) * F - 10))
