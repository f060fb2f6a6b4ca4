"""GPU parity of the autoregressive decoder scan with several row groups in one launch.

decoder_scan_kernel stages 32 rows at a time and runs up to four such groups under the same barriers of a frame;
each CTA computes two prenet columns of every row.  These tests put 100 and 128 ragged rows in one launch and check
the rows at the group edges (0, 31, 32, 63, 64, 95, 96 and the last row):

  * MASK mode: against the CPU oracle run on the row alone (mel L-inf <= 1e-3 after the scan, as test_gpu_nat.py),
    and against the same row run alone on the GPU (bit for bit);
  * SEED mode: against the oracle fed the masks rebuilt from the documented threefry stream, which is keyed by the row
    index, so rows of groups 2-4 must draw their own masks.

Utterances are short (6-21 frames, ending at different frames within each group) so that the oracle stays cheap."""
import numpy as np
import pytest

from helpers.threefry import prenet_keep_masks
from oracle import nat_oracle as no
from viettts_b200 import synthetic

pytestmark = pytest.mark.gpu
MEL_LINF = 1e-3


@pytest.fixture(scope="module")
def eng(acoustic_ckpt):
    from viettts_b200.engine import Engine
    e = Engine(0)
    e.load_acoustic(acoustic_ckpt)
    yield e
    e.close()


def _batch(B):
    """B ragged utterances: 6-14 phonemes, 6-21 frames."""
    utts = []
    for b in range(B):
        tk, dur = synthetic.utterance(300 + b, 6 + (b * 5) % 9, 0.1 + 0.03 * ((b * 7) % 9))
        d, n = no.seconds_to_frames(dur)
        utts.append((np.asarray(tk, np.int32), d[0], n))
    Lmax = max(len(u[0]) for u in utts)
    tokens = np.zeros((B, Lmax), np.int32)
    dur = np.zeros((B, Lmax), np.float32)
    for b, (tk, d, _) in enumerate(utts):
        tokens[b, : len(tk)] = tk
        dur[b, : len(tk)] = d
    lens = np.array([len(u[0]) for u in utts], np.int32)
    nfs = np.array([u[2] for u in utts], np.int32)
    return utts, tokens, dur, lens, nfs


def _edge_rows(B):
    return sorted({r for r in (0, 31, 32, 63, 64, 95, 96) if r < B} | {B - 1})


@pytest.mark.parametrize("B", [128, 100])
def test_mask_mode_group_edges(eng, acoustic_ckpt, B):
    utts, tokens, dur, lens, nfs = _batch(B)
    N = int(nfs.max())
    masks = synthetic.dropout_masks(21, B, N)
    mel = eng.predict_mel(tokens, dur, lengths=lens, n_frames=nfs, masks=masks)
    for b in _edge_rows(B):
        tk, d, n = utts[b]
        ref = no.inference(acoustic_ckpt, tk[None], d[None], n, masks[b : b + 1, :n]).numpy()
        e_ref = float(np.abs(mel[b, :n] - ref[0]).max())
        alone = eng.predict_mel(tokens[b : b + 1], dur[b : b + 1], lengths=lens[b : b + 1], n_frames=nfs[b : b + 1], masks=masks[b : b + 1])
        e_alone = float(np.abs(mel[b, :n] - alone[0, :n]).max())
        print(f"B={B} row {b}: N={n} oracle {e_ref:.3e} alone {e_alone:.3e}")
        assert e_ref < MEL_LINF
        assert np.array_equal(mel[b, :n], alone[0, :n]), (b, e_alone)
        assert np.all(mel[b, n:] == 0.0)


@pytest.mark.parametrize("B", [128, 100])
def test_seed_mode_group_edges(eng, acoustic_ckpt, B):
    utts, tokens, dur, lens, nfs = _batch(B)
    seed = (11 << 32) | 4321
    mel = eng.predict_mel(tokens, dur, lengths=lens, n_frames=nfs, seed=seed)
    for b in _edge_rows(B):
        tk, d, n = utts[b]
        masks = prenet_keep_masks(seed, [b], n)
        assert 0.4 < masks.mean() < 0.6
        ref = no.inference(acoustic_ckpt, tk[None], d[None], n, masks).numpy()
        e = float(np.abs(mel[b, :n] - ref[0]).max())
        print(f"B={B} row {b}: N={n} seed-stream oracle {e:.3e}")
        assert e < MEL_LINF
