"""The reference's dropout / zoneout masks, drawn the way JAX + Haiku draw them.

The reference keeps prenet dropout live at inference and seeds it from the checkpoint's `rng`
(vietTTS/nat/model.py:95-100,132; nat/text2mel.py:65-82): Haiku's `hk.next_rng_key()` walks a split chain
(`key, sub = jax.random.split(key)`) and `hk.dropout` draws `jax.random.bernoulli(sub, 0.5, x.shape)`.  Both are
defined on the counter-based threefry2x32 generator, so the masks are a pure function of the two rng words and can be
reproduced without JAX.  This module restates that function in numpy (host side; a few hundred thousand block-cipher
evaluations per utterance).  The library draws the same masks on the device (VTTS_DROPOUT_REFERENCE, `rng=` in
`Engine`), which makes the drop-in `predict_mel` / GTA `forward_fn` sample-wise (not just statistically) equal to the
reference; this module is the host oracle the tests compare the device's masks with, and a source of explicit masks
for the VTTS_DROPOUT_MASK path.

Layout restated (jax/_src/prng.py, the classic layout, `jax_threefry_partitionable=False`, the default of every jax
release the 2021 reference can run on):
  threefry_2x32(key, counts)   counts are cut into halves x0 | x1; (y0, y1) = threefry2x32(key, (x0, x1)); concat(y0, y1)
  split(key, n)                threefry_2x32(key, arange(2n)).reshape(n, 2)
  random_bits(key, shape)      threefry_2x32(key, arange(prod(shape))).reshape(shape)
  uniform                      bitcast_f32((bits >> 9) | 0x3F800000) - 1
  bernoulli(key, p, shape)     uniform < p
Haiku (base.py PRNGSequence): `next_rng_key()` = `new = split(key, 2); key = new[0]; return new[1]`; inside
`hk.dynamic_unroll` the sequence is carried through the steps as if the loop were unrolled.

Pinned by tests/test_refshim_rng.py (Random123 known answers, JAX's documented PRNGKey(0) outputs) and by the golden
masks recorded while executing the reference's own source (tests/golden/nat_ref_*.npz).
"""
from __future__ import annotations

import numpy as np

_ROT = ((13, 15, 26, 6), (17, 29, 16, 24))


def _rotl(x, r):
    return (x << np.uint32(r)) | (x >> np.uint32(32 - r))


def threefry2x32(k0, k1, x0, x1):
    """Threefry-2x32, 20 rounds, on uint32 arrays x0, x1 with the key words k0, k1."""
    with np.errstate(over="ignore"):
        k0, k1 = np.uint32(k0), np.uint32(k1)
        ks = (k0, k1, np.uint32(0x1BD11BDA) ^ k0 ^ k1)
        x0 = np.asarray(x0, np.uint32) + ks[0]
        x1 = np.asarray(x1, np.uint32) + ks[1]
        for blk in range(5):
            for r in _ROT[blk & 1]:
                x0 = x0 + x1
                x1 = _rotl(x1, r) ^ x0
            x0 = x0 + ks[(blk + 1) % 3]
            x1 = x1 + ks[(blk + 2) % 3] + np.uint32(blk + 1)
    return x0, x1


def random_bits(key, n: int) -> np.ndarray:
    """jax random_bits(key, 32, (n,)): uint32 [n]."""
    key = np.asarray(key, np.uint32).ravel()
    m = n + (n & 1)
    c = np.arange(m, dtype=np.uint32)
    if m != n:
        c[-1] = 0
    h = m // 2
    y0, y1 = threefry2x32(key[0], key[1], c[:h], c[h:])
    return np.concatenate([y0, y1])[:n]


def split(key, num: int = 2) -> np.ndarray:
    return random_bits(key, 2 * num).reshape(num, 2)


def subkey_chain(key, n: int) -> np.ndarray:
    """The n sub-keys n consecutive hk.next_rng_key() calls return, starting from `key`: uint32 [n,2]."""
    key = np.asarray(key, np.uint32).ravel().copy()
    out = np.empty((n, 2), np.uint32)
    for i in range(n):
        new = split(key, 2)
        key, out[i] = new[0], new[1]
    return out


def bernoulli_bits(subkey, n: int) -> np.ndarray:
    """The uint32 words behind bernoulli(subkey, p, shape) with prod(shape) = n (p = 0.5 keeps where word < 2^31)."""
    return random_bits(subkey, n)


def bernoulli(subkey, p: float, shape) -> np.ndarray:
    n = int(np.prod(shape))
    bits = random_bits(subkey, n)
    u = ((bits >> np.uint32(9)) | np.uint32(0x3F800000)).view(np.float32) - np.float32(1.0)
    return (u < np.float32(p)).reshape(shape)


def rng_key(rng) -> np.ndarray:
    """The checkpoint's `rng` entry (a uint32[2] jax PRNGKey) as two words."""
    k = np.asarray(rng).astype(np.uint64).ravel()
    if k.size != 2:
        raise ValueError(f"rng must hold two uint32 words, got shape {np.asarray(rng).shape}")
    return k.astype(np.uint32)


def inference_keep_masks(rng, batch: int, n_frames: int) -> np.ndarray:
    """Keep-masks of AcousticModel.inference (model.py:123-144) for a reference call with `batch` rows:
    per decoder step two draws of shape [batch, 256] (prenet dropout 1, then 2).  uint8 [batch, n_frames, 2, 256]."""
    subs = subkey_chain(rng_key(rng), 2 * n_frames)
    out = np.empty((batch, n_frames, 2, 256), np.uint8)
    for i in range(2 * n_frames):
        out[:, i // 2, i % 2] = bernoulli(subs[i], 0.5, (batch, 256))
    return out


def teacher_forced_masks(rng, batch: int, n_frames: int):
    """Masks of AcousticModel.__call__ (model.py:146-169): prenet dropouts over [B,N,256] (two draws), then the zoneout
    masks of the state tree (layer0.hidden, layer0.cell, layer1.hidden, layer1.cell), Bernoulli(0.1) over [B,N,512].
    Returns (keep uint8 [B,N,2,256], zone uint8 [B,N,4,512]; zone 1 = keep the previous state)."""
    subs = subkey_chain(rng_key(rng), 6)
    keep = np.stack([bernoulli(subs[i], 0.5, (batch, n_frames, 256)) for i in range(2)], axis=2).astype(np.uint8)
    zone = np.stack([bernoulli(subs[2 + i], 0.1, (batch, n_frames, 512)) for i in range(4)], axis=2).astype(np.uint8)
    return keep, zone
