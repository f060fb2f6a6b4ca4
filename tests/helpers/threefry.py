"""numpy restatement of the device's VTTS_DROPOUT_SEED streams (csrc/nat.cu `threefry2x32`, `keep_scale`, `zone_keep`).

Both draws use threefry2x32 keyed by the 64-bit seed (k0 = low word, k1 = high word) with the counter
(frame, row << 12 | entry) and keep on the first output word o0:
  prenet keep   entry = layer * 256 + unit                 kept when o0 < 2^31      (p = 0.5)
  zoneout       entry = 512 + which * 512 + unit           kept when o0 < 429496730 (p = 0.1, 1 = keep the previous state)
where `which` runs over the state tree (h0, c0, h1, c1).  `row` is the row's index in the call, so a row's masks
depend on its position in the batch but not on the batch's padded frame count."""
import numpy as np

ZONE_THRESHOLD = 429496730      # 0.1 * 2^32


def threefry2x32(k0, k1, c0, c1):
    """Threefry-2x32, 20 rounds, on uint32 arrays c0, c1 (broadcast) with the key words k0, k1."""
    M = np.uint32
    k0, k1, c0, c1 = (np.asarray(v, dtype=np.uint32) for v in (k0, k1, c0, c1))
    ks = [k0, k1, M(0x1BD11BDA) ^ k0 ^ k1]
    x0, x1 = c0 + k0, c1 + k1
    R = [[13, 15, 26, 6], [17, 29, 16, 24]]
    with np.errstate(over="ignore"):
        for blk in range(5):
            for r in R[blk & 1]:
                x0 = x0 + x1
                x1 = (x1 << M(r)) | (x1 >> M(32 - r))
                x1 = x1 ^ x0
            x0 = x0 + ks[(blk + 1) % 3]
            x1 = x1 + ks[(blk + 2) % 3] + M(blk + 1)
    return x0, x1


def _draw(seed, rows, n, entries):
    """o0 of the counters (frame t, row << 12 | entry): uint32 [len(rows), n, *entries.shape]"""
    rows = np.asarray(rows, np.uint32).reshape(-1, 1, *([1] * entries.ndim))
    t = np.arange(n, dtype=np.uint32).reshape(1, n, *([1] * entries.ndim))
    e = entries.astype(np.uint32)[None, None]
    c0 = np.broadcast_to(t, (rows.shape[0], n) + entries.shape)
    c1 = (rows << np.uint32(12)) | e
    o0, _ = threefry2x32(np.uint32(seed & 0xFFFFFFFF), np.uint32(seed >> 32), c0, np.broadcast_to(c1, c0.shape))
    return o0


def prenet_keep_masks(seed, rows, n):
    """uint8 [len(rows), n, 2, 256]: the prenet keep-masks that rows `rows` of a call draw over frames 0..n-1"""
    entries = np.arange(2, dtype=np.uint32)[:, None] * 256 + np.arange(256, dtype=np.uint32)[None, :]
    return (_draw(seed, rows, n, entries) < np.uint32(0x80000000)).astype(np.uint8)


def zoneout_masks(seed, rows, n):
    """uint8 [len(rows), n, 4, 512] in the (h0, c0, h1, c1) order, 1 = keep the previous state"""
    entries = 512 + np.arange(4, dtype=np.uint32)[:, None] * 512 + np.arange(512, dtype=np.uint32)[None, :]
    return (_draw(seed, rows, n, entries) < np.uint32(ZONE_THRESHOLD)).astype(np.uint8)
