"""Integer statement of the FLAC encoder (viettts_b200/csrc/flac.cu, vtts_flac_encode) and an independent, strict FLAC
decoder that judges its output.

The contract: the device writes exactly the bytes `encode` writes, in every vtts_precision mode.  Every decision below
is made in integers or in correctly rounded fp64 (+, -, *, / and rint only, never contracted into an FMA), so numpy and
the device reach the same integers.

encode(codes_int16, rate, block) -> bytes, a native FLAC stream (RFC 9639), mono, 16 bits, in the streamable subset:
  Stream header: "fLaC", one STREAMINFO block marked last: min = max block size = `block`, min / max frame size the
    actual byte sizes of the frames (0 without frames), the rate, 1 channel, 16 bits, the total samples n, MD5 zero.
  Frames: fixed blocking, frame i holds samples [i block, min((i + 1) block, n)).  A full frame states its size by the
    table code (256 .. 4096: codes 8 .. 12); the last, short frame always by the 8-bit (code 6) or 16-bit (code 7) field.
    The rate code is explicit (the subset forbids 0000): the table code of 8k, 16k, 22.05k, 24k, 32k, 44.1k, 48k, 88.2k,
    96k, 176.4k, 192k; else 8-bit kHz; else 16-bit Hz; else 16-bit tens of Hz; any other rate is rejected.  Channel
    assignment 0 (mono), sample-size code 4 (16 bits), the frame number in the UTF-8-style coding, CRC-8 (poly 0x07) of
    the header, one subframe, zero bits to a byte boundary, CRC-16 (poly 0x8005) of the whole frame.
  Subframe of a frame of n samples x (int16):
    CONSTANT when all n samples are equal.  Otherwise the candidate with the fewest subframe bits among FIXED orders
    0..4, LPC orders 1..12 and VERBATIM, in that order, the earlier one on a tie; a predictor needs order < n, and a
    candidate whose residual leaves the int32 range is skipped.  No wasted bits.
    Residual: Rice coding with 4-bit parameters k in [0, 14] (method 0, no escapes).  The partition order p runs over
    0 .. pmax, pmax the largest p <= 8 with n divisible by 2^p and (n >> p) > order.  A partition of cnt residuals r
    with u = zigzag(r) costs 4 + min_k (sum(u >> k) + cnt (k + 1)) bits (the smaller k on a tie); the residual costs
    6 + min_p of the partition sums (the smaller p on a tie).  All of it in integers.
  LPC analysis of a frame:
    window: w[i] = w[n - 1 - i] = floor(32768 (3 a^2 D - 2 a^3) / D^3) with a = 2 i + 1, D = 2 L, L = n >> 2, for
      i < L, and 32768 (1.0 in Q15) in between: a Tukey-like taper with a smoothstep edge, in integers;
    x_w = (x w + 2^14) >> 15; autocorrelation R[l] = sum_{i >= l} x_w[i] x_w[i - l], l = 0..12, in int64 (exact);
    Levinson-Durbin in fp64 over R (as doubles, exact): err = R[0]; for order i = 1..12 while err > 0:
      acc = R[i]; acc = acc - a[j] * R[i - 1 - j] for j = 0..i-2 in turn; k = acc / err;
      a[j] = a[j] - k * a[i - 2 - j] (j < i - 1, from the old a); a[i - 1] = k; err = err * (1 - k * k);
      the predictor of order i is a[0..i-1] (x[t] ~ sum_j a[j] x[t - 1 - j]), dropped if any value is not finite;
    quantization (libFLAC's rule): precision P by n (<= 192: 7, <= 384: 8, <= 576: 9, <= 1152: 10, <= 2304: 11, else
      12); cmax = max |a[j]| (0: the order is skipped); frexp(cmax) = (m, e); shift = clamp(P - e, 0, 15);
      err = 0.0; per j in order: err = err + a[j] * 2^shift; q = clip(rint(err), -2^(P-1), 2^(P-1) - 1) (half to
      even); err = err - q;
    prediction sum_j q[j] x[t - 1 - j] in int64, shifted right arithmetically by `shift`; r = x[t] - prediction.

decode(data) -> (int16 samples, rate, streaminfo) is written from the RFC, not from the encoder, and takes more than the
encoder writes: every subframe type, wasted bits, Rice with 4- and 5-bit parameters and escapes, every block-size and
rate code, the variable-blocksize flag.  It checks the sync code, both CRCs, the reserved bits and the padding, and
rejects negative LPC shifts, precision code 15 and partition orders that do not divide the block."""
from __future__ import annotations

import math

import numpy as np

BLOCKS = (256, 512, 1024, 2048, 4096)
RATE_CODES = {88200: 1, 176400: 2, 192000: 3, 8000: 4, 16000: 5, 22050: 6, 24000: 7, 32000: 8, 44100: 9, 48000: 10, 96000: 11}
BLOCK_CODES = {256: 8, 512: 9, 1024: 10, 2048: 11, 4096: 12}
MAX_FIXED, MAX_LPC, MAX_PORDER, MAX_RICE = 4, 12, 8, 14
HEADER_BYTES = 42
SUB_CONSTANT, SUB_VERBATIM, SUB_FIXED, SUB_LPC = "constant", "verbatim", "fixed", "lpc"


# ---- CRCs --------------------------------------------------------------------------------------------------------
def _crc_table(poly: int, width: int):
    top, mask, out = 1 << (width - 1), (1 << width) - 1, []
    for b in range(256):
        c = b << (width - 8)
        for _ in range(8):
            c = ((c << 1) ^ poly) & mask if c & top else (c << 1) & mask
        out.append(c)
    return out


_CRC8, _CRC16 = _crc_table(0x07, 8), _crc_table(0x8005, 16)


def crc8(data) -> int:
    c = 0
    for b in bytes(data):
        c = _CRC8[c ^ b]
    return c


def crc16(data) -> int:
    c = 0
    for b in bytes(data):
        c = ((c << 8) & 0xFFFF) ^ _CRC16[(c >> 8) ^ b]
    return c


# ---- stream parameters -------------------------------------------------------------------------------------------
def rate_code(rate: int):
    """(4-bit code, extra bits, extra value) of the frame header's rate field; ValueError for a rate FLAC cannot state"""
    r = int(rate)
    if r != rate or r < 1:
        raise ValueError(f"flac: rate {rate} must be a positive integer")
    if r in RATE_CODES:
        return RATE_CODES[r], 0, 0
    if r % 1000 == 0 and r // 1000 <= 255:
        return 12, 8, r // 1000
    if r <= 65535:
        return 13, 16, r
    if r % 10 == 0 and r // 10 <= 65535:
        return 14, 16, r // 10
    raise ValueError(f"flac: rate {rate} has no frame-header code (a table rate, kHz <= 255, Hz <= 65535 or tens of Hz "
                     f"<= 655350)")


def check_block(block: int) -> int:
    if block not in BLOCKS:
        raise ValueError(f"flac: block {block} must be one of {', '.join(map(str, BLOCKS))}")
    return int(block)


def utf8_number(v: int) -> bytes:
    """the UTF-8-style coding of a frame (< 2^31) or sample (< 2^36) number"""
    if v < 0x80:
        return bytes([v])
    n = 2
    while v >= 1 << (5 * n + 1):
        n += 1
    out = [0x80 | ((v >> (6 * i)) & 0x3F) for i in range(n - 1)][::-1]
    return bytes([((0xFF00 >> n) & 0xFF) | (v >> (6 * (n - 1)))] + out)


def precision_of(n: int) -> int:
    for lim, p in ((192, 7), (384, 8), (576, 9), (1152, 10), (2304, 11)):
        if n <= lim:
            return p
    return 12


def bound(S: int, block: int) -> int:
    """bytes of a row of S samples that no output exceeds: the stream header and VERBATIM frames with the longest header"""
    nf = -(-int(S) // check_block(block))
    return HEADER_BYTES + nf * (15 + 1 + 2) + 2 * int(S)


# ---- bit packing -------------------------------------------------------------------------------------------------
def _pack(values, nbits) -> bytes:
    """MSB-first concatenation of fields: values (< 2^min(nbits, 63)) in nbits bits each, zero bits to a byte"""
    v = np.asarray(values, np.uint64)
    nb = np.asarray(nbits, np.int64)
    end = np.cumsum(nb)
    total = int(end[-1]) if end.size else 0
    bits = np.zeros(-(-total // 8) * 8, np.uint8)
    for j in range(64):
        sel = (nb > j) & (((v >> np.uint64(j)) & np.uint64(1)) == 1)
        if not sel.any():
            if not ((v >> np.uint64(j)) != 0).any():
                break
            continue
        bits[end[sel] - 1 - j] = 1
    return np.packbits(bits).tobytes()


def _signed(v, bits):
    return int(v) & ((1 << bits) - 1)


# ---- analysis ----------------------------------------------------------------------------------------------------
def window(n: int) -> np.ndarray:
    w = np.full(n, 32768, np.int64)
    L = n >> 2
    if L:
        a = 2 * np.arange(L, dtype=np.int64) + 1
        D = 2 * L
        e = (32768 * (3 * a * a * D - 2 * a * a * a)) // (D * D * D)
        w[:L] = e
        w[n - L:] = e[::-1]
    return w


def autocorrelation(x: np.ndarray) -> list:
    xw = (x.astype(np.int64) * window(x.size) + (1 << 14)) >> 15
    return [int(np.dot(xw[l:], xw[: xw.size - l])) if l < xw.size else 0 for l in range(MAX_LPC + 1)]


def levinson(R) -> dict:
    """{order: predictor coefficients (Python floats)} for the orders 1..12 the recursion reaches"""
    out = {}
    err = float(R[0])
    a: list = []
    for i in range(1, MAX_LPC + 1):
        if not err > 0.0:
            break
        acc = float(R[i])
        for j in range(i - 1):
            acc = acc - a[j] * float(R[i - 1 - j])
        k = acc / err
        a = [a[j] - k * a[i - 2 - j] for j in range(i - 1)] + [k]
        err = err * (1.0 - k * k)
        if not all(math.isfinite(c) for c in a):
            break
        out[i] = list(a)
    return out


def quantize(a, P: int):
    """(q list, shift) of predictor a at precision P, or None when every coefficient is 0"""
    cmax = max(abs(c) for c in a)
    if not cmax > 0.0:
        return None
    _, e = math.frexp(cmax)
    shift = min(max(P - e, 0), 15)
    qmax, qmin = (1 << (P - 1)) - 1, -(1 << (P - 1))
    scale, err, q = float(1 << shift), 0.0, []
    for c in a:
        err = err + c * scale
        v = min(max(int(np.rint(err)), qmin), qmax)
        err = err - float(v)
        q.append(v)
    return q, shift


def fixed_residual(x: np.ndarray, order: int) -> np.ndarray:
    x = x.astype(np.int64)
    r = x.copy()
    for _ in range(order):
        r = np.diff(r)
    return r   # r[t - order] for t = order .. n-1


def lpc_residual(x: np.ndarray, q, shift: int) -> np.ndarray:
    x = x.astype(np.int64)
    o, n = len(q), x.size
    pred = np.zeros(n - o, np.int64)
    for j, c in enumerate(q):
        pred += int(c) * x[o - 1 - j: n - 1 - j]
    return x[o:] - (pred >> shift)


def zigzag(r: np.ndarray) -> np.ndarray:
    r = r.astype(np.int64)
    return np.where(r >= 0, 2 * r, -2 * r - 1)


def max_porder(n: int, order: int) -> int:
    p = 0
    while p < MAX_PORDER and n % (2 << p) == 0 and (n >> (p + 1)) > order:
        p += 1
    return p


def rice_plan(r: np.ndarray, n: int, order: int):
    """(bits of the residual section, partition order, k per partition)"""
    ks = np.arange(MAX_RICE + 1, dtype=np.int64)
    u = np.concatenate([np.zeros(order, np.int64), zigzag(r)])   # the warm-up samples add 0 to every sum
    pmax = max_porder(n, order)
    sums = (u.reshape(1 << pmax, n >> pmax)[:, :, None] >> ks).sum(axis=1)   # [partitions, k] at order pmax
    best = None
    for p in range(pmax, -1, -1):
        cnt = np.full(1 << p, n >> p, np.int64)
        cnt[0] -= order
        cost = sums + cnt[:, None] * (ks + 1)
        kk = np.argmin(cost, axis=1)          # the first minimum: the smaller k on a tie
        bits = 6 + int((4 + cost[np.arange(1 << p), kk]).sum())
        if best is None or bits <= best[0]:   # p descends: the smaller p on a tie
            best = (bits, p, kk.tolist())
        if p:
            sums = sums.reshape(-1, 2, ks.size).sum(axis=1)
    return best


def choose(x: np.ndarray) -> dict:
    """the subframe of a frame of int16 samples x, as a dict (type, order, bits, ...)"""
    n = x.size
    if np.all(x == x[0]):
        return {"type": SUB_CONSTANT, "bits": 8 + 16}
    best = None

    def consider(c):
        nonlocal best
        if best is None or c["bits"] < best["bits"]:
            best = c

    for o in range(MAX_FIXED + 1):
        if o >= n:
            break
        r = fixed_residual(x, o)
        if r.size and (r.min() < -2**31 or r.max() > 2**31 - 1):
            continue
        rb, p, ks = rice_plan(r, n, o)
        consider({"type": SUB_FIXED, "order": o, "bits": 8 + 16 * o + rb, "porder": p, "ks": ks, "residual": r})
    P = precision_of(n)
    preds = levinson(autocorrelation(x))
    for o in range(1, MAX_LPC + 1):
        if o >= n or o not in preds:
            continue
        qs = quantize(preds[o], P)
        if qs is None:
            continue
        q, shift = qs
        r = lpc_residual(x, q, shift)
        if r.size and (r.min() < -2**31 or r.max() > 2**31 - 1):
            continue
        rb, p, ks = rice_plan(r, n, o)
        consider({"type": SUB_LPC, "order": o, "bits": 8 + 16 * o + 4 + 5 + P * o + rb, "porder": p, "ks": ks,
                  "residual": r, "q": q, "shift": shift, "precision": P})
    consider({"type": SUB_VERBATIM, "bits": 8 + 16 * n})
    return best


def _subframe_fields(x: np.ndarray, sf: dict):
    vals, nb = [], []

    def put(v, b):
        vals.append(v)
        nb.append(b)

    t = sf["type"]
    if t == SUB_CONSTANT:
        put(0, 8)
        put(_signed(x[0], 16), 16)
        return vals, nb
    if t == SUB_VERBATIM:
        put(1 << 1, 8)
        vals.extend(x.astype(np.int64) & 0xFFFF)
        nb.extend([16] * x.size)
        return vals, nb
    o = sf["order"]
    put(((0x08 | o) if t == SUB_FIXED else (0x20 | (o - 1))) << 1, 8)
    for i in range(o):
        put(_signed(x[i], 16), 16)
    if t == SUB_LPC:
        P = sf["precision"]
        put(P - 1, 4)
        put(sf["shift"], 5)
        for c in sf["q"]:
            put(_signed(c, P), P)
    put(0, 2)
    put(sf["porder"], 4)
    u = zigzag(sf["residual"])
    n, p = x.size, sf["porder"]
    m = n >> p
    for j, k in enumerate(sf["ks"]):
        lo, hi = (0 if j == 0 else j * m - o), (j + 1) * m - o
        seg = u[lo:hi]
        put(k, 4)
        vals.extend(((1 << k) | (seg & ((1 << k) - 1))).tolist())
        nb.extend(((seg >> k) + 1 + k).tolist())
    return vals, nb


def frame_header(n: int, number: int, rate: int, block: int, variable: bool = False) -> bytes:
    """frame header with its CRC-8: a full frame (n == block) by the table code, a short one by the 8/16-bit field"""
    rc, rbits, rval = rate_code(rate)
    if n == block and block in BLOCK_CODES:
        bc, extra = BLOCK_CODES[block], b""
    elif n <= 256:
        bc, extra = 6, bytes([n - 1])
    else:
        bc, extra = 7, (n - 1).to_bytes(2, "big")
    h = bytes([0xFF, 0xF8 | int(variable), (bc << 4) | rc, 0x08]) + utf8_number(number) + extra
    h += rval.to_bytes(rbits // 8, "big") if rbits else b""
    return h + bytes([crc8(h)])


def encode_frame(x, number: int, rate: int, block: int) -> bytes:
    """one frame of int16 samples x (1 <= len <= block) with frame number `number`"""
    x = np.asarray(x, np.int64)
    sf = choose(x)
    vals, nb = _subframe_fields(x, sf)
    f = frame_header(x.size, number, rate, block) + _pack(vals, nb)
    return f + crc16(f).to_bytes(2, "big")


def streaminfo(block: int, rate: int, n: int, min_frame: int, max_frame: int) -> bytes:
    v = (block << 16 | block) << 48 | min_frame << 24 | max_frame
    w = rate << 44 | 0 << 41 | 15 << 36 | n
    return b"fLaC" + bytes([0x80, 0, 0, 34]) + v.to_bytes(10, "big") + w.to_bytes(8, "big") + bytes(16)


def unknown_totals(data: bytes) -> bytes:
    """`data` with STREAMINFO's min / max frame size and total samples set to 0: what a stream slot writes"""
    v = bytearray(data)
    v[12:18] = bytes(6)
    v[21] &= 0xF0
    v[22:26] = bytes(4)
    return bytes(v)


def encode(codes_int16, rate: int, block: int = 4096) -> bytes:
    """native FLAC stream of the int16 samples of one row"""
    rate_code(rate)
    block = check_block(block)
    x = np.asarray(codes_int16).astype(np.int64).ravel()
    frames = [encode_frame(x[i: i + block], i // block, rate, block) for i in range(0, x.size, block)]
    sizes = [len(f) for f in frames]
    head = streaminfo(block, int(rate), x.size, min(sizes, default=0), max(sizes, default=0))
    return head + b"".join(frames)


def frames_of(data: bytes) -> list:
    """the frames of one of our streams, split by walking the decoder (for the per-frame tests)"""
    return decode(data, _frames=True)


# ---- decoder -----------------------------------------------------------------------------------------------------
class FlacError(ValueError):
    pass


_BITS = bytes.maketrans(b"\x00\x01", b"01")


class _Bits:
    def __init__(self, data: bytes, pos: int = 0):
        self.raw = np.unpackbits(np.frombuffer(data, np.uint8)).tobytes()
        self.p = pos * 8

    def u(self, n: int) -> int:
        if n == 0:
            return 0
        if self.p + n > len(self.raw):
            raise FlacError("flac: read past the end of the stream")
        v = int(self.raw[self.p: self.p + n].translate(_BITS), 2)
        self.p += n
        return v

    def s(self, n: int) -> int:
        v = self.u(n)
        return v - (1 << n) if n and v >> (n - 1) else v

    def unary(self) -> int:
        i = self.raw.find(b"\x01", self.p)
        if i < 0:
            raise FlacError("flac: unterminated unary code")
        q = i - self.p
        self.p = i + 1
        return q

    def align(self):
        r = self.p % 8
        if r:
            if self.u(8 - r):
                raise FlacError("flac: non-zero padding")

    @property
    def byte(self) -> int:
        assert self.p % 8 == 0
        return self.p // 8


def _utf8(b: _Bits, max_bytes: int) -> int:
    c = b.u(8)
    if c < 0x80:
        return c
    n = 0
    while c & (0x80 >> n):
        n += 1
    if n < 2 or n > max_bytes:
        raise FlacError(f"flac: bad coded number lead byte {c:#x}")
    v = c & (0x7F >> n)
    for _ in range(n - 1):
        d = b.u(8)
        if d >> 6 != 2:
            raise FlacError("flac: bad coded number continuation byte")
        v = v << 6 | (d & 0x3F)
    return v


def _residual(b: _Bits, n: int, order: int) -> list:
    method = b.u(2)
    if method > 1:
        raise FlacError(f"flac: reserved residual coding method {method}")
    pbits, esc = (4, 15) if method == 0 else (5, 31)
    p = b.u(4)
    if n % (1 << p):
        raise FlacError(f"flac: partition order {p} does not divide the block of {n}")
    m = n >> p
    if m < order:
        raise FlacError(f"flac: partition order {p} leaves fewer than {order} samples in partition 0")
    out = []
    for j in range(1 << p):
        cnt = m - order if j == 0 else m
        k = b.u(pbits)
        if k == esc:
            w = b.u(5)
            out.extend(b.s(w) for _ in range(cnt))
            continue
        for _ in range(cnt):
            u = b.unary() << k | b.u(k)
            out.append((u >> 1) ^ -(u & 1))
    return out


def _subframe(b: _Bits, n: int, bps: int) -> np.ndarray:
    if b.u(1):
        raise FlacError("flac: subframe padding bit set")
    t = b.u(6)
    wasted = b.unary() + 1 if b.u(1) else 0
    sbps = bps - wasted
    if sbps < 1:
        raise FlacError("flac: more wasted bits than bits")
    if t == 0:
        x = np.full(n, b.s(sbps), np.int64)
    elif t == 1:
        x = np.array([b.s(sbps) for _ in range(n)], np.int64)
    elif 8 <= t <= 12:
        o = t - 8
        if o > n:
            raise FlacError("flac: fixed order above the block size")
        x = [b.s(sbps) for _ in range(o)]
        r = _residual(b, n, o)
        coef = {0: (), 1: (1,), 2: (2, -1), 3: (3, -3, 1), 4: (4, -6, 4, -1)}[o]
        for e in r:
            x.append(e + sum(c * x[-1 - j] for j, c in enumerate(coef)))
        x = np.array(x, np.int64)
    elif t >= 32:
        o = t - 31
        if o > n:
            raise FlacError("flac: lpc order above the block size")
        x = [b.s(sbps) for _ in range(o)]
        pc = b.u(4)
        if pc == 15:
            raise FlacError("flac: invalid lpc precision code 15")
        P = pc + 1
        shift = b.s(5)
        if shift < 0:
            raise FlacError(f"flac: negative lpc shift {shift}")
        q = [b.s(P) for _ in range(o)]
        r = _residual(b, n, o)
        for e in r:
            x.append(e + (sum(c * x[-1 - j] for j, c in enumerate(q)) >> shift))
        x = np.array(x, np.int64)
    else:
        raise FlacError(f"flac: reserved subframe type {t}")
    if x.size and (x.min() < -(1 << (sbps - 1)) or x.max() >= 1 << (sbps - 1)):
        raise FlacError("flac: decoded sample outside the sample size")
    return x << wasted


_BS_TABLE = {1: 192, 2: 576, 3: 1152, 4: 2304, 5: 4608, 8: 256, 9: 512, 10: 1024, 11: 2048, 12: 4096, 13: 8192, 14: 16384,
             15: 32768}
_RATE_TABLE = {v: k for k, v in RATE_CODES.items()}
_BPS_TABLE = {1: 8, 2: 12, 4: 16, 5: 20, 6: 24, 7: 32}


def decode_frame(data: bytes, pos: int, si: dict, expect: int | None = None):
    """(samples, end position, header dict) of the frame at byte `pos`"""
    b = _Bits(data, pos)
    sync = b.u(14)
    if sync != 0x3FFE:
        raise FlacError(f"flac: bad frame sync {sync:#x} at byte {pos}")
    if b.u(1):
        raise FlacError("flac: reserved bit after the sync code set")
    variable = b.u(1)
    bc, rc, ch, ss = b.u(4), b.u(4), b.u(4), b.u(3)
    if b.u(1):
        raise FlacError("flac: reserved bit after the sample size set")
    if ch != 0:
        raise FlacError(f"flac: channel assignment {ch} (only mono is decoded)")
    if bc == 0 or rc == 15 or ss == 3:
        raise FlacError(f"flac: reserved block-size / rate / sample-size code ({bc}, {rc}, {ss})")
    number = _utf8(b, 7 if variable else 6)
    if bc == 6:
        n = b.u(8) + 1
    elif bc == 7:
        n = b.u(16) + 1
    else:
        n = _BS_TABLE[bc]
    if rc == 0:
        rate = si["rate"]
    elif rc <= 11:
        rate = _RATE_TABLE[rc]
    else:
        rate = b.u(8) * 1000 if rc == 12 else (b.u(16) if rc == 13 else b.u(16) * 10)
    bps = si["bps"] if ss == 0 else _BPS_TABLE[ss]
    hb = b.byte
    if b.u(8) != crc8(data[pos:hb]):
        raise FlacError(f"flac: frame header CRC-8 mismatch at byte {pos}")
    if bps != 16 or si["bps"] != 16:
        raise FlacError(f"flac: {bps} bits per sample (16-bit streams are decoded)")
    if expect is not None and number != expect:
        raise FlacError(f"flac: frame / sample number {number}, expected {expect}")
    x = _subframe(b, n, bps)
    b.align()
    end = b.byte
    if b.u(16) != crc16(data[pos:end]):
        raise FlacError(f"flac: frame CRC-16 mismatch at byte {pos}")
    return x, end + 2, {"n": n, "rate": rate, "number": number, "variable": bool(variable), "block_code": bc, "rate_code": rc}


def parse_streaminfo(data: bytes):
    """(streaminfo dict, byte offset of the first frame)"""
    if data[:4] != b"fLaC":
        raise FlacError("flac: no fLaC marker")
    pos, si = 4, None
    while True:
        if pos + 4 > len(data):
            raise FlacError("flac: truncated metadata")
        last, typ, ln = data[pos] >> 7, data[pos] & 0x7F, int.from_bytes(data[pos + 1: pos + 4], "big")
        body = data[pos + 4: pos + 4 + ln]
        if si is None:
            if typ != 0 or ln != 34:
                raise FlacError("flac: the first metadata block is not STREAMINFO")
            v = int.from_bytes(body[:18], "big")
            si = {"min_block": v >> 128, "max_block": (v >> 112) & 0xFFFF, "min_frame": (v >> 88) & 0xFFFFFF,
                  "max_frame": (v >> 64) & 0xFFFFFF, "rate": (v >> 44) & 0xFFFFF, "channels": ((v >> 41) & 7) + 1,
                  "bps": ((v >> 36) & 31) + 1, "total": v & ((1 << 36) - 1), "md5": bytes(body[18:34])}
        pos += 4 + ln
        if last:
            return si, pos


def decode(data: bytes, _frames: bool = False):
    """(int16 samples, rate, streaminfo dict) of a mono 16-bit FLAC stream; FlacError (a ValueError) on any fault"""
    data = bytes(data)
    si, pos = parse_streaminfo(data)
    if si["channels"] != 1:
        raise FlacError(f"flac: {si['channels']} channels (only mono is decoded)")
    out, frames, rate, k, sample = [], [], si["rate"], 0, 0
    sizes = []
    while pos < len(data):
        x, end, h = decode_frame(data, pos, si)
        want = sample if h["variable"] else k
        if h["number"] != want:
            raise FlacError(f"flac: frame {k} carries number {h['number']}, expected {want}")
        if si["max_block"] and h["n"] > si["max_block"]:
            raise FlacError(f"flac: block of {h['n']} above STREAMINFO's maximum {si['max_block']}")
        frames.append(data[pos:end])
        sizes.append(end - pos)
        out.append(x)
        rate, k, sample, pos = h["rate"], k + 1, sample + h["n"], end
    if _frames:
        return frames
    y = np.concatenate(out) if out else np.zeros(0, np.int64)
    if si["total"] and si["total"] != y.size:
        raise FlacError(f"flac: {y.size} samples decoded, STREAMINFO states {si['total']}")
    if si["min_frame"] and sizes and min(sizes) < si["min_frame"] or si["max_frame"] and sizes and max(sizes) > si["max_frame"]:
        raise FlacError("flac: a frame size lies outside STREAMINFO's range")
    return y.astype(np.int16), rate, si
