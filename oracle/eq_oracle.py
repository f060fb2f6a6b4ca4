"""Float64 statement of the equalizer (viettts_b200/csrc/eq.cu, vtts_eq*): a cascade of K <= 8 second-order sections.

A filter is sos, float64 [K][6] rows b0 b1 b2 a0 a1 a2 (scipy's layout).  For one mono row x of n samples the output is
y = scipy.signal.sosfilt(sos, x) in float64 from zero state at sample 0, not clipped; outputs past n are 0.

Every section runs on the device as the trapezoidal state-variable filter (Simper's linear SVF) of its own bilinear
transform, with parameters g, k and output mix m0, m1, m2 (`svf_params`).  `emulate` restates the kernels' fp32
arithmetic in numpy: 1024-sample blocks of 32 lanes x 32 samples, per-section lane scans, the block chain
s_k+1 = M s_k + e_k and the output pass; `emulate_stream` runs the same arithmetic push by push as the stream does.

Also here: an independent numpy statement of every designer of vtts_eq_design (Butterworth through scipy, the RBJ
Audio EQ Cookbook formulas written out) and the stability rule."""
from __future__ import annotations

import numpy as np
from scipy import signal

KMAX = 8
SEG = 32
Q = 32 * SEG
POLE_MARGIN = 1e-6
HIGHPASS, LOWPASS, LOWSHELF, HIGHSHELF, PEAKING, NOTCH = range(6)


def sosfilt(sos, x) -> np.ndarray:
    return signal.sosfilt(np.asarray(sos, np.float64), np.asarray(x, np.float64))


# ---- designers -------------------------------------------------------------------------------------------------------

def butter(btype: str, order: int, f0: float, rate: int) -> np.ndarray:
    return signal.butter(order, f0, btype, fs=rate, output="sos")


def _rbj(b, a) -> np.ndarray:
    b, a = np.asarray(b, np.float64), np.asarray(a, np.float64)
    return np.concatenate([b / a[0], a / a[0]])[None]


def _w0(f0, rate):
    w0 = 2 * np.pi * f0 / rate
    return np.cos(w0), np.sin(w0)


def shelf(high: bool, f0: float, gain_db: float, S: float, rate: int) -> np.ndarray:
    A = 10 ** (gain_db / 40)
    cw, sw = _w0(f0, rate)
    alpha = sw / 2 * np.sqrt((A + 1 / A) * (1 / S - 1) + 2)
    ra = 2 * np.sqrt(A) * alpha
    if not high:
        return _rbj([A * ((A + 1) - (A - 1) * cw + ra), 2 * A * ((A - 1) - (A + 1) * cw), A * ((A + 1) - (A - 1) * cw - ra)],
                    [(A + 1) + (A - 1) * cw + ra, -2 * ((A - 1) + (A + 1) * cw), (A + 1) + (A - 1) * cw - ra])
    return _rbj([A * ((A + 1) + (A - 1) * cw + ra), -2 * A * ((A - 1) + (A + 1) * cw), A * ((A + 1) + (A - 1) * cw - ra)],
                [(A + 1) - (A - 1) * cw + ra, 2 * ((A - 1) - (A + 1) * cw), (A + 1) - (A - 1) * cw - ra])


def peaking(f0: float, q: float, gain_db: float, rate: int) -> np.ndarray:
    A = 10 ** (gain_db / 40)
    cw, sw = _w0(f0, rate)
    alpha = sw / (2 * q)
    return _rbj([1 + alpha * A, -2 * cw, 1 - alpha * A], [1 + alpha / A, -2 * cw, 1 - alpha / A])


def notch(f0: float, q: float, rate: int) -> np.ndarray:
    cw, sw = _w0(f0, rate)
    alpha = sw / (2 * q)
    return _rbj([1, -2 * cw, 1], [1 + alpha, -2 * cw, 1 - alpha])


# ---- validity and the state-variable form ----------------------------------------------------------------------------

def pole_radius(a1: float, a2: float) -> float:
    return float(np.abs(np.roots([1.0, a1, a2])).max()) if a2 != 0 or a1 != 0 else 0.0


def valid(sos) -> bool:
    """1 <= K <= 8 finite sections with a0 != 0, each strictly stable with every pole radius <= 1 - POLE_MARGIN"""
    sos = np.asarray(sos, np.float64)
    if sos.ndim != 2 or sos.shape[1] != 6 or not 1 <= sos.shape[0] <= KMAX or not np.all(np.isfinite(sos)):
        return False
    for row in sos:
        if row[3] == 0:
            return False
        a1, a2 = row[4] / row[3], row[5] / row[3]
        if not (abs(a2) < 1 and abs(a1) < 1 + a2) or pole_radius(a1, a2) > 1 - POLE_MARGIN:
            return False
    return True


def svf_params(sos) -> np.ndarray:
    """[K][5]: g, k, m0, m1, m2 of every section: H(s) = (m0 (s^2 + k s + 1) + m1 s + m2) / (s^2 + k s + 1) with
    s = (z - 1) / (g (z + 1)) is the section's transfer function"""
    out = []
    for row in np.asarray(sos, np.float64):
        b0, b1, b2, a1, a2 = row[0] / row[3], row[1] / row[3], row[2] / row[3], row[4] / row[3], row[5] / row[3]
        c0 = 1 + a1 + a2
        g = np.sqrt(c0 / (1 - a1 + a2))
        k = 2 * g * (1 - a2) / c0
        n2, n1, n0 = g * g * (b0 - b1 + b2) / c0, 2 * g * (b0 - b2) / c0, (b0 + b1 + b2) / c0
        out.append([g, k, n2, n1 - n2 * k, n0 - n2])
    return np.array(out)


def svf_response(params, w) -> np.ndarray:
    """the cascade's response at digital frequencies w (rad / sample) from svf_params"""
    s = 1j * np.tan(np.asarray(w, np.float64) / 2)
    h = np.ones_like(s)
    for g, k, m0, m1, m2 in params:
        sa = s / g
        D = sa * sa + k * sa + 1
        h = h * (m0 * D + m1 * sa + m2) / D
    return h


def kernel_coeffs(sos) -> np.ndarray:
    """[K][6] float64: d, g d, g^2 d, m0, m1, m2 per section (d = 1 / (1 + g (g + k))), before the fp32 rounding"""
    P = svf_params(sos)
    g, k = P[:, 0], P[:, 1]
    d = 1 / (1 + g * (g + k))
    return np.stack([d, g * d, g * g * d, P[:, 2], P[:, 3], P[:, 4]], axis=1)


def transitions(sos):
    """(A [2K][2K] one-sample zero-input transition of the cascade, c [K][6]) in float64"""
    c = kernel_coeffs(sos)
    K = c.shape[0]
    A = np.zeros((2 * K, 2 * K))
    for col in range(2 * K):
        s = np.zeros(2 * K)
        s[col] = 1.0
        _step64(c, s, 0.0)
        A[:, col] = s
    return A, c


def _step64(c, s, x):
    for j in range(c.shape[0]):
        d, gd, g2d, m0, m1, m2 = c[j]
        s1, s2 = s[2 * j], s[2 * j + 1]
        v3 = x - s2
        v1 = d * s1 + gd * v3
        v2 = s2 + gd * s1 + g2d * v3
        s[2 * j], s[2 * j + 1] = 2 * v1 - s1, 2 * v2 - s2
        x = m0 * x + m1 * v1 + m2 * v2
    return x


def impulse_l1(sos) -> float:
    """||h||_1 of the cascade's impulse response, run until it has decayed below 1e-13 of its peak"""
    r = max(pole_radius(row[4] / row[3], row[5] / row[3]) for row in np.asarray(sos, np.float64))
    n = int(min(4_000_000, max(4096, 32 * np.log(1e-13) / np.log(max(r, 1e-3)))))
    x = np.zeros(n)
    x[0] = 1.0
    return float(np.abs(sosfilt(sos, x)).sum())


# ---- fp32 emulation of eq.cu -----------------------------------------------------------------------------------------

class Fp32Filter:
    """the fp32 parameters of the kernels, rounded once from float64"""

    def __init__(self, sos):
        A, c = transitions(sos)
        self.K = c.shape[0]
        self.c = c.astype(np.float32)
        self.seg = np.zeros((self.K, 5, 2, 2), np.float32)
        for j in range(self.K):
            Aj = A[2 * j:2 * j + 2, 2 * j:2 * j + 2]
            for d in range(5):
                self.seg[j, d] = np.linalg.matrix_power(Aj, SEG << d).astype(np.float32)
        self.blk = np.linalg.matrix_power(A, Q).astype(np.float32)


def _svf32(c, s1, s2, x):
    f = np.float32
    v3 = f(x - s2) if np.isscalar(x) else (x - s2).astype(f)
    v1 = (c[1] * v3 + c[0] * s1).astype(f)
    v2 = (c[2] * v3 + (c[1] * s1 + s2).astype(f)).astype(f)
    s1n = (f(2) * v1 - s1).astype(f)
    s2n = (f(2) * v2 - s2).astype(f)
    y = (c[5] * v2 + (c[4] * v1 + c[3] * x).astype(f)).astype(f)
    return s1n, s2n, y


def _blocks32(F: Fp32Filter, X, enter):
    """X f32 [nb, 32 lanes, 32] block samples, enter f32 [nb, 2K] (zeros: the zero-state pass).  Returns (Y, end) with
    end [nb, 2K] the state the last lane leaves each section with."""
    f = np.float32
    Y = X.copy()
    nb = X.shape[0]
    end = np.zeros((nb, 2 * F.K), f)
    lane = np.arange(32)
    for j in range(F.K):
        c = F.c[j]
        n1 = np.zeros((nb, 32), f)
        n2 = np.zeros((nb, 32), f)
        n1[:, 0], n2[:, 0] = enter[:, 2 * j], enter[:, 2 * j + 1]
        s1, s2 = n1.copy(), n2.copy()
        for i in range(SEG):
            s1, s2, _ = _svf32(c, s1, s2, Y[:, :, i])
        for d in range(5):
            sh = 1 << d
            o1, o2 = np.roll(s1, sh, axis=1), np.roll(s2, sh, axis=1)
            A = F.seg[j, d]
            u1 = ((s1 + (A[0, 0] * o1).astype(f)).astype(f) + (A[0, 1] * o2).astype(f)).astype(f)
            u2 = ((s2 + (A[1, 0] * o1).astype(f)).astype(f) + (A[1, 1] * o2).astype(f)).astype(f)
            s1, s2 = np.where(lane >= sh, u1, s1), np.where(lane >= sh, u2, s2)
        s1, s2 = np.roll(s1, 1, axis=1), np.roll(s2, 1, axis=1)
        s1[:, 0], s2[:, 0] = n1[:, 0], n2[:, 0]
        for i in range(SEG):
            s1, s2, Y[:, :, i] = _svf32(c, s1, s2, Y[:, :, i])
        end[:, 2 * j], end[:, 2 * j + 1] = s1[:, 31], s2[:, 31]
    return Y, end


def _chain32(F: Fp32Filter, e, complete, s0):
    """entering states [nb, 2K] of blocks with end states e from s0; returns (states, the state after the complete ones)"""
    f = np.float32
    s = s0.astype(f).copy()
    M = F.blk
    out = np.zeros_like(e)
    for q in range(e.shape[0]):
        out[q] = s
        if complete[q]:
            acc = e[q].copy()
            for col in range(s.size):
                acc = (acc + (M[:, col] * s[col]).astype(f)).astype(f)
            s = acc
    return out, s


def _run32(F: Fp32Filter, x, n, k0, nk, carry):
    """blocks [k0, k0 + nk) of the row x (absolute samples; those at or past n read as 0) from the state carry entering
    block k0.  Returns (y over samples [k0 Q, (k0 + nk) Q), the state at the last complete block boundary)."""
    f = np.float32
    t0, t1 = k0 * Q, (k0 + nk) * Q
    seg = np.zeros(t1 - t0, f)
    hi = min(n, t1, x.size)
    if hi > t0:
        seg[:hi - t0] = x[t0:hi]
    X = seg.reshape(nk, 32, SEG)
    _, e = _blocks32(F, X, np.zeros((nk, 2 * F.K), f))
    complete = (np.arange(k0, k0 + nk) + 1) * Q <= n
    S_in, s_end = _chain32(F, e, complete, carry)
    Y, _ = _blocks32(F, X, S_in)
    return Y.reshape(-1), s_end


def emulate(sos, x) -> np.ndarray:
    """y of eq.cu's arithmetic over one row, in fp32 numpy (no FMA: the error is of the same size)"""
    F = Fp32Filter(sos)
    x = np.asarray(x, np.float32)
    n = x.size
    if n == 0:
        return np.zeros(0, np.float32)
    nk = -(-n // Q)
    y, _ = _run32(F, x, n, 0, nk, np.zeros(2 * F.K, np.float32))
    return y[:n]


def emulate_stream(sos, x, pushes) -> list:
    """the outputs of each push of a stream slot fed x in chunks of the given sizes, with the stream's arithmetic:
    every push re-runs the slot's incomplete block from the state at its last complete block boundary"""
    F = Fp32Filter(sos)
    x = np.asarray(x, np.float32)
    carry = np.zeros(2 * F.K, np.float32)
    P0, out = 0, []
    for k in pushes:
        P1 = P0 + int(k)
        if P1 == P0:
            out.append(np.zeros(0, np.float32))
            continue
        k0 = P0 // Q
        nk = (P1 - 1) // Q - k0 + 1
        y, carry = _run32(F, x, P1, k0, nk, carry)
        out.append(y[P0 - k0 * Q:P1 - k0 * Q].copy())
        P0 = P1
    return out
