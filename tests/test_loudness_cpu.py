"""CPU: the loudness meter's definition, its filter, its stream schedule and the tolerance the GPU tests hold it to.

The oracle (oracle/loudness_oracle.py) is pinned against BS.1770-4's tabulated 48 kHz coefficients, its calibration tone
and signals whose gated loudness has a closed form; vtts_loudness_filter against the oracle; the stream's peak schedule
against counting; and L_TOL -- the bound on |reading - float64 reading| in LU -- against an fp32 numpy emulation of
the kernels' warp-segment scheme."""
import numpy as np
import pytest

from oracle import loudness_oracle as lo

RATES = [8000, 16000, 22050, 24000, 44100, 48000]
L_TOL = 2e-4     # LU, integrated / momentary / short-term (see test_bound_has_headroom_over_the_emulation)


def sine(freq, seconds, rate, amp=1.0, phase=0.3):
    t = np.arange(int(round(seconds * rate))) / rate
    return amp * np.sin(2 * np.pi * freq * t + phase)


def noise(seconds, rate, seed=0, amp=0.3):
    return amp * np.random.default_rng(seed).standard_normal(int(seconds * rate))


def bursts(seconds, rate, seed=0):
    """sine bursts of varying level and pitch over faint noise: what the gates see in speech"""
    rng = np.random.default_rng(seed)
    n = int(seconds * rate)
    x = 1e-4 * rng.standard_normal(n)
    t = 0
    while t < n:
        d = int(rng.uniform(0.05, 0.6) * rate)
        if rng.random() < 0.6:
            x[t:t + d] += rng.uniform(0.01, 0.9) * np.sin(2 * np.pi * rng.uniform(60, 6000) * np.arange(min(d, n - t)) / rate)
        t += d + int(rng.uniform(0.0, 0.3) * rate)
    return x


# ---- fp32 emulation of loudness.cu ---------------------------------------------------------------------------------

def kernel_params(rate):
    """kw_step's nine parameters in double: the shelf's b0 b1 b2 a1 a2, then the high-pass as a TPT state-variable
    filter: g = tan(pi f0 / r), g + 1 / Q, 1 / (1 + g (g + 1 / Q)), and the output scale a0"""
    c = lo.coeffs10(rate)
    g = np.tan(np.pi * lo.HP_F0 / rate)
    kq = 1.0 / lo.HP_Q
    return np.array([*c[:5], g, g + kq, 1.0 / (1.0 + g * (g + kq)), 1.0 + g * kq + g * g])


def _step(c, s, x):
    """kw_step on arrays (s [..., 4], x [...]) in the dtype of c"""
    y1 = c[0] * x + s[..., 0]
    z1 = c[1] * x + (-c[3] * y1 + s[..., 1])
    z2 = c[2] * x + (-c[4]) * y1
    hp = (y1 - (c[6] * s[..., 2] + s[..., 3])) * c[7]
    v1 = c[5] * hp
    bp = v1 + s[..., 2]
    v2 = c[5] * bp
    return np.stack([z1, z2, bp + v1, (v2 + s[..., 3]) + v2], axis=-1).astype(c.dtype), (c[8] * hp).astype(c.dtype)


def _state_matrix(p):
    return _step(p, np.eye(4), np.zeros(4))[0].T


def emulate(x, rate):
    """(integrated, momentary, short-term) through the kernels' fp32 arithmetic: per sub-block 32 lane segments
    filtered from zero, a constant-matrix scan of the lane end states, a re-filter from each lane's entering state, the
    state chain s_k+1 = A^m s_k + e_k, and the gate's fp32 sums"""
    f = np.float32
    cd = kernel_params(rate)
    c = cd.astype(f)
    A = _state_matrix(cd)
    m = rate // 10
    seg = -(-m // 32)
    Mseg = [np.linalg.matrix_power(A, seg << d).astype(f) for d in range(5)]
    Mblk = np.linalg.matrix_power(A, m).astype(f)
    x = np.asarray(x, f)
    K = x.size // m
    if K == 0:
        return -np.inf, -np.inf, -np.inf
    X = np.zeros((K, 32 * seg), f)
    X[:, :m] = x[: K * m].reshape(K, m)
    X = X.reshape(K, 32, seg)
    lens = np.clip(m - seg * np.arange(32), 0, seg)

    def run(enter0, energy):
        st = np.zeros((K, 32, 4), f)
        st[:, 0] = enter0
        for i in range(seg):
            act = (i < lens)[None, :, None]
            nst, _ = _step(c, st, X[:, :, i])
            st = np.where(act, nst, st)
        for d in range(5):
            o = np.zeros_like(st)
            o[:, 1 << d:] = st[:, : 32 - (1 << d)]
            upd = (st + o @ Mseg[d].T).astype(f)
            st[:, 1 << d:] = upd[:, 1 << d:]
        s = np.zeros_like(st)
        s[:, 1:] = st[:, :31]
        s[:, 0] = enter0
        acc = np.zeros((K, 32), f)
        for i in range(seg):
            act = i < lens
            ns, y = _step(c, s, X[:, :, i])
            s = np.where(act[None, :, None], ns, s)
            acc = np.where(act[None, :], (acc + y * y).astype(f), acc)
        if energy:
            return acc.sum(axis=1, dtype=f)
        last = int(np.flatnonzero(lens > 0)[-1])
        return s[:, last]

    e = run(np.zeros((K, 4), f), False)
    sk = np.zeros((K, 4), f)
    s = np.zeros(4, f)
    for k in range(K):
        sk[k] = s
        s = (e[k] + Mblk @ s).astype(f)
    E = run(sk, True)
    J = max(0, K - 3)
    z = ((((E[:J] + E[1:J + 1]) + E[2:J + 2]) + E[3:J + 3]) * f(1.0 / (4 * m))).astype(f)
    with np.errstate(divide="ignore"):
        l = (f(-0.691) + f(10) * np.log10(z)).astype(f)
    a = l > -70
    if not a.any():
        L = -np.inf
    else:
        g = f(-0.691) + f(10) * np.log10(f(z[a].sum(dtype=f) / f(a.sum()))) - f(10)
        r = a & (l > g)
        L = float(f(-0.691) + f(10) * np.log10(f(z[r].sum(dtype=f) / f(r.sum()))))
    mom = float(l[J - 1]) if J else -np.inf
    st = float(f(-0.691) + f(10) * np.log10(E[K - 30:].sum(dtype=f) / f(30 * m))) if K >= 30 else -np.inf
    return L, mom, st


def reading_error(got, ref):
    """|got - ref| in LU over the three readings, 0 where both are -inf (inf if only one is)"""
    err = 0.0
    for a, b in zip(got, ref):
        if np.isinf(a) or np.isinf(b):
            err = max(err, 0.0 if a == b else np.inf)
        else:
            err = max(err, abs(a - b))
    return err


# ---- tests ---------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("rate", RATES)
def test_library_filter_matches_the_oracle(rate):
    import ctypes
    from viettts_b200 import _lib, build
    build.build()
    lib = _lib.load()
    c = (ctypes.c_double * 10)()
    assert lib.vtts_loudness_filter(rate, c) == 0
    assert np.abs(np.array(c[:]) - lo.coeffs10(rate)).max() <= 1e-12


def test_filter_at_48k_is_the_bs1770_table():
    import ctypes
    from viettts_b200 import _lib, build
    build.build()
    lib = _lib.load()
    c = (ctypes.c_double * 10)()
    assert lib.vtts_loudness_filter(48000, c) == 0
    bs, as_, bh, ah = lo.BS1770_48K
    table = np.concatenate([bs, as_[1:], bh, ah[1:]])
    assert np.abs(np.array(c[:]) - table).max() <= 1e-12
    assert np.abs(lo.coeffs10(48000) - table).max() <= 1e-12


@pytest.mark.parametrize("rate", [11025, 7990, 192010, 16005, 0, -16000])
def test_filter_rejects_rates_without_whole_100ms(rate):
    import ctypes
    from viettts_b200 import _lib, build
    build.build()
    c = (ctypes.c_double * 10)()
    assert _lib.load().vtts_loudness_filter(rate, c) == -1
    with pytest.raises(ValueError):
        lo.design(rate)


def test_calibration_tone():
    """a full-scale 997 Hz sine measures -3.01 LKFS at 48 kHz (BS.1770-4 section 2.1)"""
    L = lo.measure(sine(997, 10, 48000), 48000)[0]
    assert abs(L + 3.0103) <= 0.005, L
    assert abs(lo.measure(sine(997, 10, 16000), 16000)[0] + 2.970) <= 0.005


def test_absolute_gate_drops_silence():
    rate = 16000
    tone = sine(1000, 4, rate, 0.5)
    alone = lo.measure(tone, rate)[0]
    with_silence = lo.measure(np.concatenate([tone, np.zeros(6 * rate)]), rate)[0]
    # the blocks overlapping the tone's end carry part of its energy; the rest is silent and gated out
    assert abs(with_silence - alone) <= 0.3
    E = lo.energies(np.concatenate([tone, np.zeros(6 * rate)]), rate)
    m = rate // 10
    J = E.size - 3
    z = (E[:J] + E[1:J + 1] + E[2:J + 2] + E[3:J + 3]) / (4 * m)
    l = lo.lufs(z)
    assert (l[50:] <= -70).all()               # blocks starting 1 s after the tone hold only the filter's decayed tail
    a = l > -70
    r = a & (l > lo.lufs(z[a].mean()) - 10)
    assert abs(with_silence - lo.lufs(z[r].mean())) <= 1e-12


def test_relative_gate_drops_a_quiet_passage():
    """a tone followed by the same tone 25 LU quieter measures as the loud tone alone: the quiet blocks are above the
    absolute gate but more than 10 LU below the mean"""
    rate = 48000
    loud = sine(1000, 5, rate, 0.5)
    quiet = sine(1000, 5, rate, 0.5 * 10 ** (-25 / 20), phase=0.3 + 2 * np.pi * 1000 * 5)
    both = lo.measure(np.concatenate([loud, quiet]), rate)[0]
    m = rate // 10
    E = lo.energies(np.concatenate([loud, quiet]), rate)
    J = E.size - 3
    z = (E[:J] + E[1:J + 1] + E[2:J + 2] + E[3:J + 3]) / (4 * m)
    l = lo.lufs(z)
    assert (l[-5:] > -70).all() and (l[-5:] < l[:5].max() - 20).all()
    g = lo.lufs(z.mean()) - 10
    assert abs(both - lo.lufs(z[l > g].mean())) <= 1e-12
    # only the three blocks straddling the step carry part of the quiet passage's level
    assert abs(both - lo.measure(loud, rate)[0]) <= 0.2


@pytest.mark.parametrize("rate", [8000, 44100])
def test_block_count_at_the_edges(rate):
    m = rate // 10
    for n, J in ((4 * m - 1, 0), (4 * m, 1), (4 * m + 1, 1), (5 * m - 1, 1), (5 * m, 2)):
        E = lo.energies(noise(1, rate)[:n] if n <= rate else noise(n / rate + 1, rate)[:n], rate)
        assert max(0, E.size - 3) == J == max(0, n // m - 3), n
        L, mom, _ = lo.gate(E, m)
        assert np.isfinite(mom) == (J > 0) and np.isfinite(L) == (J > 0), n


@pytest.mark.parametrize("n", [0, 1, 1599, 6399])
def test_rows_shorter_than_400ms_are_minus_inf(n):
    x = noise(1, 16000)[:n]
    L, mom, st, _ = lo.measure(x, 16000)
    assert L == mom == st == -np.inf


def test_silence_is_minus_inf_and_gain_zero():
    x = np.zeros(5 * 16000)
    assert lo.measure(x, 16000)[:3] == (-np.inf, -np.inf, -np.inf)
    assert lo.true_peak(x) == -np.inf
    assert lo.gain(x, 16000, -16.0, -1.0) == 0.0


def test_true_peak_includes_the_sample_peak():
    """the interpolator reproduces the input samples only approximately; a sample peak it reads below still counts"""
    x = noise(0.2, 16000, 4)
    u = lo.oversample(x)
    assert np.abs(u[::4] - x).max() > 1e-4
    step = np.concatenate([np.zeros(500), 0.8 * np.ones(500)])
    assert np.abs(lo.oversample(step)).max() > 0.8
    for v in (x, step, np.array([0.5]), np.array([0.0, -0.25, 0.0])):
        assert lo.true_peak(v) == 20 * np.log10(max(np.abs(v).max(), np.abs(lo.oversample(v)).max()))


@pytest.mark.parametrize("rate", RATES)
def test_kernel_realization_is_the_k_filter(rate):
    """kw_step in double (shelf TDF2, high-pass TPT state-variable form) computes the oracle's lfilter cascade"""
    x = noise(0.5, rate, 9)
    p = kernel_params(rate)
    s = np.zeros(4)
    y = np.empty_like(x)
    for t in range(x.size):
        s, y[t] = _step(p, s, x[t])
    assert np.abs(y - lo.kweight(x, rate)).max() <= 1e-12


def test_stream_peak_schedule_matches_counting():
    """before END the running peak covers max(0, 4P - 40) oversampled outputs: every output whose inputs have arrived"""
    for P in range(0, 3000):
        assert lo.peak_covered_closed_form(P) == lo.peak_covered(P), P
    from oracle import resample_oracle as ro
    assert ro.lookahead(1, lo.OS) == lo.LOOKAHEAD == 10
    assert ro.emitted_closed_form(777, 1, lo.OS) == lo.peak_covered(777)
    assert lo.peak_covered(5, end=True) == 20


def test_meter_lookahead_from_the_library():
    from viettts_b200 import _lib, build
    build.build()
    lib = _lib.load()
    for rate in RATES:
        assert lib.vtts_loudness_stream_lookahead(rate) == lo.LOOKAHEAD
    assert lib.vtts_loudness_stream_lookahead(11025) == -1


def emulation_cases():
    for rate in RATES:
        yield rate, noise(6.05, rate, rate)
        yield rate, bursts(8, rate, rate + 1)
        yield rate, sine(50, 4, rate, 0.7)             # the high-pass's region, where fp32 coefficients matter most
    yield 16000, bursts(185, 16000, 3)


def test_bound_has_headroom_over_the_emulation():
    """L_TOL is at least 4x the worst error of the fp32 emulation and no looser than 1e-3 LU (EBU Tech 3341 allows
    0.1 LU)"""
    worst = 0.0
    for rate, x in emulation_cases():
        ref = lo.gate(lo.energies(x, rate), rate // 10)
        worst = max(worst, reading_error(emulate(x, rate), ref))
    print(f"fp32 emulation {worst:.2e} LU (L_TOL {L_TOL:.0e})")
    assert 4 * worst <= L_TOL <= 1e-3, worst
