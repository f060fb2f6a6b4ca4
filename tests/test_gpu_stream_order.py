"""GPU: the calls of one context run in the order they are issued, whatever CUDA stream each is given.

A context's calls share its workspace, its tensor-core tile-scheduler counters and its error flag.  Tensor calls and
stream pushes run on the caller's stream, `*_host` calls and `push` on the context's own non-blocking stream, so a
caller mixing them (or two torch streams) must still get every call's single-stream bits.  Each case computes every
call's output alone first (one stream, synchronised; the other GPU test files pin those outputs against float64), then
issues the same calls interleaved across streams with no synchronisation in between, and asserts np.array_equal for
every output.  After each case one more plain call must equal its reference: a tile-scheduler pair left non-zero by an
overlap would make every later tensor-core launch skip tiles.  The work is sized so the calls overlap on the device
when nothing orders them: the generator at B = 32 and 300 frames, the audio stages on 32 rows of 5 s."""
import numpy as np
import pytest
import torch

from viettts_b200 import config, synthetic

pytestmark = pytest.mark.gpu
HOP = config.HOP
B, T = 32, 300                    # generator batch: tens of ms on an H100
SA = 5 * config.SAMPLE_RATE       # audio rows of 5 s
WRAP_TILES = 4 * 132              # tiles of a launch several times the SM count of an H100 SXM


@pytest.fixture(scope="module")
def eng(hifigan_params, acoustic_ckpt):
    from viettts_b200.engine import Engine
    e = Engine(0)
    e.load_hifigan(hifigan_params)
    e.load_acoustic(acoustic_ckpt)
    e.load_duration(synthetic.duration_ckpt(1234))
    yield e
    torch.cuda.synchronize()
    e.close()


@pytest.fixture
def modes(eng):
    """restores the default precision and fused pairs after a case"""
    yield
    eng.set_precision("bf16x3")
    eng.set_fused_pairs(True)


def dev(a):
    t = torch.from_numpy(np.ascontiguousarray(a)).cuda()
    torch.cuda.synchronize()
    return t


def alone(call):
    """the output of a tensor call issued on its own on torch's current stream, synchronised, as a host array"""
    out = call()
    torch.cuda.synchronize()
    return out.cpu().numpy()


def mels(seed, b=B, t=T):
    return synthetic.mel_input(seed, b, t)


def audio(seed, b=32, s=SA):
    """seeded speech-band test rows: a few partials under noise, at varied levels"""
    rng = np.random.default_rng(seed)
    n = np.arange(s) / config.SAMPLE_RATE
    f0 = rng.uniform(90, 300, size=(b, 1))
    x = sum(np.sin(2 * np.pi * k * f0 * n + rng.uniform(0, 6.3, size=(b, 1))) / k for k in (1, 2, 3, 5))
    x = x + 0.3 * rng.standard_normal((b, s))
    return (x * rng.uniform(0.02, 0.5, size=(b, 1))).astype(np.float32)


def generator_tiles_lower_bound(b, t):
    """tiles of one stage-3 launch at least: 256 t output rows per batch row, a tensor-core tile holds at most 256"""
    return b * t


# ---- a. tensor call and host call ---------------------------------------------------------------------------------

@pytest.mark.parametrize("fused", [True, False], ids=["fused", "unfused"])
@pytest.mark.parametrize("mode", ["bf16x3", "fp16"])
@pytest.mark.parametrize("order", ["tensor_then_host", "host_then_tensor"])
def test_tensor_call_and_host_call(eng, modes, mode, fused, order):
    """hifigan_forward on torch's current stream and mel2wave (the own stream) of a different mel of the same shape,
    so both use the same workspace layout.  A host call returns once its work is done, so in the second order the
    tensor call follows a finished host call and a host call follows it while it may still run."""
    eng.set_precision(mode)
    eng.set_fused_pairs(fused)
    ma, mb = mels(1), mels(2)
    ma_t = dev(ma)
    ref_a = alone(lambda: eng.hifigan_forward(ma_t))
    ref_b = eng.mel2wave(mb)
    if order == "tensor_then_host":
        wa_t = eng.hifigan_forward(ma_t)
        wb = eng.mel2wave(mb)
        wb2 = wb
    else:
        wb = eng.mel2wave(mb)
        wa_t = eng.hifigan_forward(ma_t)
        wb2 = eng.mel2wave(mb)
    torch.cuda.synchronize()
    assert np.array_equal(wa_t.cpu().numpy(), ref_a)
    assert np.array_equal(wb, ref_b) and np.array_equal(wb2, ref_b)
    assert np.array_equal(alone(lambda: eng.hifigan_forward(ma_t)), ref_a)


# ---- b. two side streams ------------------------------------------------------------------------------------------

@pytest.mark.parametrize("mode", ["bf16x3", "fp16"])
def test_two_side_streams(eng, modes, mode):
    """hifigan_forward on two torch streams issued back to back, at different B and T so their tile counts differ, one
    of them with launches of far more than 4 x 132 tiles"""
    eng.set_precision(mode)
    assert generator_tiles_lower_bound(B, T) > WRAP_TILES
    shapes = [(B, T), (7, 123), (B, T), (3, 57)]
    ms = [mels(10 + i, b, t) for i, (b, t) in enumerate(shapes)]
    ms_t = [dev(m) for m in ms]
    refs = [alone(lambda: eng.hifigan_forward(m_t)) for m_t in ms_t]
    s = [torch.cuda.Stream(), torch.cuda.Stream()]
    outs = []
    for i, m_t in enumerate(ms_t):
        with torch.cuda.stream(s[i % 2]):
            outs.append(eng.hifigan_forward(m_t))
    torch.cuda.synchronize()
    for o, r in zip(outs, refs):
        assert np.array_equal(o.cpu().numpy(), r)
    assert np.array_equal(alone(lambda: eng.hifigan_forward(ms_t[0])), refs[0])


# ---- c. audio stages without tensor cores -------------------------------------------------------------------------

def test_audio_stages_across_streams(eng):
    """denoise_forward on one side stream, loudness (host), limit_forward on another side stream: three users of the
    workspace; the workspace is grown by the reference calls first, so none of the interleaved calls reallocates it"""
    x, y, z = audio(1), audio(2), audio(3)
    x_t, z_t = dev(x), dev(z)
    dn_ref = eng.denoise_forward(x_t, 0.7).cpu().numpy()
    ln_ref = eng.loudness(y)
    lm_ref = [a.cpu().numpy() for a in eng.limit_forward(z_t, -3.0, gain_db=12.0)]
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    with torch.cuda.stream(s1):
        dn_t = eng.denoise_forward(x_t, 0.7)
    ln = eng.loudness(y)
    with torch.cuda.stream(s2):
        lm_t = eng.limit_forward(z_t, -3.0, gain_db=12.0)
    ln2 = eng.loudness(y)
    torch.cuda.synchronize()
    assert np.array_equal(dn_t.cpu().numpy(), dn_ref)
    for got in (ln, ln2):
        for a, r in zip(got, ln_ref):
            assert np.array_equal(a, r)
    for a, r in zip(lm_t, lm_ref):
        assert np.array_equal(a.cpu().numpy(), r)
    assert np.array_equal(eng.denoise_forward(x_t, 0.7).cpu().numpy(), dn_ref)


def test_stage_stream_push_device_between_host_calls(eng):
    """a denoise stream's push_device on a side stream, push by push between limit (host) calls: the slots' audio
    equals the one-shot denoise of each slot's whole input, and every limit call its reference"""
    S, F, n_push = 4, 4000, 20
    x = audio(5, S, F * n_push)
    ref = eng.denoise(x, 0.7)
    z = audio(6, 32, SA)
    lm_ref = eng.limit(z, -3.0, gain_db=12.0)
    side = torch.cuda.Stream()
    with eng.open_denoise_stream(S, F, 0.7) as ds:
        xs = [dev(x[:, i * F:(i + 1) * F]) for i in range(n_push)] + [dev(np.zeros((S, F), np.float32))]   # END, no new samples
        ys = [torch.empty((S, ds.out_pitch), device="cuda") for _ in xs]
        torch.cuda.synchronize()
        counts, lms = [], []
        for i in range(n_push + 1):
            n = np.full(S, F if i < n_push else 0, np.int32)
            flags = np.full(S, (1 if i == 0 else 0) | (2 if i == n_push else 0), np.uint8)
            with torch.cuda.stream(side):
                counts.append(ds.push_device(xs[i], n, flags, ys[i]))
            lms.append(eng.limit(z, -3.0, gain_db=12.0))
        torch.cuda.synchronize()
    for s in range(S):
        got = np.concatenate([y[s, : int(c[s])].cpu().numpy() for y, c in zip(ys, counts)])
        assert np.array_equal(got, ref[s])
    for lm in lms:
        for a, r in zip(lm, lm_ref):
            assert np.array_equal(a, r)


# ---- d. stream handles ----------------------------------------------------------------------------------------------

@pytest.mark.parametrize("mode", ["bf16x3", "fp16"])
def test_vocoder_stream_between_host_calls(eng, modes, mode):
    """a vocoder stream's push_device on a side stream, push by push between mel2wave host calls; each slot's audio
    equals mel2wave of its whole mel (fused pairs off: the stream runs each ResBlock pair as two convs)"""
    eng.set_precision(mode)
    eng.set_fused_pairs(False)
    S, F, n_push = 3, 32, 8
    m = mels(20, S, F * n_push)
    refs = [eng.mel2wave(m[s:s + 1])[0] for s in range(S)]
    mo = mels(21)
    ref_o = eng.mel2wave(mo)
    side = torch.cuda.Stream()
    with eng.open_vocoder_stream(S, F) as vs:
        ms_t = [dev(m[:, i * F:(i + 1) * F]) for i in range(n_push)] + [dev(np.zeros((S, F, 80), np.float32))]   # END, no new frames
        outs = [torch.empty((S, vs.wav_ld), device="cuda") for _ in ms_t]
        torch.cuda.synchronize()
        counts, others = [], []
        for i in range(n_push + 1):
            n = np.full(S, F if i < n_push else 0, np.int32)
            flags = np.full(S, (1 if i == 0 else 0) | (2 if i == n_push else 0), np.uint8)
            with torch.cuda.stream(side):
                counts.append(vs.push_device(ms_t[i], n, flags, outs[i]))
            others.append(eng.mel2wave(mo))
        torch.cuda.synchronize()
    for s in range(S):
        got = np.concatenate([o[s, : int(c[s]) * HOP].cpu().numpy() for o, c in zip(outs, counts)])
        assert np.array_equal(got, refs[s]), s
    for o in others:
        assert np.array_equal(o, ref_o)
    assert np.array_equal(eng.mel2wave(m[:1]), refs[0][None])


def tts_tokens(seed, L):
    rng = np.random.default_rng(seed)
    t = rng.integers(4, 90, size=L).astype(np.int32)
    t[4::5] = 3
    t[0] = t[-1] = 0
    return t


def test_tts_stream_steps_between_side_stream_calls(eng, modes):
    """a TtsStream step() loop with a hifigan_forward on a side stream between steps: each slot's audio equals `tts` of
    its tokens, each side-stream call its reference"""
    eng.set_precision("bf16x3")
    eng.set_fused_pairs(False)
    lens = [30, 7, 55]
    tok = np.zeros((3, max(lens)), np.int32)
    for b, n in enumerate(lens):
        tok[b, :n] = tts_tokens(60 + b, n)
    waves, _ = eng.tts(tok, lens, silence_duration=0.1)
    mo = mels(22)
    ref_o = eng.mel2wave(mo)
    mo_t = dev(mo)
    side = torch.cuda.Stream()
    others = []
    with eng.open_tts_stream(4, 16, 2000, 100) as ts:
        for b in range(3):
            ts.begin(b, tok[b, : lens[b]], silence_duration=0.1)
        pieces = {b: [] for b in range(3)}
        while ts.busy().any():
            for s, w in ts.step().items():
                pieces[s].append(w)
            with torch.cuda.stream(side):
                others.append(eng.hifigan_forward(mo_t))
        torch.cuda.synchronize()
    for b in range(3):
        assert np.array_equal(np.concatenate(pieces[b]), waves[b]), b
    for o in others:
        assert np.array_equal(o.cpu().numpy(), ref_o)


# ---- e. acoustic and duration models --------------------------------------------------------------------------------

def utts(seed, b, n):
    """tokens [b,L] and durations in frames [b,L] of rows of exactly n frames each (n_frames passed explicitly)"""
    rng = np.random.default_rng(seed)
    L = 40
    tok = rng.integers(4, 90, size=(b, L)).astype(np.int32)
    d = rng.uniform(0.5, 1.5, size=(b, L))
    d = (d * (n + 0.5) / d.sum(1, keepdims=True)).astype(np.float32)
    return tok, d


def test_acoustic_forward_then_predict_mel(eng):
    """acoustic_forward on a side stream, then predict_mel (host) of other rows: the decoder scans of the two calls
    share the workspace's grid-barrier counter"""
    N = 200
    ta, da = utts(30, 16, N)
    tb, db = utts(31, 16, N)
    nf = np.full(16, N, np.int32)
    ta_t, da_t, nf_t = dev(ta), dev(da), dev(nf)
    ref_a = alone(lambda: eng.acoustic_forward(ta_t, da_t, N, n_frames_t=nf_t))
    ref_b = eng.predict_mel(tb, db, n_frames=nf)
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        ma_t = eng.acoustic_forward(ta_t, da_t, N, n_frames_t=nf_t)
    mb = eng.predict_mel(tb, db, n_frames=nf)
    torch.cuda.synchronize()
    assert np.array_equal(ma_t.cpu().numpy(), ref_a)
    assert np.array_equal(mb, ref_b)
    assert np.array_equal(alone(lambda: eng.acoustic_forward(ta_t, da_t, N, n_frames_t=nf_t)), ref_a)


def test_duration_forward_between_tts_plans(eng):
    """duration_forward on a side stream, interleaved with tts_plan (host) of other rows"""
    tok = np.stack([tts_tokens(70 + b, 60) for b in range(32)])
    tok2 = np.stack([tts_tokens(170 + b, 60) for b in range(32)])
    tok_t = dev(tok)
    ref_d = alone(lambda: eng.duration_forward(tok_t))
    ref_p = eng.tts_plan(tok2, silence_duration=0.1)
    side = torch.cuda.Stream()
    outs, plans = [], []
    for _ in range(3):
        with torch.cuda.stream(side):
            outs.append(eng.duration_forward(tok_t))
        plans.append(eng.tts_plan(tok2, silence_duration=0.1))
    torch.cuda.synchronize()
    for o in outs:
        assert np.array_equal(o.cpu().numpy(), ref_d)
    for p in plans:
        for a, r in zip(p, ref_p):
            assert np.array_equal(a, r)
    assert np.array_equal(alone(lambda: eng.duration_forward(tok_t)), ref_d)


# ---- f. graph capture -----------------------------------------------------------------------------------------------

def captured(fn):
    """fn() captured in one CUDA graph after an eager warm-up call (as scripts/bench_encode.py graph_ms), replayed once"""
    fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    g.replay()
    torch.cuda.synchronize()
    return g


def test_graph_capture_replays_the_eager_call(eng):
    """encode_forward and hifigan_forward captured in torch.cuda.graph: a capturing stream neither waits on nor records
    the context's last call, and the replay equals the eager call; the next eager call is still ordered"""
    x_t = dev(audio(40))
    ref_c = eng.encode_forward(x_t, "ulaw").cpu().numpy()
    c_t = torch.empty_like(x_t, dtype=torch.uint8)
    g1 = captured(lambda: eng.encode_forward(x_t, "ulaw", out=c_t))
    m = mels(41)
    ref_w = eng.mel2wave(m)
    m_t = dev(m)
    w_t = torch.empty((B, T * HOP), device="cuda")
    g2 = captured(lambda: eng.hifigan_forward(m_t, out=w_t))
    c_t.zero_()
    w_t.zero_()
    g1.replay()
    g2.replay()
    torch.cuda.synchronize()
    assert np.array_equal(c_t.cpu().numpy(), ref_c)
    assert np.array_equal(w_t.cpu().numpy(), ref_w)
    assert np.array_equal(eng.mel2wave(m), ref_w)
    assert np.array_equal(eng.encode_forward(x_t, "ulaw").cpu().numpy(), ref_c)
