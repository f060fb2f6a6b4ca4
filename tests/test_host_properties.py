"""Property tests (hypothesis) of the host-side logic around the kernels: sharding / bucketing invariants, text
normalisation, PCM conversion, converter layout algebra, duration fix-ups."""
import numpy as np
from hypothesis import given, settings
from hypothesis import strategies as st

from viettts_b200 import config, parallel, synthesizer
from viettts_b200.hifigan import convert
from viettts_b200.nat import text2mel as t2m

LENGTHS = st.lists(st.integers(1, 2000), min_size=1, max_size=200)


@given(LENGTHS, st.integers(1, 8))
@settings(max_examples=60, deadline=None)
def test_lpt_shard_is_a_partition_with_bounded_imbalance(costs, world):
    shards = parallel.lpt_shard(costs, world)
    assert len(shards) == world
    flat = sorted(i for s in shards for i in s)
    assert flat == list(range(len(costs)))
    loads = [sum(costs[i] for i in s) for s in shards]
    assert max(loads) - min(loads) <= max(costs)          # LPT: no rank is ahead by more than one item
    for s in shards:
        assert [costs[i] for i in s] == sorted((costs[i] for i in s), reverse=True)


@given(LENGTHS, st.floats(0.0, 0.5), st.integers(1, 64))
@settings(max_examples=60, deadline=None)
def test_buckets_cover_everything_within_the_padding_budget(nf, pad, rows):
    buckets = parallel.bucket_by_length(nf, pad, rows)
    assert sorted(i for b in buckets for i in b) == list(range(len(nf)))
    for b in buckets:
        assert 1 <= len(b) <= rows
        longest = max(nf[i] for i in b)
        padded = longest * len(b)
        assert padded - sum(nf[i] for i in b) <= pad * padded + 1e-9


@given(st.text(alphabet=st.sampled_from(list("abcđêơ .,:;?!\n\t\"'  ")), max_size=80))
@settings(max_examples=200, deadline=None)
def test_normalised_text_is_clean_and_stable(text):
    out = synthesizer.nat_normalize_text(text)
    assert out == out.strip() and "  " not in out and "\n" not in out and '"' not in out
    assert not any(ch in out for ch in ".,:;?!")
    assert synthesizer.nat_normalize_text(out) == out      # idempotent on its own output


@given(st.lists(st.floats(-4.0, 4.0, allow_nan=False, width=32), min_size=1, max_size=300))
@settings(max_examples=100, deadline=None)
def test_pcm16_is_monotone_bounded_and_odd(xs):
    x = np.asarray(xs, np.float32)
    p = synthesizer.float_to_pcm16(x).astype(np.int64)
    assert p.min() >= -32768 and p.max() <= 32767
    order = np.argsort(x, kind="stable")
    assert np.all(np.diff(p[order]) >= 0)                  # monotone
    inside = np.abs(x) <= 1.0
    assert np.array_equal(synthesizer.float_to_pcm16(-x[inside]).astype(np.int64), -p[inside])   # odd symmetry (round half even)
    assert np.all(np.abs(p[inside] - x[inside].astype(np.float64) * 32767.0) <= 0.5 + 1e-6)


@given(st.integers(1, 5), st.integers(1, 6), st.integers(1, 7), st.integers(0, 2 ** 31 - 1))
@settings(max_examples=50, deadline=None)
def test_converter_layout_algebra(co, ci, k, seed):
    """Conv1d: hk[k, i, o] == torch[o, i, k].  ConvTranspose1d: hk[k, o, i] == torch[i, o, K-1-k]."""
    rng = np.random.default_rng(seed)
    wc = rng.standard_normal((co, ci, k)).astype(np.float32)
    wt = rng.standard_normal((ci, co, k)).astype(np.float32)
    sd = {"conv_pre.weight": wc, "conv_pre.bias": np.zeros(co, np.float32), "ups.0.weight": wt, "ups.0.bias": np.zeros(co, np.float32)}
    hk = convert.state_dict_to_haiku(sd)
    a, b = hk["generator/~/conv1_d"]["w"], hk["generator/~/ups_0"]["w"]
    assert a.shape == (k, ci, co) and b.shape == (k, co, ci)
    for kk in range(k):
        assert np.array_equal(a[kk], wc[:, :, kk].T)
        assert np.array_equal(b[kk], wt[:, :, k - 1 - kk].T)
    # the reference's formulation: rot90(k=1, axes=(0, 2)) / swapaxes(0, 2)
    assert np.array_equal(b, np.rot90(wt, k=1, axes=(0, 2))) and np.array_equal(a, np.swapaxes(wc, 0, 2))


@given(st.lists(st.integers(0, 92), min_size=2, max_size=60), st.floats(-1.0, 0.5), st.integers(0, 2 ** 31 - 1))
@settings(max_examples=80, deadline=None)
def test_duration_fixups(tokens, silence, seed):
    rng = np.random.default_rng(seed)
    d = rng.uniform(0.001, 0.4, (1, len(tokens))).astype(np.float32)
    out = t2m.adjust_durations(tokens, d, silence)
    tok = np.asarray(tokens)
    assert out.dtype == np.float32 and out.shape == d.shape
    assert np.all(out[0, tok == config.WORD_END_INDEX] == 0)
    sil = tok == config.SIL_INDEX
    assert np.all(out[0, sil] >= np.float32(silence)) and np.all(out[0, sil] >= d[0, sil])
    rest = ~sil & (tok != config.WORD_END_INDEX)
    assert np.array_equal(out[0, rest], d[0, rest])
    frames, n = t2m.seconds_to_frames(out)
    assert n == int(np.float32(sum(float(f) for f in frames[0]))) and frames.dtype == np.float32


def test_balanced_buckets_equal_cost_and_padding_bound():
    """parallel.balanced_buckets (BASELINE configs[4]): every utterance placed exactly once, whole-workload padding within
    the bound, at most 32 rows per bucket (one decoder scan), predicted per-rank cost within 5 % of the mean at 8 ranks."""
    import numpy as np
    from viettts_b200 import parallel
    rng = np.random.default_rng(3)
    for trial in range(5):
        n = (rng.integers(50, 301, size=256) * 3.125).astype(np.int64)
        for world in (1, 2, 8):
            buckets, shards = parallel.balanced_buckets(n, world)
            flat = sorted(i for b in buckets for i in b)
            assert flat == list(range(len(n)))
            assert sorted(i for s in shards for i in s) == list(range(len(buckets)))
            assert max(len(b) for b in buckets) <= 32
            padded = sum(len(b) * int(n[b].max()) for b in buckets)
            assert 1.0 - n.sum() / padded <= 0.08
            loads = [sum(parallel.batch_cost_us(n[buckets[i]]) for i in s) for s in shards]
            if world == 8:
                assert max(loads) / np.mean(loads) <= 1.05, (trial, world, max(loads) / np.mean(loads))
