"""CPU: the slot-stream driver (tests/helpers/slot_streams.py) against a numpy fake stream, so that the checks every GPU
stream test relies on are shown to pass a correct stream and to catch each way a stream can break its contract.

The fake is y[t] = g (x[t] + x[t-1] / 2) (x[-1] = 0 at BEGIN, g the slot's BEGIN value) released D samples behind its
input until END, with the running max of |x| since BEGIN as its reduction."""
import numpy as np
import pytest
import torch

from helpers import slot_streams as ss
from viettts_b200.engine import STREAM_BEGIN, STREAM_END


class FakeStream:
    def __init__(self, S, F, D, flaw=None):
        self.max_chunk_samples, self.out_pitch, self.D, self.flaw = F, F + D, D, flaw
        self.inp = [np.zeros(0, np.float32)] * S
        self.carry, self.E, self.gain = [np.float32(0)] * S, [0] * S, np.ones(S, np.float32)
        self.reduction_db = np.zeros(S, np.float32)

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        pass

    def _step(self, x, n_new, flags, gain):
        ys = []
        for s, (n, f) in enumerate(zip(n_new, flags)):
            if n == 0 and f == 0:
                ys.append(np.zeros(0, np.float32))
                continue
            new = x[s, :n].copy()
            if f & STREAM_BEGIN:
                if self.flaw != "state":
                    self.carry[s], self.reduction_db[s] = np.float32(0), 0
                elif self.inp[s].size:
                    self.carry[s] = self.inp[s][-1]
                self.inp[s], self.E[s], self.gain[s] = np.zeros(0, np.float32), 0, gain[s]
            elif self.flaw == "drop" and n:
                new = np.append(new[1:], np.float32(0))
            if self.flaw == "past" and 0 < n < x.shape[1]:
                new[-1] += 0 * x[s, n]
            a = self.inp[s] = np.concatenate([self.inp[s], new])
            if a.size:
                self.reduction_db[s] = max(self.reduction_db[s], np.abs(a).max())
            e = a.size if f & STREAM_END else max(0, a.size - self.D)
            prev = np.concatenate([[self.carry[s]], a[:-1]]).astype(np.float32)
            y = self.gain[s] * (a + np.float32(0.5) * prev)
            ys.append(np.concatenate([y[self.E[s]:e], [0] if self.flaw == "n_out" and f & STREAM_END else []]).astype(np.float32))
            self.E[s] = e
        return ys

    def push(self, x, n_new, begin, end, gain=None):
        flags = np.asarray(begin, np.uint8) * STREAM_BEGIN | np.asarray(end, np.uint8) * STREAM_END
        return self._step(np.asarray(x, np.float32), n_new, flags, gain)

    def push_device(self, x_t, n_new, flags, out_t, red_t, gain=None):
        ys = self._step(x_t.numpy().copy(), n_new, flags, gain)
        for s, y in enumerate(ys):
            if self.flaw == "idle":
                out_t[s] = 0
            out_t[s, :y.size] = torch.from_numpy(y)
        red_t.copy_(torch.from_numpy(self.reduction_db))
        return np.array([y.size for y in ys], np.int32)


def one_shot(x, g):
    prev = np.concatenate([[0], x[:-1]]).astype(np.float32)
    return (np.float32(g) * (x + np.float32(0.5) * prev)).astype(np.float32), (np.abs(x).max() if x.size else 0)


def fake(S, F, D=5, flaw=None, in_place=False):
    st = ss.Stage(None, "fake", lambda: FakeStream(S, F, D, flaw), lambda P, end, v: P if end else max(0, P - D), one_shot,
                  param="gain", reduction=True, in_place=in_place)
    st.device = "cpu"
    return st


def signal(s, u, n):
    return np.random.default_rng(100 * s + u).uniform(-1, 1, n).astype(np.float32)


def gains(plans, rng):
    return [[float(rng.uniform(0.5, 2)) for _ in p] for p in plans]


@pytest.mark.parametrize("D,in_place", [(5, False), (0, True)])
@pytest.mark.parametrize("host", [False, True])
def test_a_correct_stream_passes_every_plan_kind(host, D, in_place):
    F = 600                        # the "short" kind pushes 513 samples
    rng = np.random.default_rng(1)
    plans = [ss.push_plan(k, F, rng) for k in ss.KINDS]
    out = ss.run(fake(len(plans), F, D, in_place=in_place), plans, signal, gains(plans, rng), host=host)
    assert [len([o for o in row if o is not None]) for row in out] == [1, 1, 1, 1, 1, 1, 3, 2, 1, 0]


@pytest.mark.parametrize("host", [False, True])
@pytest.mark.parametrize("kind", ["one", "full", "random"])
def test_a_correct_stream_passes_every_pattern(kind, host):
    F, rng = 64, np.random.default_rng(2)
    plans = [[ss.pattern(kind, n, F, rng) for n in lengths] for lengths in ([0, 200], [1, 64, 65], [129])]
    out = ss.run(fake(3, F), plans, signal, gains(plans, rng), host=host)
    assert [o[2].size for row in out for o in row] == [0, 200, 1, 64, 65, 129]


@pytest.mark.parametrize("flaw,check,host", [("n_out", "n_out", True), ("n_out", "n_out", False),
                                              ("drop", "one-shot", True), ("idle", "idle slot's row", False),
                                              ("past", "read past n_new", True), ("past", "read past n_new", False),
                                              ("state", "one-shot", False)])
def test_a_broken_stream_is_caught(flaw, check, host):
    F, rng = 600, np.random.default_rng(3)
    plans = [ss.push_plan(k, F, rng) for k in ("reuse", "idle", 255, "late", "short")]
    with pytest.raises(AssertionError, match=check):
        ss.run(fake(len(plans), F, flaw=flaw), plans, signal, gains(plans, rng), host=host)
