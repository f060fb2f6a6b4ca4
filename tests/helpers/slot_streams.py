"""The library's per-slot sample streams as the tests drive them: one table of stages, the push plans, and one driver.

Every stream's contract: a slot's outputs, concatenated over one utterance (BEGIN ... END), equal the stage's one-shot
call on the utterance's whole input bit for bit, and each push emits exactly what the stage's counting formula
E(P, end, v) gives (outputs after P inputs, v the slot's BEGIN value).  `run` holds a stream to it on every push."""
import numpy as np

from oracle import denoise_oracle as do
from oracle import resample_oracle as ro
from oracle import time_stretch_oracle as tso
from viettts_b200 import config
from viettts_b200.engine import STREAM_BEGIN, STREAM_END, reverb_stream_emitted

SR = config.SAMPLE_RATE
SENTINEL = np.float32(12345.0)      # fills an output buffer before a device push: what an idle slot's row must keep


def floats(vals):
    """float32 [S]: each slot's BEGIN value, NaN for the slots a push does not begin (the stream must not read it)"""
    return np.array([np.nan if v is None else v for v in vals], np.float32)


class Stage:
    """One sample stream: `open()` gives its handle (S slots, chunk F, the stage's spec); `emitted(P, end, v)` its
    counting formula; `one_shot(x, v)` its one-shot call on one row, (y, reduction or None); `param` its BEGIN keyword
    and `begin(vals)` the push's keywords for per-slot values `vals` (None: the slot does not begin), with the values
    the slots actually take; `reduction` / `meter` what else a push writes; `in_place` whether a device push runs with
    out_t = x_t; `launches` the launches of every push, where the stage states them; `device` where its buffers live."""
    device = "cuda"

    def __init__(self, eng, name, open_, emitted, one_shot, param=None, begin=None, reduction=False, meter=False,
                 in_place=False, launches=None):
        self.eng, self.name, self.open, self.emitted, self.one_shot = eng, name, open_, emitted, one_shot
        self.param, self.reduction, self.meter, self.in_place, self.launches = param, reduction, meter, in_place, launches
        if begin is not None:
            self.begin = begin

    def begin(self, vals):
        return ({} if self.param is None else {self.param: floats(vals)}), vals

    def push_device(self, st, x_t, n_new, flags, y_t, red_t, kw):
        """n_out of a device push (None for the meter, which fills y_t with its readings)"""
        if self.meter:
            st.push_device(x_t, n_new, flags, y_t)
            return None
        return st.push_device(x_t, n_new, flags, y_t, *((red_t,) if self.reduction else ()), **kw)


def stage(eng, name, S, F, rate=SR, **spec):
    """the table: stream `name` with S slots of chunk F at `rate` Hz and its spec (the keywords its open call takes)"""
    def hop(P, end, v=None):
        return P if end else do.emitted_closed_form(P)

    def no_lookahead(P, end, v=None):
        return P

    if name == "resample":
        rates = (rate, spec["out_rate"])
        return Stage(eng, name, lambda: eng.open_resample_stream(S, F, rates[1], in_rate=rate),
                     lambda P, end, v=None: ro.out_len(P, *rates) if end else ro.emitted_closed_form(P, *rates),
                     lambda x, v: (eng.resample(x, rates[1], in_rate=rate), None), launches=2)
    if name == "denoise":
        return Stage(eng, name, lambda: eng.open_denoise_stream(S, F, spec["strength"], bias=spec["bias"]), hop,
                     lambda x, v: (eng.denoise(x, spec["strength"], bias=spec["bias"]), None), launches=3)
    if name == "pitch":
        return Stage(eng, name, lambda: eng.open_pitch_shift_stream(S, F), hop,
                     lambda x, v: (eng.pitch_shift(x, v), None), param="semitones", launches=5)
    if name == "voice_shift":
        return Stage(eng, name, lambda: eng.open_voice_shift_stream(S, F), hop,
                     lambda x, v: (eng.pitch_shift(x, v[0], formant=v[1]), None), begin=voice_begin, launches=5)
    if name == "time_stretch":
        return Stage(eng, name, lambda: eng.open_time_stretch_stream(S, F),
                     lambda P, end, v: tso.stretch_emitted(P, v, end),
                     lambda x, v: (eng.time_stretch(x, v), None), param="tempo", launches=5)
    if name == "limiter":
        la_ms, rel_ms = spec.get("lookahead_ms", 5.0), spec.get("release_ms", 100.0)
        la = eng.limiter_stream_lookahead(rate, la_ms)
        return Stage(eng, name, lambda: eng.open_limiter_stream(S, F, rate, spec["ceiling"], la_ms, rel_ms),
                     lambda P, end, v=None: P if end else max(0, P - la),
                     lambda x, v: eng.limit(x, spec["ceiling"], rate, gain_db=v, lookahead_ms=la_ms, release_ms=rel_ms),
                     param="gain_db", reduction=True)
    if name == "eq":
        return Stage(eng, name, lambda: eng.open_eq_stream(S, F, spec["eq"], rate), no_lookahead,
                     lambda x, v: (eng.equalize(x, spec["eq"], rate), None), in_place=True)
    if name in ("compressor", "deesser"):
        open_, call = ((eng.open_compressor_stream, eng.compress) if name == "compressor" else
                       (eng.open_deesser_stream, eng.deess))
        return Stage(eng, name, lambda: open_(S, F, spec["spec"], rate), no_lookahead,
                     lambda x, v: call(x, spec["spec"], rate), reduction=True, in_place=True)
    if name == "reverb":
        return Stage(eng, name, lambda: eng.open_reverb_stream(S, F, spec["spec"], rate),
                     lambda P, end, v=None: reverb_stream_emitted(P, end),
                     lambda x, v: (eng.reverb(x, spec["spec"], rate), None))
    if name == "watermark":
        return Stage(eng, name, lambda: eng.open_watermark_stream(S, F, spec["spec"]), hop,
                     lambda x, v: (eng.watermark(x, spec["spec"]), None))
    if name == "bed":
        bank = eng.prepare_beds(spec["bed"], rate)
        tail = bank.params[0]["Tt"]

        def mix(x, v):          # a row of zero samples still gets the bed's tail
            y, red = eng.mix_bed(x[None] if x.size else np.zeros((1, 1), np.float32), bank, rate, lengths=[x.size],
                                 index=[v])
            return y[0, :x.size + (tail if v >= 0 else 0)], red[0]
        return Stage(eng, name, lambda: eng.open_bed_stream(S, F, bank, rate),
                     lambda P, end, v=0: P + (tail if end and v >= 0 else 0), mix, param="bed",
                     begin=lambda vals: ({"bed": np.array([0 if v is None else v for v in vals], np.int32)}, vals),
                     reduction=True)
    if name == "loudness":
        return Stage(eng, name, lambda: eng.open_loudness_meter(S, F, rate, max_seconds=spec["max_seconds"]), None,
                     lambda x, v: (None, eng.loudness(x, rate)), meter=True)
    raise KeyError(name)


def voice_begin(vals):
    """values (semitones, formant or None: the formants follow the pitch).  A push that passes formants gives one to
    every slot it begins (NaN is rejected with BEGIN), so there the slots drawn to follow the pitch keep their formants
    (formant 0)."""
    if all(v is None or v[1] is None for v in vals):
        return {"semitones": floats([None if v is None else v[0] for v in vals]), "formant": None}, vals
    vals = [v if v is None or v[1] is not None else (v[0], 0.0) for v in vals]
    return {"semitones": floats([None if v is None else v[0] for v in vals]),
            "formant": floats([None if v is None else v[1] for v in vals])}, vals


# ---- plans: per slot, a list of utterances, each a list of push sizes --------------------------------------------------
# BEGIN goes with an utterance's first push and END with its last; a size None is a push the slot sits out (no flags),
# and a size 0 between them is an idle push of an open slot.

KINDS = ["ones", 255, 256, 1000, "max", "end_empty", "short", "reuse", "late", "idle"]


def push_plan(kind, F, rng):
    """the utterances of one slot of plan kind `kind` ("late" sits out a few pushes before it begins)"""
    if kind == "ones":
        return [[1] * int(rng.integers(1100, 1500))]
    if kind in (255, 256, 1000):
        return [[min(kind, F)] * int(rng.integers(4, 12))]
    if kind == "max":
        return [[F] * int(rng.integers(2, 5)) + [int(rng.integers(1, F))]]
    if kind == "end_empty":
        return [[int(v) for v in rng.integers(1, F + 1, size=4)] + [0]]
    if kind == "short":
        return [[int(rng.integers(1, 200)), int(rng.integers(0, 200))], [512], [513]]
    if kind == "reuse":
        return [[int(v) for v in rng.integers(1, F + 1, size=3)], [int(v) for v in rng.integers(1, F + 1, size=5)]]
    if kind == "late":
        return [[None] * int(rng.integers(2, 6)), [int(v) for v in rng.integers(1, F + 1, size=6)]]
    assert kind == "idle", kind
    return []


def pattern(kind, n, F, rng):
    """one utterance of n samples in `kind` pushes: "one" sample, "full" chunks of F, or "random" sizes in [0, F]"""
    sizes = []
    while n > 0 or not sizes:
        k = 1 if kind == "one" else F if kind == "full" else int(rng.integers(0, F + 1))
        sizes.append(min(k, n))
        n -= sizes[-1]
    return sizes


def _pushes(plan):
    """[(n_new, flags, utterance) or None] of one slot's plan"""
    out = []
    for u, sizes in enumerate(plan):
        real = [q for q, n in enumerate(sizes) if n is not None]
        for q, n in enumerate(sizes):
            if n is not None:
                out.append((n, (STREAM_BEGIN if q == real[0] else 0) | (STREAM_END if q == real[-1] else 0), u))
            else:
                out.append(None)
    return out


# ---- the driver ----------------------------------------------------------------------------------------------------------

def run(stage, plans, signal, values=None, host=False):
    """Pushes `plans` (one per slot) through `stage`, through `push` (host) or `push_device`; `signal(s, u, n)` is the
    input of slot s's utterance u (n samples) and `values[s][u]` its BEGIN value.  Every input past n_new is NaN.  On
    every push: n_out is the counting formula's; an idle slot (n_new = 0, no flags) emits nothing and leaves its output
    row (device) and its reduction as they were; no output is NaN, so none read an input past n_new; the launches are
    the stage's.  At END: the utterance's outputs, concatenated, and its reduction equal the one-shot call bit for bit.
    Returns per slot and utterance (input, BEGIN value, outputs, reduction at END), None for one with no pushes."""
    import torch
    S = len(plans)
    pushes = [_pushes(p) for p in plans]
    xs = [[signal(s, u, sum(n for n in sizes if n)) for u, sizes in enumerate(p)] for s, p in enumerate(plans)]
    value = [[None if values is None else values[s][u] for u in range(len(p))] for s, p in enumerate(plans)]
    got = [[[] for _ in p] for p in plans]
    out = [[None] * len(p) for p in plans]
    P, E, pos = [0] * S, [0] * S, [0] * S
    red_prev = None
    with stage.open() as st:
        F = st.max_chunk_samples
        x_t = torch.zeros((S, F), dtype=torch.float32, device=stage.device)
        y_t = x_t if stage.in_place else torch.empty((S, st.out_pitch), dtype=torch.float32, device=stage.device)
        red_t = torch.zeros(S, dtype=torch.float32, device=stage.device) if stage.reduction else None
        for c in range(max(map(len, pushes))):
            n_new, flags = np.zeros(S, np.int32), np.zeros(S, np.uint8)
            x = np.full((S, F), np.nan, np.float32)
            begins = [None] * S
            for s in range(S):
                p = pushes[s][c] if c < len(pushes[s]) else None
                if p is None:
                    continue
                n_new[s], flags[s], u = p
                if flags[s] & STREAM_BEGIN:
                    pos[s] = P[s] = E[s] = 0
                    begins[s] = value[s][u]
                x[s, :n_new[s]] = xs[s][u][pos[s]:pos[s] + n_new[s]]
                pos[s] += n_new[s]
            kw, taken = stage.begin(begins)
            for s in np.flatnonzero(flags & STREAM_BEGIN):
                value[s][pushes[s][c][2]] = taken[s]
            c0 = stage.eng.launch_count() if stage.launches else 0
            if host:
                ys = st.push(x, n_new, (flags & STREAM_BEGIN) != 0, (flags & STREAM_END) != 0, **kw)
                n_out = [y.size for y in ys]
                red = st.reduction_db.copy() if stage.reduction else None
            else:
                x_t.copy_(torch.from_numpy(x))
                if not stage.in_place:
                    y_t.fill_(float(SENTINEL))
                n_out = stage.push_device(st, x_t, n_new, flags, y_t, red_t, kw)
                y = y_t.cpu().numpy()
                ys = [y[s, :n_out[s]] for s in range(S)]
                red = red_t.cpu().numpy().copy() if stage.reduction else None
            if stage.launches:
                assert stage.eng.launch_count() - c0 == stage.launches, ("launches", stage.name, c)
            for s in range(S):
                what = (stage.name, s, c, int(n_new[s]), int(flags[s]))
                if n_new[s] == 0 and flags[s] == 0:
                    assert n_out[s] == 0, ("n_out of an idle slot",) + what
                    if not host:
                        before = x[s] if stage.in_place else np.full(y.shape[1], SENTINEL)
                        assert np.array_equal(y[s].view(np.uint32), before.view(np.uint32)), ("idle slot's row",) + what
                    if red_prev is not None:
                        assert red[s] == red_prev[s], ("idle slot's reduction",) + what
                    continue
                u = pushes[s][c][2]
                end = bool(flags[s] & STREAM_END)
                P[s] += int(n_new[s])
                e = stage.emitted(P[s], end, value[s][u])
                assert n_out[s] == e - E[s], ("n_out", P[s], int(n_out[s]), e - E[s]) + what
                E[s] = e
                assert not np.isnan(ys[s]).any(), ("an output read past n_new",) + what
                got[s][u].append(ys[s].copy())
                if end:
                    y_u = np.concatenate(got[s][u])
                    ref, rref = stage.one_shot(xs[s][u], value[s][u])
                    assert y_u.shape == ref.shape and np.array_equal(y_u, ref), ("one-shot",) + what + (u, value[s][u])
                    if stage.reduction:
                        assert red[s] == rref, ("one-shot reduction", float(red[s]), float(rref)) + what
                    out[s][u] = (xs[s][u], value[s][u], y_u, red[s] if stage.reduction else None)
            red_prev = red
    return out
