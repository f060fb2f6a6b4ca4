"""CPU: every call of a context orders itself after the context's previous call (CallOrder, vtts_internal.cuh), whatever
stream it runs on.  Read from the sources: each entry point include/viettts_b200.h declares with a `void* stream` opens
a CallOrder on that stream before it uses the stream for anything else, or hands the stream to a helper that does; the
host-staging path (HostStage) opens one on the context's own stream when it is constructed; and every `*_host` entry
point reaches a HostStage.  A new entry point that skipped the ordering would fail here before it could race another
call in the shared workspace or tile-scheduler counters."""
import re
from pathlib import Path

import pytest

REPO = Path(__file__).resolve().parents[1]
CSRC = REPO / "viettts_b200" / "csrc"


def _strip(text):
    """the source without comments and string literals"""
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    text = re.sub(r"//[^\n]*", "", text)
    return re.sub(r'"(?:\\.|[^"\\])*"', '""', text)


def _declared():
    """{name: parameter text} of every function the header declares"""
    text = _strip((REPO / "include" / "viettts_b200.h").read_text())
    return {m.group(1): m.group(2) for m in re.finditer(r"\b(vtts_[a-z0-9_]+)\s*\(([^;{]*?)\)\s*;", text, flags=re.S)}


def _definitions():
    """{name: (parameter text, body)} of every int function defined at the top level of a .cu file"""
    out = {}
    for f in sorted(CSRC.glob("*.cu")):
        text = _strip(f.read_text())
        for m in re.finditer(r'^(?:static\s+|extern\s+""\s+)?int\s+(\w+)\s*\(([^;{]*?)\)\s*\{', text, flags=re.M | re.S):
            depth, i = 1, m.end()
            while depth:
                depth += {"{": 1, "}": -1}.get(text[i], 0)
                i += 1
            out.setdefault(m.group(1), (m.group(2), text[m.end():i - 1]))
    return out


DECLARED = _declared()
DEFS = _definitions()
STREAM_ENTRIES = sorted(n for n, p in DECLARED.items() if re.search(r"void\s*\*\s*stream\b", p))
HOST_ENTRIES = sorted(n for n in DECLARED if n.endswith("_host"))


def _orders_first(body, var):
    """True if the first use of `var` in `body` opens the CallOrder, or passes `var` to a function that orders on its
    own stream parameter first"""
    m = re.search(rf"\b{var}\b", body)
    if not m:
        return False
    line = body[body.rfind("\n", 0, m.start()) + 1:body.find("\n", m.end())]
    if re.search(rf"\bCallOrder\s+order\s*\(\s*ctx\s*,\s*{var}\s*\)", line):
        return True
    call = re.search(r"(\w+)\s*\([^;]*$", body[:m.start()])
    if not call or call.group(1) not in DEFS:
        return False
    params, helper = DEFS[call.group(1)]
    hvar = re.search(r"(?:void\s*\*|cudaStream_t)\s*(\w+)\s*$", params.strip())
    return bool(hvar) and _orders_first(helper, hvar.group(1))


def test_the_sources_are_parsed():
    assert len(STREAM_ENTRIES) >= 40 and len(HOST_ENTRIES) >= 40
    assert "vtts_hifigan_forward" in STREAM_ENTRIES and "vtts_vocoder_stream_push" in STREAM_ENTRIES
    missing = [n for n in STREAM_ENTRIES + HOST_ENTRIES if n not in DEFS]
    assert not missing, f"declared but not defined in {CSRC}: {missing}"


@pytest.mark.parametrize("name", STREAM_ENTRIES)
def test_stream_entry_point_orders_its_call(name):
    assert _orders_first(DEFS[name][1], "stream"), (
        f"{name} uses its stream before `const CallOrder order(ctx, stream);` (or a helper that opens it)")


def test_host_stage_orders_on_the_own_stream():
    text = _strip((CSRC / "stream_common.cuh").read_text())
    cls = text[text.index("class HostStage"):]
    cls = cls[:cls.index("\n};")]
    assert re.search(r"explicit HostStage\(vtts_ctx\* c\)\s*:[^{]*\border\(c, c->own_stream\)", cls)
    assert re.search(r"\bconst CallOrder order;", cls)
    # every launch and copy of a host call goes through `st`, the stream the CallOrder waits on
    assert re.search(r"\bst\(c->own_stream\)", cls)


def _reaches_host_stage(name, seen):
    if name in seen or name not in DEFS:
        return False
    seen.add(name)
    body = DEFS[name][1]
    if re.search(r"\bHostStage\s+hs\s*\(\s*ctx\s*\)", body):
        return True
    return any(_reaches_host_stage(c, seen) for c in re.findall(r"\b(\w+)\s*\(", body))


@pytest.mark.parametrize("name", HOST_ENTRIES)
def test_host_entry_point_stages_through_host_stage(name):
    assert _reaches_host_stage(name, set()), f"{name} never constructs a HostStage, so its call is not ordered"


def test_call_order_waits_and_records_the_tail():
    text = _strip((CSRC / "vtts_internal.cuh").read_text())
    cls = text[text.index("class CallOrder"):]
    cls = cls[:cls.index("\n};")]
    ctor = cls[cls.index("CallOrder(vtts_ctx*"):cls.index("~CallOrder")]
    dtor = cls[cls.index("~CallOrder"):]
    assert "cudaStreamWaitEvent(st, ctx->tail, 0)" in ctor and "cudaStreamIsCapturing" in ctor
    assert "cudaEventRecord(ctx->tail, st)" in dtor
    api = _strip((CSRC / "api.cu").read_text())
    assert "cudaEventCreateWithFlags(&ctx->tail, cudaEventDisableTiming)" in api and "cudaEventDestroy(ctx->tail)" in api
