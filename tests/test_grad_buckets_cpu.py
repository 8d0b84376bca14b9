"""The backward-event contract that `GradSync`'s overlapped all-reduce relies on, checked on the launch trace of lm_step.cu
without a GPU (tests/lm_schedule: every launch with its arguments, pointers as <buffer>+<byte offset>).

`GradSync` reduces bucket (lo..hi) on a side stream as soon as backward event `lo` has fired, and the tail (final norm,
tables, head) after the whole backward pass.  That is only correct if
  * every launch that writes a gradient of layer l is enqueued before `cudaEventRecord(bwd_events[l])`, in every decoder
    variant, and the events are recorded L..0, once each, on the compute stream;
  * `GradSync.layer_start` (the `layers.l.ln1` offsets, then `final_norm`, or `embed` for a post-LN OPT) bounds each
    layer's tensors, and its bucket plan plus the tail covers the flat buffer exactly once with ranges the peer-memory
    kernel accepts.
A gradient write is a non-const pointer parameter of the launcher's kernels.h declaration, `C` / `C_lo` / `aux_out` of
an `SkGemmEx`, or a `cudaMemsetAsync` destination, that points into `grads`.  Models with fp32 master weights are not
covered: `GradSync` refuses them for more than one rank (their `sk_widen_grads` reads `grads` after event 0)."""
import os
import re
import shutil
import types

import numpy as np
import pytest

import test_lm_schedule_cpu as S

# the bf16 training variants of tests/lm_schedule/driver.cpp
VARIANTS = ["qwen2", "qwen2 untied, no qkv bias", "qwen2 chunked head (SK_HEAD_CHUNK)", "qwen2 large vocabulary",
            "opt", "opt untied", "opt chunked head",
            "opt post-ln", "opt post-ln chunked head", "opt post-ln proj", "opt post-ln proj chunked head",
            "neox", "neox chunked head"]
GEMM_WRITES = ("C", "C_lo", "aux_out")
# pointer parameters that only read the gradient buffer
READS = {("*", "residual"), ("sk_widen_grads_launch", "g16")}
EVENTS_ON = "-- sk_lm_set_backward_events(lm, events.data(), L + 1)"
EVENTS_OFF = "-- sk_lm_set_backward_events(lm, nullptr, 0)"

pytestmark = pytest.mark.skipif(S.NVCC is None or shutil.which("g++") is None, reason="needs nvcc and g++")


def written_params():
    """{launcher: [names of its non-const pointer parameters, in declaration order]} from kernels.h"""
    header = S._strip_comments(open(os.path.join(S.CSRC, "kernels.h")).read())
    out = {}
    for m in re.finditer(r"^(extern \"C\" )?(int|size_t|SkGemmEx)\s+(sk_\w+)\(([^)]*)\)\s*;", header, re.M):
        params = S._params(m.group(4))
        out[m.group(3)] = [(i, n) for i, (t, n) in enumerate(params)
                           if "*" in t and not t.startswith("const") and ("*", n) not in READS and (m.group(3), n) not in READS]
    return out


def _args(line):
    return line[line.index("(") + 1:line.rindex(")")].split(", ")


def _grad_elem(arg):
    m = re.fullmatch(r"grads\+(\d+)", arg.strip())
    return int(m.group(1)) // 2 if m else None


def parse(text):
    """{variant: (tensors {name: (offset, elements)}, n_params, [("write", launch, first, end) | ("event", k, stream)])}
    with the events and writes of the one forward-backward pass that runs with backward events set."""
    writes = written_params()
    out, cur = {}, None
    for name, lines in S.phases(text):
        variant, phase = name.split(": ", 1)
        if phase == "create":
            tensors, n_params = {}, None
            for ln in lines:
                m = re.match(r"tensor (\S+) off=(\d+) \[(\d+), (\d+)\]$", ln)
                if m:
                    tensors[m.group(1)] = (int(m.group(2)), int(m.group(3)) * int(m.group(4)))
                m = re.match(r"param_count (\d+)$", ln)
                if m:
                    n_params = int(m.group(1))
            cur = out[variant] = (tensors, n_params, [])
        if phase != "training":
            continue
        on = False
        for ln in lines:
            if ln == EVENTS_ON:
                on = True
                continue
            if ln == EVENTS_OFF:
                break
            if not on or ln.startswith("-- ") or ln.startswith("-> "):
                continue
            fn = ln[:ln.index("(")] if "(" in ln else ln
            if fn == "cudaEventRecord":
                ev, stream = _args(ln)
                cur[2].append(("event", int(re.fullmatch(r"events\+(\d+)", ev).group(1)), stream))
            elif fn == "cudaMemsetAsync":
                dst, _, nbytes, _ = _args(ln)
                e = _grad_elem(dst)
                if e is not None:
                    cur[2].append(("write", ln, e, e + int(nbytes) // 2))
            elif fn == "sk_gemm_ex_launch":
                for field in GEMM_WRITES:
                    e = _grad_elem(re.search(rf"\b{field}=(\S+)", ln).group(1))
                    if e is not None:
                        cur[2].append(("write", ln, e, e + 1))
            elif fn in writes:
                args = _args(ln)
                for i, _ in writes[fn]:
                    e = _grad_elem(args[i])
                    if e is not None:
                        cur[2].append(("write", ln, e, e + 1))
    return out


@pytest.fixture(scope="module")
def traced(tmp_path_factory):
    return parse(S.trace(str(tmp_path_factory.mktemp("lm_schedule"))))


def _sync(tensors, n_params, n_layers, layers_per_bucket):
    """The product GradSync on a stand-in model with this layout (one process: nothing is reduced)."""
    from slamkit_b200.trainer import GradSync
    model = types.SimpleNamespace(config=types.SimpleNamespace(n_layers=n_layers), n_params=n_params, grads=None,
                                  tensors={k: (o, 1, n) for k, (o, n) in tensors.items()}, master=False)
    return GradSync(model, layers_per_bucket=layers_per_bucket, overlap=True)


def _layer(name):
    m = re.match(r"layers\.(\d+)\.", name)
    return int(m.group(1)) if m else None


def test_every_bf16_training_variant_is_traced(traced):
    assert set(VARIANTS) <= set(traced), sorted(set(VARIANTS) - set(traced))
    written = written_params()
    for fn, names in (("sk_rmsnorm_bwd_launch", {"dx", "dw"}), ("sk_layernorm_bwd_launch", {"dw", "db"}),
                      ("sk_embed_bwd_launch", {"dE"}), ("sk_colsum_launch", {"out"})):
        assert names <= {n for _, n in written[fn]}, fn          # the parser sees the launchers' outputs


@pytest.mark.parametrize("variant", VARIANTS)
def test_backward_events_follow_every_gradient_write_of_their_layer(traced, variant):
    tensors, n_params, log = traced[variant]
    L = max(_layer(n) for n in tensors if _layer(n) is not None) + 1
    events = [(x[1], x[2]) for x in log if x[0] == "event"]
    assert [k for k, _ in events] == list(range(L, -1, -1)), events       # L..0, once each, in backward order
    assert all(s == "stream+0" for _, s in events), events                # on the compute stream
    fired = set()
    n_writes = {l: 0 for l in range(L)}
    for x in log:
        if x[0] == "event":
            fired.add(x[1])
            continue
        _, line, lo, hi = x
        owners = [n for n, (o, sz) in tensors.items() if o <= lo and hi <= o + sz]
        assert len(owners) == 1, f"gradient write outside the layout (elements [{lo}, {hi})): {line}"
        l = _layer(owners[0])
        if l is not None:
            assert l not in fired, f"{owners[0]} is written after backward event {l} was recorded: {line}"
            n_writes[l] += 1
    assert all(n_writes.values()), n_writes                                # the parser found every layer's writes


@pytest.mark.parametrize("variant", VARIANTS)
def test_layer_start_bounds_every_layer_and_the_buckets_cover_the_buffer(traced, variant):
    from slamkit_b200.p2p import PeerAllReduce
    tensors, n_params, _ = traced[variant]
    L = max(_layer(n) for n in tensors if _layer(n) is not None) + 1
    spans = sorted((o, o + sz, n) for n, (o, sz) in tensors.items())
    assert spans[-1][1] <= n_params and all(a[1] <= b[0] for a, b in zip(spans, spans[1:])), "tensors overlap"
    for lpb in (1, 2, 4):
        sync = _sync(tensors, n_params, L, lpb)
        start = sync.layer_start
        assert len(start) == L + 1
        for name, (o, sz) in tensors.items():
            l = _layer(name)
            if l is not None:
                assert start[l] <= o and o + sz <= start[l + 1], (name, o, sz, start)
            else:
                assert o >= start[L], (name, o, start)
        cover = np.zeros(n_params, dtype=np.int32)
        ranges = [(lo, hi) for _, lo, hi in sync.buckets] + [sync.tail]
        for lo, hi in ranges:
            assert PeerAllReduce.supports(lo, hi), (lo, hi)          # no bucket of a real layout falls back to NCCL
            cover[lo:hi] += 1
        assert (cover == 1).all(), f"layers_per_bucket={lpb}: {ranges}"
        assert [ev for ev, _, _ in sync.buckets] == sorted({max(0, h - lpb) for h in range(L, 0, -lpb)}, reverse=True)
