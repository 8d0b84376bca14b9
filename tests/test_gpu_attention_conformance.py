"""Conformance of the attention kernels (attention.cu, decode.cu) per element, against the references of tests/attn_ref.py.

Every entry point: sk_attn_tc_fwd / sk_attn_tc_bwd (causal, plain and packed), sk_attn_fwd / sk_attn_bwd (also
bidirectional), the split-bf16 HuBERT forward sk_attn_tc_fwd_split and sk_attn_decode.  Exact modes are compared bit for
bit over T in {1, 2, 63, 64, 65, 127, 128, 129, 200, 255, 257, 1024, 2048} (and a packed 8192-token row) and the GQA
groups the configs use; random data with adversarial score patterns against the per-element contract; isolation of
documents, future rows and batch rows bit for bit; decode against the prefill kernel; pitched inputs with NaN padding
and outputs inside sentinel-filled buffers; dependent launches back to back; argument checks in a child process.
"""
import ctypes as C
import os
import subprocess
import sys

import pytest
import torch

import attn_ref as A

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
BF = torch.bfloat16
T_SWEEP = [1, 2, 63, 64, 65, 127, 128, 129, 200, 255, 257, 1024, 2048]
HEADS = [(14, 2), (12, 12), (2, 1), (16, 2), (12, 2)]
SENT16 = 0x7FB5                       # a NaN payload no kernel produces
SENT32 = 0x7FC0DEAD


def _lib():
    from slamkit_b200 import _lib as L
    return L, L.require_cuda()


def _p(t, off=0):
    return C.c_void_p(t.data_ptr() + off * t.element_size()) if t is not None else C.c_void_p(0)


def run_fwd(entry, qkv, B, T, H, KVH, causal=True, scale=0.125, seg=None, o=None, lse=None):
    """entry "tc" (sk_attn_tc_fwd, fused projection) or "plain" (sk_attn_fwd, three column slices)."""
    L, lib = _lib()
    o = torch.empty(B * T, H * 64, dtype=BF, device=DEV) if o is None else o
    lse = torch.empty(B, H, T, dtype=torch.float32, device=DEV) if lse is None else lse
    if entry == "tc":
        L.check(lib.sk_attn_tc_fwd(_p(qkv), _p(o), _p(lse), B, T, H, KVH, qkv.stride(0), o.stride(0), int(causal),
                                   L.f32(scale), _p(seg), L.stream_ptr()))
    else:
        assert seg is None
        L.check(lib.sk_attn_fwd(_p(qkv), _p(qkv, H * 64), _p(qkv, (H + KVH) * 64), _p(o), _p(lse), B, T, H, KVH,
                                qkv.stride(0), o.stride(0), int(causal), L.f32(scale), L.stream_ptr()))
    return o, lse


def run_bwd(entry, qkv, o, do, lse, B, T, H, KVH, causal=True, scale=0.125, seg=None, seg_end=None, dqkv=None):
    L, lib = _lib()
    assert o.stride(0) == do.stride(0)
    dqkv = torch.empty(B * T, (H + 2 * KVH) * 64, dtype=BF, device=DEV) if dqkv is None else dqkv
    delta = torch.empty(B * H * T, dtype=torch.float32, device=DEV)
    if entry == "tc":
        L.check(lib.sk_attn_tc_bwd(_p(qkv), _p(o), _p(do), _p(lse), _p(delta), None, _p(dqkv), B, T, H, KVH, qkv.stride(0),
                                   o.stride(0), dqkv.stride(0), int(causal), L.f32(scale), _p(seg), _p(seg_end),
                                   L.stream_ptr()))
    else:
        assert seg is None
        L.check(lib.sk_attn_bwd(_p(qkv), _p(qkv, H * 64), _p(qkv, (H + KVH) * 64), _p(o), _p(do), _p(lse), _p(delta),
                                _p(dqkv), _p(dqkv, H * 64), _p(dqkv, (H + KVH) * 64), B, T, H, KVH, qkv.stride(0),
                                o.stride(0), dqkv.stride(0), int(causal), L.f32(scale), L.stream_ptr()))
    return dqkv


def run_decode(q, kc, vc, lens, H, KVH, scale=0.125, o=None, ldq=None):
    L, lib = _lib()
    B, Tc = kc.shape[0], kc.shape[2]
    o = torch.empty(B, H * 64, dtype=BF, device=DEV) if o is None else o
    part = torch.empty(int(lib.sk_attn_decode_partial_bytes(B, H, Tc)) // 4, dtype=torch.float32, device=DEV)
    L.check(lib.sk_attn_decode(_p(q), ldq or q.stride(0), _p(kc), _p(vc), _p(lens), _p(o), o.stride(0), _p(part), B, H, KVH,
                               Tc, L.f32(scale), L.stream_ptr()))
    return o


def _check(rep):
    assert rep is None, str(rep)


def _seg_dev(seg):
    """(seg_start, seg_end) int32 [B*T] on the device, via sk_seg_bounds from position ids (the LM's path), checked
    against the reference's document starts."""
    from slamkit_b200 import ops
    B, T = seg.shape
    pos = torch.arange(T)[None].expand(B, T) - seg
    ss, se = ops.seg_bounds(pos.to(DEV))
    assert torch.equal(ss.cpu().view(B, T).long(), seg)
    return ss, se


def _onehot(B, T, H, KVH, causal=True, seg=None, seed=0):
    lo, hi = A.bounds(B, T, causal, seg)
    modes = A.modes_for(H)
    tg = A.onehot_targets(lo, hi, modes)
    q, k = A.onehot_q(tg, modes), A.onehot_k(B, T, KVH)
    v = A.int_values((B, T, KVH, 64), 8, seed + T + H)
    return q, k, v, tg, lo, hi


def _exact_fwd(entry, B, T, H, KVH, causal, seg=None, tag=""):
    """one-hot and uniform forward, bit for bit (lse: 0 exactly, log n within 2 ulps)"""
    G = H // KVH
    segd = _seg_dev(seg)[0] if seg is not None else None
    q, k, v, tg, lo, hi = _onehot(B, T, H, KVH, causal, seg)
    o, lse = run_fwd(entry, A.fuse(q, k, v, device=DEV), B, T, H, KVH, causal, seg=segd)
    want_o, _ = A.expect_onehot_fwd(v, tg, G)
    what = f"{entry} causal={causal} B={B} T={T} H={H} KVH={KVH}{tag}"
    _check(A.mismatch_exact(A.heads(o, B, T, H), want_o, f"one-hot O {what}"))
    lse_c = A.lse_bth(lse)
    _check(A.mismatch_exact(lse_c, torch.zeros_like(lse_c), f"one-hot lse {what}"))
    vu = A.int_values((B, T, KVH, 64), 64, T + 1)
    o, lse = run_fwd(entry, A.fuse(torch.zeros_like(q), k, vu, device=DEV), B, T, H, KVH, causal, seg=segd)
    want_o, want_l = A.expect_uniform_fwd(vu, lo, hi, G)
    _check(A.mismatch_exact(A.heads(o, B, T, H), want_o, f"uniform O {what}"))
    _check(A.mismatch_lse_exact(A.lse_bth(lse), want_l, f"uniform lse {what}"))


def _exact_bwd(entry, B, T, H, KVH, causal, seg=None, tag=""):
    """one-hot backward with o = 0 (dS = dP / 8 on the target) and with the true o (dQ = dK = 0), bit for bit"""
    G = H // KVH
    ss, se = _seg_dev(seg) if seg is not None else (None, None)
    q, k, _, tg, lo, hi = _onehot(B, T, H, KVH, causal, seg)
    v, do = A.onehot_bwd_inputs(tg, KVH, T, seed=T + 7)
    qkv = A.fuse(q, k, v, device=DEV)
    dod = do.reshape(B * T, H * 64).to(BF).to(DEV)
    what = f"{entry} causal={causal} B={B} T={T} H={H} KVH={KVH}{tag}"
    zero_o = torch.zeros(B * T, H * 64, dtype=BF, device=DEV)
    zero_l = torch.zeros(B, H, T, dtype=torch.float32, device=DEV)
    for true_o in (False, True):
        if true_o:
            o, lse = run_fwd(entry, qkv, B, T, H, KVH, causal, seg=ss)
        else:
            o, lse = zero_o, zero_l
        dqkv = run_bwd(entry, qkv, o, dod, lse, B, T, H, KVH, causal, seg=ss, seg_end=se)
        dq, dk, dv = A.expect_onehot_bwd(q, k, v, do, tg, G, true_o=true_o)
        gq, gk, gv = A.unfuse(dqkv, B, T, H, KVH)
        w = f"{what} {'true o' if true_o else 'o = 0'}"
        _check(A.mismatch_exact(gq, dq, f"dQ {w}"))
        _check(A.mismatch_exact(gk, dk, f"dK {w}", rows="key"))
        _check(A.mismatch_exact(gv, dv, f"dV {w}", rows="key"))


# --------------------------------------------------------------------------------------------------- exact modes
@pytest.mark.parametrize("H,KVH", HEADS, ids=[f"H{h}KV{k}" for h, k in HEADS])
@pytest.mark.parametrize("T", T_SWEEP)
def test_exact_forward(T, H, KVH):
    for entry in ("tc", "plain"):
        _exact_fwd(entry, 2, T, H, KVH, True)
    _exact_fwd("plain", 2, T, H, KVH, False)


@pytest.mark.parametrize("H,KVH", HEADS, ids=[f"H{h}KV{k}" for h, k in HEADS])
@pytest.mark.parametrize("T", T_SWEEP)
def test_exact_backward(T, H, KVH):
    for entry in ("tc", "plain"):
        _exact_bwd(entry, 2, T, H, KVH, True)
    _exact_bwd("plain", 2, T, H, KVH, False)


# boundaries at tile offsets 0, +-1, 63/64/65, 127/128/129; length-1 documents at a tile start (64) and a tile end
# (63, 127); a document filling a whole tile ([192, 256)); a ragged tail
PACKED = {
    "boundaries": [[63, 1, 1, 63, 1, 128, 143], [1, 126, 1, 1, 63, 64, 144]],
    "tail": [[129, 1, 1, 70], [64, 64, 64, 9]],
}


def _cfg4_docs(seed=0):
    g = torch.Generator().manual_seed(seed)
    docs, t = [], 0
    while t < 8192:
        n = int(torch.randint(512, 2049, (1,), generator=g))
        n = 8192 - t if 8192 - t < 512 + 512 else min(n, 8192 - t - 512)
        docs.append(n)
        t += n
    return [docs]


@pytest.mark.parametrize("H,KVH", [(14, 2), (2, 1)], ids=["H14KV2", "H2KV1"])
@pytest.mark.parametrize("layout", list(PACKED) + ["cfg4"])
def test_exact_packed(layout, H, KVH):
    docs = _cfg4_docs() if layout == "cfg4" else PACKED[layout]
    B, T = len(docs), sum(docs[0])
    seg = A.doc_starts(B, T, docs)
    _exact_fwd("tc", B, T, H, KVH, True, seg, f" packed {layout}")
    _exact_bwd("tc", B, T, H, KVH, True, seg, f" packed {layout}")


def test_exact_t8192_unpacked_forward():
    """One 8192-token document: the longest rows, lse = log(8192) counts every key."""
    _exact_fwd("tc", 1, 8192, 2, 1, True)


# --------------------------------------------------------------------------------------------------- isolation
def _rand(shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return A.bf16(torch.randn(shape, generator=g) * scale)


def _fwd_bwd(qkv, do, B, T, H, KVH, seg=None):
    ss, se = _seg_dev(seg) if seg is not None else (None, None)
    o, lse = run_fwd("tc", qkv, B, T, H, KVH, True, seg=ss)
    dqkv = run_bwd("tc", qkv, o, do, lse, B, T, H, KVH, True, seg=ss, seg_end=se)
    return o.cpu(), lse.cpu(), dqkv.cpu()


def test_isolation_of_documents():
    """Changing every other document's q / k / v / dO (finite values) leaves a document's O, lse, dQ, dK, dV unchanged."""
    H, KVH = 14, 2
    docs = PACKED["boundaries"]
    B, T = 2, sum(docs[0])
    seg = A.doc_starts(B, T, docs)
    W = (H + 2 * KVH) * 64
    x, do = _rand((B * T, W), 1, 2.0), _rand((B * T, H * 64), 2)
    base = _fwd_bwd(x.to(BF).to(DEV), do.to(BF).to(DEV), B, T, H, KVH, seg)
    starts = sorted(set(seg[0].tolist())) + [T]
    for a, e in zip(starts[:-1], starts[1:]):
        keep = torch.zeros(B * T, dtype=torch.bool)
        keep[a:e] = True                                                   # document [a, e) of batch row 0
        x2 = torch.where(keep[:, None], x, _rand((B * T, W), 3 + a, 3.0))
        do2 = torch.where(keep[:, None], do, _rand((B * T, H * 64), 4 + a))
        got = _fwd_bwd(x2.to(BF).to(DEV), do2.to(BF).to(DEV), B, T, H, KVH, seg)
        for name, g, w in zip(("O", "lse", "dqkv"), got, base):
            if name == "lse":
                g, w = g[0, :, a:e], w[0, :, a:e]
            else:
                g, w = g[a:e], w[a:e]
            assert torch.equal(g, w), f"{name} of document [{a}, {e}) changed when the other documents did"


@pytest.mark.parametrize("t", [0, 63, 100, 128, 511])
def test_isolation_of_future_rows(t):
    """Changing rows > t leaves O, lse and dQ of rows <= t unchanged."""
    B, T, H, KVH = 2, 600, 12, 2
    W = (H + 2 * KVH) * 64
    x, do = _rand((B, T, W), 5, 2.0), _rand((B, T, H * 64), 6)
    base = _fwd_bwd(x.reshape(B * T, W).to(BF).to(DEV), do.reshape(B * T, -1).to(BF).to(DEV), B, T, H, KVH)
    x2, do2 = x.clone(), do.clone()
    x2[:, t + 1:] = _rand((B, T - t - 1, W), 7, 3.0)
    do2[:, t + 1:] = _rand((B, T - t - 1, H * 64), 8)
    o, lse, dqkv = _fwd_bwd(x2.reshape(B * T, W).to(BF).to(DEV), do2.reshape(B * T, -1).to(BF).to(DEV), B, T, H, KVH)
    rows = (torch.arange(B)[:, None] * T + torch.arange(t + 1)[None]).reshape(-1)
    assert torch.equal(o[rows], base[0][rows]), "O of earlier rows changed"
    assert torch.equal(lse[:, :, :t + 1], base[1][:, :, :t + 1]), "lse of earlier rows changed"
    assert torch.equal(dqkv[rows, :H * 64], base[2][rows, :H * 64]), "dQ of earlier rows changed"


def test_isolation_of_batch_rows():
    """A batch row's O, lse and dqkv do not depend on the other rows: B = 3 with changed neighbours, and B = 1."""
    B, T, H, KVH = 3, 333, 14, 2
    W = (H + 2 * KVH) * 64
    x, do = _rand((B, T, W), 9, 2.0), _rand((B, T, H * 64), 10)
    flat = lambda t: t.reshape(-1, t.shape[-1]).to(BF).to(DEV)
    base = _fwd_bwd(flat(x), flat(do), B, T, H, KVH)
    x2, do2 = x.clone(), do.clone()
    x2[[0, 2]] = _rand((2, T, W), 11, 3.0)
    do2[[0, 2]] = _rand((2, T, H * 64), 12)
    other = _fwd_bwd(flat(x2), flat(do2), B, T, H, KVH)
    alone = _fwd_bwd(flat(x[1:2]), flat(do[1:2]), 1, T, H, KVH)
    r = slice(T, 2 * T)
    for name, o, lse, g in (("neighbours changed", other[0][r], other[1][1], other[2][r]),
                            ("B = 1", alone[0], alone[1][0], alone[2])):
        assert torch.equal(o, base[0][r]), f"O of batch row 1 changed ({name})"
        assert torch.equal(lse, base[1][1]), f"lse of batch row 1 changed ({name})"
        assert torch.equal(g, base[2][r]), f"dqkv of batch row 1 changed ({name})"


# --------------------------------------------------------------------------------------------------- random mode
RANDOM_CASES = {
    # name: (inputs, B, T, H, KVH, scale, docs)
    "rising": ("rising", 2, 700, 4, 2, 0.125, None),
    "wide40": ("wide", 2, 513, 14, 2, 0.125, None),
    "midtile-docs": ("wide", 2, 400, 4, 2, 0.125, [[37, 100, 29, 234], [129, 5, 266]]),
    "scale0.1": ("wide", 2, 300, 12, 12, 0.1, None),
}


@pytest.mark.parametrize("name", list(RANDOM_CASES))
def test_random_per_element(name):
    """fp64 reference with the contract bounds of attn_ref (forward; backward from the kernel's own o and lse)."""
    kind, B, T, H, KVH, scale, docs = RANDOM_CASES[name]
    q, k, v = (A.rising_inputs if kind == "rising" else A.wide_inputs)(B, T, H, KVH, seed=21)
    seg = A.doc_starts(B, T, docs) if docs else None
    lo, hi = A.bounds(B, T, True, seg)
    ss, se = _seg_dev(seg) if seg is not None else (None, None)
    qkv = A.fuse(q, k, v, device=DEV)
    do = _rand((B, T, H, 64), 22)
    o, lse = run_fwd("tc", qkv, B, T, H, KVH, True, scale, seg=ss)
    dqkv = run_bwd("tc", qkv, o, do.reshape(B * T, -1).to(BF).to(DEV), lse, B, T, H, KVH, True, scale, ss, se)
    O, L, bo, bl = A.fwd_reference(q, k, v, lo, hi, scale, True)
    oc, lc = A.heads(o, B, T, H), A.lse_bth(lse)
    _check(A.mismatch_bound(oc, O, bo, f"O {name}"))
    _check(A.mismatch_bound(lc, L, bl, f"lse {name}"))
    rq, rk, rv, bq, bk, bv = A.bwd_reference(q, k, v, oc, do, lc, lo, hi, scale, True)
    gq, gk, gv = A.unfuse(dqkv, B, T, H, KVH)
    _check(A.mismatch_bound(gq, rq, bq, f"dQ {name}"))
    _check(A.mismatch_bound(gk, rk, bk, f"dK {name}", rows="key"))
    _check(A.mismatch_bound(gv, rv, bv, f"dV {name}", rows="key"))


def test_random_bidirectional_per_element():
    B, T, H, KVH, scale = 2, 300, 4, 2, 0.125
    q, k, v = A.wide_inputs(B, T, H, KVH, seed=23)
    lo, hi = A.bounds(B, T, False)
    qkv = A.fuse(q, k, v, device=DEV)
    do = _rand((B, T, H, 64), 24)
    o, lse = run_fwd("plain", qkv, B, T, H, KVH, False, scale)
    dqkv = run_bwd("plain", qkv, o, do.reshape(B * T, -1).to(BF).to(DEV), lse, B, T, H, KVH, False, scale)
    O, L, bo, bl = A.fwd_reference(q, k, v, lo, hi, scale, False)
    oc, lc = A.heads(o, B, T, H), A.lse_bth(lse)
    _check(A.mismatch_bound(oc, O, bo, "O bidirectional"))
    _check(A.mismatch_bound(lc, L, bl, "lse bidirectional"))
    rq, rk, rv, bq, bk, bv = A.bwd_reference(q, k, v, oc, do, lc, lo, hi, scale, False)
    gq, gk, gv = A.unfuse(dqkv, B, T, H, KVH)
    _check(A.mismatch_bound(gq, rq, bq, "dQ bidirectional"))
    _check(A.mismatch_bound(gk, rk, bk, "dK bidirectional", rows="key"))
    _check(A.mismatch_bound(gv, rv, bv, "dV bidirectional", rows="key"))


# --------------------------------------------------------------------------------------------------- split (HuBERT)
def _split_run(parts, B, T, H):
    from slamkit_b200 import ops
    qh, ql, kh, kl, vh, vl = parts
    hi = torch.cat([qh, kh, vh], 2).reshape(B * T, 3 * H * 64).to(BF).to(DEV)
    lo = torch.cat([ql, kl, vl], 2).reshape(B * T, 3 * H * 64).to(BF).to(DEV)
    o_hi, o_lo = ops.attn_tc_fwd_split(hi, lo, B, T, H, 0.125)
    return A.heads(o_hi, B, T, H), A.heads(o_lo, B, T, H)


@pytest.mark.parametrize("T", [1, 2, 63, 64, 65, 129, 200, 1024])
def test_split_exact(T):
    B, H = 2, 12
    parts, (want_hi, want_lo) = A.split_onehot(B, T, H, A.modes_for(H), seed=T)
    got_hi, got_lo = _split_run(parts, B, T, H)
    _check(A.mismatch_exact(got_hi, want_hi, f"split one-hot hi T={T}"))
    _check(A.mismatch_exact(got_lo, want_lo, f"split one-hot lo T={T}"))
    parts, (want_hi, want_lo) = A.split_uniform(B, T, H, seed=T)
    got_hi, got_lo = _split_run(parts, B, T, H)
    _check(A.mismatch_exact(got_hi, want_hi, f"split uniform hi T={T}"))
    _check(A.mismatch_exact(got_lo, want_lo, f"split uniform lo T={T}"))


def test_split_random_per_element():
    B, T, H = 2, 300, 4
    g = torch.Generator().manual_seed(31)
    parts = []
    for _ in range(3):
        x = torch.randn(B, T, H, 64, generator=g) * 2.0
        xh = A.bf16(x)
        parts += [xh, A.bf16(x - xh)]
    got_hi, got_lo = _split_run(parts, B, T, H)
    q, k, v = parts[0] + parts[1], parts[2] + parts[3], parts[4] + parts[5]
    lo, hi = A.bounds(B, T, False)
    O, _, bo, _ = A.fwd_reference(q, k, v, lo, hi, 0.125, False, split=True)
    _check(A.mismatch_bound(got_hi.double() + got_lo.double(), O, bo, "split random hi + lo"))


# --------------------------------------------------------------------------------------------------- decode
DECODE_HEADS = HEADS + [(16, 1)]


@pytest.mark.parametrize("H,KVH", DECODE_HEADS, ids=[f"H{h}KV{k}" for h, k in DECODE_HEADS])
def test_decode_exact(H, KVH):
    """lens in {1, 63, 64, 65, 128, 129, T_cache, 0}; keys at and past lens are NaN (never read); lens = 0 gives 0."""
    Tc = 1024
    lens = torch.tensor([1, 63, 64, 65, 128, 129, Tc, 0])
    B = len(lens)
    q, k, v, want = A.decode_onehot(B, H, KVH, Tc, lens, A.modes_for(H), seed=H)
    vu = A.int_values((B, KVH, Tc, 64), 64, H + 1)
    for b in range(B):
        k[b, :, int(lens[b]):] = float("nan")
        v[b, :, int(lens[b]):] = float("nan")
        vu[b, :, int(lens[b]):] = float("nan")
    lens_d = lens.to(torch.int32).to(DEV)
    qkv = torch.full((B, (H + 2 * KVH) * 64), float("nan"), dtype=BF)         # q as a column slice of a projection
    qkv[:, :H * 64] = q.reshape(B, -1).to(BF)
    kd, vd = k.to(BF).to(DEV), v.to(BF).to(DEV)
    o = run_decode(qkv.to(DEV), kd, vd, lens_d, H, KVH)
    got = o.cpu().float().view(B, 1, H, 64)
    _check(A.mismatch_exact(got, want.view(B, 1, H, 64), f"decode one-hot H={H} KVH={KVH}", rows="batch-row"))
    assert torch.equal(run_decode(qkv.to(DEV), kd, vd, lens_d, H, KVH), o), "decode is not bit-identical run to run"
    qz = torch.zeros_like(qkv)
    o = run_decode(qz.to(DEV), kd, vu.to(BF).to(DEV), lens_d, H, KVH)
    want_u = A.expect_decode_uniform(vu, lens, H)
    _check(A.mismatch_exact(o.cpu().float().view(B, 1, H, 64), want_u.view(B, 1, H, 64), f"decode uniform H={H} KVH={KVH}",
                            rows="batch-row"))


@pytest.mark.parametrize("H,KVH", [(14, 2), (16, 1)], ids=["H14KV2", "H16KV1"])
def test_decode_equals_prefill_row(H, KVH):
    """Exact modes: row t of the causal forward equals decode over the same keys with lens = t + 1, bit for bit."""
    T = 300
    q, k, v, tg, lo, hi = _onehot(1, T, H, KVH)
    o, _ = run_fwd("tc", A.fuse(q, k, v, device=DEV), 1, T, H, KVH, True)
    rows = [0, 62, 63, 64, 127, 128, 129, 299]
    B = len(rows)
    qd = q[0, rows].reshape(B, H * 64).to(BF).to(DEV)
    kc = k[0].permute(1, 0, 2)[None].expand(B, -1, -1, -1).contiguous().to(BF).to(DEV)
    vc = v[0].permute(1, 0, 2)[None].expand(B, -1, -1, -1).contiguous().to(BF).to(DEV)
    lens = torch.tensor([t + 1 for t in rows], dtype=torch.int32, device=DEV)
    od = run_decode(qd, kc, vc, lens, H, KVH)
    assert torch.equal(od.cpu(), o.cpu()[rows]), "decode differs from the prefill row"
    vu = A.int_values((1, T, KVH, 64), 64, 3)
    o, _ = run_fwd("tc", A.fuse(torch.zeros_like(q), k, vu, device=DEV), 1, T, H, KVH, True)
    vcu = vu[0].permute(1, 0, 2)[None].expand(B, -1, -1, -1).contiguous().to(BF).to(DEV)
    od = run_decode(torch.zeros_like(qd), kc, vcu, lens, H, KVH)
    assert torch.equal(od.cpu(), o.cpu()[rows]), "uniform decode differs from the prefill row"


# --------------------------------------------------------------------------------------------------- guard bands
def _sentinel_bf16(rows, cols):
    return torch.full((rows, cols), SENT16, dtype=torch.int16, device=DEV).view(BF)


@pytest.mark.parametrize("entry", ["tc", "plain"])
def test_guard_bands(entry):
    """Inputs at pitch ld > (H + 2 KVH) 64 with NaN padding; O, lse and dqkv inside larger sentinel-filled buffers
    (ldo > H 64, ldg > width, column and element offsets): exact results, every sentinel intact."""
    B, T, H, KVH = 2, 200, 14, 2
    W = (H + 2 * KVH) * 64
    q, k, v, tg, lo, hi = _onehot(B, T, H, KVH)
    qkv = A.fuse(q, k, v, ld=W + 72, device=DEV)
    obuf = _sentinel_bf16(B * T + 3, H * 64 + 40)
    o = obuf[1:1 + B * T, 8:8 + H * 64]
    lbuf = torch.full((B * H * T + 64,), SENT32, dtype=torch.int32, device=DEV)
    lse = lbuf[32:32 + B * H * T].view(torch.float32).view(B, H, T)
    ob, lb = obuf.clone(), lbuf.clone()
    run_fwd(entry, qkv, B, T, H, KVH, True, o=o, lse=lse)
    _check(A.mismatch_exact(A.heads(o, B, T, H), A.expect_onehot_fwd(v, tg, H // KVH)[0], f"pitched O {entry}"))
    _check(A.mismatch_exact(A.lse_bth(lse), torch.zeros(B, T, H), f"pitched lse {entry}"))
    inside = torch.zeros_like(obuf, dtype=torch.bool)
    inside[1:1 + B * T, 8:8 + H * 64] = True
    assert torch.equal(obuf.view(torch.int16)[~inside], ob.view(torch.int16)[~inside]), "O written outside its block"
    assert torch.equal(lbuf[:32], lb[:32]) and torch.equal(lbuf[32 + B * H * T:], lb[32 + B * H * T:]), "lse written outside"
    # backward: dO shares O's pitch; dqkv inside a sentinel buffer
    vb, do = A.onehot_bwd_inputs(tg, KVH, T, seed=5)
    qkv = A.fuse(q, k, vb, ld=W + 72, device=DEV)
    dobuf = torch.full((B * T, H * 64 + 40), float("nan"), dtype=BF, device=DEV)
    dod = dobuf[:, 8:8 + H * 64]
    dod.copy_(do.reshape(B * T, -1).to(BF))
    zo = torch.zeros_like(dobuf)[:, 8:8 + H * 64]
    gbuf = _sentinel_bf16(B * T + 2, W + 40)
    dqkv = gbuf[1:1 + B * T, 8:8 + W]
    gb = gbuf.clone()
    run_bwd(entry, qkv, zo, dod, torch.zeros(B, H, T, device=DEV), B, T, H, KVH, True, dqkv=dqkv)
    dq, dk, dv = A.expect_onehot_bwd(q, k, vb, do, tg, H // KVH)
    gq, gk, gv = A.unfuse(dqkv, B, T, H, KVH)
    _check(A.mismatch_exact(gq, dq, f"pitched dQ {entry}"))
    _check(A.mismatch_exact(gk, dk, f"pitched dK {entry}", rows="key"))
    _check(A.mismatch_exact(gv, dv, f"pitched dV {entry}", rows="key"))
    inside = torch.zeros_like(gbuf, dtype=torch.bool)
    inside[1:1 + B * T, 8:8 + W] = True
    assert torch.equal(gbuf.view(torch.int16)[~inside], gb.view(torch.int16)[~inside]), "dqkv written outside its block"


# --------------------------------------------------------------------------------------------------- chains
def test_chain_and_determinism():
    """fwd -> bwd -> fwd on the backward's output, back to back on one stream, equals the run with a synchronisation
    after every launch; two backward runs are bit-identical."""
    B, T, H, KVH = 2, 333, 14, 2
    W = (H + 2 * KVH) * 64
    x = _rand((B * T, W), 41, 2.0).to(BF).to(DEV)
    do = _rand((B * T, H * 64), 42).to(BF).to(DEV)

    def chain(sync):
        s = torch.cuda.synchronize if sync else (lambda: None)
        o, lse = run_fwd("tc", x, B, T, H, KVH)
        s()
        g = run_bwd("tc", x, o, do, lse, B, T, H, KVH)
        s()
        g2 = run_bwd("tc", x, o, do, lse, B, T, H, KVH)
        s()
        o2, lse2 = run_fwd("tc", g * 64, B, T, H, KVH)                # reads the backward's output
        s()
        return [t.cpu() for t in (o, lse, g, g2, o2, lse2)]

    torch.cuda.synchronize()
    fast = chain(False)
    slow = chain(True)
    for name, a, b in zip(("o", "lse", "dqkv", "dqkv again", "o of dqkv", "lse of dqkv"), fast, slow):
        assert torch.equal(a, b), f"{name}: back-to-back launches differ from the synchronised run"
    assert torch.equal(fast[2], fast[3]), "two backward runs differ"


# --------------------------------------------------------------------------------------------------- argument checks
def argument_child():
    """Runs in a child process: every bad call returns an error with a message and launches nothing."""
    L, lib = _lib()
    B, T, H, KVH = 2, 64, 4, 2
    W = (H + 2 * KVH) * 64
    qkv = torch.zeros(B * T + 8, W + 64, dtype=BF, device=DEV)
    o = torch.zeros(B * T + 8, H * 64 + 64, dtype=BF, device=DEV)
    lse = torch.zeros(B * H * T + 64, dtype=torch.float32, device=DEV)
    delta = torch.zeros_like(lse)
    g = torch.zeros_like(qkv)
    seg = torch.zeros(B * T, dtype=torch.int32, device=DEV)
    base = dict(B=B, T=T, H=H, KVH=KVH, ld=W, ldo=H * 64, ldg=W, seg=None, seg_end=None)

    def fwd(a):
        return lib.sk_attn_fwd(_p(qkv), _p(qkv, a["H"] * 64), _p(qkv, (a["H"] + a["KVH"]) * 64), _p(o), _p(lse), a["B"],
                               a["T"], a["H"], a["KVH"], a["ld"], a["ldo"], 1, L.f32(0.125), L.stream_ptr())

    def tc_fwd(a):
        return lib.sk_attn_tc_fwd(_p(qkv), _p(o), _p(lse), a["B"], a["T"], a["H"], a["KVH"], a["ld"], a["ldo"], 1,
                                  L.f32(0.125), _p(a["seg"]), L.stream_ptr())

    def bwd(a):
        return lib.sk_attn_bwd(_p(qkv), _p(qkv, a["H"] * 64), _p(qkv, (a["H"] + a["KVH"]) * 64), _p(o), _p(o), _p(lse),
                               _p(delta), _p(g), _p(g, a["H"] * 64), _p(g, (a["H"] + a["KVH"]) * 64), a["B"], a["T"], a["H"],
                               a["KVH"], a["ld"], a["ldo"], a["ldg"], 1, L.f32(0.125), L.stream_ptr())

    def tc_bwd(a):
        return lib.sk_attn_tc_bwd(_p(qkv), _p(o), _p(o), _p(lse), _p(delta), None, _p(g), a["B"], a["T"], a["H"], a["KVH"],
                                  a["ld"], a["ldo"], a["ldg"], 1, L.f32(0.125), _p(a["seg"]), _p(a["seg_end"]),
                                  L.stream_ptr())

    def split(a):
        return lib.sk_attn_tc_fwd_split(_p(qkv), _p(qkv), _p(o), _p(o), a["B"], a["T"], a["H"], a["ld"], a["ldo"],
                                        L.f32(0.125), L.stream_ptr())

    def decode(a):
        kc = torch.zeros(1, 2, 64, 64, dtype=BF, device=DEV)
        part = torch.zeros(4096, dtype=torch.float32, device=DEV)
        lens = torch.ones(1, dtype=torch.int32, device=DEV)
        return lib.sk_attn_decode(_p(qkv), W, _p(kc), _p(kc), _p(lens), _p(o), H * 64, _p(part), 1, a["H"], 2, 64,
                                  L.f32(0.125), L.stream_ptr())

    entries = {"fwd": fwd, "tc_fwd": tc_fwd, "bwd": bwd, "tc_bwd": tc_bwd}
    bad = {"KVH=0": dict(KVH=0), "H%KVH": dict(H=3), "B=0": dict(B=0), "T=0": dict(T=0), "H=0": dict(H=0),
           "B<0": dict(B=-1), "T<0": dict(T=-5), "ld%8": dict(ld=W + 4), "ldo%8": dict(ldo=H * 64 + 2)}
    cases = [(e, n, m) for e in entries for n, m in bad.items()]
    cases += [("bwd", "ldg odd", dict(ldg=W + 1)), ("tc_bwd", "ldg odd", dict(ldg=W + 1)),
              ("tc_bwd", "seg_end without seg_start", dict(seg_end=seg)),
              ("tc_bwd", "seg_start without seg_end", dict(seg=seg))]
    entries.update(split=split, decode=decode)
    cases += [("split", "B=0", dict(B=0)), ("split", "T=0", dict(T=0)), ("split", "H=0", dict(H=0)),
              ("split", "ld%8", dict(ld=W + 4)), ("decode", "G=17", dict(H=34))]
    for e in ("fwd", "tc_fwd", "bwd", "tc_bwd"):
        assert entries[e](base) == 0, f"{e}: the valid call failed: {lib.sk_last_error().decode()}"
    torch.cuda.synchronize()
    n0 = lib.sk_launch_count()
    failed = []
    for e, n, m in cases:
        rc = entries[e](dict(base, **m))
        msg = lib.sk_last_error().decode()
        if rc == 0 or not msg:
            failed.append(f"{e} {n}: rc={rc} {msg!r}")
        print(f"{e:7s} {n:28s} rc={rc} {msg}")
    assert lib.sk_launch_count() == n0, "a refused call launched a kernel"
    torch.cuda.synchronize()
    assert not failed, failed
    print(f"{len(cases)} bad calls refused")


def test_rejects_bad_arguments():
    """KVH = 0, H % KVH != 0, B / T / H <= 0, misaligned ld / ldo / ldg, seg_end without seg_start and decode groups over
    16 are refused on the host.  In a child process, so that a host crash reports instead of ending the session."""
    code = (f"import sys; sys.path[:0] = [{ROOT!r}, {HERE!r}]; import test_gpu_attention_conformance as t; "
            f"t.argument_child()")
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, capture_output=True, text=True, timeout=600)
    print(r.stdout)
    assert r.returncode == 0, f"child exit {r.returncode}\n" + r.stdout[-4000:] + r.stderr[-4000:]
