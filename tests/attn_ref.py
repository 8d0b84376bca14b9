"""Reference, input generators and checker for the attention kernels (attention.cu, decode.cu), compared per element.

Layout used throughout: q [B, T, H, 64], k / v [B, T, KVH, 64] (float tensors holding bf16 values), q head h reads kv
head h // G with G = H / KVH.  Which keys a query row may see is an interval [lo, hi] per (batch, row):
causal [document start, t], bidirectional [0, T - 1], decode [0, lens - 1].

Exact modes (head_dim 64, scale = 1/8).  The inputs are built so that a correct flash-style kernel's bf16 output is
known bit for bit.  They rely on the kernels evaluating p = exp2f(s * sl2 - m * sl2) (one FMA) on fp32 scores and
1.0f / l being IEEE division, and on the target's score being exactly 0, which leaves no FMA residue.

- One-hot ("latest" / "earliest" per head).  k_j carries the base-16 digits of j in columns 0..3 and 1 in columns
  4..7; q_t carries sg * 2^(10+4d) in column d and -sg * 2^(10+4d) * digit_d(target(t)) in column 4 + d, with sg = +1
  ("latest": target = hi) or -1 ("earliest": target = lo).  All are bf16 values, and s(t, j) = sg * 2^10 * (j -
  target(t)) exactly in fp32 for T <= 8192 in any summation order (every partial sum is a multiple of 2^10 below
  2^27).  The target scores 0, so p = exp2f(0) = 1, l = 1 and lse = 0; every other allowed key is at least
  2^10 * 2^-3 * log2(e) = 184.7 below it in the exponent, so its p and every earlier tile's rescaling factor underflow
  to exactly 0: O = v[target] bit for bit.  A leaked key past the target (latest) or before it (earliest) scores
  higher and wins; V holds small integers that differ per kv head, so a wrong head, row, column or tile shows.
- Uniform (q = 0).  Every allowed score is 0, p = 1, l = n (the size of the allowed interval) and
  O = bf16(fl(sum v) * fl(1 / n)) with the sum exact (integers); lse = logf(n) within two fp32 ulps.  A mask that is
  off by one key changes n, hence lse, by 1/n (thousands of ulps at n = 8192).
- Backward one-hot.  o = 0 gives delta = 0; lse = 0; V and dO in {-1, 0, 1} with one non-zero dO column per row.  Then
  P = 1 on the target and 0 elsewhere, dS = dP / 8 on the target only, and dV, dQ, dK are small multiples of powers
  of two.  dO is non-zero on at most one row per (head, target), so at most G terms meet in a dK / dV row and every
  expected value is a bf16 value (asserted).  With the true o (= v[target]) delta = dP and dQ = dK = 0 exactly.
- Split bf16 (HuBERT).  The same scores, carried as (hi, lo) pairs that exercise every partial product the kernel
  forms (Qh Kh + Qh Kl + Ql Kh; Ql Kl is zero by construction); V = Vh + Vl with Vl a multiple of 2^-6, so
  O = Vh + Vl exactly and the output pair is hi = bf16(O), lo = bf16(O - hi).
- Decode.  q is pre-multiplied by scale * log2(e) per element, so scores are not exact; the row max is the target's
  own computed score, so p(target) = exp2f(0) = 1, and the margin still zeroes every other key and split.
  decode_scores emulates the kernel's fp32 FMA chain to assert that margin.
- Decode over an fp32 cache (sk_attn_decode_split).  The query arrives as a bf16 pair, q = fl(q_hi + q_lo) (the one-hot
  query split as in split_onehot; the target stays the maximum whatever q_lo is, so only random mode sees a dropped
  q_lo); K holds the one-hot digits plus fp32 values that are not bf16 values in columns where q is 0; V = Vh + Vl
  with Vl on the 2^-6 grid, so O = V[target] exactly and the output pair is o_hi = bf16(O), o_lo = bf16(O - o_hi).
  Uniform (q = 0): O = fl(sum V) * fl(1 / n), the sum exact (|sum| < 2^15 on the 2^-6 grid).

Random mode (any finite data, any scale): fp64 reference and a per-element bound that any valid flash implementation
meets, whatever its key-tile order: P (and dS) may be rounded to bf16 once, relative to any running max; scores and
sums are fp32.  With pi the fp64 softmax row, n the allowed keys, Sd = scale * sum_d |q_d k_d| and the per-row
exponent error
    D = 64 * 2^-23 * max_j Sd_j + 2^-20 * (max_j |s_j| + 1)          (fp32 scores in any order, sl2 / m*sl2 rounding,
                                                                       FMA residue, exp2f ulps)
  forward   |O - O*| <= (e^(2D) - 1) sum_j pi_j |v_j - O*|            (weights perturbed by e^(+-D), renormalised;
                                                                       sum pi |v - O*| <= sum pi (|v| + |O*|) is used)
                        + 2^-9 sum_j pi_j (|v_j| + |O*|)               (bf16 P in the numerator, fp32 l)
                        + (3n + 8) 2^-23 sum_j pi_j (|v_j| + |O*|)     (fp32 sums, per-tile rescaling, 1 / l)
                        + half a bf16 ulp of the output;
            |lse - lse*| <= D + (3n + 8) 2^-23 + 2^-21 (|lse*| + 1).
  backward  (the reference takes the kernel's own o and lse: P = exp(s - lse), delta = rowsum(dO * o) in fp64)
            eP = 2^-8 + e^(D + 2^-21 |lse|) - 1 bounds the relative error of P (one bf16 rounding, exponent error);
            dS = P (dP - delta) scale with |dS~ - dS| <= E = P scale (|dP - delta| (eP + 2^-9) + (e_dP + e_delta)(1 + eP)),
            e_dP = 64 2^-23 sum |dO||v|, e_delta = 64 2^-23 sum |dO||o| (fp32 dot products);
            |dV - dV*| <= sum P |dO| (eP + N 2^-23),  |dK - dK*| <= sum (E + N 2^-23 (|dS| + E)) |q|,
            |dQ - dQ*| <= sum (E + N 2^-23 (|dS| + E)) |k|, each plus half a bf16 ulp, N = terms in the sum.
  split     the same with 2^-16 in place of 2^-9 (P and V carried as pairs, Pl Vl dropped) and the dropped Ql Kl term
            added to the score error (2^-16 * Sd); the output is hi + lo, within 2^-17 |O*| of its pair rounding.
  decode, fp32 cache (q = q_hi + q_lo exact in fp32, P and V fp32): the bf16-P term drops out,
            |O - O*| <= (e^(2D) - 1 + (3n + 8) 2^-23) sum_j pi_j (|v_j| + |O*|) + 2^-17 |O*|
            for the output o_hi + o_lo (2^-17 |O*|: the pair rounding of the fp32 result).

Checker: every comparison reports the number of mismatches and the first few as (batch, head, row, column, 64-row
tile, 16-row warp slice), for dK / dV with the key tile as the row tile.  Works on CPU and GPU tensors alike.
"""
from __future__ import annotations

import math
from typing import List, Optional, Sequence

import torch

HD = 64
LOG2E = 1.4426950408889634
EXACT_SCALE = 0.125
MARGIN = 2.0 ** 10 * EXACT_SCALE * LOG2E      # exponent gap of the nearest non-target key in the one-hot modes
UNDERFLOW = 150.0                              # exp2f(x) == 0 for x < -150


# ----------------------------------------------------------------------------------------------------- rounding
def bf16(x: torch.Tensor) -> torch.Tensor:
    """-> float32 holding the bf16 round-to-nearest-even of x"""
    return x.float().to(torch.bfloat16).float()


def f32(x: torch.Tensor) -> torch.Tensor:
    return x.to(torch.float32)


def ulp_bf16(x: torch.Tensor) -> torch.Tensor:
    x = x.double().abs()
    _, e = torch.frexp(x)
    return torch.where(x < 2.0 ** -126, torch.full_like(x, 2.0 ** -133), torch.ldexp(torch.ones_like(x), e - 8))


def ulp_f32(x: torch.Tensor) -> torch.Tensor:
    x = x.double().abs()
    _, e = torch.frexp(x)
    return torch.where(x < 2.0 ** -126, torch.full_like(x, 2.0 ** -149), torch.ldexp(torch.ones_like(x), e - 24))


def fma32(a: torch.Tensor, b: torch.Tensor, c: torch.Tensor) -> torch.Tensor:
    """fp32 fused multiply-add: a * b + c formed in float64 (exact for the operands used here), rounded once."""
    return torch.addcmul(c.double(), a.double(), b.double()).float()


def is_bf16(x: torch.Tensor) -> bool:
    return bool(torch.equal(bf16(x), x.float()))


# ----------------------------------------------------------------------------------------------------- masks
def doc_starts(B: int, T: int, docs: Optional[Sequence[Sequence[int]]] = None) -> torch.Tensor:
    """int64 [B, T]: in-row index of the first token of each token's document (docs[b] = document lengths of row b,
    summing to T; None = one document per row)."""
    seg = torch.zeros(B, T, dtype=torch.int64)
    if docs is None:
        return seg
    for b, lens in enumerate(docs):
        assert sum(lens) == T and all(n > 0 for n in lens), (b, lens)
        t = 0
        for n in lens:
            seg[b, t:t + n] = t
            t += n
    return seg


def bounds(B: int, T: int, causal: bool, seg: Optional[torch.Tensor] = None):
    """(lo, hi) int64 [B, T]: query row t of batch row b may see keys lo <= j <= hi."""
    t = torch.arange(T).expand(B, T)
    if causal:
        lo = seg.clone() if seg is not None else torch.zeros(B, T, dtype=torch.int64)
        return lo, t.clone()
    assert seg is None
    return torch.zeros(B, T, dtype=torch.int64), torch.full((B, T), T - 1, dtype=torch.int64)


def modes_for(H: int) -> List[str]:
    """Alternate the one-hot modes over the heads, so that a wrong q head or kv head changes the output."""
    return ["latest" if h % 2 == 0 else "earliest" for h in range(H)]


def int_values(shape, amax: int, seed: int) -> torch.Tensor:
    g = torch.Generator().manual_seed(seed)
    return torch.randint(-amax, amax + 1, shape, generator=g).float()


# ----------------------------------------------------------------------------------------------------- one-hot mode
def _digits(x: torch.Tensor) -> torch.Tensor:
    """[..., 4] base-16 digits of int tensor x (x < 16^4)"""
    return torch.stack([(x >> (4 * d)) & 15 for d in range(4)], -1).float()


def onehot_k(B: int, T: int, KVH: int) -> torch.Tensor:
    assert T <= 8192
    k = torch.zeros(B, T, KVH, HD)
    k[..., :4] = _digits(torch.arange(T))[None, :, None, :]
    k[..., 4:8] = 1.0
    return k


def onehot_q(target: torch.Tensor, modes: Sequence[str]) -> torch.Tensor:
    """target int64 [..., H] -> q [..., H, 64] with s(j) = sg * 2^10 * (j - target) against onehot_k."""
    sg = torch.tensor([1.0 if m == "latest" else -1.0 for m in modes])
    p = torch.tensor([2.0 ** (10 + 4 * d) for d in range(4)])
    q = torch.zeros(*target.shape, HD)
    q[..., :4] = sg[:, None] * p
    q[..., 4:8] = -sg[:, None] * p * _digits(target)
    return q


def onehot_targets(lo: torch.Tensor, hi: torch.Tensor, modes: Sequence[str]) -> torch.Tensor:
    """int64 [B, T, H]: hi for "latest" heads, lo for "earliest" ones"""
    return torch.stack([hi if m == "latest" else lo for m in modes], -1)


def onehot_scores(q: torch.Tensor, k: torch.Tensor, G: int) -> torch.Tensor:
    """fp32 scores of the one-hot inputs [B, H, T, T], asserting they are exact (fp64 == fp32 of every partial sum
    bound) -- small shapes only."""
    kk = k.repeat_interleave(G, dim=2)
    s64 = torch.einsum("bthd,bjhd->bhtj", q.double(), kk.double())
    bound = torch.einsum("bthd,bjhd->bhtj", q.double().abs(), kk.double().abs())
    assert float(bound.max()) < 2.0 ** 27 and bool((torch.remainder(s64, 2.0 ** 10) == 0).all())
    return s64.float()


def check_onehot_claims(q, k, target, lo, hi, G, scale=EXACT_SCALE, rows=None) -> None:
    """The generator's arithmetic claims, in fp32 with the FMA emulated: target exponent exactly 0, every other allowed
    key below -UNDERFLOW, operands bf16 values.  rows: optional subset of query rows (long rows)."""
    assert is_bf16(q) and is_bf16(k)
    if rows is not None:
        q, target, lo, hi = q[:, rows], target[:, rows], lo[:, rows], hi[:, rows]
    s = onehot_scores(q, k, G)                                           # [B, H, T, T]
    sl2 = torch.tensor(scale * LOG2E, dtype=torch.float32)
    e = fma32(s, sl2, torch.zeros(()))                                   # m = 0: exponent of every key
    j = torch.arange(s.shape[-1])
    tgt = target.permute(0, 2, 1)[..., None]                             # [B, H, T, 1]
    allowed = (j >= lo[:, None, :, None]) & (j <= hi[:, None, :, None])
    is_t = j == tgt
    assert bool((e[is_t & allowed] == 0).all()), "the target's exponent is not exactly 0"
    assert bool((is_t & allowed).sum(-1).eq(1).all()), "every row has exactly one allowed target"
    others = e[allowed & ~is_t]
    assert others.numel() == 0 or float(others.max()) <= -MARGIN + 1e-3 < -UNDERFLOW
    assert float(torch.exp2(others).max() if others.numel() else 0.0) == 0.0


def expect_onehot_fwd(v: torch.Tensor, target: torch.Tensor, G: int):
    """(O [B, T, H, 64], lse [B, T, H]) of the one-hot mode: O = v[target] of the head's kv head, lse = 0."""
    B, T, H = target.shape
    kv = torch.arange(H) // G
    o = v[torch.arange(B)[:, None, None], target, kv[None, None, :]]
    return o.clone(), torch.zeros(B, T, H)


# ----------------------------------------------------------------------------------------------------- uniform mode
def expect_uniform_fwd(v: torch.Tensor, lo: torch.Tensor, hi: torch.Tensor, G: int):
    """(O, lse) with q = 0: O = bf16(fl(sum_{lo..hi} v) * fl(1 / n)), lse = log(n) (fp64, compare within 2 ulps)."""
    assert bool((v == v.round()).all()) and float(v.abs().sum(1).max()) < 2 ** 24
    B, T, KVH, _ = v.shape
    c = torch.zeros(B, T + 1, KVH, HD, dtype=torch.float64)
    c[:, 1:] = v.double().cumsum(1)
    bi = torch.arange(B)[:, None]
    ssum = (c[bi, hi + 1] - c[bi, lo]).float()                          # [B, T, KVH, 64], exact integers
    n = (hi - lo + 1).float()
    inv = torch.ones(()) / n                                             # IEEE fp32 division
    o = bf16(ssum * inv[..., None, None]).repeat_interleave(G, dim=2)
    lse = torch.log(n.double())[..., None].expand(B, T, KVH * G).clone()
    return o, lse


# ----------------------------------------------------------------------------------------------------- backward one-hot
def onehot_bwd_inputs(target: torch.Tensor, KVH: int, T: int, seed: int):
    """v [B, T, KVH, 64] and dO [B, T, H, 64] in {-1, 0, 1}: one non-zero dO column per row, and for each (head, target)
    at most one row with a non-zero dO."""
    B, _, H = target.shape
    g = torch.Generator().manual_seed(seed)
    v = torch.randint(-1, 2, (B, T, KVH, HD), generator=g).float()
    col = torch.randint(0, HD, (B, T, H), generator=g)
    sign = torch.randint(0, 2, (B, T, H), generator=g).float() * 2 - 1
    keep = torch.zeros(B, T, H, dtype=torch.bool)
    order = torch.randperm(T, generator=g)
    for b in range(B):
        for h in range(H):
            tg = target[b, order, h]
            _, inv = torch.unique(tg, return_inverse=True)
            seen = torch.full((int(inv.max()) + 1,), T, dtype=torch.int64)
            seen.scatter_reduce_(0, inv, torch.arange(T), reduce="amin")
            first = seen[inv] == torch.arange(T)
            keep[b, order, h] = first
    do = torch.zeros(B, T, H, HD)
    do.scatter_(-1, col[..., None], (sign * keep.float())[..., None])
    return v, do


def expect_onehot_bwd(q, k, v, do, target, G, true_o: bool = False, scale=EXACT_SCALE):
    """(dq [B,T,H,64], dk [B,T,KVH,64], dv [B,T,KVH,64]) of the one-hot mode with o = 0 (or the true o: dq = dk = 0)."""
    B, T, H, _ = q.shape
    KVH = H // G
    bi = torch.arange(B)[:, None, None]
    kv = (torch.arange(H) // G)[None, None, :]
    vt = v[bi, target, kv]                                               # [B, T, H, 64]
    dp = (do.double() * vt.double()).sum(-1)                             # [B, T, H]
    ds = dp * scale if not true_o else torch.zeros_like(dp)
    dq = ds[..., None] * k.double()[bi, target, kv]
    dk = torch.zeros(B, T, KVH, HD, dtype=torch.float64)
    dv = torch.zeros(B, T, KVH, HD, dtype=torch.float64)
    flat = (torch.arange(B)[:, None, None] * T + target) * KVH + kv      # [B, T, H] row of the [B*T*KVH] key table
    dk.view(-1, HD).index_add_(0, flat.reshape(-1), (ds[..., None] * q.double()).reshape(-1, HD))
    dv.view(-1, HD).index_add_(0, flat.reshape(-1), do.double().reshape(-1, HD))
    for name, t in (("dq", dq), ("dk", dk), ("dv", dv)):
        assert is_bf16(t.float()) and bool((t.float().double() == t).all()), f"expected {name} is not a bf16 value"
    return dq.float(), dk.float(), dv.float()


# ----------------------------------------------------------------------------------------------------- split bf16
def split_onehot(B: int, T: int, H: int, modes: Sequence[str], seed: int):
    """One-hot inputs of the split (HuBERT) kernel, bidirectional: returns (q_hi, q_lo, k_hi, k_lo, v_hi, v_lo) as
    [B, T, H, 64] and the expected (o_hi, o_lo).  Ql is non-zero only where Kl is zero and vice versa."""
    lo, hi = bounds(B, T, False)
    tgt = onehot_targets(lo, hi, modes)
    q = onehot_q(tgt, modes)
    k = onehot_k(B, T, H)
    q_hi, q_lo = q.clone(), torch.zeros_like(q)
    sg = torch.tensor([1.0 if m == "latest" else -1.0 for m in modes])
    p = torch.tensor([2.0 ** (10 + 4 * d) for d in range(4)])
    q_lo[..., 4:8] = sg[:, None] * p                                     # q = q_hi + q_lo, column 4 + d
    q_hi[..., 4:8] = q[..., 4:8] - q_lo[..., 4:8]
    k_hi, k_lo = k.clone(), torch.zeros_like(k)
    k_lo[..., :4] = -1.0                                                  # k = k_hi + k_lo, columns 0..3
    k_hi[..., :4] = k[..., :4] + 1.0
    for t in (q_hi, q_lo, k_hi, k_lo):
        assert is_bf16(t)
    assert float((q_lo[..., :4].abs() * k_lo[..., :4].abs()).max()) == 0 and float(k_lo[..., 4:].abs().max()) == 0
    v_hi = int_values((B, T, H, HD), 16, seed)
    v_lo = int_values((B, T, H, HD), 16, seed + 1) / 64.0
    o = expect_onehot_fwd(v_hi + v_lo, tgt, 1)[0]                        # exact in fp32: |v| < 2^5, step 2^-6
    o_hi = bf16(o)
    return (q_hi, q_lo, k_hi, k_lo, v_hi, v_lo), (o_hi, bf16(o - o_hi))


def split_uniform(B: int, T: int, H: int, seed: int):
    """q = 0 in the split kernel: O = fl(sum (Vh + Vl)) * fl(1/T), the sum exact (|sum| < 2^17, step 2^-6)."""
    z = torch.zeros(B, T, H, HD)
    k_hi = int_values((B, T, H, HD), 4, seed)
    v_hi = int_values((B, T, H, HD), 16, seed + 1)
    v_lo = int_values((B, T, H, HD), 16, seed + 2) / 64.0
    ssum = (v_hi.double() + v_lo.double()).sum(1, keepdim=True).float()
    o = (ssum * (torch.ones(()) / torch.tensor(float(T)))).expand(B, T, H, HD)
    o_hi = bf16(o)
    return (z, z, k_hi, torch.zeros_like(k_hi), v_hi, v_lo), (o_hi, bf16(o - o_hi))


# ----------------------------------------------------------------------------------------------------- decode
def decode_scores(q: torch.Tensor, k: torch.Tensor, scale: float, q_lo: Optional[torch.Tensor] = None) -> torch.Tensor:
    """The decode kernel's scaled scores, emulated: a = fl(q * fl(scale * log2 e)) per element (q = fl(q + q_lo) for a
    split query), then a sequential fp32 FMA chain over the 64 dims.  q [B, H, 64], k [B, KVH, Tc, 64] -> [B, H, Tc]."""
    B, H, _ = q.shape
    KVH = k.shape[1]
    sl2 = torch.tensor(scale, dtype=torch.float32) * torch.tensor(LOG2E, dtype=torch.float32)
    qf = q.float() if q_lo is None else q.float() + q_lo.float()          # fp32 sum
    a = qf * sl2                                                          # fp32 product
    kk = k.float().repeat_interleave(H // KVH, dim=1)                    # [B, H, Tc, 64]
    acc = torch.zeros(kk.shape[:3])
    for d in range(HD):
        acc = fma32(a[:, :, d, None], kk[..., d], acc)
    return acc


def decode_onehot(B: int, H: int, KVH: int, T_cache: int, lens: torch.Tensor, modes: Sequence[str], seed: int):
    """(q [B, H, 64], k, v [B, KVH, T_cache, 64], expected o [B, H, 64]) with target lens - 1 (latest) or 0 (earliest);
    asserts the margin on the emulated fp32 scores.  Rows with lens = 0 expect 0."""
    lens = lens.long()
    lo = torch.zeros(B, 1, dtype=torch.int64)
    hi = (lens - 1).clamp_min(0)[:, None]
    tgt = onehot_targets(lo, hi, modes)[:, 0]                          # [B, H]
    q = onehot_q(tgt, modes)
    k = onehot_k(B, T_cache, KVH).permute(0, 2, 1, 3).contiguous()
    v = int_values((B, KVH, T_cache, HD), 8, seed)
    _check_decode_margin(decode_scores(q, k, EXACT_SCALE), tgt, lens)
    kv = torch.arange(H) // (H // KVH)
    o = v[torch.arange(B)[:, None], kv[None, :], tgt]
    o[lens == 0] = 0.0
    return q, k, v, o


def _check_decode_margin(e: torch.Tensor, tgt: torch.Tensor, lens: torch.Tensor) -> None:
    """e [B, H, Tc] emulated exponents: every allowed non-target key lies more than UNDERFLOW below the target."""
    for b in range(e.shape[0]):
        n = int(lens[b])
        if n == 0:
            continue
        eb = e[b, :, :n]
        st = eb.gather(1, tgt[b][:, None])
        gap = eb - st
        gap.scatter_(1, tgt[b][:, None], -math.inf)
        if n > 1:
            assert float(gap.max()) < -UNDERFLOW, f"decode margin {float(gap.max())}"


def _pair(x: torch.Tensor):
    hi = bf16(x)
    return hi, bf16(x - hi)


def decode_split_onehot(B: int, H: int, T_cache: int, lens: torch.Tensor, modes: Sequence[str], seed: int):
    """One-hot inputs of the fp32-cache decode (KVH = H): (q_hi, q_lo [B, H, 64], k, v fp32 [B, H, T_cache, 64]) and
    the expected (o_hi, o_lo) [B, H, 64]; asserts the margin on the emulated scores.  k = k_hi + k_lo and
    v = v_hi + v_lo exactly (bf16 pairs), so the same keys can be fed to the split-bf16 prefill kernel."""
    lens = lens.long()
    lo = torch.zeros(B, 1, dtype=torch.int64)
    hi = (lens - 1).clamp_min(0)[:, None]
    tgt = onehot_targets(lo, hi, modes)[:, 0]                          # [B, H]
    q = onehot_q(tgt, modes)
    sg = torch.tensor([1.0 if m == "latest" else -1.0 for m in modes])
    p = torch.tensor([2.0 ** (10 + 4 * d) for d in range(4)])
    q_lo = torch.zeros_like(q)
    q_lo[..., 4:8] = sg[:, None] * p
    q_hi = q - q_lo
    assert is_bf16(q_hi) and is_bf16(q_lo) and torch.equal(q_hi + q_lo, q)
    g = torch.Generator().manual_seed(seed)
    k = onehot_k(B, T_cache, H).permute(0, 2, 1, 3).contiguous()
    k[..., 8:16] = sum(_pair(torch.randn(B, H, T_cache, 8, generator=g)))   # fp32, never multiplied by a non-zero q
    v = int_values((B, H, T_cache, HD), 8, seed) + int_values((B, H, T_cache, HD), 16, seed + 1) / 64.0
    _check_decode_margin(decode_scores(q_hi, k, EXACT_SCALE, q_lo), tgt, lens)
    o = v[torch.arange(B)[:, None], torch.arange(H)[None, :], tgt]
    o[lens == 0] = 0.0
    return (q_hi, q_lo, k, v), _pair(o)


def decode_split_uniform(B: int, H: int, T_cache: int, lens: torch.Tensor, seed: int):
    """q = 0 over an fp32 cache: (k, v [B, H, T_cache, 64]) and the expected (o_hi, o_lo) of
    O = fl(sum_{j < lens} v) * fl(1 / lens), the sum exact; 0 for lens = 0."""
    g = torch.Generator().manual_seed(seed)
    k = sum(_pair(torch.randn(B, H, T_cache, HD, generator=g) * 4))
    v = int_values((B, H, T_cache, HD), 8, seed) + int_values((B, H, T_cache, HD), 16, seed + 1) / 64.0
    o = torch.zeros(B, H, HD)
    for b in range(B):
        n = int(lens[b])
        if n:
            s = v[b, :, :n].double().sum(1)
            assert float(s.abs().max()) < 2 ** 15
            o[b] = s.float() * (torch.ones(()) / torch.tensor(float(n)))
    return (k, v), _pair(o)


def decode_f32_reference(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, lens: torch.Tensor, scale: float):
    """fp64 decode over an fp32 cache with the per-element bound of the module docstring: q [B, H, 64] (fp32 value of
    the pair), k / v [B, H, Tc, 64] -> (O* [B, H, 64], bound)."""
    B, H, _ = q.shape
    O = torch.zeros(B, H, HD, dtype=torch.float64)
    bo = torch.zeros_like(O)
    for b in range(B):
        n = int(lens[b])
        if n == 0:
            continue
        qb, kb, vb = q[b].double(), k[b, :, :n].double(), v[b, :, :n].double()
        s = torch.einsum("hd,hjd->hj", qb, kb) * scale
        sd = torch.einsum("hd,hjd->hj", qb.abs(), kb.abs()) * scale
        pi = torch.softmax(s, -1)
        o = torch.einsum("hj,hjd->hd", pi, vb)
        D = 64 * 2.0 ** -23 * sd.max(-1).values + 2.0 ** -20 * (s.abs().max(-1).values + 1)
        spread = torch.einsum("hj,hjd->hd", pi, vb.abs()) + o.abs()
        O[b] = o
        bo[b] = (torch.expm1(2 * D)[:, None] + (3 * n + 8) * 2.0 ** -23) * spread + 2.0 ** -17 * o.abs()
    return O, bo


def expect_decode_uniform(v: torch.Tensor, lens: torch.Tensor, H: int):
    """q = 0 in decode: O = bf16(fl(sum_{j < lens} v) * fl(1 / lens)); 0 for lens = 0."""
    B, KVH, Tc, _ = v.shape
    o = torch.zeros(B, H, HD)
    for b in range(B):
        n = int(lens[b])
        if n:
            s = v[b, :, :n].double().sum(1).float()
            o[b] = bf16(s * (torch.ones(()) / torch.tensor(float(n)))).repeat_interleave(H // KVH, dim=0)
    return o


# ----------------------------------------------------------------------------------------------------- random mode
def _docs_of(lo: torch.Tensor, hi: torch.Tensor, causal: bool):
    """Per batch row, the [a, e) spans inside which every row's allowed keys stay (documents, or the whole row)."""
    B, T = lo.shape
    out = []
    for b in range(B):
        if not causal:
            out.append([(0, T)])
            continue
        starts = sorted(set(lo[b].tolist()))
        out.append(list(zip(starts, starts[1:] + [T])))
    return out


def fwd_reference(q, k, v, lo, hi, scale: float, causal: bool, split: bool = False):
    """fp64 forward with its per-element contract bounds: (O*, lse*, bound_o, bound_lse); per head and per document."""
    B, T, H, _ = q.shape
    G = H // k.shape[2]
    c_p = 2.0 ** -16 if split else 2.0 ** -9
    O = torch.zeros(B, T, H, HD, dtype=torch.float64)
    bo = torch.zeros_like(O)
    lse = torch.zeros(B, T, H, dtype=torch.float64)
    bl = torch.zeros_like(lse)
    for b, spans in enumerate(_docs_of(lo, hi, causal)):
        for a, e in spans:
            keys = torch.arange(a, e)
            allowed = (keys[None] >= lo[b, a:e, None]) & (keys[None] <= hi[b, a:e, None])
            n = allowed.sum(-1).double()
            for h in range(H):
                qh = q[b, a:e, h].double()
                kh, vh = k[b, a:e, h // G].double(), v[b, a:e, h // G].double()
                s = (qh @ kh.t()) * scale
                sd = (qh.abs() @ kh.abs().t()) * scale
                s = s.masked_fill(~allowed, -math.inf)
                m = s.max(-1, keepdim=True).values
                w = torch.exp(s - m)
                pi = w / w.sum(-1, keepdim=True)
                o = pi @ vh
                ls = (m + torch.log(w.sum(-1, keepdim=True))).squeeze(-1)
                sabs = s.masked_fill(~allowed, 0).abs().max(-1).values
                D = 64 * 2.0 ** -23 * sd.masked_fill(~allowed, 0).max(-1).values + 2.0 ** -20 * (sabs + 1)
                if split:
                    D = D + 2.0 ** -16 * sd.masked_fill(~allowed, 0).max(-1).values
                spread = pi @ vh.abs() + o.abs()          # sum pi (|v| + |O*|), which also bounds sum pi |v - O*|
                bnd = (torch.expm1(2 * D)[:, None] + c_p + (3 * n + 8)[:, None] * 2.0 ** -23) * spread
                O[b, a:e, h] = o
                bo[b, a:e, h] = bnd
                lse[b, a:e, h] = ls
                bl[b, a:e, h] = D + (3 * n + 8) * 2.0 ** -23 + 2.0 ** -21 * (ls.abs() + 1)
    bo = bo + (2.0 ** -17 * O.abs() if split else 0.5 * ulp_bf16(O.abs() + bo))
    return O, lse, bo, bl


def bwd_reference(q, k, v, o, do, lse, lo, hi, scale: float, causal: bool):
    """fp64 backward from the kernel's own o and lse, with per-element bounds: (dq*, dk*, dv*, bq, bk, bv)."""
    B, T, H, _ = q.shape
    KVH = k.shape[2]
    G = H // KVH
    f64 = lambda t: t.double()
    dq = torch.zeros(B, T, H, HD, dtype=torch.float64)
    dk = torch.zeros(B, T, KVH, HD, dtype=torch.float64)
    dv = torch.zeros_like(dk)
    bq, bk, bv = torch.zeros_like(dq), torch.zeros_like(dk), torch.zeros_like(dk)
    ek = torch.zeros_like(dk)       # accumulated sum |dS| |q| for the fp32 summation term of dK (N applied below)
    ev = torch.zeros_like(dk)
    for b, spans in enumerate(_docs_of(lo, hi, causal)):
        for a, e in spans:
            keys = torch.arange(a, e)
            allowed = (keys[None] >= lo[b, a:e, None]) & (keys[None] <= hi[b, a:e, None])
            n = allowed.sum(-1).double()
            for h in range(H):
                g = h // G
                qh, kh, vh = f64(q[b, a:e, h]), f64(k[b, a:e, g]), f64(v[b, a:e, g])
                oh, doh, lh = f64(o[b, a:e, h]), f64(do[b, a:e, h]), f64(lse[b, a:e, h])
                s = (qh @ kh.t()) * scale
                sd = (qh.abs() @ kh.abs().t()) * scale
                sabs = s.masked_fill(~allowed, 0).abs().max(-1).values
                D = 64 * 2.0 ** -23 * sd.masked_fill(~allowed, 0).max(-1).values + 2.0 ** -20 * (sabs + 1)
                P = torch.exp(s - lh[:, None]).masked_fill(~allowed, 0)
                eP = (2.0 ** -8 + torch.expm1(D + 2.0 ** -21 * lh.abs()))[:, None]
                dP = doh @ vh.t()
                e_dP = 64 * 2.0 ** -23 * (doh.abs() @ vh.abs().t())
                delta = (doh * oh).sum(-1, keepdim=True)
                e_del = 64 * 2.0 ** -23 * (doh.abs() * oh.abs()).sum(-1, keepdim=True)
                dS = P * (dP - delta) * scale
                E = P * scale * ((dP - delta).abs() * (eP + 2.0 ** -9) + (e_dP + e_del) * (1 + eP))
                # dQ: sum over the n allowed keys
                dq[b, a:e, h] = dS @ kh
                bq[b, a:e, h] = (E + (n[:, None] + 2) * 2.0 ** -23 * (dS.abs() + E)) @ kh.abs()
                # dK / dV: sums over the group's queries (N applied after the loop)
                dk[b, a:e, g] += dS.t() @ qh
                dv[b, a:e, g] += P.t() @ doh
                bk[b, a:e, g] += E.t() @ qh.abs()
                ek[b, a:e, g] += (dS.abs() + E).t() @ qh.abs()
                bv[b, a:e, g] += (P * eP).t() @ doh.abs()
                ev[b, a:e, g] += P.t() @ doh.abs()
    N = float(G * T + 2) * 2.0 ** -23
    bk = bk + N * ek
    bv = bv + N * ev
    bq, bk, bv = (bd + 0.5 * ulp_bf16(r.abs() + bd) for r, bd in ((dq, bq), (dk, bk), (dv, bv)))
    return dq, dk, dv, bq, bk, bv


# ----------------------------------------------------------------------------------------------------- adversarial data
def rising_inputs(B: int, T: int, H: int, KVH: int, seed: int, top: float = 30.0):
    """Random q / k / v whose scaled scores (scale 1/8) rise tile by tile from about -top to +top along the keys, so the
    running max moves at every 64-key tile and each tile's rescaling factor matters."""
    g = torch.Generator().manual_seed(seed)
    q = torch.randn(B, T, H, HD, generator=g)
    k = torch.randn(B, T, KVH, HD, generator=g)
    v = torch.randn(B, T, KVH, HD, generator=g)
    q[..., 0] = 8.0                                                       # scaled score = k[..., 0] + N(0, ~1)
    k[..., 0] = torch.linspace(-top, top, T)[None, :, None]
    return bf16(q), bf16(k), bf16(v)


def wide_inputs(B: int, T: int, H: int, KVH: int, seed: int, span: float = 40.0):
    """Random inputs whose scaled scores (scale 1/8) spread over about +-span."""
    g = torch.Generator().manual_seed(seed)
    sd = math.sqrt(span / 3.0)                                               # s / 8 has standard deviation span / 3
    q = torch.randn(B, T, H, HD, generator=g) * sd
    k = torch.randn(B, T, KVH, HD, generator=g) * sd
    v = torch.randn(B, T, KVH, HD, generator=g)
    return bf16(q), bf16(k), bf16(v)


# ----------------------------------------------------------------------------------------------------- CPU flash model
def flash_emulate(q, k, v, lo, hi, scale: float, *, causal_shift: int = 0, lo_shift: int = 0, drop_last_tile=False,
                  wrong_kv_head: Optional[int] = None, no_corr_tile: Optional[int] = None, scale_mult: float = 1.0,
                  shift_warp: Optional[int] = None):
    """A straightforward fp32 flash forward in 64-key tiles with bf16 P, the FMA of the exponent emulated: the model of
    what the kernels compute (bit-exact on the exact modes), with injectable defects:
      causal_shift  the row's last allowed key moves by this many keys (mask off by one);
      lo_shift      the document start moves by this many keys;
      drop_last_tile  the last key tile is skipped when T is not a multiple of 64;
      wrong_kv_head q head that reads the next kv head;
      no_corr_tile  key tile whose rescaling of the running output is skipped;
      scale_mult    scale error;
      shift_warp    16-row slice (of the first 64-row tile) whose rows are written one row down.
    Returns (O [B, T, H, 64] bf16 values, lse [B, T, H] fp32)."""
    B, T, H, _ = q.shape
    KVH = k.shape[2]
    G = H // KVH
    scale = scale * scale_mult
    kvh = torch.arange(H) // G
    if wrong_kv_head is not None:
        kvh[wrong_kv_head] = (kvh[wrong_kv_head] + 1) % KVH
    kk, vv = k.float()[:, :, kvh], v.float()[:, :, kvh]                  # [B, T, H, 64]
    qf = q.float()
    sl2 = torch.tensor(scale, dtype=torch.float32) * torch.tensor(LOG2E, dtype=torch.float32)
    hi2, lo2 = (hi + causal_shift)[:, None, :, None], (lo + lo_shift)[:, None, :, None]
    m = torch.full((B, H, T), -math.inf)
    l = torch.zeros(B, H, T)
    acc = torch.zeros(B, H, T, HD)
    n_tiles = (T + 63) // 64
    for jt in range(n_tiles):
        if drop_last_tile and jt == n_tiles - 1 and T % 64:
            continue
        j0, j1 = jt * 64, min(T, jt * 64 + 64)
        key = torch.arange(j0, j1)
        s = torch.einsum("bthd,bjhd->bhtj", qf, kk[:, j0:j1])
        ok = (key >= lo2) & (key <= hi2)
        s = s.masked_fill(~ok, -math.inf)
        mx = torch.maximum(m, s.max(-1).values)
        corr = torch.where(m == -math.inf, torch.zeros(()), torch.exp2((m - mx) * sl2))
        mb = torch.where(mx == -math.inf, torch.zeros(()), mx * sl2)
        p = torch.exp2(fma32(s, sl2, -mb[..., None]))
        l = l * corr + p.sum(-1)
        c = torch.ones_like(corr) if no_corr_tile == jt else corr
        acc = acc * c[..., None] + torch.einsum("bhtj,bjhd->bhtd", bf16(p), vv[:, j0:j1])
        m = mx
    inv = torch.where(l > 0, torch.ones(()) / l, torch.zeros(()))
    o = bf16(acc * inv[..., None]).permute(0, 2, 1, 3).contiguous()
    lse = (m * torch.tensor(scale, dtype=torch.float32) + torch.log(l)).permute(0, 2, 1).contiguous()
    if shift_warp is not None:
        r0 = 16 * shift_warp
        o[:, r0 + 1:r0 + 16] = o[:, r0:r0 + 15].clone()
    return o, lse


# ----------------------------------------------------------------------------------------------------- checker
class Mismatch:
    """Flagged elements of a [B, rows, heads, cols] comparison: count, first locations, and a readable message."""

    def __init__(self, what: str, bad: torch.Tensor, got: torch.Tensor, want: torch.Tensor, rows: str, limit: int = 6):
        self.count = int(bad.sum())
        idx = bad.nonzero()
        self.locs = [tuple(int(x) for x in r) for r in idx[:limit].tolist()]
        self.rows = sorted(set(idx[:, 1].tolist()))
        self.heads = sorted(set(idx[:, 2].tolist()))
        self.batches = sorted(set(idx[:, 0].tolist()))
        lines = [f"{what}: {self.count} of {bad.numel()} elements differ; first (batch, head, {rows}, col, "
                 f"{rows} tile64, warp16 slice): got / want"]
        for loc in self.locs:
            b, r, h = loc[0], loc[1], loc[2]
            c = loc[3] if len(loc) > 3 else -1
            g = float(got[loc]) if got is not None else float("nan")
            w = float(want[loc])
            lines.append(f"  ({b}, {h}, {r}, {c}, {r // 64}, {(r % 64) // 16}): {g!r} / {w!r}")
        lines.append(f"  flagged {rows}s [{self.rows[0]}, {self.rows[-1]}] heads {self.heads} batches {self.batches}")
        self.message = "\n".join(lines)

    def __str__(self):
        return self.message


def _prep(got, want):
    assert got.shape == want.shape, (tuple(got.shape), tuple(want.shape))
    return got.detach().cpu().double(), want.detach().cpu().double()


def mismatch_exact(got, want, what="attention", rows="row") -> Optional[Mismatch]:
    """Element-wise equality (NaN never equals anything); got / want [B, rows, heads(, cols)]."""
    g, w = _prep(got, want)
    bad = ~(g == w)
    return Mismatch(what, bad, g, w, rows) if bool(bad.any()) else None


def mismatch_bound(got, want, bound, what="attention", rows="row") -> Optional[Mismatch]:
    """|got - want| <= bound per element (NaN fails)."""
    g, w = _prep(got, want)
    bad = ~((g - w).abs() <= bound.cpu().double())
    return Mismatch(what, bad, g, w, rows) if bool(bad.any()) else None


def mismatch_lse_exact(got, n_or_zero, what="lse", ulps: int = 2) -> Optional[Mismatch]:
    """lse against an fp64 value within `ulps` fp32 ulps (log of the uniform mode, or 0 of the one-hot mode)."""
    g, w = _prep(got, n_or_zero)
    return mismatch_bound(g, w, ulps * ulp_f32(w), what)


# ----------------------------------------------------------------------------------------------------- device layout
def fuse(q, k, v, ld: Optional[int] = None, fill=float("nan"), device="cpu") -> torch.Tensor:
    """[B*T, ld] bf16 fused projection (q heads, k heads, v heads), padding columns past the heads filled with `fill`."""
    B, T, H, _ = q.shape
    KVH = k.shape[2]
    w = (H + 2 * KVH) * HD
    ld = ld or w
    buf = torch.full((B * T, ld), fill, dtype=torch.bfloat16)
    buf[:, :H * HD] = q.reshape(B * T, -1).to(torch.bfloat16)
    buf[:, H * HD:(H + KVH) * HD] = k.reshape(B * T, -1).to(torch.bfloat16)
    buf[:, (H + KVH) * HD:w] = v.reshape(B * T, -1).to(torch.bfloat16)
    return buf.to(device)


def unfuse(x: torch.Tensor, B: int, T: int, H: int, KVH: int):
    """[B*T, >= (H + 2 KVH) 64] -> (q [B,T,H,64], k, v [B,T,KVH,64]) as float on the CPU"""
    x = x.detach().cpu().float()
    q = x[:, :H * HD].reshape(B, T, H, HD)
    k = x[:, H * HD:(H + KVH) * HD].reshape(B, T, KVH, HD)
    v = x[:, (H + KVH) * HD:(H + 2 * KVH) * HD].reshape(B, T, KVH, HD)
    return q, k, v


def heads(x: torch.Tensor, B: int, T: int, H: int) -> torch.Tensor:
    """[B*T, >= H*64] -> [B, T, H, 64] float on the CPU"""
    return x.detach().cpu().float()[:, :H * HD].reshape(B, T, H, HD)


def lse_bth(lse: torch.Tensor) -> torch.Tensor:
    """kernel lse [B, H, T] -> [B, T, H] on the CPU"""
    return lse.detach().cpu().double().permute(0, 2, 1)
