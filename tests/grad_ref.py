"""References and per-element checkers for the gradient path of the train step: the cross-entropy gradient, the
fixed-point table gradients, column sums, the LayerNorm weight gradients, the gradient norm and clip coefficient, both
AdamW kernels, the ReLU backward and the widening of bf16 gradients into fp32.

Most of these kernels get an exact reference because their operands can be chosen:
  - integer operands make every fp32 sum exact (column sums, LayerNorm dw / db, sums of squares);
  - the table gradients sum rint(dx * 2^40) in 64-bit integers, so `table_fix_sum` below restates them exactly for any
    input, and for dx on a k * 2^-j grid (j <= 40) that sum is the fp64 index_add itself;
  - `adamw_master` restates ATen's fused adam_math in numpy.float32, one rounding per operation.
The cross-entropy gradient is compared per element with float64 softmax - onehot under `ce_bound`, a bound derived from
the kernel's arithmetic; a bf16 output then has to be one of the bf16 roundings of [ref - bound, ref + bound] (at most
two values, and one unless ref sits that close to a rounding boundary).

Checkers return a list of located failures (empty when the output conforms), so the GPU suite can print where a kernel
went wrong and the CPU suite can show that each checker flags an injected defect.
"""
from __future__ import annotations

import math
from typing import List, Optional, Sequence

import numpy as np
import torch

U = 2.0 ** -24                 # unit roundoff of fp32
FIX = 2.0 ** 40                # fixed-point scale of the table gradients
LOG2E = 1.4426950408889634


# ----------------------------------------------------------------------------------------------------- bf16 helpers
def bf16(x) -> np.ndarray:
    """Round float32 values to bf16 (nearest even), returned as float32."""
    t = torch.from_numpy(np.ascontiguousarray(np.asarray(x, dtype=np.float32)))
    return t.to(torch.bfloat16).float().numpy()


def bf16_from64(x) -> np.ndarray:
    """bf16 rounding of float64 values with one rounding: the float32 conversion rounds to odd first, which keeps the
    nearest-even bf16 result of the exact value."""
    x = np.asarray(x, dtype=np.float64)
    f = x.astype(np.float32)
    lost = (f.astype(np.float64) != x) & np.isfinite(x)
    bits = f.view(np.uint32).copy()
    # round to odd: a float32 that is not exact keeps an odd last bit (the exact value lies strictly between neighbours)
    trunc = np.where(np.abs(f.astype(np.float64)) > np.abs(x), bits - 1, bits).astype(np.uint32)
    bits = np.where(lost, trunc | 1, bits).astype(np.uint32)
    return bf16(bits.view(np.float32))


def locate(mask: np.ndarray, got, want, what: str, limit: int = 5) -> List[str]:
    idx = np.argwhere(mask)
    out = [f"{what}: {len(idx)} element(s) off"] if len(idx) else []
    g, w = np.asarray(got), np.asarray(want)
    for i in idx[:limit]:
        t = tuple(int(v) for v in i)
        out.append(f"  at {t}: got {float(g[t])!r}, want {float(w[t])!r}")
    return out


def check_exact(got, want, what: str) -> List[str]:
    """Bit for bit (NaN matches NaN; +0 and -0 are different)."""
    g = np.asarray(got, dtype=np.float32)
    w = np.asarray(want, dtype=np.float32)
    bad = g.view(np.uint32) != w.view(np.uint32)
    return locate(bad, g, w, what)


def check_bf16_interval(got, ref64, bound, what: str) -> List[str]:
    """got (bf16 values) must be a bf16 rounding of some value within `bound` of the float64 reference."""
    g = np.asarray(got, dtype=np.float32)
    r = np.asarray(ref64, dtype=np.float64)
    lo, hi = bf16_from64(r - bound), bf16_from64(r + bound)
    bad = ~((g >= lo) & (g <= hi))
    return locate(bad, g, r, what)


# ----------------------------------------------------------------------------------------------------- cross entropy
def ce_reference(logits, labels, T: int, V: int, grad_scale: float, row_weight=None):
    """float64 reference of the CE kernels over bf16 logits [M, ldl] (float32 array of bf16 values) with shifted
    labels: row m predicts labels[m + 1] unless m is the last position of its sequence; a target outside [0, V) (the
    ignore index -100, or V and above) makes the row invalid.  Returns (dlogits before bf16 rounding [M, ldl] with
    padding columns and invalid rows 0, row nll [M] (0 when invalid), valid [M], lse [M], max - min logit per row,
    softmax [M, ldl], the fp32 gradient scale of each row [M])."""
    x = np.asarray(logits, dtype=np.float64)
    M, ldl = x.shape
    lab = np.asarray(labels, dtype=np.int64)
    tgt = np.full(M, -100, dtype=np.int64)
    m = np.arange(M)
    has = (m % T) < T - 1
    tgt[has] = lab[m[has] + 1]
    valid = (tgt >= 0) & (tgt < V)
    v = x[:, :V]
    mx = v.max(axis=1, keepdims=True)
    e = np.exp(v - mx)
    se = e.sum(axis=1, keepdims=True)
    p = e / se
    lse = (mx + np.log(se))[:, 0]
    nll = np.where(valid, lse - v[m, np.clip(tgt, 0, V - 1)], 0.0)
    d = np.zeros((M, ldl))
    d[:, :V] = p
    pfull = d.copy()
    d[m[valid], tgt[valid]] -= 1.0
    gs = np.full(M, float(np.float32(grad_scale)), dtype=np.float64)
    if row_weight is not None:
        gs = (np.float32(grad_scale) * np.asarray(row_weight, dtype=np.float32)).astype(np.float64)
    d *= gs[:, None]
    d[~valid] = 0.0
    spread = (mx[:, 0] - v.min(axis=1))
    return d, nll, valid, lse, spread, pfull, gs


def ce_bound(kernel: str, p, dref, lse, spread, ldl: int, gs) -> np.ndarray:
    """Per-element bound on |fp32 gradient - float64 reference| before the bf16 rounding; p is the float64 softmax.

    warp (ldl <= 512, expf): each exp is within 2 ulp (4u) plus u * |v - max| from its rounded argument; a lane sums
    16 terms, then 5 shuffle levels; 1 / se and the product add u each.
    block (ex2.approx.ftz): each 2^x is within 2 ulp, and its argument x * log2(e) - lse * log2(e) carries about
    u * (|x - max| + 3 |lse|) * log2(e) absolute; the online sum rescales once per 8-column step of a thread (ldl / 2048
    of them) and once per shuffle and block level.
    The target column adds the rounding of p - 1, the scale one rounding more."""
    g = np.abs(np.asarray(gs, dtype=np.float64)).reshape(-1, 1)
    s = np.asarray(spread, dtype=np.float64).reshape(-1, 1)
    L = np.abs(np.asarray(lse, dtype=np.float64)).reshape(-1, 1)
    if kernel == "warp":
        rel = (4 + 16 + 5 + 2 + 4 + 2 * s) * U
    else:
        steps = math.ceil(ldl / 8 / 256)
        rel = (steps * 18 + 13 * 10 + 8 + 2 * LOG2E * (s + 3 * L)) * 4 * U
    d = np.abs(np.asarray(dref, dtype=np.float64))
    # subnormal exp results carry their own absolute rounding (a few 2^-149)
    return rel * np.asarray(p, dtype=np.float64) * g + 2 * U * d + 8 * 2.0 ** -149 * (1 + g)


def check_ce_grad(got, dref, valid, V: int, bound) -> List[str]:
    """Every element within the bound; padding columns, invalid rows exactly 0."""
    g = np.asarray(got, dtype=np.float32)
    out = check_bf16_interval(np.where(valid[:, None], g, 0.0)[:, :V], np.asarray(dref)[:, :V], np.asarray(bound)[:, :V],
                              "dlogits")
    out += locate(g[:, V:] != 0, g[:, V:], np.zeros_like(g[:, V:]), "dlogits padding column not 0")
    inval = g[~valid]
    out += locate(inval != 0, inval, np.zeros_like(inval), "dlogits of an ignored row not 0")
    return out


# ----------------------------------------------------------------------------------------------------- table gradients
def grid_values(shape, j: int, kmax: int, seed: int) -> np.ndarray:
    """k * 2^-j with integer |k| <= kmax (0 included): bf16-exact for kmax <= 256 and fixed-point exact for j <= 40."""
    r = np.random.default_rng(seed)
    return (r.integers(-kmax, kmax + 1, size=shape) * 2.0 ** -j).astype(np.float32)


def opt_pos_rows(pos_ids, M: int, T: int, n_pos: int) -> np.ndarray:
    """The position-table row each token reads: min(max(pos + 2, 0), n_pos - 1), pos = pos_ids or m % T."""
    pos = np.asarray(pos_ids, dtype=np.int64).reshape(-1) if pos_ids is not None else np.arange(M) % T
    return np.clip(pos + 2, 0, n_pos - 1)


def table_fix_sum(rows, dx, n_rows: int) -> np.ndarray:
    """The fixed-point scatter: sum over m with rows[m] in [0, n_rows) of rint(dx[m] * 2^40), exact in int64, as the
    float64 value the kernels convert ((double) sum * 2^-40)."""
    dx = np.asarray(dx, dtype=np.float32)
    q = np.rint(dx.astype(np.float64) * FIX).astype(np.int64)
    r = np.asarray(rows, dtype=np.int64)
    keep = (r >= 0) & (r < n_rows)
    acc = np.zeros((n_rows, dx.shape[1]), dtype=np.int64)
    np.add.at(acc, r[keep], q[keep])
    return acc.astype(np.float64) / FIX


def table_grad_bf16(rows, dx, n_rows: int, old=None) -> np.ndarray:
    """bf16 table gradient: bf16(float(S) (+ float(old) when accumulating)), S = table_fix_sum."""
    s = table_fix_sum(rows, dx, n_rows).astype(np.float32)
    if old is not None:
        s = (s + np.asarray(old, dtype=np.float32)).astype(np.float32)
    return bf16(s)


def table_grad_f32(rows, dx, n_rows: int, head=None, old=None) -> np.ndarray:
    """fp32 table gradient: (old +) (float(head) + float(S)), each sum rounded once in fp32, in that order."""
    s = table_fix_sum(rows, dx, n_rows).astype(np.float32)
    if head is not None:
        s = (np.asarray(head, dtype=np.float32) + s).astype(np.float32)
    if old is not None:
        s = (np.asarray(old, dtype=np.float32) + s).astype(np.float32)
    return s


def index_add64(rows, dx, n_rows: int) -> np.ndarray:
    r = np.asarray(rows, dtype=np.int64)
    keep = (r >= 0) & (r < n_rows)
    acc = np.zeros((n_rows, np.asarray(dx).shape[1]))
    np.add.at(acc, r[keep], np.asarray(dx, dtype=np.float64)[keep])
    return acc


# ----------------------------------------------------------------------------------------------------- column sums / LN
def colsum_ref(x, old=None, out_f32: bool = False) -> np.ndarray:
    """Column sums of integer-valued rows (exact in fp32 below 2^24), (+ old) rounded once, bf16 unless out_f32."""
    s = np.asarray(x, dtype=np.float64).sum(axis=0).astype(np.float32)
    if old is not None:
        s = (s + np.asarray(old, dtype=np.float32)).astype(np.float32)
    return s if out_f32 else bf16(s)


def ln_bwd_ref(dy, x, w, mean, rstd, dy2=None, w2=None):
    """float64 LayerNorm backward from the given mean / rstd: (dx [M, D], dw, db, dw2, db2)."""
    dy, x, w = (np.asarray(a, dtype=np.float64) for a in (dy, x, w))
    xh = (x - np.asarray(mean, dtype=np.float64)[:, None]) * np.asarray(rstd, dtype=np.float64)[:, None]
    g = dy * w
    if dy2 is not None:
        g = g + np.asarray(dy2, dtype=np.float64) * np.asarray(w2, dtype=np.float64)
    D = x.shape[1]
    m1 = g.sum(axis=1, keepdims=True) / D
    m2 = (g * xh).sum(axis=1, keepdims=True) / D
    dx = np.asarray(rstd, dtype=np.float64)[:, None] * (g - m1 - xh * m2)
    out = [dx, (dy * xh).sum(axis=0), dy.sum(axis=0)]
    if dy2 is not None:
        d2 = np.asarray(dy2, dtype=np.float64)
        out += [(d2 * xh).sum(axis=0), d2.sum(axis=0)]
    return out


def ln_dx_bound(dy, x, w, mean, rstd, dy2=None, w2=None) -> np.ndarray:
    """Bound on the fp32 dx of the LayerNorm backward: m1 and m2 are exact sums divided by D (one rounding each),
    g - m1 - xhat * m2 carries at most three roundings (with or without contraction), times rstd one more."""
    dy, x, w = (np.asarray(a, dtype=np.float64) for a in (dy, x, w))
    xh = (x - np.asarray(mean)[:, None]) * np.asarray(rstd)[:, None]
    g = np.abs(dy * w)
    if dy2 is not None:
        g = g + np.abs(np.asarray(dy2, dtype=np.float64) * np.asarray(w2, dtype=np.float64))
    m1 = np.abs(g.sum(axis=1, keepdims=True)) / x.shape[1]
    m2 = (g * np.abs(xh)).sum(axis=1, keepdims=True) / x.shape[1]
    return 6 * U * np.asarray(rstd)[:, None] * (g + m1 + np.abs(xh) * m2)


# ----------------------------------------------------------------------------------------------------- norm and clip
def clip_grad_norm_ref(grads: Sequence[torch.Tensor], max_norm: float):
    """torch.nn.utils.clip_grad_norm_(error_if_nonfinite=False) restated as oracle/lm_oracle.py does (foreach norms in
    the gradient dtype): (per-tensor norms, total, coef) as tensors of the gradient dtype.  max_norm <= 0 is the
    Trainer's 'no clipping' (coef 1)."""
    norms = [torch.linalg.vector_norm(g, 2.0) for g in grads]
    total = torch.linalg.vector_norm(torch.stack(norms), 2.0)
    if max_norm <= 0:
        return norms, total, torch.ones((), dtype=total.dtype)
    coef = torch.clamp(max_norm / (total + 1e-6), max=1.0)
    return norms, total, coef


def chunk_tables(sizes: Sequence[int], chunk: int, align: int = 64):
    """Flat layout of tensors of the given sizes (each start rounded up to `align`) and its norm chunk tables:
    (offsets, total length, chunk_start int64, chunk_len int32, tensor_chunk_begin int32)."""
    offs, cs, cl, tb = [], [], [], [0]
    o = 0
    for n in sizes:
        offs.append(o)
        for s in range(0, n, chunk):
            cs.append(o + s)
            cl.append(min(chunk, n - s))
        if n == 0:
            cs.append(o)
            cl.append(0)
        tb.append(len(cs))
        o += -(-n // align) * align
    return offs, o, np.array(cs, np.int64), np.array(cl, np.int32), np.array(tb, np.int32)


# ----------------------------------------------------------------------------------------------------- AdamW
def adamw_master(p, g, m, v, *, lr, beta1, beta2, eps, wd, step, coef=1.0):
    """ATen fused adam_math (ADAMW) on fp32 tensors, every operation rounded to fp32 on its own; the hyperparameters
    formed in double and rounded once, as Python does before torch sees them.  Returns (p, m, v, bf16 shadow)."""
    f = np.float32
    p, g, m, v = (np.asarray(a, dtype=np.float32).copy() for a in (p, g, m, v))
    bc1 = 1.0 - float(f(beta1)) ** step
    lr_wd, omb1 = f(float(f(lr)) * float(f(wd))), f(1.0 - float(f(beta1)))
    omb2, step_size = f(1.0 - float(f(beta2))), f(float(f(lr)) / bc1)
    bc2s = f(math.sqrt(1.0 - float(f(beta2)) ** step))
    with np.errstate(all="ignore"):
        grad = (g * f(coef)).astype(f)
        p = (p - (lr_wd * p).astype(f)).astype(f)
        m = (m + (omb1 * (grad - m).astype(f)).astype(f)).astype(f)
        v = ((f(beta2) * v).astype(f) + ((omb2 * grad).astype(f) * grad).astype(f)).astype(f)
        denom = ((np.sqrt(v).astype(f) / bc2s).astype(f) + f(eps)).astype(f)
        p = (p - ((step_size * m).astype(f) / denom).astype(f)).astype(f)
    return p, m, v, bf16(p)


def adamw_groups(p, g, m, v, layout, *, wd, **hp):
    """sk_lm_optimizer_step's decay groups on flat fp32 buffers: for each (offset, rows, cols) tensor, adamw_master over
    its ALIGN_ELEMS-padded range with weight decay 0 when rows == 1 (biases and norm weights, HF Trainer's
    no-decay group), wd otherwise.  Returns (p, m, v, shadow)."""
    p, g, m, v = (np.asarray(a, dtype=np.float32).copy() for a in (p, g, m, v))
    for off, rows, cols in layout:
        n = -(-rows * cols // 64) * 64
        s = slice(off, off + n)
        p[s], m[s], v[s], _ = adamw_master(p[s], g[s], m[s], v[s], wd=0.0 if rows == 1 else wd, **hp)
    return p, m, v, bf16(p)


def adamw_bf16_ref(p, g, m, v, *, lr, beta1, beta2, eps, wd, step, coef=1.0):
    """float64 evaluation of the bf16 kernel's fp32 formula (the clip scale rounded to bf16 first, as the kernel and
    torch on bf16 gradients do).  Returns the float64 (p, m, v) before their bf16 rounding."""
    p, g, m, v = (np.asarray(a, dtype=np.float64) for a in (p, g, m, v))
    if coef != 1.0:
        g = bf16((g * np.float32(coef)).astype(np.float32)).astype(np.float64)
    f = lambda a: float(np.float32(a))
    # the launcher forms the bias corrections in double from the fp32 betas it receives
    bc1 = np.float64(np.float32(1.0 - f(beta1) ** step))
    bc2s = np.float64(np.float32(math.sqrt(1.0 - f(beta2) ** step)))
    p = p - f(lr) * f(wd) * p
    m = m + (1 - f(beta1)) * (g - m)
    v = f(beta2) * v + (1 - f(beta2)) * g * g
    p = p - (f(lr) / bc1) * m / (np.sqrt(v) / bc2s + f(eps))
    return p, m, v


def adamw_bf16_bound(p, g, m, v, *, lr, beta1, beta2, eps, wd, step):
    """Bound on |fp32 result - float64 reference| of each bf16 AdamW output (each operation rounded or contracted)."""
    p, g, m, v = (np.abs(np.asarray(a, dtype=np.float64)) for a in (p, g, m, v))
    bm = 6 * U * (m + g)
    bv = 6 * U * (v + g * g)
    mm = m + g
    vv = v + g * g
    bc2s = math.sqrt(1.0 - beta2 ** step)
    den = np.sqrt(vv) / bc2s + eps
    upd = (lr / (1.0 - beta1 ** step)) * mm / den
    bp = 4 * U * p + upd * (12 * U + bm / np.maximum(mm, 1e-300)
                            + (bv / np.maximum(vv, 1e-300)) * 0.5 * (np.sqrt(vv) / bc2s) / den)
    return bp, bm, bv
