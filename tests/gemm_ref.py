"""Reference and checker for the wgmma GEMM: C = A @ B^T with its epilogues, compared per element.

Exact-integer mode: A and B hold small integers stored in bf16 with K * max|a| * max|b| < 2^24, so every product and
every fp32 partial sum is exact.  The fp32 accumulator is then the same for every tile width, split, stream-K range
and summation order, a float64 matmul gives it exactly, and the epilogue's declared rounding points (emulated below
in fp32 with bf16 round-to-nearest-even) give the output bit for bit.

Random-data mode: bf16 normal operands, compared per element within half a bf16 ulp of the output plus the worst-case
fp32 accumulation error K * 2^-23 * sum_k |a_k b_k|.

GELU: the kernel evaluates erf with the Abramowitz-Stegun 7.1.26 polynomial (|error| <= 1.5e-7 * |y| / 2 on gelu);
it is compared with the exact-erf GELU of the exact pre-activation within one bf16 ulp plus 1.5e-7 * |y|.

Every check reports the number of mismatches and the first few as (row, col, tile row, tile col, 64-column chunk,
32-row quadrant), so that a failure points at the part of the schedule that produced it.  Works on CPU and GPU
tensors alike.
"""
from __future__ import annotations

import math
from typing import Optional

import torch

BM = 128     # tile rows
BK = 64      # k-block
EXACT_LIMIT = 1 << 24


# ----------------------------------------------------------------------------------------------------- operands
def int_operand(rows: int, cols: int, amax: int, seed: int, device="cpu") -> torch.Tensor:
    """[rows, cols] uniform integers in [-amax, amax], stored in bf16 (exact for amax <= 256)."""
    g = torch.Generator(device=device).manual_seed(seed)
    return torch.randint(-amax, amax + 1, (rows, cols), generator=g, device=device).to(torch.bfloat16)


def acc_scale(K: int, amax: int) -> float:
    """Standard deviation of a sum of K products of independent uniform integers in [-amax, amax]."""
    var = ((2 * amax + 1) ** 2 - 1) / 12.0
    return math.sqrt(K) * var


def real_operand(shape, scale: float, seed: int, device="cpu") -> torch.Tensor:
    """bf16 normal values of the given scale (bias / residual on the accumulator's scale: not integers, so every
    rounding point of the epilogue changes some outputs)."""
    g = torch.Generator(device=device).manual_seed(seed)
    return (torch.randn(shape, generator=g, device=device) * scale).to(torch.bfloat16)


def exact_acc(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """float64 [M, N] accumulator of integer operands a [M, K], b [N, K]; asserts that the fp32 sums are exact."""
    K = a.shape[1]
    amax, bmax = float(a.float().abs().max()), float(b.float().abs().max())
    assert K * amax * bmax < EXACT_LIMIT, f"fp32 accumulation is not exact: K={K} max|a|={amax} max|b|={bmax}"
    assert torch.equal(a.float(), a.float().round()) and torch.equal(b.float(), b.float().round()), "operands must be integers"
    return a.double() @ b.double().t()


# ----------------------------------------------------------------------------------------------------- epilogue
def bf16_round(x: torch.Tensor) -> torch.Tensor:
    """fp32 -> bf16 (round to nearest even) -> fp32"""
    return x.float().to(torch.bfloat16).float()


def ulp_bf16(x: torch.Tensor) -> torch.Tensor:
    """Spacing of bf16 values at |x| (float64)."""
    x = x.double().abs()
    _, e = torch.frexp(x)                        # x = m * 2^e, m in [0.5, 1)
    ulp = torch.ldexp(torch.ones_like(x), e - 8)
    return torch.where(x < 2.0 ** -126, torch.full_like(x, 2.0 ** -133), ulp)


def epilogue(acc: torch.Tensor, bias: Optional[torch.Tensor] = None, residual: Optional[torch.Tensor] = None,
             round_before_res: bool = False, out_f32: bool = False) -> torch.Tensor:
    """The GEMM's declared rounding points, in fp32:  v = acc + bias;  v = (bf16(v) if round_before_res else v) + res;
    out = bf16(v), or v when out_f32.  acc must be exact in fp32 (exact_acc)."""
    v = acc.float()
    if bias is not None:
        v = v + bias.float()
    if residual is not None:
        v = (bf16_round(v) if round_before_res else v) + residual.float()
    return v if out_f32 else bf16_round(v)


def rope_epilogue(acc: torch.Tensor, bias: Optional[torch.Tensor], cos: torch.Tensor, sin: torch.Tensor,
                  pos: torch.Tensor, rope_cols: int) -> torch.Tensor:
    """Bias + RoPE epilogue of sk_linear_rope: x = bf16(acc + bias); each 64-column head below rope_cols is rotated
    (rotate_half) as sk_rope does it, out1 = bf16(bf16(x1 c) + bf16(-x2 s)), out2 = bf16(bf16(x2 c) + bf16(x1 s)),
    with pos clamped to the rows of the tables."""
    x = epilogue(acc, bias)
    pos = pos.long().clamp(0, cos.shape[0] - 1)
    c, s = cos.float()[pos], sin.float()[pos]    # [M, 32]
    out = x.clone()
    for h0 in range(0, rope_cols, 64):
        x1, x2 = x[:, h0:h0 + 32], x[:, h0 + 32:h0 + 64]
        out[:, h0:h0 + 32] = bf16_round(bf16_round(x1 * c) + bf16_round(-x2 * s))
        out[:, h0 + 32:h0 + 64] = bf16_round(bf16_round(x2 * c) + bf16_round(x1 * s))
    return out


def gelu_exact(v: torch.Tensor) -> torch.Tensor:
    v = v.double()
    return 0.5 * v * (1.0 + torch.erf(v / math.sqrt(2.0)))


# ----------------------------------------------------------------------------------------------------- checker
def report(bad: torch.Tensor, out: torch.Tensor, want: torch.Tensor, bn: int, what: str, limit: int = 6) -> Optional[str]:
    """None when no element is flagged, else a message with the count and the first `limit` mismatches."""
    n = int(bad.sum())
    if n == 0:
        return None
    idx = bad.nonzero()[:limit].tolist()
    lines = [f"{what}: {n} of {bad.numel()} elements differ; first (row, col, tile row, tile col, chunk64, quadrant): got / want"]
    for r, c in idx:
        lines.append(f"  ({r}, {c}, {r // BM}, {c // bn}, {(c % bn) // 64}, {(r % BM) // 32}): "
                     f"{float(out[r, c])!r} / {float(want[r, c])!r}")
    rows = bad.any(dim=1).nonzero().flatten()
    cols = bad.any(dim=0).nonzero().flatten()
    lines.append(f"  flagged rows [{int(rows.min())}, {int(rows.max())}], columns [{int(cols.min())}, {int(cols.max())}]")
    return "\n".join(lines)


def mismatch_exact(out: torch.Tensor, want: torch.Tensor, bn: int = 256, what: str = "gemm") -> Optional[str]:
    """Element-wise equality (NaN never equals anything)."""
    assert out.shape == want.shape, (out.shape, want.shape)
    o, w = out.float(), want.float().to(out.device)
    return report(o != w, o, w, bn, what)


def mismatch_bound(out: torch.Tensor, want: torch.Tensor, bound: torch.Tensor, bn: int = 256,
                   what: str = "gemm") -> Optional[str]:
    """|out - want| <= bound per element (NaN fails)."""
    assert out.shape == want.shape, (out.shape, want.shape)
    o, w = out.double(), want.double().to(out.device)
    bad = ~((o - w).abs() <= bound.to(out.device))
    return report(bad, o, w, bn, what)


def random_bound(a: torch.Tensor, b: torch.Tensor, ref: torch.Tensor, out_f32: bool = False) -> torch.Tensor:
    """Per-element bound of a bf16 GEMM on arbitrary operands: fp32 accumulation of K products in any order
    (K * 2^-23 * sum_k |a_k b_k|, twice the sequential round-to-nearest bound), plus half a bf16 ulp of the output."""
    K = a.shape[1]
    absacc = a.double().abs() @ b.double().abs().t()
    acc_err = K * 2.0 ** -23 * absacc + 2.0 ** -23 * ref.double().abs()
    if out_f32:
        return acc_err
    return acc_err + 0.5 * ulp_bf16(ref.double().abs() + acc_err)


def mismatch_random(out: torch.Tensor, a: torch.Tensor, b: torch.Tensor, bn: int = 256, out_f32: bool = False,
                    what: str = "gemm") -> Optional[str]:
    ref = a.double() @ b.double().t()
    return mismatch_bound(out, ref, random_bound(a, b, ref, out_f32), bn, what)


def mismatch_gelu(out: torch.Tensor, v: torch.Tensor, bn: int = 256, what: str = "gelu") -> Optional[str]:
    """out against the exact-erf GELU of the fp32 pre-activation v (= acc + bias)."""
    g = gelu_exact(v)
    bound = ulp_bf16(g) + 1.5e-7 * v.double().abs()
    return mismatch_bound(out, g, bound, bn, what)


# ----------------------------------------------------------------------------------------------------- schedules
def streamk_contributors(plan: dict, K: int) -> list:
    """Per stream-K unit: the CTA groups whose K range starts strictly inside it (the owner's contributors), as the
    kernel's WorkIter::n_contrib counts them."""
    num_kb = (K + BK - 1) // BK
    total = plan["sk_units"] * num_kb
    starts = [total * g // plan["sk_groups"] for g in range(plan["sk_groups"])]
    return [sum(1 for s in starts if u * num_kb < s < (u + 1) * num_kb) for u in range(plan["sk_units"])]


def schedule_kind(plan: dict, K: int) -> str:
    """plain64 / plain128 / plain256 / splitk / streamk1 (one contributor per split tile) / streamk2 (two or more)."""
    if plan["splits"] > 1:
        return "splitk"
    if plan["sk_units"] > 0:
        most = max(streamk_contributors(plan, K))
        return "streamk1" if most == 1 else ("streamk2" if most >= 2 else "streamk0")
    return f"plain{plan['bn']}"
