"""References and per-element checkers for the Qwen2 layer's own kernels: RMSNorm forward and backward, RoPE forward and
inverse (full and partial rotary), and SwiGLU forward and backward, standalone or fused into the GEMM epilogues.

Each reference is HF's formula (Qwen2RMSNorm, apply_rotary_pos_emb, Qwen2MLP with torch's SiLU) with the rounding points
the kernels declare:
  - RMSNorm   y = bf16(w * bf16(x * rstd)),  rstd = rsqrt(mean(x^2) + eps);
  - RoPE      out = bf16(bf16(q * cos) + bf16(rotate_half(q) * sin)), and its autograd for the inverse;
  - SwiGLU    act = bf16(bf16(silu(g)) * u),  d_gate = bf16(bf16(d_act * u) * silu'(g)),  d_up = bf16(d_act * bf16(silu(g))).
RoPE is exact: it is restated with torch bf16 operations.  RMSNorm's fp32 reduction and rsqrtf, and SwiGLU's
ex2.approx / rcp.approx, cannot be bit-exact, so those references are float64 with a bound derived from the kernel's
arithmetic (docstrings below).  Every bound holds whether or not nvcc contracts a*b + c into an FMA.  Where an
intermediate is rounded to bf16 before it is multiplied, the checker takes the (one or two) bf16 roundings of the
bounded interval as candidates and applies the rest of the formula to each: the products of two bf16 values are exact
in fp32, so the result stays nearly bit-exact.

Checkers return a list of located failures (empty when the output conforms), as tests/grad_ref.py does.
"""
from __future__ import annotations

import math
from typing import List, Optional

import numpy as np
import torch

from grad_ref import U, bf16, bf16_from64, check_bf16_interval, check_exact, colsum_ref, locate

F32_MAX = float(np.finfo(np.float32).max)
TINY = 2.0 ** -149                # smallest fp32 subnormal


def _f32(x) -> np.ndarray:
    """float64 -> float32 with one rounding (subnormals kept, overflow to inf)."""
    with np.errstate(over="ignore"):
        return np.asarray(x, dtype=np.float64).astype(np.float32)


def _bf16_of_f32_product(a, b) -> np.ndarray:
    """bf16(fp32(a * b)): the kernels' product of two fp32 values, rounded to fp32 and then to bf16."""
    with np.errstate(all="ignore"):
        return bf16(_f32(np.asarray(a, np.float64) * np.asarray(b, np.float64)))


def _between(got, a, b, what: str, want=None) -> List[str]:
    """got must lie in [min(a, b), max(a, b)] elementwise; NaN in a or b requires NaN in got."""
    g = np.asarray(got, np.float32)
    lo, hi = np.minimum(a, b), np.maximum(a, b)
    nan = np.isnan(a) | np.isnan(b)
    with np.errstate(invalid="ignore"):
        ok = np.where(nan, np.isnan(g), (g >= lo) & (g <= hi))
    return locate(~ok, g, want if want is not None else a, what)


# ----------------------------------------------------------------------------------------------------- RMSNorm
def rstd_bound(D: int) -> float:
    """Relative bound on the kernel's fp32 rstd against the float64 one.

    The sum of squares adds positive, exactly representable terms (a bf16 square has 16 significant bits): each lane
    adds at most 8 * ceil(D / 256) of them one after another (two per step when contracted), then a 5-level butterfly,
    so the sum is within (n + 5) u of the exact one (n additions on the longest path, positive terms).  The division by
    D and the add of eps round once each (eps > 0 only shrinks the relative error).  rstd = (ms + eps)^-1/2 halves the
    relative error of its argument, and rsqrtf adds its 2 ulp (4 u)."""
    n = 8 * math.ceil(D / 256)
    return ((n + 5 + 2) / 2 + 4) * U * 1.001


def rmsnorm_fwd_ref(x, w, eps: float):
    """-> (candidate outputs ylo, yhi, float64 rstd [M], relative bound).  Each output is bf16(w * c) for c one of the
    bf16 roundings of x * rstd * (1 +- (eps_rel + u)) (the fp32 product x * rstd adds u); w * c is exact in fp32."""
    x64 = np.asarray(x, np.float64)
    D = x64.shape[1]
    rstd = 1.0 / np.sqrt((x64 * x64).sum(axis=1) / D + float(np.float32(eps)))
    e = rstd_bound(D)
    t = x64 * rstd[:, None]
    lo, hi = t * (1 - e - U), t * (1 + e + U)
    clo, chi = bf16_from64(np.minimum(lo, hi)), bf16_from64(np.maximum(lo, hi))
    w32 = np.asarray(w, np.float32)[None, :]
    return bf16(clo * w32), bf16(chi * w32), rstd, e


def check_rmsnorm_fwd(y, rstd_out, x, w, eps: float) -> List[str]:
    ylo, yhi, rstd, e = rmsnorm_fwd_ref(x, w, eps)
    out = _between(y, ylo, yhi, "rmsnorm y", ylo)
    if rstd_out is not None:
        r = np.asarray(rstd_out, np.float64)
        out += locate(~(np.abs(r - rstd) <= e * rstd), r, rstd, "rmsnorm rstd")
    return out


def rmsnorm_two_candidates(x, w, eps: float) -> int:
    """How many outputs have two candidates (x * rstd within the bound of a bf16 rounding boundary)."""
    ylo, yhi, _, _ = rmsnorm_fwd_ref(x, w, eps)
    return int((ylo != yhi).sum())


def rmsnorm_bwd_ref(dy, x, w, rstd, dres=None):
    """float64 backward of y = w * bf16(x * rstd) from the given rstd, as autograd runs it on HF's bf16 module:
    g = bf16(dy * w) (bf16 multiply), dx = rstd g - rstd^2 x mean(g * xhat) (+ dres), one rounding to bf16;
    dw = sum over rows of dy * bf16(fp32(x * rstd)).  Returns (dx64, dw64, g, xhat)."""
    dy, x, w = (np.asarray(a, np.float32) for a in (dy, x, w))
    r32 = np.asarray(rstd, np.float32)[:, None]
    g = bf16(dy * w[None, :]).astype(np.float64)
    r = r32.astype(np.float64)
    xhat = x.astype(np.float64) * r
    D = x.shape[1]
    dot = (g * xhat).sum(axis=1, keepdims=True) / D
    dx = r * g - r * r * x * dot
    # (+ dres): the kernel adds +0 without one, so a zero dx is +0
    dx = dx + (np.asarray(dres, np.float64) if dres is not None else 0.0)
    xb = bf16((x * r32).astype(np.float32)).astype(np.float64)
    dw = (dy.astype(np.float64) * xb).sum(axis=0)
    return dx, dw, g, xhat


def rmsnorm_dx_bound(dy, x, w, rstd, dres=None) -> np.ndarray:
    """Bound on the fp32 dx before its bf16 rounding.  xhat = x * rstd rounds once; the dot product sums
    n = 8 * ceil(D / 256) fma terms per lane and 5 butterfly levels ((n + 6) u of sum |g xhat|, counting the rounding of
    xhat); / D, rstd * rstd and the product with dot round once each; rstd * g, the fma and the add of dres once each."""
    dx, _, g, xhat = rmsnorm_bwd_ref(dy, x, w, rstd, dres)
    D = np.asarray(x).shape[1]
    n = 8 * math.ceil(D / 256)
    r = np.asarray(rstd, np.float64)[:, None]
    s = (np.abs(g) * np.abs(xhat)).sum(axis=1, keepdims=True) / D
    c2x = r * r * np.abs(np.asarray(x, np.float64)) * s
    rg = r * np.abs(g)
    dr = np.abs(np.asarray(dres, np.float64)) if dres is not None else 0.0
    return ((n + 6 + 3) * c2x + 2 * rg + 2 * (rg + c2x + dr)) * U * 1.001


def rmsnorm_dw_bound(dy, x, rstd, blocks: int, old=None) -> np.ndarray:
    """Bound on the fp32 column sums of dy * bf16(xhat): each warp adds its rows (ceil(M / (8 blocks)) fma steps), the
    block adds its 8 warps, and the reduction adds the blocks (ceil(blocks / 32) per thread, then a 5-level tree), each
    step rounding once; (+ old) one more rounding."""
    M = np.asarray(x).shape[0]
    xb = bf16((np.asarray(x, np.float32) * np.asarray(rstd, np.float32)[:, None]).astype(np.float32))
    a = (np.abs(np.asarray(dy, np.float64)) * np.abs(xb.astype(np.float64))).sum(axis=0)
    depth = math.ceil(M / (8 * blocks)) + 8 + math.ceil(blocks / 32) + 5 + 1
    extra = np.abs(np.asarray(old, np.float64)) if old is not None else 0.0
    return depth * U * (a + extra) * 1.001


def check_rmsnorm_bwd(dx, dw, dy, x, w, rstd, dres=None, dw_old=None, blocks: int = 528) -> List[str]:
    """dx per element within rmsnorm_dx_bound, dw within rmsnorm_dw_bound (+ dw_old when accumulating)."""
    ref, dw64, _, _ = rmsnorm_bwd_ref(dy, x, w, rstd, dres)
    out = check_bf16_interval(dx, ref, rmsnorm_dx_bound(dy, x, w, rstd, dres), "rmsnorm dx")
    if dw_old is not None:
        dw64 = dw64 + np.asarray(dw_old, np.float64)
    out += check_bf16_interval(dw, dw64, rmsnorm_dw_bound(dy, x, rstd, blocks, dw_old), "rmsnorm dw")
    return out


def rmsnorm_bwd_exact(dy, x, w, rstd, dres=None, dw_old=None):
    """Bit-exact (dx, dw) when every intermediate is exact: rstd a power of two, dy, x, w, dres on integer grids small
    enough that every fp32 product and sum is exact, and each row's sum of g * x a multiple of D (or D a power of two),
    so that the kernel's / D does not round.  Then dx is the bf16 rounding of the exact value and dw the bf16 column
    sum (grad_ref.colsum_ref)."""
    dx, _, g, _ = rmsnorm_bwd_ref(dy, x, w, rstd, dres)
    xb = bf16((np.asarray(x, np.float32) * np.asarray(rstd, np.float32)[:, None]).astype(np.float32))
    return bf16_from64(dx), colsum_ref(np.asarray(dy, np.float64) * xb, dw_old)


def exact_rmsnorm_bwd_operands(M: int, D: int, seed: int, k: int = 2):
    """Operands for rmsnorm_bwd_exact: x in [-16, 16], dy and w in [-8, 8] (|g| <= 64), rstd = 2^-k, dres on the
    2^-3k grid, and the first columns (w = 1 there) adjusted per row so that sum_i g_i x_i is a multiple of D."""
    r = np.random.default_rng(seed)
    x = r.integers(-16, 17, size=(M, D)).astype(np.float32)
    dy = r.integers(-8, 9, size=(M, D)).astype(np.float32)
    w = r.integers(-8, 9, size=D).astype(np.float32)
    J = min(D, math.ceil(D / 32) + 1)          # |target| <= D / 2 spread over J columns of |x| <= 16
    w[:J] = 1.0
    dy[:, :J] = 1.0
    g = dy * w[None, :]
    rest = (g[:, J:] * x[:, J:]).sum(axis=1).astype(np.int64)
    for m in range(M):
        t = int((-rest[m]) % D)
        if t > D // 2:
            t -= D
        q, rem = divmod(abs(t), J)
        col = np.full(J, q) + (np.arange(J) < rem)
        x[m, :J] = np.sign(t) * col
    assert np.abs(x).max() <= 16 and (((g * x).sum(axis=1)) % D == 0).all()
    rstd = np.full(M, 2.0 ** -k, np.float32)
    dres = (r.integers(-64, 65, size=(M, D)) * 2.0 ** (-3 * k)).astype(np.float32)
    return dy, x, w, rstd, dres


# ----------------------------------------------------------------------------------------------------- RoPE
def rope_positions(M: int, T: int, max_pos: int, pos_ids=None) -> torch.Tensor:
    """The table row each token reads: pos_ids (or m % T when None), clamped to [0, max_pos - 1]."""
    pos = torch.as_tensor(np.asarray(pos_ids)).long().reshape(-1) if pos_ids is not None else torch.arange(M) % T
    return pos.clamp(0, max_pos - 1)


def _rope_parts(qkv: torch.Tensor, n_rot_heads: int, head_dim: int, rot: int):
    M = qkv.shape[0]
    h = qkv[:, :n_rot_heads * head_dim].reshape(M, n_rot_heads, head_dim)
    return h[..., :rot], h[..., rot:]


def rope_ref(qkv, cos, sin, pos: torch.Tensor, n_rot_heads: int, head_dim: int, rot: Optional[int] = None,
             inverse: bool = False) -> torch.Tensor:
    """HF apply_rotary_pos_emb on bf16 tensors (CPU): q_rot * cos + rotate_half(q_rot) * sin on the first `rot`
    columns of each of the first n_rot_heads heads (cos / sin tables [max_pos, rot / 2], both halves of a row the same,
    as HF's cat(freqs, freqs)); every other column is returned as it is.  inverse: the autograd of that forward for an
    incoming gradient q, dq1 = bf16(bf16(g1 c) + bf16(g2 s)), dq2 = bf16(bf16(g2 c) - bf16(g1 s))."""
    rot = rot or head_dim
    qkv = torch.as_tensor(qkv).to(torch.bfloat16)
    c = cos.to(torch.bfloat16)[pos][:, None, :]                  # [M, 1, rot / 2]
    s = sin.to(torch.bfloat16)[pos][:, None, :]
    q, _ = _rope_parts(qkv, n_rot_heads, head_dim, rot)
    h = rot // 2
    x1, x2 = q[..., :h], q[..., h:]
    if not inverse:
        o1 = x1 * c + (-x2) * s
        o2 = x2 * c + x1 * s
    else:
        o1 = x1 * c + x2 * s
        o2 = x2 * c - x1 * s
    out = qkv.clone()
    view = out[:, :n_rot_heads * head_dim].view(qkv.shape[0], n_rot_heads, head_dim)
    view[..., :h] = o1
    view[..., h:rot] = o2
    return out


def rope_autograd(qkv, cos, sin, pos: torch.Tensor, n_rot_heads: int, head_dim: int, grad, rot: Optional[int] = None):
    """torch autograd of HF's forward in bf16 (cat(freqs, freqs) tables, rotate_half): the gradient of the rotated
    columns for the incoming gradient `grad` (same layout as qkv)."""
    rot = rot or head_dim
    M = qkv.shape[0]
    q, _ = _rope_parts(torch.as_tensor(qkv).to(torch.bfloat16), n_rot_heads, head_dim, rot)
    q = q.detach().clone().requires_grad_(True)
    c = cos.to(torch.bfloat16)[pos][:, None, :]
    s = sin.to(torch.bfloat16)[pos][:, None, :]
    c, s = torch.cat([c, c], -1), torch.cat([s, s], -1)
    rh = torch.cat([-q[..., rot // 2:], q[..., :rot // 2]], -1)
    out = q * c + rh * s
    g, _ = _rope_parts(torch.as_tensor(grad).to(torch.bfloat16), n_rot_heads, head_dim, rot)
    out.backward(g)
    return q.grad.reshape(M, n_rot_heads, rot)


def check_rope(got, want, what: str = "rope") -> List[str]:
    return check_exact(torch.as_tensor(got).float().numpy(), torch.as_tensor(want).float().numpy(), what)


# ----------------------------------------------------------------------------------------------------- SwiGLU
def sigmoid64(g) -> np.ndarray:
    """torch's sigmoid inside silu (x / (1 + exp(-x)), opmath fp32) evaluated in float64 with fp32's range: exp(-x)
    overflows to inf above 88.72, and values below 2^-149 become 0."""
    x = np.asarray(g, np.float64)
    with np.errstate(over="ignore", invalid="ignore"):
        e = np.exp(-x)
        e = np.where(e > F32_MAX, np.inf, e)
        s = 1.0 / (1.0 + e)
    return np.where(np.abs(s) < TINY / 2, 0.0 * s, s)


def silu64(g) -> np.ndarray:
    x = np.asarray(g, np.float64)
    with np.errstate(over="ignore", invalid="ignore"):
        e = np.exp(-x)
        e = np.where(e > F32_MAX, np.inf, e)
        v = x / (1.0 + e)
    return np.where(np.abs(v) < TINY / 2, 0.0 * v, v)


def dsilu64(g) -> np.ndarray:
    """torch's silu_backward factor s * (1 + x * (1 - s)) in float64 with fp32's range."""
    x = np.asarray(g, np.float64)
    s = sigmoid64(x)
    with np.errstate(over="ignore", invalid="ignore"):
        v = s * (1.0 + x * (1.0 - s))
    return np.where(np.abs(v) < TINY / 2, 0.0 * v, v)


def sigmoid_abs_bound(g) -> np.ndarray:
    """Bound on |sigmoid_f(x) - s| for the kernels' 1 / (1 + ex2.approx(x * -log2 e)) through rcp.approx.

    e = 2^(x * -log2 e): the fp32 constant and the product each carry u relative, 2 u |x| absolute in the exponent and
    hence 2 u |x| relative in e, and ex2.approx adds 2 ulp (4 u); an error of r in e moves s by r (1 - s) relative.
    1 + e rounds with at most min(u, e) relative (the kernel forms (1 + e) 2^-32 in one fma: the same rounding, scaled);
    rcp.approx is within 1 ulp (2 u) and exact at a power of two (for e < 2^-25, 1 + e rounds to 1 and the kernel's
    sigmoid is exactly 1).  The scaling back by 2^-32 is exact, or one rounding of a subnormal sigmoid (2^-149)."""
    x = np.asarray(g, np.float64)
    s = sigmoid64(x)
    with np.errstate(over="ignore", invalid="ignore"):
        one_m = np.where(np.isfinite(x), 1.0 - s, 0.0)
        e = np.where(s > 0, one_m / np.where(s > 0, s, 1.0), np.inf)
        rel = (2 * np.abs(x) + 8) * U * one_m + np.minimum(U, e) + np.where(e >= 2.0 ** -25, 2 * U, 0.0)
    return np.where(np.isfinite(x), s * rel * 1.01 + np.where(s > 0, 2 * TINY, 0.0), 0.0)


def silu_abs_bound(g) -> np.ndarray:
    """x * sigmoid_f(x) rounded once: |x| times the sigmoid bound, u of the product and 2^-149 for a subnormal one."""
    x = np.asarray(g, np.float64)
    with np.errstate(invalid="ignore"):
        b = np.abs(x) * sigmoid_abs_bound(x) + U * np.abs(silu64(x)) + TINY
    return np.where(np.isfinite(x), b, 0.0)


def dsilu_abs_bound(g) -> np.ndarray:
    """s (1 + x (1 - s)) from the kernel's s: an error d in s moves it by d |1 + x (1 - 2 s)|; 1 - s, x (1 - s),
    1 + x (1 - s) and the product round once each (fewer when contracted).  Absolute, so it covers the zero of silu'
    at x = -1.278."""
    x = np.asarray(g, np.float64)
    s = sigmoid64(x)
    with np.errstate(over="ignore", invalid="ignore"):
        t = np.abs(x) * (1.0 - s)
        b = sigmoid_abs_bound(x) * np.abs(1.0 + x * (1.0 - 2.0 * s)) + 4 * U * s * (1.0 + 2.0 * t) + 2 * TINY
    return np.where(np.isfinite(x), b * 1.01, 0.0)


def silu_candidates(g):
    """(lo, hi): the bf16 roundings the kernel's bf16(silu(g)) may take (NaN where torch's silu is NaN)."""
    v = silu64(g)
    b = silu_abs_bound(g)
    with np.errstate(invalid="ignore"):
        lo, hi = bf16_from64(v - b), bf16_from64(v + b)
    inf = np.isinf(v)
    return np.where(inf, v, lo).astype(np.float32), np.where(inf, v, hi).astype(np.float32)


def swiglu_fwd_candidates(g, u):
    """act = bf16(c * u) for c in silu_candidates(g): the interval of its possible values (monotone in c)."""
    clo, chi = silu_candidates(g)
    return _bf16_of_f32_product(clo, u), _bf16_of_f32_product(chi, u)


def check_swiglu_fwd(act, g, u, what: str = "swiglu act") -> List[str]:
    a, b = swiglu_fwd_candidates(g, u)
    return _between(act, a, b, what, a)


def check_swiglu_bwd(d_gate, d_up, g, u, d_act, what: str = "swiglu") -> List[str]:
    """d_up = bf16(d_act * bf16(silu(g))) over the silu candidates; d_gate = bf16(p * silu'(g)) with p = bf16(d_act * u)
    exact, within |p| times dsilu_abs_bound plus the fp32 product's rounding; NaN exactly where torch gives NaN."""
    clo, chi = silu_candidates(g)
    out = _between(d_up, _bf16_of_f32_product(d_act, clo), _bf16_of_f32_product(d_act, chi), what + " d_up")
    p = _bf16_of_f32_product(d_act, u).astype(np.float64)
    ds = dsilu64(g)
    with np.errstate(invalid="ignore", over="ignore"):
        ref = p * ds
        bound = np.abs(p) * dsilu_abs_bound(g) + U * np.abs(ref) + TINY
    dg = np.asarray(d_gate, np.float32)
    nan = np.isnan(ref)
    inf = np.isinf(ref) & ~nan
    fin = ~(nan | inf)
    out += locate(nan & ~np.isnan(dg), dg, ref, what + " d_gate not NaN where torch's is")
    out += locate(inf & (dg != ref), dg, ref, what + " d_gate infinite")
    lo, hi = bf16_from64(np.where(fin, ref - bound, 0.0)), bf16_from64(np.where(fin, ref + bound, 0.0))
    with np.errstate(invalid="ignore"):
        ok = (dg >= lo) & (dg <= hi)
    out += locate(fin & ~ok, dg, ref, what + " d_gate")
    return out


def torch_swiglu(g, u, d_act=None):
    """HF Qwen2MLP on bf16 tensors: (act, d_gate, d_up) from torch's F.silu and its autograd (CPU)."""
    gt = torch.as_tensor(np.asarray(g, np.float32)).to(torch.bfloat16).requires_grad_(True)
    ut = torch.as_tensor(np.asarray(u, np.float32)).to(torch.bfloat16).requires_grad_(True)
    act = torch.nn.functional.silu(gt) * ut
    if d_act is None:
        return act.detach().float().numpy(), None, None
    act.backward(torch.as_tensor(np.asarray(d_act, np.float32)).to(torch.bfloat16))
    return act.detach().float().numpy(), gt.grad.float().numpy(), ut.grad.float().numpy()


def all_bf16() -> np.ndarray:
    """Every bf16 bit pattern (65,536 values, ±0, subnormals, ±inf and NaNs) as float32."""
    return torch.arange(-32768, 32768, dtype=torch.int32).to(torch.int16).view(torch.bfloat16).float().numpy()
