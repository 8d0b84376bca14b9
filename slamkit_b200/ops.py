"""Thin torch-tensor wrappers over the op-level C ABI (one function per entry point of include/slamkit_b200.h).

These exist for tests, for host-side composition of the HuBERT path and for users who want a single kernel; the
train step itself is driven through the handle API (slamkit_b200.lm.B200UnitLM).  Every function launches the
hand-written CUDA kernel on the current torch stream -- there is no torch fallback.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional, Tuple

import torch

from . import _lib as L


def _bf16(t: torch.Tensor) -> torch.Tensor:
    assert t.is_cuda and t.dtype == torch.bfloat16, "expected a CUDA bf16 tensor"
    return t


_gemm_ws = {}


def gemm_workspace(device) -> torch.Tensor:
    """Per-device GEMM scratch (stream-K partial tiles + flag words; zeroed once, re-armed by the kernel)."""
    lib = L.require_cuda()
    key = torch.device(device).index or 0
    if key not in _gemm_ws:
        _gemm_ws[key] = torch.zeros(int(lib.sk_gemm_ws_bytes()) + (64 << 20), dtype=torch.uint8, device=device)
    return _gemm_ws[key]


def _gemm_args(a, b, a_mn, b_mn, bias, residual, out, out_f32, round_before_res, act, force_bn):
    """Leading arguments of sk_gemm_bf16 / sk_gemm_bf16_ws / sk_gemm_plan (M .. force_bn); out may be None (plan only)."""
    _bf16(a), _bf16(b)
    assert a.dim() == 2 and b.dim() == 2 and a.stride(1) == 1 and b.stride(1) == 1
    M, K = (a.shape[1], a.shape[0]) if a_mn else (a.shape[0], a.shape[1])
    N, Kb = (b.shape[1], b.shape[0]) if b_mn else (b.shape[0], b.shape[1])
    assert K == Kb, f"contraction mismatch {K} vs {Kb}"
    assert out is None or out.stride(1) == 1
    return (M, N, K, L.ptr(a), a.stride(0), int(a_mn), L.ptr(b), b.stride(0), int(b_mn), L.ptr(out),
            out.stride(0) if out is not None else N, int(out_f32), L.ptr(bias), L.ptr(residual),
            residual.stride(0) if residual is not None else 0, int(round_before_res), act, force_bn)


def gemm(a: torch.Tensor, b: torch.Tensor, *, a_mn: bool = False, b_mn: bool = False,
         bias: Optional[torch.Tensor] = None, residual: Optional[torch.Tensor] = None,
         out: Optional[torch.Tensor] = None, out_f32: bool = False, round_before_res: bool = False,
         act: int = 0, force_bn: int = 0, streamk: bool = False) -> torch.Tensor:
    """C = A @ B^T (+bias) (+residual).  a: [M,K] (or [K,M] if a_mn); b: [N,K] (or [K,N] if b_mn).
    streamk=True hands the kernel the per-device scratch (sk_gemm_bf16_ws: split-K for few tiles and a long K loop,
    stream-K balancing for a partial last wave)."""
    lib = L.require_cuda()
    if out is None:
        M = a.shape[1] if a_mn else a.shape[0]
        N = b.shape[1] if b_mn else b.shape[0]
        out = torch.empty((M, N), device=a.device, dtype=torch.float32 if out_f32 else torch.bfloat16)
    M, N, K, pa, lda, am, pb, ldb, bm, pc, ldc, f32, pbias, pres, ldr, rbr, act, fbn = _gemm_args(
        a, b, a_mn, b_mn, bias, residual, out, out_f32, round_before_res, act, force_bn)
    if streamk:
        ws = gemm_workspace(a.device)
        L.check(lib.sk_gemm_bf16_ws(M, N, K, pa, lda, am, pb, ldb, bm, pc, ldc, f32, pbias, pres, ldr, rbr, act, fbn,
                                    L.ptr(ws), C.c_int64(ws.numel()), L.stream_ptr()))
        return out
    L.check(lib.sk_gemm_bf16(M, N, K, pa, lda, am, pb, ldb, bm, pc, ldc, f32, pbias, pres, ldr, rbr, act, fbn,
                             L.stream_ptr()))
    return out


def gemm_plan(a: torch.Tensor, b: torch.Tensor, *, a_mn: bool = False, b_mn: bool = False,
              bias: Optional[torch.Tensor] = None, residual: Optional[torch.Tensor] = None,
              out: Optional[torch.Tensor] = None, out_f32: bool = False, round_before_res: bool = False,
              act: int = 0, force_bn: int = 0, streamk: bool = False) -> dict:
    """The schedule gemm() runs for the same arguments (sk_gemm_plan): bn, epi_warps, splits, sk_units, sk_groups,
    sk_G, sk_colunits, tma_store, grid.  Nothing is launched.  Pass `out` when it matters (residual is out, pitch)."""
    lib = L.require_cuda()
    M, N, K, pa, lda, am, pb, ldb, bm, pc, ldc, f32, pbias, pres, ldr, rbr, act, fbn = _gemm_args(
        a, b, a_mn, b_mn, bias, residual, out, out_f32, round_before_res, act, force_bn)
    ws = gemm_workspace(a.device) if streamk else None
    plan = L.SkGemmPlan()
    L.check(lib.sk_gemm_plan(M, N, K, pa, lda, am, pb, ldb, bm, pc, ldc, f32, pbias, pres, ldr, rbr, act, fbn, L.ptr(ws),
                             C.c_int64(ws.numel() if ws is not None else 0), C.byref(plan)))
    return {name: int(getattr(plan, name)) for name, _ in L.SkGemmPlan._fields_}


def gemm_splitk(a: torch.Tensor, b: torch.Tensor, out: torch.Tensor, *, a_mn: bool, b_mn: bool, accumulate: bool,
                ws_bytes: int = 64 << 20) -> torch.Tensor:
    """Weight-gradient style GEMM with deterministic split-K (sk_gemm_bf16_splitk)."""
    lib = L.require_cuda()
    M, K = (a.shape[1], a.shape[0]) if a_mn else (a.shape[0], a.shape[1])
    N = b.shape[1] if b_mn else b.shape[0]
    ws = torch.zeros(ws_bytes, dtype=torch.uint8, device=a.device)
    L.check(lib.sk_gemm_bf16_splitk(M, N, K, L.ptr(a), a.stride(0), int(a_mn), L.ptr(b), b.stride(0), int(b_mn), L.ptr(out),
                                    out.stride(0), int(accumulate), L.ptr(ws), C.c_int64(ws_bytes), L.stream_ptr()))
    return out


def embed_fwd(ids: torch.Tensor, table: torch.Tensor, vocab: int) -> torch.Tensor:
    lib = L.require_cuda()
    M, D = ids.numel(), table.shape[1]
    out = torch.empty((M, D), device=table.device, dtype=torch.bfloat16)
    L.check(lib.sk_embed_fwd(L.ptr(ids), L.ptr(table), L.ptr(out), M, D, vocab, L.stream_ptr()))
    return out


def embed_bwd(ids: torch.Tensor, dx: torch.Tensor, dtable: torch.Tensor, vocab: int, accumulate: bool) -> None:
    lib = L.require_cuda()
    M, D = dx.shape
    scratch = torch.empty((dtable.shape[0], D), device=dx.device, dtype=torch.int64)   # 64-bit fixed-point accumulators
    L.check(lib.sk_embed_bwd(L.ptr(ids), L.ptr(dx), L.ptr(scratch), L.ptr(dtable), M, D, vocab, dtable.shape[0],
                             int(accumulate), L.stream_ptr()))


def rmsnorm_fwd(x: torch.Tensor, w: torch.Tensor, eps: float) -> Tuple[torch.Tensor, torch.Tensor]:
    lib = L.require_cuda()
    M, D = x.shape
    y = torch.empty_like(x)
    rstd = torch.empty((M,), device=x.device, dtype=torch.float32)
    L.check(lib.sk_rmsnorm_fwd(L.ptr(x), L.ptr(w), L.ptr(y), L.ptr(rstd), M, D, L.f32(eps), L.stream_ptr()))
    return y, rstd


def rmsnorm_bwd(dy, x, w, rstd, dres: Optional[torch.Tensor], dw: torch.Tensor, accumulate_dw: bool) -> torch.Tensor:
    lib = L.require_cuda()
    M, D = x.shape
    dx = torch.empty_like(x)
    partial = torch.empty((lib.sk_rmsnorm_bwd_blocks() * D,), device=x.device, dtype=torch.float32)
    L.check(lib.sk_rmsnorm_bwd(L.ptr(dy), L.ptr(x), L.ptr(w), L.ptr(rstd), L.ptr(dres), L.ptr(dx), L.ptr(dw),
                               L.ptr(partial), M, D, int(accumulate_dw), L.stream_ptr()))
    return dx


def layernorm_fwd(x: torch.Tensor, w: torch.Tensor, b: torch.Tensor, eps: float):
    """-> (y bf16 [M, D], mean fp32 [M], rstd fp32 [M])"""
    lib = L.load()
    M, D = x.shape
    y = torch.empty_like(x)
    mean = torch.empty(M, device=x.device, dtype=torch.float32)
    rstd = torch.empty(M, device=x.device, dtype=torch.float32)
    L.check(lib.sk_layernorm_fwd(L.ptr(x), L.ptr(w), L.ptr(b), L.ptr(y), L.ptr(mean), L.ptr(rstd), M, D, L.f32(eps),
                                 L.stream_ptr()))
    return y, mean, rstd


def layernorm_bwd(dy, x, w, mean, rstd, dres: Optional[torch.Tensor], dw: torch.Tensor, db: torch.Tensor,
                  accumulate: bool) -> torch.Tensor:
    """-> dx; dw / db written (or added to)"""
    lib = L.load()
    M, D = x.shape
    dx = torch.empty_like(x)
    n = lib.sk_layernorm_bwd_blocks() * D
    pw = torch.empty(n, device=x.device, dtype=torch.float32)
    pb = torch.empty(n, device=x.device, dtype=torch.float32)
    L.check(lib.sk_layernorm_bwd(L.ptr(dy), L.ptr(x), L.ptr(w), L.ptr(mean), L.ptr(rstd), L.ptr(dres), L.ptr(dx), L.ptr(dw),
                                 L.ptr(db), L.ptr(pw), L.ptr(pb), M, D, int(accumulate), L.stream_ptr()))
    return dx


def colsum(x: torch.Tensor, out: torch.Tensor, accumulate: bool) -> torch.Tensor:
    lib = L.require_cuda()
    M, N = x.shape
    partial = torch.empty((lib.sk_colsum_splits() * N,), device=x.device, dtype=torch.float32)
    L.check(lib.sk_colsum(L.ptr(x), L.ptr(out), L.ptr(partial), M, N, x.stride(0), int(accumulate), L.stream_ptr()))
    return out


def rope_(qkv: torch.Tensor, cos: torch.Tensor, sin: torch.Tensor, T: int, n_rot_heads: int, head_dim: int,
          inverse: bool = False, pos_ids: Optional[torch.Tensor] = None) -> torch.Tensor:
    lib = L.require_cuda()
    M = qkv.shape[0]
    L.check(lib.sk_rope(L.ptr(qkv), L.ptr(cos), L.ptr(sin), L.ptr(pos_ids), M, T, qkv.stride(0), n_rot_heads, head_dim,
                        int(inverse), cos.shape[0], L.stream_ptr()))
    return qkv


def block_gate_up(w_gate: torch.Tensor, w_up: torch.Tensor) -> torch.Tensor:
    """[F, K] gate / up weights (or [M, F] activations, transposed use) -> the [2F, K] 128-row block layout of the fused
    SwiGLU linears: rows [256b, 256b+128) = gate rows [128b, 128b+128), rows [256b+128, 256b+256) = up rows."""
    F = w_gate.shape[0]
    assert F % 128 == 0 and w_up.shape == w_gate.shape
    g = w_gate.view(F // 128, 128, -1)
    u = w_up.view(F // 128, 128, -1)
    return torch.stack([g, u], dim=1).reshape(2 * F, -1).contiguous()


def linear_swiglu_fwd(x: torch.Tensor, w_gu_blocked: torch.Tensor):
    """-> (gu [M, 2F] in block layout, act [M, F])"""
    lib = L.require_cuda()
    M, K = x.shape
    F = w_gu_blocked.shape[0] // 2
    gu = torch.empty((M, 2 * F), device=x.device, dtype=torch.bfloat16)
    act = torch.empty((M, F), device=x.device, dtype=torch.bfloat16)
    L.check(lib.sk_linear_swiglu_fwd(M, F, K, L.ptr(x), L.ptr(w_gu_blocked), L.ptr(gu), L.ptr(act), L.stream_ptr()))
    return gu, act


def linear_swiglu_bwd(dy: torch.Tensor, w_down: torch.Tensor, gu_blocked: torch.Tensor) -> torch.Tensor:
    """dy [M, N], w_down [N, F], gu [M, 2F] (block layout) -> d_gu [M, 2F] (block layout)"""
    lib = L.require_cuda()
    M, N = dy.shape
    F = w_down.shape[1]
    dgu = torch.empty((M, 2 * F), device=dy.device, dtype=torch.bfloat16)
    L.check(lib.sk_linear_swiglu_bwd(M, N, F, L.ptr(dy), L.ptr(w_down), L.ptr(gu_blocked), L.ptr(dgu), L.stream_ptr()))
    return dgu


def linear_rope(x: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor], cos: torch.Tensor, sin: torch.Tensor, T: int,
                rope_cols: int, pos_ids: Optional[torch.Tensor] = None) -> torch.Tensor:
    lib = L.require_cuda()
    M, K = x.shape
    N = w.shape[0]
    out = torch.empty((M, N), device=x.device, dtype=torch.bfloat16)
    L.check(lib.sk_linear_rope(M, N, K, L.ptr(x), L.ptr(w), L.ptr(bias), L.ptr(out), L.ptr(cos), L.ptr(sin), L.ptr(pos_ids),
                               T, rope_cols, cos.shape[0], L.stream_ptr()))
    return out


def swiglu_fwd(gu: torch.Tensor) -> torch.Tensor:
    lib = L.require_cuda()
    M, F2 = gu.shape
    act = torch.empty((M, F2 // 2), device=gu.device, dtype=torch.bfloat16)
    L.check(lib.sk_swiglu_fwd(L.ptr(gu), L.ptr(act), M, F2 // 2, L.stream_ptr()))
    return act


def swiglu_bwd(gu: torch.Tensor, dact: torch.Tensor) -> torch.Tensor:
    lib = L.require_cuda()
    M, F2 = gu.shape
    dgu = torch.empty_like(gu)
    L.check(lib.sk_swiglu_bwd(L.ptr(gu), L.ptr(dact), L.ptr(dgu), M, F2 // 2, L.stream_ptr()))
    return dgu


def ce_fwd_bwd(logits: torch.Tensor, labels: torch.Tensor, T: int, vocab: int, num_items: float, dloss: float = 1.0,
               want_grad: bool = True):
    """Returns (stats[3] = loss, n_valid, nll_sum ; dlogits or None ; row_nll)."""
    lib = L.require_cuda()
    M, ldl = logits.shape
    dlogits = torch.empty_like(logits) if want_grad else None
    partial = torch.empty((2 * lib.sk_ce_blocks(M),), device=logits.device, dtype=torch.float32)
    row_nll = torch.empty((M,), device=logits.device, dtype=torch.float32)
    stats = torch.empty((3,), device=logits.device, dtype=torch.float32)
    L.check(lib.sk_ce_fwd_bwd(L.ptr(logits), L.ptr(labels), L.ptr(dlogits), L.ptr(partial), L.ptr(row_nll),
                              L.ptr(stats), M, T, vocab, ldl, L.f32(num_items), L.f32(dloss), L.stream_ptr()))
    return stats, dlogits, row_nll


def attn_fwd(qkv: torch.Tensor, B: int, T: int, H: int, KVH: int, causal: bool, scale: float):
    """qkv: [B*T, (H+2*KVH)*64] fused projection output. Returns (o [B*T, H*64], lse [B,H,T])."""
    lib = L.require_cuda()
    hd = 64
    o = torch.empty((B * T, H * hd), device=qkv.device, dtype=torch.bfloat16)
    lse = torch.empty((B, H, T), device=qkv.device, dtype=torch.float32)
    q, k, v = qkv, qkv[:, H * hd:], qkv[:, (H + KVH) * hd:]
    L.check(lib.sk_attn_fwd(L.ptr(q), L.ptr(k), L.ptr(v), L.ptr(o), L.ptr(lse), B, T, H, KVH, qkv.stride(0), o.stride(0),
                            int(causal), L.f32(scale), L.stream_ptr()))
    return o, lse


def seg_bounds(pos_ids: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """Document bounds of a packed batch from position_ids [B, T] (sk_seg_bounds): (seg_start, seg_end) int32 [B*T]."""
    lib = L.require_cuda()
    B, T = pos_ids.shape
    pos = pos_ids.to(torch.int32).contiguous()
    ss = torch.empty(B * T, device=pos.device, dtype=torch.int32)
    se = torch.empty(B * T, device=pos.device, dtype=torch.int32)
    L.check(lib.sk_seg_bounds(L.ptr(pos), L.ptr(ss), L.ptr(se), B, T, L.stream_ptr()))
    return ss, se


def attn_tc_fwd(qkv: torch.Tensor, B: int, T: int, H: int, KVH: int, causal: bool, scale: float,
                seg_start: Optional[torch.Tensor] = None):
    """Flash-attention forward on the fused projection (sk_attn_tc_fwd); same contract as attn_fwd.  seg_start (from seg_bounds) makes
    it block-diagonal causal for packed batches."""
    lib = L.require_cuda()
    o = torch.empty((B * T, H * 64), device=qkv.device, dtype=torch.bfloat16)
    lse = torch.empty((B, H, T), device=qkv.device, dtype=torch.float32)
    L.check(lib.sk_attn_tc_fwd(L.ptr(qkv), L.ptr(o), L.ptr(lse), B, T, H, KVH, qkv.stride(0), o.stride(0), int(causal),
                               L.f32(scale), L.ptr(seg_start), L.stream_ptr()))
    return o, lse


def attn_tc_bwd(qkv, o, d_o, lse, B, T, H, KVH, causal: bool, scale: float, seg_start: Optional[torch.Tensor] = None,
                seg_end: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Flash-attention backward on the fused projection (sk_attn_tc_bwd); same contract as attn_bwd."""
    lib = L.require_cuda()
    dqkv = torch.empty_like(qkv)
    delta = torch.empty_like(lse)
    L.check(lib.sk_attn_tc_bwd(L.ptr(qkv), L.ptr(o), L.ptr(d_o), L.ptr(lse), L.ptr(delta), L.ptr(None), L.ptr(dqkv),
                               B, T, H, KVH, qkv.stride(0), o.stride(0), dqkv.stride(0), int(causal), L.f32(scale),
                               L.ptr(seg_start), L.ptr(seg_end), L.stream_ptr()))
    return dqkv


def attn_tc_fwd_split(qkv_hi: torch.Tensor, qkv_lo: torch.Tensor, B: int, T: int, H: int, scale: float):
    """Split-bf16 bidirectional forward of the HuBERT encoder (sk_attn_tc_fwd_split).  qkv_hi / qkv_lo: [B*T, 3*H*64]
    (H q-, k- and v-heads) with the same row pitch.  Returns (o_hi, o_lo) [B*T, H*64]."""
    lib = L.require_cuda()
    assert qkv_hi.stride(0) == qkv_lo.stride(0)
    o_hi = torch.empty((B * T, H * 64), device=qkv_hi.device, dtype=torch.bfloat16)
    o_lo = torch.empty_like(o_hi)
    L.check(lib.sk_attn_tc_fwd_split(L.ptr(qkv_hi), L.ptr(qkv_lo), L.ptr(o_hi), L.ptr(o_lo), B, T, H, qkv_hi.stride(0),
                                     o_hi.stride(0), L.f32(scale), L.stream_ptr()))
    return o_hi, o_lo


def attn_bwd(qkv, o, d_o, lse, B, T, H, KVH, causal: bool, scale: float) -> torch.Tensor:
    lib = L.require_cuda()
    hd = 64
    dqkv = torch.empty_like(qkv)
    delta = torch.empty_like(lse)
    q, k, v = qkv, qkv[:, H * hd:], qkv[:, (H + KVH) * hd:]
    dq, dk, dv = dqkv, dqkv[:, H * hd:], dqkv[:, (H + KVH) * hd:]
    L.check(lib.sk_attn_bwd(L.ptr(q), L.ptr(k), L.ptr(v), L.ptr(o), L.ptr(d_o), L.ptr(lse), L.ptr(delta), L.ptr(dq),
                            L.ptr(dk), L.ptr(dv), B, T, H, KVH, qkv.stride(0), o.stride(0), dqkv.stride(0), int(causal),
                            L.f32(scale), L.stream_ptr()))
    return dqkv


def adamw_step(p, g, m, v, lr, beta1, beta2, eps, wd, step, clip_stats: Optional[torch.Tensor] = None) -> None:
    lib = L.require_cuda()
    L.check(lib.sk_adamw_step(L.ptr(p), L.ptr(g), L.ptr(m), L.ptr(v), C.c_int64(p.numel()), L.f32(lr), L.f32(beta1),
                              L.f32(beta2), L.f32(eps), L.f32(wd), int(step), L.ptr(clip_stats), L.stream_ptr()))
