/* slamkit_b200 -- C ABI of the H100-native (sm_90a) hot paths of slp-rl/slamkit.
 *
 * The reference has no native code and no FFI of its own (SURVEY.md §0, §8b): both hot paths enter third-party
 * Python libraries through two plugin ABCs.  This header is therefore the interface a binding for those two plugin
 * points would use; each entry point cites the reference call site it replaces (paths relative to the reference
 * repo; "HF:" = transformers 5.5.0, "SK:" = scikit-learn 1.9.0).
 *
 * Conventions (all entry points):
 *   - plain pointers and sizes only; every pointer is caller-owned DEVICE memory unless the name ends in _host;
 *   - no allocation and no synchronisation inside compute calls: work is enqueued on `stream` (a cudaStream_t passed
 *     as void*) and ordered with the caller's other work on that stream;
 *   - return 0 on success, <0 on error (-1 bad argument, -2 CUDA error); sk_last_error() returns a message;
 *   - bf16 tensors are passed as void* (uint16 storage), row-major, with explicit leading dimensions (in elements);
 *   - handles are re-entrant per handle, not thread-safe across threads sharing one handle.
 */
#ifndef SLAMKIT_B200_H
#define SLAMKIT_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ---- library ------------------------------------------------------------------------------------------------ */
const char* sk_last_error(void);
int sk_version(void);                       /* 100*major + minor */
int sk_device_sm_count(void);               /* multiprocessor count of the current device (132 on H100 SXM) */
int sk_device_cc(void);                     /* 10*major + minor of the current device; kernels require 90 */

/* ---- tensor-core GEMM (wgmma + TMA) ---------------------------------------------------------------------------
 * C[M,N] = A * B^T (+ bias[N]) (+ residual[M,N]); bf16 operands, fp32 accumulation, bf16 (or fp32) output.
 *   a_mn = 0: A is [M,K] row-major (lda = row pitch);  a_mn = 1: A is stored transposed as [K,M] (lda = its pitch).
 *   b_mn = 0: B is [N,K] row-major (a torch Linear weight);  b_mn = 1: B is stored as [K,N].
 *   act: 0 none, 1 GELU(erf), 2 ReLU on (acc+bias).  round_before_res: round (acc+bias) to bf16 before adding the residual
 *   (bit-matches an unfused bf16 linear followed by a bf16 add).  force_bn: 0 auto, else 64/128/192/224/256.
 * Replaces every torch.nn.Linear / F.linear on both hot paths (HF:models/qwen2/modeling_qwen2.py:35-48,187-246;
 * HF:models/hubert/modeling_hubert.py:216-231,262-405) and their autograd dgrad/wgrad GEMMs. */
int sk_gemm_bf16(int M, int N, int K, const void* A, int lda, int a_mn, const void* B, int ldb, int b_mn, void* C,
                 int ldc, int out_f32, const void* bias, const void* residual, int ldr, int round_before_res, int act,
                 int force_bn, void* stream);

/* Same GEMM with a caller-provided fp32 scratch: when the output has few tiles and K is long (weight gradients
 * dW = dY^T X with K = tokens) the K loop is split over idle SMs into fp32 slabs that are reduced in a fixed order
 * (deterministic).  accumulate=1 adds into C (gradient accumulation).  Falls back to the plain kernel when the shape
 * does not benefit or the scratch is too small. */
int sk_gemm_bf16_splitk(int M, int N, int K, const void* A, int lda, int a_mn, const void* B, int ldb, int b_mn, void* C,
                        int ldc, int accumulate, void* splitk_ws, int64_t splitk_ws_bytes, void* stream);

/* General form with a scratch buffer.  With ws_bytes >= sk_gemm_ws_bytes() the launch is load-balanced stream-K style:
 * the K loops of the tiles that would form a last, partial wave are laid end to end and cut evenly over all SMs, fp32
 * partial tiles meet in the scratch and are added in a fixed order (deterministic, bit-identical run to run).  The last 4096 bytes of the scratch are flag words: they must be zero before
 * the first call and are left zero by every call.  One scratch buffer serves one stream at a time. */
int sk_gemm_bf16_ws(int M, int N, int K, const void* A, int lda, int a_mn, const void* B, int ldb, int b_mn, void* C,
                    int ldc, int out_f32, const void* bias, const void* residual, int ldr, int round_before_res, int act,
                    int force_bn, void* ws, int64_t ws_bytes, void* stream);
int64_t sk_gemm_ws_bytes(void);
/* Test hook: the schedule sk_gemm_bf16_ws would run for these arguments (sk_gemm_bf16 = the same call with ws = NULL),
 * after the same argument checks.  Nothing is launched and no pointer is dereferenced: only the shapes, the flags,
 * ws_bytes, which of bias / residual / ws are NULL and whether residual == C matter. */
typedef struct SkGemmPlan {
  int32_t bn;                /* tile width: 64, 128, 192, 224 or 256 (tiles are 128 rows) */
  int32_t epi_warps;         /* 4, or 8 (two per 32-row quadrant): warps of the parked epilogue.  One-pass TMA-store
                                plans with epi_warps == 4 and the plain convert or SwiGLU-forward epilogue finish each
                                tile from the wgmma registers on all 8 consumer warps instead */
  int32_t splits;            /* > 1: split-K into this many K ranges, fp32 slabs summed by a second kernel */
  int32_t sk_units;          /* > 0: stream-K over the last sk_units units (rows of tiles, or columns: sk_colunits) */
  int32_t sk_groups;         /* CTA groups that share the stream-K iteration space (cut into equal K ranges) */
  int32_t sk_G;              /* tiles per unit = CTAs per group */
  int32_t sk_colunits;       /* 1: a stream-K unit is a column of tiles (<= 8 tile rows, > 8 tile columns) */
  int32_t tma_store;         /* 1: bf16 output through TMA stores; 0: direct stores (fp32 output, split-K slabs) */
  int32_t grid;              /* CTAs of the GEMM kernel */
} SkGemmPlan;
int sk_gemm_plan(int M, int N, int K, const void* A, int lda, int a_mn, const void* B, int ldb, int b_mn, const void* C,
                 int ldc, int out_f32, const void* bias, const void* residual, int ldr, int round_before_res, int act,
                 int force_bn, const void* ws, int64_t ws_bytes, SkGemmPlan* plan);
/* Test hooks: the batched / split-bf16 form of the GEMM that the HuBERT path runs (sk_hubert_*), so that its features
 * can be checked on their own.  C[b*M + m, n] = act(sum over the passes + bias) (+ residual), with
 *   passes 1: A*B^T;  passes 3: A*B^T + A*B_lo^T + A_lo*B^T (split-bf16, fp32-grade products);
 *   a_rows > 0: A is the 3-D K-major view (a_inner elements per row, a_rows rows a_row_stride apart, batch items
 *     a_batch_stride apart): row m of batch item b is A[b*a_batch_stride + m*a_row_stride, + K) (strided-window conv);
 *   a_mode 1 (needs the 3-D view; 64-column tiles): k-block kb of row m, column tile n reads A[b][m + kb][64n, 64n + 64)
 *     (grouped positional conv on a [B, T + halo, G*64] staging buffer);
 *   col_gin > 0: accumulator column c goes to output column (c / col_gin) * col_gout + c % col_gin and is dropped when
 *     c % col_gin >= col_gout (bias is read at c, residual at the output column);
 *   out_f32: C is fp32; else C (and C_lo when non-NULL: lo = bf16(v - bf16(v))) are bf16;
 *   bias_f32: bias is fp32; residual_lo (optional) is added after residual.
 * All elements counts and pitches are in elements.  sk_gemm_split_plan reports the schedule after the same argument
 * checks, without launching or dereferencing anything. */
typedef struct SkGemmSplitDesc {
  int32_t M, N, K, batch, a_mode, passes;
  const void* A;
  const void* A_lo;
  int32_t lda, a_mn;
  int64_t a_inner, a_rows, a_row_stride, a_batch_stride;
  const void* B;
  const void* B_lo;
  int32_t ldb;
  void* C;
  void* C_lo;
  int32_t ldc, out_f32;
  const void* bias;
  int32_t bias_f32;
  const void* residual;
  const void* residual_lo;
  int32_t ldr, act, col_gin, col_gout, force_bn;
} SkGemmSplitDesc;
int sk_gemm_split(const SkGemmSplitDesc* desc, void* stream);
int sk_gemm_split_plan(const SkGemmSplitDesc* desc, SkGemmPlan* plan);

/* Linears of the LM step with the following element-wise op fused into the GEMM epilogue (no extra pass over HBM).
 * sk_linear_swiglu_fwd: gu[M,2F] = x[M,K] * w_gu[2F,K]^T and act[M,F] = bf16(bf16(silu(gate)) * up)  (Qwen2MLP,
 *   HF:models/qwen2/modeling_qwen2.py:35-48).  w_gu -- and therefore gu -- is stored in 128-row blocks: rows
 *   [256b, 256b+128) = gate_proj rows [128b, 128b+128), rows [256b+128, 256b+256) = the same rows of up_proj; F % 128 == 0.
 * sk_linear_swiglu_bwd: d_gu[M,2F] (same block layout) from d_act = dy[M,N] * w_down[N,F] and the saved gu; d_act is
 *   never written.
 * sk_linear_rope: out[M,N] = x[M,K] * w[N,K]^T + bias[N], then every 64-column head with column < rope_cols is rotated
 *   (HF apply_rotary_pos_emb, :102-146); pos_ids int32 [M] or NULL (position = row % T), clamped to [0, max_positions). */
int sk_linear_swiglu_fwd(int M, int F, int K, const void* x, const void* w_gu, void* gu, void* act, void* stream);
int sk_linear_swiglu_bwd(int M, int N, int F, const void* dy, const void* w_down, const void* gu, void* dgu, void* stream);
int sk_linear_rope(int M, int N, int K, const void* x, const void* w, const void* bias, void* out, const void* cos_t,
                   const void* sin_t, const int32_t* pos_ids, int T, int rope_cols, int max_positions, void* stream);
/* GPT-NeoX epilogues (HF:models/gpt_neox/modeling_gpt_neox.py):
 * sk_linear_rope_partial: sk_linear_rope where only the first rot_dims (16, 32 or 64) columns of each rotated head turn,
 *   element i with i + rot_dims/2, with bf16 tables [max_positions, rot_dims/2]; rot_dims = 64 is sk_linear_rope.
 * sk_linear_gelu_fwd: pre[M,F] = bf16(x[M,K] * w1[F,K]^T + b1) and act[M,F] = bf16(gelu_erf(pre)); F % 64 == 0.
 * sk_linear_gelu_bwd: dpre[M,F] = bf16(bf16(dy[M,N] * w2[N,F]) * gelu'(pre)); d_act is never written.
 * sk_linear_res2: out[M,N] = bf16(bf16(bf16(x * w^T + bias) + res2) + res) (mlp + attn + x in HF's order; out may be res).
 *   ws / ws_bytes: optional stream-K scratch as for sk_gemm_bf16_ws. */
int sk_linear_rope_partial(int M, int N, int K, const void* x, const void* w, const void* bias, void* out, const void* cos_t,
                           const void* sin_t, const int32_t* pos_ids, int T, int rope_cols, int max_positions, int rot_dims,
                           void* stream);
int sk_linear_gelu_fwd(int M, int F, int K, const void* x, const void* w1, const void* b1, void* pre, void* act, void* stream);
int sk_linear_gelu_bwd(int M, int N, int F, const void* dy, const void* w2, const void* pre, void* dpre, void* stream);
int sk_linear_res2(int M, int N, int K, const void* x, const void* w, const void* bias, const void* res2, const void* res,
                   void* out, void* ws, int64_t ws_bytes, void* stream);
/* Test hook: the schedule of a fused linear for an M x N x K problem (the GEMM's own M, N, K); nothing is launched.
 * kind 0 rope_partial, 1 gelu_fwd, 2 gelu_bwd, 3 res2 with the scratch of sk_gemm_ws_bytes() when with_ws;
 * 4 sk_linear_swiglu_fwd (N = 2F), 5 sk_linear_swiglu_bwd (N = F, K = the dy width), 6 sk_linear_rope. */
int sk_neox_gemm_plan(int kind, int M, int N, int K, int with_ws, SkGemmPlan* plan);

/* ---- causal-LM element-wise / reduction kernels (path (ii)) --------------------------------------------------- */
/* Embedding lookup, HF:models/qwen2/modeling_qwen2.py:332-415 (embed_tokens). ids int64 [M]. */
int sk_embed_fwd(const int64_t* ids, const void* table, void* out, int M, int D, int V, void* stream);
/* dTable[ids[m]] += dx[m]; scratch: Vpad*D 64-bit words (2 floats each: the rows are summed in 64-bit fixed point, so
 * the result does not depend on the order the atomics land in); accumulate=1 keeps the existing bf16 gradient. */
int sk_embed_bwd(const int64_t* ids, const void* dx, float* scratch, void* dtable, int M, int D, int V, int Vpad,
                 int accumulate, void* stream);
/* Qwen2RMSNorm, HF:models/qwen2/modeling_qwen2.py:249-262. rstd (fp32 [M]) may be NULL. */
int sk_rmsnorm_fwd(const void* x, const void* w, void* y, float* rstd, int M, int D, float eps, void* stream);
/* dx = d(rmsnorm)(dy) (+ dres);  dw (+)= sum_rows dy*xhat.  dw_partial: fp32 [sk_rmsnorm_bwd_blocks()*D]. */
int sk_rmsnorm_bwd_blocks(void);
int sk_rmsnorm_bwd(const void* dy, const void* x, const void* w, const float* rstd, const void* dres, void* dx,
                   void* dw, float* dw_partial, int M, int D, int accumulate_dw, void* stream);
/* nn.LayerNorm with affine weight w and bias b (the OPT decoder's, HF:models/opt/modeling_opt.py:195-200): fp32 inside,
 * y = bf16((x - mean) * rstd * w + b).  mean / rstd (fp32 [M], may be NULL) are what the backward reads.  D <= 2048. */
int sk_layernorm_fwd(const void* x, const void* w, const void* b, void* y, float* mean, float* rstd, int M, int D, float eps,
                     void* stream);
/* dx = d(layernorm)(dy) (+ dres); dw (+)= sum_rows dy * xhat, db (+)= sum_rows dy, through fixed-order per-block partials
 * (deterministic).  dw_partial / db_partial: fp32 [sk_layernorm_bwd_blocks() * D] each. */
int sk_layernorm_bwd_blocks(void);
int sk_layernorm_bwd(const void* dy, const void* x, const void* w, const float* mean, const float* rstd, const void* dres,
                     void* dx, void* dw, void* db, float* dw_partial, float* db_partial, int M, int D, int accumulate,
                     void* stream);
/* GPT-NeoX parallel residual: y1 = LN(x; w1, b1) and y2 = LN(x; w2, b2) from one read of x, each bit-identical to
 * sk_layernorm_fwd; mean / rstd (fp32 [M], may be NULL) are shared.  The backward forms, in fp32,
 * dx = dres + LN'(w1 * dy1 + w2 * dy2) and dw1 / db1 / dw2 / db2 (+)= their row sums through fixed-order per-block
 * partials (deterministic).  partial: fp32 [4 * sk_layernorm_bwd_blocks() * D].  D <= 2048. */
int sk_layernorm2_fwd(const void* x, const void* w1, const void* b1, const void* w2, const void* b2, void* y1, void* y2,
                      float* mean, float* rstd, int M, int D, float eps, void* stream);
int sk_layernorm2_bwd(const void* dy1, const void* dy2, const void* x, const void* w1, const void* w2, const float* mean,
                      const float* rstd, const void* dres, void* dx, void* dw1, void* db1, void* dw2, void* db2,
                      float* partial, int M, int D, int accumulate, void* stream);
/* Column sums of a bf16 matrix (bias gradient). partial: fp32 [sk_colsum_splits()*N]. */
int sk_colsum_splits(void);
int sk_colsum(const void* x, void* out, float* partial, int M, int N, int ld, int accumulate, void* stream);
/* Rotary embedding (rotate_half form) in place on the first n_rot_heads heads of each row,
 * HF:models/qwen2/modeling_qwen2.py:102-146 (apply_rotary_pos_emb). cos/sin: bf16 [maxpos, head_dim/2].
 * pos_ids: int32 [M] or NULL (position = row % T), clamped to [0, max_positions) = the rows of the tables.
 * inverse=1 applies the transposed rotation (backward). */
int sk_rope(void* qkv, const void* cos_t, const void* sin_t, const int32_t* pos_ids, int M, int T, int ld,
            int n_rot_heads, int head_dim, int inverse, int max_positions, void* stream);
/* sk_rope with GPT-NeoX partial rotary: the first rot_dims (16, 32 or head_dim = 64) columns of each head turn, tables
 * bf16 [max_positions, rot_dims/2]; the other columns are left as they are. */
int sk_rope_partial(void* qkv, const void* cos_t, const void* sin_t, const int32_t* pos_ids, int M, int T, int ld,
                    int n_rot_heads, int head_dim, int rot_dims, int inverse, int max_positions, void* stream);
/* Qwen2MLP activation down(silu(gate)*up), HF:models/qwen2/modeling_qwen2.py:35-48. gu = [gate | up], each F wide. */
int sk_swiglu_fwd(const void* gu, void* act, int M, int F, void* stream);
int sk_swiglu_bwd(const void* gu, const void* dact, void* dgu, int M, int F, void* stream);
/* compute_loss, slamkit/model/unit_lm.py:13-29: fp32 upcast, shift, CE(ignore_index=-100), sum/num_items (or mean
 * over valid tokens when num_items <= 0).  logits bf16 [B*T, ldl] with V valid columns; labels int64 [B*T];
 * dlogits (bf16, may be NULL) = d loss / d logits * dloss; partial: fp32 [2*sk_ce_blocks(M)]; row_nll fp32 [M] or
 * NULL; stats: fp32[3] = {loss, n_valid_targets, nll_sum}. */
int sk_ce_blocks(int M);
int sk_ce_fwd_bwd(const void* logits, const int64_t* labels, void* dlogits, float* partial, float* row_nll,
                  float* stats, int M, int T, int V, int ldl, float num_items, float dloss, void* stream);
/* Test hooks over the launchers the train step uses.  sk_ce_fwd_bwd_weighted: sk_ce_fwd_bwd with the gradient of row m
 * scaled by row_weight[m] (fp32 [M], the DPO path's per-sequence weights).  sk_ce_chunk: the chunked lm_head's CE on rows
 * [row0, row0 + rows) whose logits sit at logits_chunk ([rows, ldl]; dlogits_chunk may equal it), one (nll, valid) pair
 * per global row in partial fp32 [2 * M]; grad_scale multiplies the gradient.  sk_ce_finalize sums the pairs into stats. */
int sk_ce_fwd_bwd_weighted(const void* logits, const int64_t* labels, void* dlogits, float* partial, float* row_nll,
                           const float* row_weight, float* stats, int M, int T, int V, int ldl, float num_items, float dloss,
                           void* stream);
int sk_ce_chunk(const void* logits_chunk, const int64_t* labels, void* dlogits_chunk, float* partial, int row0, int rows,
                int M, int T, int V, int ldl, float grad_scale, void* stream);
int sk_ce_finalize(const float* partial, int M, float num_items, float* stats, void* stream);
/* OPT learned positions: dP[row(m)] (+)= dx[m] in the fixed point of sk_embed_bwd, row(m) = min(max(pos + 2, 0), n_pos - 1)
 * with pos = pos_ids[m] (int32 [M]) or m % T when pos_ids is NULL.  scratch: n_pos * D 64-bit words. */
int sk_opt_pos_bwd(const int32_t* pos_ids, const void* dx, float* scratch, void* dP, int M, int T, int D, int n_pos,
                   int accumulate, void* stream);
/* ReLU backward in place, torch threshold_backward(g, a, 0): g = a <= 0 ? 0 : g (bf16 [n], n a multiple of 8). */
int sk_relu_bwd(void* g, const void* a, int64_t n, void* stream);

/* ---- attention -------------------------------------------------------------------------------------------------
 * softmax(q k^T * scale [causal]) v with grouped-query heads, head_dim 64; q/k/v are column slices (pitch ld) of the
 * fused projection output, o is [B*T, ldo]; lse fp32 [B,H,T].  Replaces SDPA/FA2 behind HF Qwen2Attention
 * (HF:models/qwen2/modeling_qwen2.py:187-246) and HubertAttention (HF:models/hubert/modeling_hubert.py:262-345). */
int sk_attn_fwd(const void* q, const void* k, const void* v, void* o, float* lse, int B, int T, int H, int KVH, int ld,
                int ldo, int causal, float scale, void* stream);
/* The same forward on the fused projection (optionally block-diagonal over packed documents).
 * qkv points at the fused [B*T, ld] projection: H q-heads, then KVH k-heads, then KVH v-heads, 64 columns each. */
int sk_attn_tc_fwd(const void* qkv, void* o, float* lse, int B, int T, int H, int KVH, int ld, int ldo, int causal,
                   float scale, const int32_t* seg_start, void* stream);
/* Document bounds of packed batches (DataCollatorWithFlattening, slamkit/data/hf_dataset.py:61-62): a document starts at
 * column 0 and wherever position_ids == 0, exactly how HF derives cu_seqlens for its varlen flash-attention path
 * (HF:modeling_flash_attention_utils.py prepare_fa_kwargs_from_position_ids).  seg_start[b*T+t] = in-row index of the
 * first token of t's document, seg_end = one past its last.  Passing them (NULL = one document per row) to
 * sk_attn_tc_fwd / sk_attn_tc_bwd makes attention block-diagonal causal. */
int sk_seg_bounds(const int32_t* pos_ids, int32_t* seg_start, int32_t* seg_end, int B, int T, void* stream);
/* Backward on the fused projection: dqkv (same fused layout as qkv, pitch ldg) from d_o; delta fp32 [B,H,T] is caller
 * scratch; partial is accepted for ABI compatibility, unused, and may be NULL.  Deterministic (dK / dV summed over
 * the GQA group in a fixed order). */
int sk_attn_tc_bwd(const void* qkv, const void* o, const void* d_o, const float* lse, float* delta, float* partial,
                   void* dqkv, int B, int T, int H, int KVH, int ld, int ldo, int ldg, int causal, float scale,
                   const int32_t* seg_start, const int32_t* seg_end, void* stream);
int sk_attn_bwd(const void* q, const void* k, const void* v, const void* o, const void* d_o, const float* lse,
                float* delta, void* dq, void* dk, void* dv, int B, int T, int H, int KVH, int ld, int ldo, int ldg,
                int causal, float scale, void* stream);
/* Split-bf16 bidirectional forward of the HuBERT encoder: each value is an fp32-grade (hi, lo) bf16 pair.  qkv_hi /
 * qkv_lo point at [B*T, ld] projections with H q-heads, then H k-heads, then H v-heads (64 columns each); o_hi / o_lo are
 * [B*T, ldo].  S = Qh Kh^T + Qh Kl^T + Ql Kh^T and O = Ph Vh + Ph Vl + Pl Vh in fp32; the output pair is
 * hi = bf16(o), lo = bf16(o - hi). */
int sk_attn_tc_fwd_split(const void* qkv_hi, const void* qkv_lo, void* o_hi, void* o_lo, int B, int T, int H, int ld,
                         int ldo, float scale, void* stream);
/* The causal instance of the same kernel (fp32 OPT inference): row t attends to keys 0..t of its batch row.  No key tile
 * past a query tile's diagonal is read. */
int sk_attn_tc_fwd_split_causal(const void* qkv_hi, const void* qkv_lo, void* o_hi, void* o_lo, int B, int T, int H, int ld,
                                int ldo, float scale, void* stream);

/* ---- optimiser ----------------------------------------------------------------------------------------------------
 * Gradient clipping + AdamW as HF Trainer runs them (HF:trainer.py clip_grad_norm_ then torch.optim.AdamW(fused)):
 * config/training_args/default.yaml:4-9 (lr 1e-3, max_grad_norm 0.5), betas (0.9,0.999), eps 1e-8, wd 0.
 * bf16 parameters AND bf16 moment buffers (params are created in bf16: config/model/slam.yaml:9). */
/* chunk tables (device): chunk_start int64[n_chunks], chunk_len int32[n_chunks], tensor_chunk_begin int32[n_tensors+1];
 * partial fp32[n_chunks]; stats fp32[3] = {total_norm, clip_coef, exact_fp32_norm}. emulate_bf16=1 rounds per-tensor
 * norms, the total and the coefficient to bf16 like torch does on bf16 gradients. */
int sk_grad_norm(const void* grads, const int64_t* chunk_start, const int32_t* chunk_len, int n_chunks,
                 const int32_t* tensor_chunk_begin, int n_tensors, float* partial, float max_norm, int emulate_bf16,
                 float* stats, void* stream);
/* One fused pass over the flat parameter buffer (14 B/param). clip_stats: the stats buffer of sk_grad_norm or NULL. */
int sk_adamw_step(void* params, const void* grads, void* exp_avg, void* exp_avg_sq, int64_t n, float lr, float beta1,
                  float beta2, float eps, float weight_decay, int step, const float* clip_stats, void* stream);
/* fp32 master weights (see sk_lm_set_master).  sk_grad_norm_f32: sk_grad_norm over fp32 gradients, fp32 throughout (no
 * bf16 rounding).  sk_adamw_master_step: AdamW on fp32 params / grads / moments (n a multiple of 8, 16-byte aligned)
 * with torch's fp32 element arithmetic, each operation rounded once; 1 - beta, lr * weight_decay, lr / (1 - beta1^step)
 * and sqrt(1 - beta2^step) are formed in double from the fp32 arguments; also writes shadow = bf16(params) [n]. */
int sk_grad_norm_f32(const float* grads, const int64_t* chunk_start, const int32_t* chunk_len, int n_chunks,
                     const int32_t* tensor_chunk_begin, int n_tensors, float* partial, float max_norm, float* stats, void* stream);
int sk_adamw_master_step(float* params, void* shadow, const float* grads, float* exp_avg, float* exp_avg_sq, int64_t n, float lr,
                         float beta1, float beta2, float eps, float weight_decay, int step, const float* clip_stats, void* stream);
/* OPT master weights: residual add + LayerNorm on fp32 rows, one warp per row (D a multiple of 8, <= 2048):
 * xo = x + float(y) (y bf16 [M, D] or NULL: no add, xo unused), h = bf16(LN(xo) * w + b) with fp32 w, b; mean / rstd
 * fp32 [M] (may be NULL).  Backward: dres_out = dres_in + LN'(float(dy) * w) in fp32 (dres_in NULL reads zeros; may
 * alias dres_out), dres16 = bf16(dres_out), dw / db fp32 [D] (+)= (accumulate) through partial fp32
 * [2 * sk_layernorm_bwd_blocks() * D] in a fixed order. */
int sk_add_layernorm_f32(const float* x, const void* y, const float* w, const float* b, float* xo, void* h, float* mean, float* rstd,
                         int M, int D, float eps, void* stream);
int sk_layernorm_bwd_f32(const void* dy, const float* x, const float* w, const float* mean, const float* rstd, const float* dres_in,
                         float* dres_out, void* dres16, float* dw, float* db, float* partial, int M, int D, int accumulate,
                         void* stream);
/* Test hooks over the master step's table and widening launchers.  sk_table_bwd_f32: fp32 table gradient from fp32 rows
 * dx [M, D] in the 64-bit fixed point of sk_embed_bwd: ids given, row(m) = ids[m] (ids outside [0, n_rows) skipped) and
 * head (bf16 [n_rows_padded, D] or NULL) is added; ids NULL, row(m) is the OPT position row of sk_opt_pos_bwd.
 * dtable = (keep ? dtable : 0) + (float(head) + sum); scratch: n_rows_padded * D 64-bit words.
 * sk_widen_grads: g32 (+)= float(g16) over the chunks [chunk_start[c], + chunk_len[c]) (device tables as sk_grad_norm;
 * starts and lengths multiples of 8). */
int sk_table_bwd_f32(const int64_t* ids, const int32_t* pos_ids, const float* dx, float* scratch, float* dtable, const void* head,
                     int M, int T, int D, int n_rows, int n_rows_padded, int keep, void* stream);
int sk_widen_grads(const void* g16, float* g32, const int64_t* chunk_start, const int32_t* chunk_len, int n_chunks, int keep,
                   void* stream);

/* ---- causal-LM train step (path (ii)) ---------------------------------------------------------------------------
 * One object per model replica; replaces UnitLM.forward + compute_loss + autograd backward
 * (slamkit/model/unit_lm.py:13-29,135-182 -> HF Qwen2ForCausalLM, HF:models/qwen2/modeling_qwen2.py:417-487) and,
 * with sk_grad_norm/sk_adamw_step, the HF Trainer inner step (HF:trainer.py:1867-2014). */
typedef struct SkLmConfig {
  int32_t vocab_size;        /* 502 for unit_hubert_25 (slamkit/tokeniser/unit_tokeniser.py:33-47) */
  int32_t hidden;            /* 896 */
  int32_t n_layers;          /* 24 */
  int32_t n_heads;           /* 14 */
  int32_t n_kv_heads;        /* 2 */
  int32_t head_dim;          /* 64 (only 64 is supported) */
  int32_t ffn;               /* 4864 */
  int32_t max_positions;     /* rows of the RoPE tables */
  float rms_eps;             /* 1e-6 */
  int32_t tie_embeddings;    /* 1: lm_head shares the embedding table */
  int32_t qkv_bias;          /* 1 for Qwen2 */
} SkLmConfig;
typedef struct SkLm SkLm;

int sk_lm_create(const SkLmConfig* cfg, SkLm** out);
/* Pre-LayerNorm OPT decoder (HF OPTForCausalLM with do_layer_norm_before = True and word_embed_proj_dim = hidden, e.g.
 * facebook/opt-125m, the base of config/model/twist.yaml and gslm.yaml; HF:models/opt/modeling_opt.py):
 *   x0 = bf16(embed_tokens[id] + embed_positions[pos + 2]);  per layer  h = LN1(x);  q|k|v = h W + b;  causal MHA with
 *   scale 1/8 (HF multiplies q by 1/8, a power of two);  x += o W_o + b_o;  h = LN2(x);  x += relu(h W_1 + b_1) W_2 + b_2;
 *   final LN, tied (or separate) lm_head without bias.  LayerNorms are affine, fp32 inside, rounded once to bf16.
 * Returns the same SkLm handle type: every sk_lm_* entry point runs this decoder on it.  Differences from a Qwen2 handle:
 *   - the flat layout (sk_lm_tensor_info) lists per layer ln1, ln1_b, wqkv [3*hidden, hidden], bqkv, wo, bo, ln2, ln2_b,
 *     w1 [ffn, hidden], b1, w2 [hidden, ffn], b2; then final_norm, final_norm_b, embed [Vpad, hidden],
 *     pos_embed [max_positions + 2, hidden] and, untied, lm_head;
 *   - sk_lm_bind takes NULL RoPE tables;
 *   - positions (row % T, pos_ids, or the decode step's pos[b]) select table row position + 2, clamped to the table;
 *   - the gradient-norm groups are OPTForCausalLM's parameters: q, k, v, out_proj, fc1, fc2 weights and biases and the
 *     LayerNorm weights and biases each count as one tensor;
 *   - the KV cache holds n_heads K/V heads per layer (same layout as above with n_kv_heads = n_heads).
 * post_ln = 1 selects the post-LayerNorm OPT (do_layer_norm_before = False, e.g. facebook/opt-350m), optionally with the
 * bias-free project_in / project_out pair (proj_dim = word_embed_proj_dim, 0 or hidden: none):
 *   e = embed_tokens[id] [proj_dim];  x0 = bf16(bf16(e W_in^T) + embed_positions[pos + 2]);  per layer
 *   s1 = bf16(bf16(attn(x) W_o + b_o) + x), y1 = LN1(s1);  s2 = bf16(bf16(relu(y1 W_1 + b_1) W_2 + b_2) + y1), x' = LN2(s2);
 *   h = bf16(x_L W_out^T);  logits = h E^T (tied: K = proj_dim).  There is no decoder-level final LayerNorm.
 * Its flat layout has embed [Vpad, proj_dim], proj_in [hidden, proj_dim] and proj_out [proj_dim, hidden] (when
 * projecting) and no final_norm / final_norm_b; its gradient-norm groups add project_out and project_in.  It trains in
 * bf16 and runs fp32 inference (sk_lm_set_fp32); sk_lm_set_master refuses it.  Zero in both fields (what an 8-field
 * initialiser leaves) is the pre-LayerNorm decoder above; pre-LN with proj_dim != hidden is refused. */
typedef struct SkOptConfig {
  int32_t vocab_size;        /* 502 for unit_hubert_25 */
  int32_t hidden;            /* 768 for opt-125m; n_heads * 64, <= 2048 */
  int32_t n_layers;          /* 12 */
  int32_t n_heads;           /* 12 */
  int32_t ffn;               /* 3072; a multiple of 8 */
  int32_t max_positions;     /* max_position_embeddings (2048): the position table has max_positions + 2 rows */
  float ln_eps;              /* 1e-5 */
  int32_t tie_embeddings;    /* 1: lm_head shares the token embedding table */
  int32_t post_ln;           /* 0: pre-LayerNorm (opt-125m); 1: post-LayerNorm (opt-350m) */
  int32_t proj_dim;          /* word_embed_proj_dim: 0 or hidden = no projections; else a multiple of 64, < hidden */
} SkOptConfig;
int sk_lm_create_opt(const SkOptConfig* cfg, SkLm** out);
/* GPT-NeoX decoder with the parallel residual (HF GPTNeoXForCausalLM, use_parallel_residual = True, e.g. the Pythia
 * models with head_dim 64: pythia-70m / -160m / -410m; HF:models/gpt_neox/modeling_gpt_neox.py):
 *   x0 = embed_in[id];  per layer  h1 = LN1(x), h2 = LN2(x);  q|k|v = h1 W + b;  RoPE on the first rot_dims columns of
 *   each q / k head;  causal MHA with scale 1/8;  attn = o W_o + b_o;  mlp = gelu(h2 W_1 + b_1) W_2 + b_2;
 *   x = bf16(bf16(mlp + attn) + x);  final LN, untied embed_out without bias.
 * Differences from a Qwen2 handle:
 *   - the flat layout lists per layer ln1, ln1_b, ln2, ln2_b, wqkv [3*hidden, hidden] in [Q;K;V] row order (HF stores
 *     per-head [q|k|v] blocks: the caller permutes), bqkv, wo, bo, w1 [ffn, hidden], b1, w2 [hidden, ffn], b2; then
 *     final_norm, final_norm_b, embed [Vpad, hidden], lm_head [Vpad, hidden];
 *   - sk_lm_bind takes RoPE tables of bf16 [max_positions, rot_dims/2];
 *   - the gradient-norm groups are GPTNeoXForCausalLM's parameters (query_key_value weight and bias are one tensor each);
 *   - the KV cache holds n_heads K/V heads per layer. */
typedef struct SkNeoxConfig {
  int32_t vocab_size;        /* 502 for unit_hubert_25 */
  int32_t hidden;            /* 768 for pythia-160m; n_heads * 64, <= 2048 */
  int32_t n_layers;
  int32_t n_heads;
  int32_t ffn;               /* intermediate_size (4 * hidden); a multiple of 64 */
  int32_t max_positions;     /* rows of the RoPE tables */
  int32_t rot_dims;          /* head_dim * partial_rotary_factor: 16, 32 or 64 */
  float ln_eps;              /* layer_norm_eps, 1e-5 */
} SkNeoxConfig;
int sk_lm_create_neox(const SkNeoxConfig* cfg, SkLm** out);
void sk_lm_destroy(SkLm* lm);
/* Flat parameter layout (bf16 elements). Tensors are enumerated in a fixed order; name_buf receives e.g.
 * "layers.3.wqkv". Returns the number of tensors when idx < 0. */
int64_t sk_lm_param_count(const SkLm* lm);
int sk_lm_tensor_info(const SkLm* lm, int idx, char* name_buf, int name_cap, int64_t* offset, int32_t* rows,
                      int32_t* cols);
int64_t sk_lm_workspace_bytes(const SkLm* lm, int B, int T);
/* Bind caller-owned memory: params/grads are flat bf16 [param_count]; rope tables bf16 [max_positions, head_dim/2];
 * workspace >= sk_lm_workspace_bytes(B,T) for the largest (B,T) used. */
int sk_lm_bind(SkLm* lm, void* params, void* grads, const void* rope_cos, const void* rope_sin, void* workspace,
               int64_t workspace_bytes);
/* OPT handles only, after sk_lm_bind: train fp32 master weights, as HF OPTForCausalLM with fp32 parameters runs under
 * torch.autocast(bfloat16) (the reference's default recipe, torch_dtype null and bf16: true).  params32 / grads32 are
 * caller-owned flat fp32 [param_count] buffers in the bf16 layout (grads32 may be NULL for a forward-only handle); the
 * bound bf16 `params` become the shadow bf16(params32) that the GEMMs read (the caller fills it once; the optimiser step
 * rewrites it), the bound bf16 `grads` the per-micro-batch scratch of the linear gradients.  From then on:
 *   - the residual stream is fp32: x0 = E[id] + P[pos + 2] from the fp32 tables, x += float(bf16 branch output), every
 *     LayerNorm reads fp32 x, gamma, beta and rounds its output once to bf16 for the next linear;
 *   - sk_lm_forward_backward accumulates into grads32: linear weight / bias gradients are computed in bf16 and widened,
 *     LayerNorm and table gradients are fp32, the residual gradient is fp32 (its bf16 copy feeds the GEMMs);
 *   - sk_lm_optimizer_step takes fp32 exp_avg / exp_avg_sq, clips over the fp32 grads32 (emulate_bf16_norm is ignored)
 *     and writes params32, the moments and the bf16 shadow;
 *   - sk_lm_workspace_bytes reports the larger fp32-residual workspace: bind it again before the next forward pass;
 *   - sk_lm_prefill / sk_lm_decode_step refuse the handle (generation runs on the saved checkpoint).
 * Qwen2 and GPT-NeoX handles are refused. */
int sk_lm_set_master(SkLm* lm, float* params32, float* grads32);
/* The chunks whose bf16 gradients the master step widens into grads32 (see sk_widen_grads), copied to host arrays of
 * capacity cap; returns the number of chunks, or -1. */
int sk_lm_widen_chunks(const SkLm* lm, int64_t* chunk_start, int32_t* chunk_len, int cap);
/* OPT handles only, after sk_lm_bind: fp32 inference, as the reference scores and generates a float32 checkpoint (HF
 * OPTForCausalLM in fp32, no autocast).  params32 is a caller-owned flat fp32 [param_count] buffer in the bf16 layout
 * (it stays referenced); `prepared` (>= sk_lm_fp32_prepared_bytes, 256-byte aligned) receives its split-bf16 (hi, lo)
 * copy, written on `stream`.  Call again after params32 changes.  From then on the handle is forward only:
 *   - every linear is the split-bf16 three-product GEMM with fp32 bias; activations and the residual stream are (hi, lo)
 *     pairs; LayerNorms use fp32 gamma / beta; attention is the causal split-bf16 kernel; fp32-grade throughout;
 *   - sk_lm_forward (labels and pos_ids NULL) writes fp32 logits, read through sk_lm_logits_f32 (sk_lm_logits is NULL);
 *   - sk_lm_prefill / sk_lm_decode_step write fp32 logits [B, ldl]; the KV cache is fp32 (sk_lm_kv_cache_bytes);
 *   - sk_lm_workspace_bytes and sk_lm_decode_workspace_bytes report the fp32-grade sizes: bind the workspace again;
 *   - sk_lm_forward_backward, sk_lm_forward_rows, sk_lm_backward_weighted and sk_lm_optimizer_step are refused.
 * Mutually exclusive with sk_lm_set_master.  Qwen2 and GPT-NeoX handles are refused; hidden <= 1024. */
int64_t sk_lm_fp32_prepared_bytes(const SkLm* lm);
int sk_lm_set_fp32(SkLm* lm, const float* params32, void* prepared, int64_t prepared_bytes, void* stream);
/* Forward only (eval / log-likelihood): logits stay in the workspace, see sk_lm_logits. labels may be NULL.
 * pos_ids: int32 [B*T] or NULL (positions 0..T-1 per row).  When given they drive RoPE AND mark packed documents: a
 * document starts wherever pos_ids == 0, and tokens attend only within their document (the reference's varlen
 * flash-attention path for DataCollatorWithFlattening batches, slamkit/data/hf_dataset.py:61-62; cli/train.py:43-45).
 * The same holds for every sk_lm_* entry point below that takes pos_ids. */
int sk_lm_forward(SkLm* lm, const int64_t* ids, const int64_t* labels, const int32_t* pos_ids, int B, int T,
                  float num_items, float* stats, void* stream);
/* Forward + backward of one micro-batch. accumulate=0 overwrites grads, 1 adds (gradient accumulation).
 * stats fp32[3] = {loss, n_valid_targets, nll_sum}. loss = nll_sum/num_items when num_items > 0
 * (HF:trainer.py:2092-2154 num_items_in_batch semantics), else mean over valid targets. */
int sk_lm_forward_backward(SkLm* lm, const int64_t* ids, const int64_t* labels, const int32_t* pos_ids, int B, int T,
                           float num_items, float dloss, int accumulate, float* stats, void* stream);
/* Data-parallel overlap hook: n = n_layers+1 caller-owned cudaEvent_t handles; during sk_lm_forward_backward event l is
 * recorded on the compute stream once layer l's gradients are final (event n_layers: final-norm part), so the host can
 * enqueue that bucket's all-reduce (sk_p2p_* below, or NCCL) on a side stream while the backward pass continues.
 * NULL/0 disables. */
int sk_lm_set_backward_events(SkLm* lm, void* const* events, int n);
/* Preference optimisation (DPO, cli/preference_alignment_train.py -> trl.DPOTrainer; SURVEY.md §3.4): the loss is not a
 * plain CE, but its logit gradient is a per-SEQUENCE-weighted CE gradient.  sk_lm_forward_rows runs the forward pass
 * and returns the per-position NLL (fp32 [B*T], 0 where the shifted label is -100) with all activations kept in the
 * workspace; the host turns per-sequence sums into DPO weights; sk_lm_backward_weighted then back-propagates
 * d loss / d logits[row] = row_weight[row] * (softmax - onehot) through the same activations. */
int sk_lm_forward_rows(SkLm* lm, const int64_t* ids, const int64_t* labels, const int32_t* pos_ids, int B, int T,
                       float* row_nll, float* stats, void* stream);
int sk_lm_backward_weighted(SkLm* lm, const int64_t* ids, const int64_t* labels, const int32_t* pos_ids, int B, int T,
                            const float* row_weight, int accumulate, float* stats, void* stream);
/* bf16 [B*T, sk_lm_logits_ld()] logits of the last forward (valid columns: vocab_size). */
const void* sk_lm_logits(const SkLm* lm);
int sk_lm_logits_ld(const SkLm* lm);
/* fp32 [B*T, sk_lm_logits_ld()] logits of the last forward of an fp32 inference handle (NULL on other handles). */
const float* sk_lm_logits_f32(const SkLm* lm);
/* Clip (max_norm <= 0 disables) + AdamW over the bound params/grads; moments are caller-owned flat bf16 buffers.
 * stats fp32[3] as sk_grad_norm. */
int sk_lm_optimizer_step(SkLm* lm, void* exp_avg, void* exp_avg_sq, float lr, float beta1, float beta2, float eps,
                         float weight_decay, int step, float max_grad_norm, int emulate_bf16_norm, float* stats,
                         void* stream);

/* ---- incremental decoding (TokenLM.generate with a KV cache) -----------------------------------------------------
 * Replaces HF GenerationMixin's cached greedy / sampling loop behind UnitLM.generate (slamkit/model/unit_lm.py:196-198,
 * called by SpeechLM.generate, slamkit/model/speech_lm.py:38-55).  sk_lm_decode_step and sk_select_next allocate
 * nothing, never synchronise and take the same arguments every step (positions, lengths and the step index live in
 * device memory), so one step can be captured in a CUDA graph and replayed; run one step eagerly before capturing.
 *
 * KV cache of all layers, caller-owned: [L][K|V][B][KVH][T_cache][head_dim] bf16, K stored after RoPE. */
int64_t sk_lm_kv_cache_bytes(const SkLm* lm, int B, int T_cache);
int64_t sk_lm_decode_workspace_bytes(const SkLm* lm, int B, int T_cache);
/* ids RIGHT-padded [B,T] (T <= T_cache), lens int32 [B], 1 <= lens[b] <= T real tokens at positions 0..lens[b]-1.  Runs
 * the forward pass on the bound workspace (sized for [B,T]) without the full-sequence head, copies the K/V of positions
 * < lens[b] into the cache and writes the bf16 logits of each row's last real token into logits [B, ldl]
 * (ldl >= sk_lm_logits_ld()).  Also clears the GEMM flag words of decode_ws. */
int sk_lm_prefill(SkLm* lm, const int64_t* ids, const int32_t* lens, int B, int T, void* kv_cache, int T_cache,
                  void* logits, int ldl, void* decode_ws, int64_t decode_ws_bytes, void* stream);
/* One token per row: tokens int64 [B] at positions pos int32 [B] (pos[b] < T_cache): embed, per layer RMSNorm ->
 * QKV + bias + RoPE GEMM (M = B) -> K/V appended at pos[b] -> decode attention over [0, pos[b]] -> o-proj + residual ->
 * RMSNorm -> SwiGLU GEMM -> down-proj + residual; final norm, head -> logits [B, ldl]. */
int sk_lm_decode_step(SkLm* lm, const int64_t* tokens, const int32_t* pos, int B, void* kv_cache, int T_cache,
                      void* logits, int ldl, void* decode_ws, int64_t decode_ws_bytes, void* stream);
/* Decoding restricted to n allowed ids (generate's allowed_token_ids): the compact head is rows ids[0 .. n) of the
 * handle's head (the token table when tied, else lm_head / embed_out; post-LN OPT with project_out: the proj_dim-wide
 * table) gathered into head bf16 [n_pad, head width], rows n .. n_pad - 1 zero; n_pad a multiple of 64 <= the padded
 * vocabulary.  ids int32, ascending, in [0, vocab).  Run once per generate call (not per step). */
int sk_lm_gather_head(const SkLm* lm, const int32_t* ids, int n, int n_pad, void* head, void* stream);
/* sk_lm_prefill / sk_lm_decode_step with the final GEMM on the compact head: logits [B, ld_sub] (ld_sub >= n_pad, a
 * multiple of 8), column c = the logit of ids[c], bit-identical to that id's column of the full-vocabulary call (the
 * same whole-tile GEMM, same K order per element).  Every other launch is the full call's.  bf16 handles only. */
int sk_lm_prefill_sub(SkLm* lm, const int64_t* ids, const int32_t* lens, int B, int T, void* kv_cache, int T_cache,
                      const void* head, int n_pad, void* logits, int ld_sub, void* decode_ws, int64_t decode_ws_bytes,
                      void* stream);
int sk_lm_decode_step_sub(SkLm* lm, const int64_t* tokens, const int32_t* pos, int B, void* kv_cache, int T_cache,
                          const void* head, int n_pad, void* logits, int ld_sub, void* decode_ws, int64_t decode_ws_bytes,
                          void* stream);
/* Prompt fan-out for num_return_sequences: copies positions t < lens[b] of every layer's K and V of row b of src_cache
 * (B rows) into rows b*k .. b*k + k - 1 of dst_cache (B*k rows), both with the same T_cache and the handle's layout
 * ([L][K|V][rows][KVH][T_cache][head_dim], bf16, or fp32 on fp32 inference handles).  Positions >= lens[b] of the
 * destination are not written.  src and dst must not overlap; both 16-byte aligned. */
int sk_lm_kv_fanout(const SkLm* lm, const void* src_cache, int B, int k, void* dst_cache, int T_cache, const int32_t* lens,
                    void* stream);
/* Stand-alone decode attention: o[b, h*64 .. h*64+63] (pitch ldo) = softmax(q k^T * scale) v over keys [0, lens[b]) of
 * row b; q [B, H*64] pitch ldq; k_cache / v_cache [B][KVH][T_cache][64] bf16.  Flash-decoding over fixed 64-key splits
 * (one CTA per row, kv head and split serves the H/KVH <= 16 query heads of its group) and a combine pass in split
 * order: bit-identical run to run, and no key at or past lens[b] is read.  partial: sk_attn_decode_partial_bytes. */
int64_t sk_attn_decode_partial_bytes(int B, int H, int T_cache);
int sk_attn_decode(const void* q, int ldq, const void* k_cache, const void* v_cache, const int32_t* lens, void* o, int ldo,
                   float* partial, int B, int H, int KVH, int T_cache, float scale, void* stream);
/* The same over an fp32 cache (fp32 inference): q = q_hi + q_lo (bf16 pairs, pitch ldq), k_cache / v_cache
 * [B][H][T_cache][64] fp32, the fp32 result written as the pair o_hi = bf16(o), o_lo = bf16(o - o_hi) (pitch ldo). */
int sk_attn_decode_split(const void* q_hi, const void* q_lo, int ldq, const float* k_cache, const float* v_cache,
                         const int32_t* lens, void* o_hi, void* o_lo, int ldo, float* partial, int B, int H, int T_cache,
                         float scale, void* stream);
/* Token selection settings (HF GenerationConfig fields). */
typedef struct SkSampling {
  uint64_t seed;             /* Philox key of the draws */
  double top_p;              /* >= 1: off */
  float temperature;         /* sampling only */
  int32_t do_sample;         /* 0: greedy (argmax, lowest id on ties; temperature / top-k / top-p unused) */
  int32_t top_k;             /* <= 0: off */
  int32_t n_eos;             /* 0..8 */
  int32_t eos[8];            /* a row finishes after emitting one of these */
  int32_t pad_token_id;      /* written for rows that have finished */
  int32_t max_length;        /* a row finishes once prompt + generated tokens reach this length */
} SkSampling;
/* Device-resident decode state (pointers to caller-owned device memory). */
typedef struct SkDecodeState {
  int64_t* tokens;           /* [B] last token of each row: the next decode step's input */
  int32_t* pos;              /* [B] its position */
  int32_t* finished;         /* [B] */
  int32_t* n_gen;            /* [B] tokens generated */
  int64_t* out;              /* [B, max_new] generated ids; pad_token_id once a row has finished */
  int32_t* step;             /* [2] step index and an arrival counter, both zero-initialised */
  int32_t max_new;
  int32_t reserved;
} SkDecodeState;
/* Selects the next token of every row in HF's order: bans -> (if do_sample) temperature -> top-k (keeps scores >= the
 * k-th largest) -> top-p (drops the tokens whose ascending cumulative probability is <= 1 - top_p, ties by id, keeps the
 * most likely one) -> softmax -> inverse-CDF draw in token-id order; greedy: argmax.  ban_bits: uint32 [ceil(V/32)]
 * bitmask of banned ids or NULL.  uniforms: NULL = Philox4x32-10 keyed by (seed, step, row); else one fp32 uniform in
 * [0, 1) per row.  Finished rows (or pos[b] + 1 >= max_length) only write pad_token_id.  Otherwise out[b, step],
 * n_gen[b], tokens[b], pos[b] (+1) and finished[b] (eos) are updated; the step index advances by one per call. */
int sk_select_next(const void* logits, int ldl, int V, int B, const uint32_t* ban_bits, const SkSampling* cfg,
                   const float* uniforms, const SkDecodeState* state, void* stream);
/* sk_select_next on fp32 logits [B, ldl] (fp32 inference handles); logits 16-byte aligned. */
int sk_select_next_f32(const float* logits, int ldl, int V, int B, const uint32_t* ban_bits, const SkSampling* cfg,
                       const float* uniforms, const SkDecodeState* state, void* stream);
/* sk_select_next over compact bf16 logits [B, ld_sub]: column c is token ids[c] (int32 [n], ascending, in [0, V)) and
 * every other id of the V-token vocabulary is banned.  Picks the token sk_select_next picks on the full logits with the
 * complement in ban_bits (the same per-thread sums and tie breaks); writes the token id, not the column. */
int sk_select_next_sub(const void* logits, int ld_sub, const int32_t* ids, int n, int V, int B, const SkSampling* cfg,
                       const float* uniforms, const SkDecodeState* state, void* stream);
/* History-dependent logits processors (HF GenerationConfig repetition_penalty, no_repeat_ngram_size, min_new_tokens /
 * min_length).  Row b's history is history[b, 0 .. prompt_len + step): the padded prompt exactly as the caller passed
 * it (left pads included), then the tokens selected so far (pad_token_id for finished rows). */
typedef struct SkLogitRules {
  int64_t* history;          /* [B, hist_ld]; columns < prompt_len filled by the caller, the rest appended per step */
  uint32_t* presence;        /* [B, ceil(V/32)] bit i: id i occurs in the history (sk_presence_init, then per step) */
  uint32_t* scratch;         /* [B, ceil(V/32)] per-step bans; needed when ngram > 0 or min_step > 0 */
  float penalty;             /* repetition_penalty; 1: off */
  int32_t ngram;             /* no_repeat_ngram_size; <= 0: off */
  int32_t min_step;          /* eos ids are -inf while step < min_step (needs n_eos > 0) */
  int32_t prompt_len;        /* T, the padded prompt width */
  int32_t hist_ld;           /* >= prompt_len + max_new */
  int32_t reserved;
} SkLogitRules;
/* sk_select_next / sk_select_next_f32 with rules, applied on the fp32 scores in HF's order (penalty -> n-gram bans ->
 * ban_bits -> min length), before temperature; greedy honours them too:
 *   repetition penalty: every id whose presence bit is set: s = s < 0 ? s * penalty : s / penalty (rounded once);
 *   n-gram bans (cur_len = prompt_len + step, when cur_len + 1 >= ngram): every id that followed an earlier occurrence of
 *     the row's last ngram - 1 tokens, at any position of the history, pads included, is -inf;
 *   min length: while step < min_step, every eos id is -inf.
 * After the selection every row appends its token (pad_token_id once finished) at history[b, prompt_len + step] and
 * sets its presence bit.  The step index is read from device memory: graph-capturable as sk_select_next.
 * presence may be NULL when penalty == 1; scratch may be NULL when there are no n-gram or min-length bans. */
int sk_select_next_ex(const void* logits, int ldl, int V, int B, const uint32_t* ban_bits, const SkSampling* cfg,
                      const float* uniforms, const SkDecodeState* state, const SkLogitRules* rules, void* stream);
int sk_select_next_ex_f32(const float* logits, int ldl, int V, int B, const uint32_t* ban_bits, const SkSampling* cfg,
                          const float* uniforms, const SkDecodeState* state, const SkLogitRules* rules, void* stream);
/* presence[b] = the bitmap of history[b, 0 .. prompt_len) (ids outside [0, V) are skipped); overwrites every word. */
int sk_presence_init(const int64_t* history, int hist_ld, int prompt_len, int B, int V, uint32_t* presence, void* stream);

/* ---- sequence scoring (modelling metrics of cli/eval.py) ---------------------------------------------------------------
 * The tail of UnitLM.log_likelihood (slamkit/model/unit_lm.py:184-194 -> calc_nll, slamkit/utils/calculation_utils.py:5-29)
 * with the bf16 model's rounding: for logits z bf16 [B*T, ldl] (V valid columns; e.g. sk_lm_logits after sk_lm_forward with
 * labels = NULL) and tokens ids int64 [B,T], target y = ids[b, t+1] of logits row b*T + t:
 *   banned columns (ban_bits: uint32 [ceil(V/32)] bitmask as for sk_select_next, or NULL) are -inf;
 *   y == pad_id is masked: value 0, not counted, its logits row is not read;
 *   token_nll[b, t] = -bf16((z_y - max) - log(sum exp(z - max))) with fp32 max / sum over the non-banned columns
 *                     (+inf for a banned target);
 *   ll_out[b] (bf16) = -bf16(sum_t token_nll[b, t]), or with mean_nll -bf16(bf16(sum) / count) (NaN when count = 0).
 * Every logits element of an unmasked row is read once; columns >= V are never read.  token_nll: fp32 [B, T-1],
 * caller-owned (the per-sequence pass sums it in a fixed order).  No atomics: bit-identical run to run.  V in [2, 2^20],
 * ldl % 8 == 0, logits 16-byte aligned. */
int sk_seq_loglik(const void* logits, int ldl, int V, const int64_t* ids, int B, int T, int pad_id, const uint32_t* ban_bits,
                  int mean_nll, float* token_nll, void* ll_out, void* stream);
/* The same contract on fp32 logits of an fp32 model, as calc_nll runs on them: no bf16 rounding anywhere,
 *   token_nll[b, t] = -((z_y - max) - log(sum exp(z - max))),  ll_out[b] (fp32) = -sum_t, or -(sum / count). */
int sk_seq_loglik_f32(const float* logits, int ldl, int V, const int64_t* ids, int B, int T, int pad_id,
                      const uint32_t* ban_bits, int mean_nll, float* token_nll, float* ll_out, void* stream);
/* UnitTokeniser.tokenise on the device (slamkit/tokeniser/unit_tokeniser.py:40-73 with its `<S> $0 <S>` template): sk_rle's
 * units int32 [B, T_units] and counts int32 [B] -> right-padded ids int64 [B, T_out] = [bos, units + offset..., eos, pad...].
 * T_out = max(counts) + 2 gives the batch tokenise() builds. */
int sk_units_to_tokens(const int32_t* units, const int32_t* counts, int B, int T_units, int offset, int bos, int eos, int pad,
                       int64_t* ids, int T_out, void* stream);
/* InterleavingTokeniser.build_prompt (SPEECH output) on the device, left-padded: row b of ids int64 [B, T_out] is
 * [pad..., prefix[0 .. n_prefix), unit_id[units[b, j]] for j < counts[b], marker] and mask int64 [B, T_out] is 0 on the
 * pads, 1 elsewhere.  unit_id int32 [n_units] (device) maps unit u to the id of `<Un u>`; prefix int32 (device) holds what
 * the text tokenizer puts before a string.  T_out >= n_prefix + max(counts) + 1. */
int sk_units_to_prompt(const int32_t* units, const int32_t* counts, int B, int T_units, const int32_t* unit_id, int n_units,
                       const int32_t* prefix, int n_prefix, int marker, int pad, int64_t* ids, int64_t* mask, int T_out,
                       void* stream);
/* ---- HuBERT unit extraction (path (i)) ------------------------------------------------------------------------------
 * One object per device; replaces HubertFeatureExtractor.extract + batch_cluster
 * (slamkit/feature_extractor/hubert_feature_extractor.py:40-50,73-81): F.pad(40,40) -> HF HubertModel conv encoder,
 * projection, positional conv, `n_layers` encoder layers (= the reference's `layer`, hidden_states[layer]) -> k-means
 * labels -> rel_l trim.  Weights are one flat fp32 buffer in the "prepared" layout enumerated by sk_hubert_tensor_info:
 * conv{i}.w as [C_out, k*C_in] with (tap, in-channel) order, pos.w grouped/padded [G*64, K*64] with torch weight_norm
 * already folded, fused wqkv/bqkv, km.centers zero-padded to a multiple of 64 rows. */
typedef struct SkHubertConfig {
  int32_t n_conv;                /* 8 */
  int32_t conv_dim;              /* 512 */
  int32_t conv_kernel[8];        /* 10,3,3,3,3,2,2,2 */
  int32_t conv_stride[8];        /* 5,2,2,2,2,2,2,2 */
  int32_t hidden;                /* 768 */
  int32_t n_heads;               /* 12 (head_dim must be 64) */
  int32_t ffn;                   /* 3072 */
  int32_t n_layers;              /* encoder layers to RUN = config `layer` (11 for mhubert_25) */
  int32_t pos_conv_kernel;       /* 128 */
  int32_t pos_conv_groups;       /* 16 */
  int32_t n_units;               /* 500 */
  float ln_eps;                  /* 1e-5 */
  int32_t pad;                   /* 40 */
} SkHubertConfig;
typedef struct SkHubert SkHubert;

int sk_hubert_create(const SkHubertConfig* cfg, SkHubert** out);
void sk_hubert_destroy(SkHubert* h);
int64_t sk_hubert_param_count(const SkHubert* h);            /* fp32 elements of the flat weight buffer */
int sk_hubert_tensor_info(const SkHubert* h, int idx, char* name_buf, int name_cap, int64_t* offset, int32_t* rows,
                          int32_t* cols);                    /* idx < 0 -> number of tensors */
int sk_hubert_frames(const SkHubert* h, int S);              /* frames produced for S-sample clips (after the pad) */
int64_t sk_hubert_prepared_bytes(const SkHubert* h);         /* device scratch for the split (hi, lo) weight copies */
int64_t sk_hubert_workspace_bytes(const SkHubert* h, int B, int S);
int sk_hubert_bind(SkHubert* h, const float* weights, void* prepared, int64_t prepared_bytes, void* workspace,
                   int64_t workspace_bytes, void* stream);
/* wav fp32 [B,S] (device), lens int64 [B] or NULL; ids int32 [B, sk_hubert_frames(S)] (all frames, untrimmed),
 * n_frames int32 [B] = ceil(float32(lens)/S*T) (hubert_feature_extractor.py:46). */
int sk_hubert_units(SkHubert* h, const float* wav, const int64_t* lens, int B, int S, int32_t* ids, int32_t* n_frames,
                    void* stream);
/* the fp32 layer-`n_layers` features [B*T, hidden] (parity checks against hidden_states[layer]) */
int sk_hubert_features(SkHubert* h, const float* wav, int B, int S, float* feat, void* stream);
/* Test hook: run the pass up to one stage and return that stage as fp32. stage 100+i = conv layer i output
 * [B*T_i, conv_dim]; 200 = projection [B*T, hidden]; 201 = positional conv; 0..n_layers = hidden_states[stage];
 * 300 + 10 l + j = inside encoder layer l: j = 0 qkv projection [B*T, 3 hidden], 1 attention, 2 o-proj + residual,
 * 3 first LayerNorm, 4 GELU(ff1) [B*T, ffn], 5 ff2 + residual (each [B*T, hidden] unless given). */
int sk_hubert_debug_stage(SkHubert* h, const float* wav, int B, int S, int stage, float* out, void* stream);
/* Run-length dedup of each row's first n_frames[b] labels (UnitTokeniser.audio_represent,
 * slamkit/tokeniser/unit_tokeniser.py:57): units/durations int32 [B,T], counts int32 [B]. */
int sk_rle(const int32_t* ids, const int32_t* n_frames, int32_t* units, int32_t* durations, int32_t* counts, int B, int T,
           void* stream);
/* sklearn KMeans.predict tail (SK:cluster/_k_means_lloyd.pyx:198-213): labels = first argmin_j(sqnorm[j] - 2 dot[m][j]) */
int sk_row_sqnorm(const float* x, float* out, int rows, int D, void* stream);
int sk_kmeans_argmin(const float* dot, const float* centers_sqnorm, int32_t* labels, int M, int U, int ld, void* stream);
/* conv0 statistics buffer length (doubles per clip) */
int sk_conv0_nstat(void);

/* ---- HiFi-GAN unit vocoder ---------------------------------------------------------------------------------------------
 * CodeHiFiGANVocoder.forward (slamkit/vocoder/hifigan/vocoder.py:56-88 -> CodeGenerator, generator.py:95-197) in eval
 * mode with weight norm folded, fp32-grade: convolutions run as split-bf16 (hi*hi + hi*lo + lo*hi) implicit GEMMs on the
 * tensor cores.  speaker_id = style_id = 0, as vocode() passes them; f0 conditioning and embedder_params are not
 * supported.  Rows of a batch are packed on one timeline with zero gaps wide enough that a row's waveform is
 * bit-identical alone, in any batch and at any position.  Weights are one flat fp32 buffer enumerated by
 * sk_vocoder_tensor_info with the reference's state-dict names and torch shapes (ConvTranspose1d: [Cin, Cout, k]). */
typedef struct SkVocoderConfig {
  int32_t num_embeddings;            /* code vocabulary (500) */
  int32_t embedding_dim;             /* 128; a multiple of 4 */
  int32_t model_in_dim;              /* embedding_dim * (1 + multispkr + multistyle) */
  int32_t multispkr, num_speakers;
  int32_t multistyle, num_styles;
  int32_t upsample_initial_channel;  /* 512; every stage's channel count must be a multiple of 4 */
  int32_t n_upsamples;               /* 1..8 */
  int32_t upsample_rates[8];         /* rate u, kernel k: k - u even, k <= 32 */
  int32_t upsample_kernel_sizes[8];
  int32_t n_resblocks;               /* 1..4 ResBlocks per stage, averaged */
  int32_t resblock_kernel_sizes[4];  /* odd */
  int32_t resblock_dilations[4][3];
  int32_t dur_predictor;             /* 1: VariancePredictor durations (dur_prediction=True) */
  int32_t dur_hidden;                /* var_pred_hidden_dim */
  int32_t dur_kernel;                /* var_pred_kernel_size: only 3 */
  int32_t max_rows;                  /* workspace: rows per sub-batch */
  int32_t max_frames;                /* workspace: unit frames per sub-batch (summed over its rows) */
} SkVocoderConfig;
typedef struct SkVocoder SkVocoder;

int sk_vocoder_create(const SkVocoderConfig* cfg, SkVocoder** out);
void sk_vocoder_destroy(SkVocoder* v);
int64_t sk_vocoder_param_count(const SkVocoder* v);        /* fp32 elements of the flat weight buffer */
int sk_vocoder_tensor_info(const SkVocoder* v, int idx, char* name_buf, int name_cap, int64_t* offset,
                           int64_t* numel);                /* idx < 0 -> number of tensors */
int sk_vocoder_gap(const SkVocoder* v);                    /* zero frames between packed rows */
int sk_vocoder_upsampling(const SkVocoder* v);             /* output samples per unit frame (product of the rates) */
int64_t sk_vocoder_prepared_bytes(const SkVocoder* v);     /* device scratch for the split (hi, lo) conv weights */
int64_t sk_vocoder_workspace_bytes(const SkVocoder* v);    /* for (max_rows, max_frames) */
/* weights fp32 [sk_vocoder_param_count] stays referenced; the conv weights are split into `prepared` on `stream`. */
int sk_vocoder_bind(SkVocoder* v, const float* weights, void* prepared, int64_t prepared_bytes, void* workspace,
                    int64_t workspace_bytes, void* stream);
/* codes int64 [B, ld] with counts int32 [B] entries per row; negative codes are dropped.  B <= max_rows,
 * ld <= max_frames.  dur int32 [B, ld] (per kept unit, or NULL), log_dur fp32 [B, ld] (the predictor's value before
 * exp / round, or NULL), frames int32 [B] (frames per row).  status int32 [2]: {codes >= num_embeddings, rows with more
 * units than max_frames}; such codes are read as 0 and never index out of bounds. */
int sk_vocoder_durations(SkVocoder* v, const int64_t* codes, int ld, const int32_t* counts, int B, int32_t* dur,
                         float* log_dur, int32_t* frames, int32_t* status, void* stream);
/* wave fp32 [B, ldw]: row b's frames_host[b] * sk_vocoder_upsampling() samples, then zeros.  frames_host: the frames of
 * sk_vocoder_durations on the host (the caller reads them once to size wave); rows are vocoded in sub-batches of whole
 * rows that fit the workspace.  Codes must have passed sk_vocoder_durations with status {0, 0}. */
int sk_vocoder_run(SkVocoder* v, const int64_t* codes, int ld, const int32_t* counts, int B, const int32_t* frames_host,
                   float* wave, int64_t ldw, void* stream);
/* Test hook: one convolution layer run exactly as sk_vocoder_run runs it (the same weight preparation and launcher).
 * x fp32 [T_in, Cin] is staged through leaky_relu(., slope) (slope 1: identity).  A conv (transposed 0: rate 1, odd k,
 * padding (k - 1) * dilation / 2) gives T_out = T_in; a ConvTranspose1d (stride rate, padding (k - rate) / 2, k - rate
 * even) gives T_out = T_in * rate.  weight is torch's layout (Conv1d [Cout, Cin, k], ConvTranspose1d [Cin, Cout, k]),
 * bias fp32 [Cout].  Output position o is zero when valid[o / up] == 0 (uint8 [T_out / up]); else
 *   v = acc + bias;  v += res[o] (when res);  mode 2: v = sum[o] + v;  divide > 0: v = v / divide,
 * stored to y [T_out, Cout] in mode 0, or to sum [T_out, Cout] in modes 1 and 2 (y is not written).  prep: device scratch
 * of 2 * 2 * k * round_up(Cout, 64) * round_up(Cin, 32) bytes for the split bf16 weights.  Cin and Cout are multiples of 4;
 * every argument is checked before anything is launched. */
typedef struct SkVocoderConvDesc {
  int32_t T_in, Cin, Cout, k;
  int32_t transposed, rate, dilation;
  float slope;
  const float* x;
  const float* weight;
  const float* bias;
  const uint8_t* valid;
  int32_t up, mode;
  float* y;
  const float* res;
  float* sum;
  int32_t divide;
  void* prep;
  int64_t prep_bytes;
} SkVocoderConvDesc;
int sk_vocoder_conv(const SkVocoderConvDesc* desc, void* stream);

/* ---- host-side FLAC decoding (no audio decoder exists in the image) ------------------------------------------------
 * Replaces torchaudio.info / torchaudio.load in cli/extract_features.py:45-57.  Host pointers. md5_16 receives the
 * STREAMINFO MD5 of the unencoded audio (all zero if the encoder did not set it). */
int sk_flac_info(const char* path, int32_t* sample_rate, int32_t* channels, int32_t* bits_per_sample,
                 int64_t* n_samples, uint8_t* md5_16);
/* interleaved int32 PCM into a host buffer with room for `capacity` samples per channel */
int sk_flac_decode_i32(const char* path, int32_t* pcm_host, int64_t capacity, int64_t* n_decoded);

/* ---- data-parallel gradient all-reduce over NVLink peer memory (single NVSwitch node) ----------------------------------
 * Replaces the per-bucket NCCL all-reduce of accelerate's DDP wrapper around `training_step` (HF:trainer.py:1867-2014;
 * config/training_args/default.yaml:18) for ranks that share a node: every rank maps every other rank's flat bf16
 * gradient buffer and a small flag array with CUDA IPC, and one small-footprint kernel per bucket (128-thread CTAs of
 * <= 32 registers per thread, no shared memory: they co-reside with the GEMM / attention CTAs of the backward pass)
 * reduce-scatters and all-gathers in one pass -- rank r sums the W copies of its 1/W of the bucket in rank order (fp32,
 * one rounding: bit-identical on all ranks) and stores the result into all W buffers.  Protocol per bucket (all on one side stream):
 *   sk_p2p_signal(slot, epoch)  this rank's gradients of the bucket are final (READY flag to every peer)
 *   sk_p2p_allreduce_bf16(...)  waits for every peer's READY, reduces, tells every peer when its share is written
 *   sk_p2p_wait(slots, epoch)   returns (in stream order) when every peer's share of those slots has arrived in this
 *                               rank's buffer (one call may cover all buckets of a step)
 * `epoch` must grow by one per reduction of a slot; flags are never reset.  `bufs` / `flags`: arrays of `world` device
 * pointers (own memory at [rank], IPC mappings elsewhere); ranges in bf16 elements, multiples of 8.  `err_flag`: int in
 * pinned host memory, set non-zero when a spin timed out (a peer died): check it after synchronising. */
int64_t sk_p2p_flag_bytes(void);
int sk_p2p_alloc(int64_t bytes, void** out);                 /* zeroed cudaMalloc (flag arrays) */
int sk_p2p_free(void* p);
int sk_p2p_export(const void* ptr, void* handle64, int64_t* offset);   /* IPC handle of the allocation holding ptr */
int sk_p2p_open(const void* handle64, void** base);
int sk_p2p_close(void* base);
int sk_p2p_signal(void* const* flags, int rank, int world, int slot, uint32_t epoch, void* stream);
int sk_p2p_allreduce_bf16(void* const* bufs, void* const* flags, int rank, int world, int64_t offset_elems, int64_t n_elems,
                          int slot, uint32_t epoch, int ctas, int* err_flag, void* stream);
int sk_p2p_wait(void* const* flags, int rank, int world, int slot_lo, int n_slots, uint32_t epoch, int* err_flag, void* stream);
/* Profiling hook: uint64 [257][4] device buffer that the kernels above fill with %globaltimer stamps per slot (0 READY sent,
 * 1 reduce kernel running, 2 peers ready, 3 last CTA done; row 256: wait kernel start / end); NULL switches it off. */
int sk_p2p_set_trace(void* buf);
/* Test hook: `ctas` CTAs with the reduce kernel's footprint (128 threads, <= 32 registers, no shared memory) that hold their
 * slot for `ns` nanoseconds; started_u32 counts the CTAs that got onto an SM. */
int sk_p2p_debug_hog(int ctas, int64_t ns, void* started_u32, void* stream);

/* number of kernels this library launched since load (bench.py's gpu_launches) */
int64_t sk_launch_count(void);
/* Bench-only device timing: when enabled, CUDA events are recorded on the launching stream around every launch of
 * category 0 (GEMM), 1 (attention), 2 (optimiser).  sk_prof_collect synchronises the device and returns the
 * summed milliseconds and launch-group counts per category (arrays of 4), then resets. */
int sk_prof_enable(int on);
int sk_prof_collect(double* ms_by_cat, int64_t* count_by_cat);

#ifdef __cplusplus
}
#endif
#endif /* SLAMKIT_B200_H */
