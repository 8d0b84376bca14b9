// Internal C++ launcher declarations shared by api.cu / lm_step.cu / hubert_step.cu.
// (The public, C-ABI surface is include/slamkit_b200.h.)
#pragma once
#include "common.cuh"

// gemm_tcgen05.cu
int sk_make_tmap_2d(CUtensorMap* out, const void* ptr, int elem_bytes, uint64_t inner, uint64_t outer, uint64_t ld,
                    uint32_t box_inner, uint32_t box_outer);
int sk_make_tmap_3d(CUtensorMap* out, const void* ptr, uint64_t inner, uint64_t rows, uint64_t batch, uint64_t row_stride,
                    uint64_t batch_stride, uint32_t box_rows);
int sk_pick_bn(int M, int N, int force_bn, bool fit_forced, bool fit, bool whole_heads);
size_t sk_gemm_ws_min_bytes(void);   // scratch size that enables stream-K (last 4 KB = flag words, zero on first use)
// SkGemmEx::act
constexpr int SK_ACT_NONE = 0, SK_ACT_GELU = 1, SK_ACT_RELU = 2;
// SkGemmEx::epi, the fused epilogues of the LM step (0 = none):
//   SwiGLU forward : B = gate/up weight in [128 gate rows | 128 up rows] blocks, N = 2F; C = gu [M,2F] (same block
//                    layout) and aux_out = act [M,F] = bf16(bf16(silu(gate)) * up)
//   SwiGLU backward: N = F, acc = d_act; aux = gu [M,2F]; C = d_gu [M,2F] (ldc = its pitch)
//   bias + RoPE    : 64-column heads with column < rope_cols are rotated with cos/sin[pos] (pos = rope_pos[row] or
//                    row % rope_T, clamped to [0, rope_maxpos)); the first rope_rot columns of each head rotate
//                    (0 or 64: the whole head, tables [maxpos, 32]; 16 / 32: partial rotary, tables [maxpos, rope_rot/2])
//   GELU forward   : C = pre = bf16(acc + bias) and aux_out = bf16(gelu_erf(pre)) (same shape, ld_aux_out)
//   GELU backward  : acc = d_act; aux = the saved pre; C = bf16(bf16(acc) * gelu'(pre))
//   two residuals  : C = bf16(bf16(bf16(acc + bias) + aux) + residual) (GPT-NeoX parallel residual: mlp + attn + x)
constexpr int SK_EPI_SWIGLU_FWD = 1, SK_EPI_SWIGLU_BWD = 2, SK_EPI_BIAS_ROPE = 3, SK_EPI_GELU_FWD = 4,
              SK_EPI_GELU_BWD = 5, SK_EPI_RES2 = 6;
// Extended GEMM description (HuBERT path): batched / strided-window A operands (convolutions as GEMMs without an
// im2col copy), split-bf16 3-pass accumulation, fp32 bias, hi/lo residual and outputs, grouped column compaction.
// The sk_gemm_* builders below fill it for each kind of GEMM the library launches.
struct SkGemmEx {
  int M, N, K;              // M: rows per batch item
  int batch;                // >= 1
  int a_mode;               // 0 plain, 1 shifted-window grouped conv (BN = 64 = one channel group per N tile)
  int passes;               // 1 or 3
  const void *A, *A_lo;
  int lda, a_mn;
  long a_inner, a_rows, a_row_stride, a_batch_stride;   // 3-D A view (elements), active when a_rows > 0
  const void *B, *B_lo;
  int ldb, b_mn;
  void *C, *C_lo;
  int ldc, out_f32;
  const void* bias;
  int bias_f32;
  const void *residual, *residual_lo;
  int ldr, round_before_res, act;
  int col_gin, col_gout;
  int force_bn;
  void* splitk_ws;          // optional scratch: deterministic split-K (few tiles, long K) and stream-K load balancing
  size_t splitk_ws_bytes;
  int pdl;                  // 1: launch with programmatic stream serialization (the LM step's short back-to-back GEMMs)
  int epi;                  // fused epilogue of the LM step: SK_EPI_* (0 = none)
  const void* aux;
  int ld_aux;
  void* aux_out;
  int ld_aux_out;
  const void *rope_cos, *rope_sin;
  const int* rope_pos;
  int rope_T, rope_cols, rope_maxpos;
  int rope_rot;
};
int sk_gemm_ex_launch(const SkGemmEx& g, cudaStream_t stream);
struct SkGemmPlan;
int sk_gemm_plan_ex(const SkGemmEx& g, SkGemmPlan* out);   // the decisions sk_gemm_ex_launch makes for g, nothing launched

// ---- descriptor builders: host-only, no CUDA call.  A residual's pitch (ldr) and round_before_res are set only
// together with the residual.
// A zeroed one-pass M x N x K descriptor, the start of every builder
inline SkGemmEx sk_gemm_base(int M, int N, int K) {
  SkGemmEx g{};
  g.M = M; g.N = N; g.K = K; g.batch = 1; g.passes = 1;
  return g;
}
// The plain GEMM of the C ABI (sk_gemm_bf16*, sk_gemm_plan).  A: [M,K] (a_mn=0, lda = row pitch of the [M,K] array) or
// stored [K,M] (a_mn=1, lda = row pitch of the [K,M] array).  B: [N,K] (b_mn=0) or stored [K,N] (b_mn=1).
inline SkGemmEx sk_gemm_desc(int M, int N, int K, const void* A, int lda, int a_mn, const void* B, int ldb, int b_mn, void* C,
                             int ldc, int out_f32, const void* bias, const void* residual, int ldr, int round_before_res,
                             int act, int force_bn, void* splitk_ws, size_t splitk_ws_bytes) {
  SkGemmEx g = sk_gemm_base(M, N, K);
  g.A = A; g.lda = lda; g.a_mn = a_mn;
  g.B = B; g.ldb = ldb; g.b_mn = b_mn;
  g.C = C; g.ldc = ldc; g.out_f32 = out_f32;
  g.bias = bias; g.residual = residual; g.ldr = ldr; g.round_before_res = round_before_res; g.act = act;
  g.force_bn = force_bn;
  g.pdl = 1;
  g.splitk_ws = splitk_ws;
  g.splitk_ws_bytes = splitk_ws_bytes;
  return g;
}
// The linears of the LM step (launched with programmatic stream serialization).
// y[M,N] (pitch ldy) = act(x[M,K] W[N,K]^T + bias) (+ res, same pitch as y, added to the bf16-rounded product)
inline SkGemmEx sk_gemm_linear(int M, int N, int K, const void* x, const void* W, void* y, int ldy, const void* bias,
                               const void* res, int act, void* splitk_ws = nullptr, size_t splitk_ws_bytes = 0) {
  SkGemmEx g = sk_gemm_base(M, N, K);
  g.A = x; g.lda = K;
  g.B = W; g.ldb = K;
  g.C = y; g.ldc = ldy;
  g.bias = bias;
  if (res) { g.residual = res; g.ldr = ldy; g.round_before_res = 1; }
  g.act = act;
  g.pdl = 1;
  g.splitk_ws = splitk_ws;
  g.splitk_ws_bytes = splitk_ws_bytes;
  return g;
}
// dx[M,K] = dy[M,N] W[N,K] (+ res [M,K], added to the bf16-rounded product)
inline SkGemmEx sk_gemm_dgrad(int M, int N, int K, const void* dy, const void* W, void* dx, const void* res = nullptr) {
  SkGemmEx g = sk_gemm_base(M, K, N);
  g.A = dy; g.lda = N;
  g.B = W; g.ldb = K; g.b_mn = 1;
  g.C = dx; g.ldc = K;
  if (res) { g.residual = res; g.ldr = K; g.round_before_res = 1; }
  g.pdl = 1;
  return g;
}
// dW[N,K] (+)= dy[M,N]^T x[M,K]; accumulating adds the bf16-rounded product to dW.  Scratch: split-K for the small
// weight gradients, stream-K balancing for the large ones
inline SkGemmEx sk_gemm_wgrad(int M, int N, int K, const void* dy, const void* x, void* dW, bool accumulate, void* splitk_ws,
                              size_t splitk_ws_bytes) {
  SkGemmEx g = sk_gemm_base(N, K, M);
  g.A = dy; g.lda = N; g.a_mn = 1;
  g.B = x; g.ldb = K; g.b_mn = 1;
  g.C = dW; g.ldc = K;
  if (accumulate) { g.residual = dW; g.ldr = K; g.round_before_res = 1; }
  g.pdl = 1;
  g.splitk_ws = splitk_ws;
  g.splitk_ws_bytes = splitk_ws_bytes;
  return g;
}
// gu[M,2F] = x[M,K] * Wgu[2F,K]^T with Wgu (and gu) in [128 gate | 128 up] blocks, and act[M,F] = bf16(bf16(silu(gate)) * up)
// written by the same epilogue (HF Qwen2MLP, HF:models/qwen2/modeling_qwen2.py:35-48)
inline SkGemmEx sk_gemm_swiglu_fwd(int M, int F, int K, const void* x, const void* Wgu, void* gu, void* act) {
  SkGemmEx g = sk_gemm_linear(M, 2 * F, K, x, Wgu, gu, 2 * F, nullptr, nullptr, SK_ACT_NONE);
  g.epi = SK_EPI_SWIGLU_FWD; g.aux_out = act; g.ld_aux_out = F;
  return g;
}
// d_gu[M,2F] from d_act = dy[M,N] * Wd[N,F] without materialising d_act: the epilogue turns each accumulator tile into
// d_gate / d_up with the saved gu (autograd of the SwiGLU above, same bf16 rounding points as the unfused kernels)
inline SkGemmEx sk_gemm_swiglu_bwd(int M, int N, int F, const void* dy, const void* Wd, const void* gu, void* dgu) {
  SkGemmEx g = sk_gemm_dgrad(M, N, F, dy, Wd, dgu);
  g.ldc = 2 * F;
  g.epi = SK_EPI_SWIGLU_BWD; g.aux = gu; g.ld_aux = 2 * F;
  return g;
}
// out[M,N] = x[M,K] * W[N,K]^T + bias, 64-column heads below rope_cols rotated in the epilogue (HF apply_rotary_pos_emb,
// HF:models/qwen2/modeling_qwen2.py:102-146); rope_rot: rotated columns per head (0 = all 64)
inline SkGemmEx sk_gemm_rope(int M, int N, int K, const void* x, const void* W, const void* bias, void* out, const void* cos_t,
                             const void* sin_t, const int32_t* pos_ids, int T, int rope_cols, int max_positions, int rope_rot) {
  SkGemmEx g = sk_gemm_linear(M, N, K, x, W, out, N, bias, nullptr, SK_ACT_NONE);
  g.epi = SK_EPI_BIAS_ROPE; g.rope_cos = cos_t; g.rope_sin = sin_t; g.rope_pos = pos_ids; g.rope_T = T;
  g.rope_cols = rope_cols; g.rope_maxpos = max_positions; g.rope_rot = rope_rot;
  return g;
}
// GPT-NeoX MLP (HF GPTNeoXMLP): pre[M,F] = bf16(x W1^T + b1) and act = bf16(gelu(pre)) from one epilogue
inline SkGemmEx sk_gemm_gelu_fwd(int M, int F, int K, const void* x, const void* W1, const void* b1, void* pre, void* act) {
  SkGemmEx g = sk_gemm_linear(M, F, K, x, W1, pre, F, b1, nullptr, SK_ACT_NONE);
  g.epi = SK_EPI_GELU_FWD; g.aux_out = act; g.ld_aux_out = F;
  return g;
}
// d_pre[M,F] = bf16(bf16(dy W2) * gelu'(pre)): d_act never reaches memory
inline SkGemmEx sk_gemm_gelu_bwd(int M, int N, int F, const void* dy, const void* W2, const void* pre, void* dpre) {
  SkGemmEx g = sk_gemm_dgrad(M, N, F, dy, W2, dpre);
  g.epi = SK_EPI_GELU_BWD; g.aux = pre; g.ld_aux = F;
  return g;
}
// out[M,N] = bf16(bf16(bf16(x W^T + bias) + res2) + res): GPT-NeoX's `mlp_output + attn_output + hidden_states`, rounded
// at each add in that order.  out may alias res (each element reads its residuals before it is stored).
inline SkGemmEx sk_gemm_res2(int M, int N, int K, const void* x, const void* W, const void* bias, const void* res2,
                             const void* res, void* out, void* splitk_ws = nullptr, size_t splitk_ws_bytes = 0) {
  SkGemmEx g = sk_gemm_linear(M, N, K, x, W, out, N, bias, res, SK_ACT_NONE, splitk_ws, splitk_ws_bytes);
  g.epi = SK_EPI_RES2; g.aux = res2; g.ld_aux = N;
  return g;
}
// The fp32-grade linear of the HuBERT encoder and of fp32 OPT inference: y[M,N] = act(x[M,K] W[N,K]^T + bias) (+ res),
// split-bf16 3-pass on (hi, lo) pairs of x and W, fp32 bias (or none), optional (hi, lo) residual [M, N]; the result as a
// (hi, lo) pair y_hi / y_lo, or fp32 into y32 when y32 is given; output pitch ldy.
inline SkGemmEx sk_gemm_linear_split(int M, int N, int K, const bf16* x_hi, const bf16* x_lo, const bf16* w_hi,
                                     const bf16* w_lo, const float* bias, int act, const bf16* res_hi, const bf16* res_lo,
                                     bf16* y_hi, bf16* y_lo, float* y32, int ldy) {
  SkGemmEx g = sk_gemm_base(M, N, K);
  g.passes = 3;
  g.A = x_hi; g.A_lo = x_lo; g.lda = K;
  g.B = w_hi; g.B_lo = w_lo; g.ldb = K;
  if (y32) { g.C = y32; g.out_f32 = 1; } else { g.C = y_hi; g.C_lo = y_lo; }
  g.ldc = ldy;
  if (bias) { g.bias = bias; g.bias_f32 = 1; }
  if (res_hi) { g.residual = res_hi; g.residual_lo = res_lo; g.ldr = N; }
  g.act = act;
  return g;
}

// lm_kernels.cu
int sk_embed_fwd_launch(const int64_t* ids, const bf16* E, bf16* out, int M, int D, int V, cudaStream_t s);
int sk_embed_bwd_launch(const int64_t* ids, const bf16* dx, float* scratch, bf16* dE, int M, int D, int V, int Vpad,
                        int accumulate, cudaStream_t s);
int sk_rmsnorm_fwd_launch(const bf16* x, const bf16* w, bf16* y, float* rstd, int M, int D, float eps, cudaStream_t s);
extern "C" int sk_rmsnorm_bwd_blocks(void);
int sk_rmsnorm_bwd_launch(const bf16* dy, const bf16* x, const bf16* w, const float* rstd, const bf16* dres, bf16* dx,
                          bf16* dw, float* dw_partial, int M, int D, int accumulate_dw, cudaStream_t s);
extern "C" int sk_colsum_splits(void);
int sk_colsum_launch(const bf16* x, bf16* out, float* partial, int M, int N, int ld, int accumulate, cudaStream_t s);
// rot_dims: rotated columns per head (0 = head_dim; 16 / 32 for head_dim 64: partial rotary, tables [max_pos, rot_dims/2])
int sk_rope_launch(bf16* qkv, const bf16* cos_t, const bf16* sin_t, const int* pos_ids, int M, int T, int ld,
                   int n_rot_heads, int head_dim, int inverse, int max_positions, cudaStream_t s, int rot_dims = 0);
int sk_swiglu_fwd_launch(const bf16* gu, bf16* act, int M, int F, cudaStream_t s);
int sk_swiglu_bwd_launch(const bf16* gu, const bf16* dact, bf16* dgu, int M, int F, cudaStream_t s);
extern "C" int sk_ce_blocks(int M);
int sk_ce_launch(const bf16* logits, const int64_t* labels, bf16* dlogits, float* partial, float* row_nll,
                 float* stats_out, int M, int T, int V, int ldl, float num_items, float dloss, cudaStream_t s,
                 const float* row_weight = nullptr);
int sk_ce_chunk_launch(const bf16* logits_chunk, const int64_t* labels, bf16* dlogits_chunk, float* partial, int row0, int rows,
                       int M, int T, int V, int ldl, float grad_scale, cudaStream_t s);
int sk_ce_finalize_launch(const float* partial, int M, float num_items, float* stats_out, cudaStream_t s);
int sk_gradnorm_launch(const bf16* g, const long* chunk_start, const int* chunk_len, int n_chunks,
                       const int* tensor_chunk_begin, int n_tensors, float* partial, float max_norm, int emulate_bf16,
                       float* stats_out, cudaStream_t s);
int sk_adamw_launch(bf16* p, const bf16* g, bf16* m, bf16* v, long n, float lr, float beta1, float beta2, float eps,
                    float wd, int step, const float* clip_stats, cudaStream_t s);
int sk_transpose_launch(const bf16* in, bf16* out, int M, int N, cudaStream_t s);
int sk_seg_bounds_launch(const int32_t* pos_ids, int32_t* seg_start, int32_t* seg_end, int B, int T, cudaStream_t s);
// OPT decoder: LayerNorm (fp32 mean / rstd per row saved by the forward), token + learned position embedding
// (table row = position + 2, clamped), the position-table gradient in the embedding's 64-bit fixed point, ReLU backward
int sk_layernorm_fwd_launch(const bf16* x, const bf16* w, const bf16* b, bf16* y, float* mean, float* rstd, int M, int D,
                            float eps, cudaStream_t s);
extern "C" int sk_layernorm_bwd_blocks(void);
int sk_layernorm_bwd_launch(const bf16* dy, const bf16* x, const bf16* w, const float* mean, const float* rstd, const bf16* dres,
                            bf16* dx, bf16* dw, bf16* db, float* dw_partial, float* db_partial, int M, int D, int accumulate,
                            cudaStream_t s);
int sk_opt_embed_fwd_launch(const int64_t* ids, const int32_t* pos_ids, const bf16* E, const bf16* P, bf16* out, int M, int T, int D,
                            int V, int n_pos, cudaStream_t s);
int sk_opt_pos_bwd_launch(const int32_t* pos_ids, const bf16* dx, float* scratch, bf16* dP, int M, int T, int D, int n_pos,
                          int accumulate, cudaStream_t s);
int sk_relu_bwd_launch(bf16* g, const bf16* a, long n, cudaStream_t s);
// OPT with fp32 master weights (autocast numerics): the fp32 embedding sum, the fused residual add + LayerNorm of the
// fp32 residual stream, its backward into an fp32 residual gradient (plus a bf16 copy) with fp32 dw / db (partial:
// 2 x sk_layernorm_bwd_blocks() x D floats), table gradients from fp32 rows into fp32, the widening of bf16 linear
// gradients into the fp32 gradient buffer, the fp32 gradient norm and AdamW on the fp32 masters
int sk_opt_embed_fwd_f32_launch(const int64_t* ids, const int32_t* pos_ids, const float* E, const float* P, float* out, int M,
                                int T, int D, int V, int n_pos, cudaStream_t s);
int sk_add_layernorm_f32_launch(const float* x, const bf16* y, const float* w, const float* b, float* xo, bf16* h, float* mean,
                                float* rstd, int M, int D, float eps, cudaStream_t s);
int sk_layernorm_bwd_f32_launch(const bf16* dy, const float* x, const float* w, const float* mean, const float* rstd,
                                const float* dres_in, float* dres_out, bf16* dres16, float* dw, float* db, float* partial, int M,
                                int D, int accumulate, cudaStream_t s);
int sk_table_bwd_f32_launch(const int64_t* ids, const int32_t* pos_ids, const float* dx, float* scratch, float* dtable,
                            const bf16* head, int M, int T, int D, int n_rows, int n_rows_padded, int keep, cudaStream_t s);
int sk_widen_grads_launch(const bf16* g16, float* g32, const long* chunk_start, const int* chunk_len, int n_chunks, int keep,
                          cudaStream_t s);
int sk_gradnorm_f32_launch(const float* g, const long* chunk_start, const int* chunk_len, int n_chunks,
                           const int* tensor_chunk_begin, int n_tensors, float* partial, float max_norm, float* stats_out,
                           cudaStream_t s);
int sk_adamw_master_launch(float* p, bf16* shadow, const float* g, float* m, float* v, long n, float lr, float beta1, float beta2,
                           float eps, float wd, int step, const float* clip_stats, cudaStream_t s);
// GPT-NeoX parallel residual: ln1(x) and ln2(x) from one read of x (shared fp32 mean / rstd), and the fused backward
// dx = dres + LN'(w1 * dy1 + w2 * dy2) with the four deterministic parameter gradients (partial: 4 x
// sk_layernorm_bwd_blocks() x D floats)
int sk_layernorm2_fwd_launch(const bf16* x, const bf16* w1, const bf16* b1, const bf16* w2, const bf16* b2, bf16* y1, bf16* y2,
                             float* mean, float* rstd, int M, int D, float eps, cudaStream_t s);
int sk_layernorm2_bwd_launch(const bf16* dy1, const bf16* dy2, const bf16* x, const bf16* w1, const bf16* w2, const float* mean,
                             const float* rstd, const bf16* dres, bf16* dx, bf16* dw1, bf16* db1, bf16* dw2, bf16* db2,
                             float* partial, int M, int D, int accumulate, cudaStream_t s);

// attention.cu
int sk_attn_fwd_launch(const bf16* q, const bf16* k, const bf16* v, bf16* o, float* lse, int B, int T, int H, int KVH,
                       int ld, int ldo, int causal, float scale, cudaStream_t s, const int* seg_start = nullptr);
int sk_attn_bwd_launch(const bf16* q, const bf16* k, const bf16* v, const bf16* o, const bf16* d_o, const float* lse,
                       float* delta, bf16* dq, bf16* dk, bf16* dv, int B, int T, int H, int KVH, int ld, int ldo,
                       int ldg, int causal, float scale, cudaStream_t s, const int* seg_start = nullptr);
int sk_attn_fwd_split_launch(const bf16* q_hi, const bf16* q_lo, const bf16* k_hi, const bf16* k_lo, const bf16* v_hi,
                             const bf16* v_lo, bf16* o_hi, bf16* o_lo, int B, int T, int H, int ld, int ldo, float scale,
                             cudaStream_t s, int causal = 0);

// attention.cu: entry points on the fused q|k|v projection (LM step, HuBERT encoder)
int sk_attn_tc_fwd_split_launch(const bf16* qkv_hi, const bf16* qkv_lo, bf16* o_hi, bf16* o_lo, int B, int T, int H, int ld,
                                int ldo, float scale, cudaStream_t s, int causal = 0);
// seg_start / seg_end (optional, int32 [B*T]): in-row index of the first token of each token's document and one past
// its last -- block-diagonal causal attention for packed batches (sk_seg_bounds_launch builds them from position_ids)
int sk_attn_tc_bwd_launch(const bf16* qkv, const bf16* o, const bf16* d_o, const float* lse, float* delta, float* partial,
                          bf16* dqkv, int B, int T, int H, int KVH, int ld, int ldo, int ldg, int causal, float scale,
                          cudaStream_t s, const int* seg_start = nullptr, const int* seg_end = nullptr,
                          // optional: apply the inverse rotary embedding to dq / dk on the way out (bf16 [max_pos, 32] tables)
                          const bf16* rope_cos = nullptr, const bf16* rope_sin = nullptr, const int* pos_ids = nullptr,
                          int max_pos = 0);
int sk_attn_tc_fwd_launch(const bf16* qkv, bf16* o, float* lse, int B, int T, int H, int KVH, int ld, int ldo, int causal,
                          float scale, cudaStream_t s, const int* seg_start = nullptr);

// decode.cu: KV cache, decode attention and token selection of incremental decoding (cache layout per layer:
// [K|V][B][KVH][T_cache][64] bf16)
int sk_kv_prefill_launch(const bf16* qkv, long layer_stride, int ldq, bf16* cache, const int32_t* lens, int L, int B, int T,
                         int H, int KVH, int T_cache, cudaStream_t s);
int sk_kv_append_launch(const bf16* qkv, int ldq, bf16* kc, bf16* vc, const int32_t* pos, int32_t* lens, int B, int H,
                        int KVH, int T_cache, cudaStream_t s);
int sk_gather_last_launch(const bf16* x, const int32_t* lens, bf16* out, int B, int T, int D, cudaStream_t s);
// rows ids[0 .. n) of src [V, K] into dst [n_pad, K], zero rows after them (the compact head of sk_lm_gather_head)
int sk_gather_rows_launch(const bf16* src, const int32_t* ids, int n, int n_pad, int V, int K, bf16* dst, cudaStream_t s);
// fp32 OPT inference: an fp32 cache ([K|V][B][H][T_cache][64] per layer) filled from the (hi, lo) projections of one layer,
// decode attention with a (hi, lo) query and output
int sk_kv_prefill_f32_launch(const bf16* qkv_hi, const bf16* qkv_lo, int ldq, float* cache, const int32_t* lens, int B, int T,
                             int H, int T_cache, cudaStream_t s);
int sk_kv_append_f32_launch(const bf16* qkv_hi, const bf16* qkv_lo, int ldq, float* kc, float* vc, const int32_t* pos,
                            int32_t* lens, int B, int H, int T_cache, cudaStream_t s);
int sk_attn_decode_f32_launch(const bf16* q_hi, const bf16* q_lo, int ldq, const float* kc, const float* vc, const int32_t* lens,
                              bf16* o_hi, bf16* o_lo, int ldo, float* partial, int B, int H, int T_cache, float scale,
                              cudaStream_t s);
int sk_attn_decode_splits(int T_cache);
int sk_attn_decode_launch(const bf16* q, int ldq, const bf16* kc, const bf16* vc, const int32_t* lens, bf16* o, int ldo,
                          float* partial, int B, int H, int KVH, int T_cache, float scale, cudaStream_t s);
int sk_kv_fanout_launch(const void* src, void* dst, const int32_t* lens, int L, int B, int k, int KVH, int T_cache,
                        int row_bytes, cudaStream_t s);
struct SkSampling;
struct SkDecodeState;
int sk_select_next_launch(const bf16* logits, int ldl, int V, int B, const uint32_t* ban, const SkSampling& cfg,
                          const float* uniforms, const SkDecodeState& st, cudaStream_t s);

// hubert_kernels.cu
int sk_split_f32_launch(const float* x, bf16* hi, bf16* lo, long n, cudaStream_t s);
extern "C" int sk_conv0_nstat(void);
int sk_conv0_launch(const float* wav, const float* w, const float* gamma, const float* beta, double* stats,
                    float2* affine, bf16* out_hi, bf16* out_lo, int B, int S, int pad, int T0, int C, int KW, int ST,
                    float eps, cudaStream_t s);
int sk_layernorm_hilo_launch(const bf16* a_hi, const bf16* a_lo, const bf16* b_hi, const bf16* b_lo, const float* gamma,
                             const float* beta, bf16* o_hi, bf16* o_lo, float* o_f32, int M, int D, float eps,
                             cudaStream_t s);
int sk_regroup_pad_launch(const bf16* in_hi, const bf16* in_lo, bf16* out_hi, bf16* out_lo, int B, int T, int halo,
                          int G, int cg, int cgp, cudaStream_t s);
int sk_row_sqnorm_launch(const float* c, float* out, int U, int D, cudaStream_t s);
int sk_kmeans_argmin_launch(const float* dot, const float* csq, int32_t* labels, int M, int U, int ld, cudaStream_t s);
int sk_rle_launch(const int32_t* labels, const int32_t* n_frames, int32_t* units, int32_t* durations, int32_t* counts,
                  int B, int T, cudaStream_t s);
int sk_rel_len_launch(const int64_t* lens, int32_t* n_frames, int B, int S, int T, cudaStream_t s);
int sk_hilo_to_f32_launch(const bf16* hi, const bf16* lo, float* out, long n, cudaStream_t s);

// p2p_comm.cu: bf16 gradient all-reduce over CUDA-IPC peer memory (one NVSwitch node)
size_t sk_p2p_flag_bytes_impl();
int sk_p2p_set_trace_impl(void* buf);
int sk_p2p_hog_launch(int ctas, long long ns, unsigned* started, cudaStream_t s);
int sk_p2p_alloc_impl(size_t bytes, void** out);
int sk_p2p_free_impl(void* p);
int sk_p2p_export_impl(const void* ptr, void* handle64, size_t* offset);
int sk_p2p_open_impl(const void* handle64, void** base);
int sk_p2p_close_impl(void* base);
int sk_p2p_signal_launch(void* const* flags, int rank, int world, int slot, uint32_t epoch, cudaStream_t s);
int sk_p2p_wait_launch(void* const* flags, int rank, int world, int slot_lo, int n_slots, uint32_t epoch, int* err_flag, cudaStream_t s);
int sk_p2p_allreduce_launch(void* const* bufs, void* const* flags, int rank, int world, size_t offset_elems, size_t n_elems,
                            int slot, uint32_t epoch, int ctas, int* err_flag, cudaStream_t s);
