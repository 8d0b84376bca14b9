// extern "C" surface of libslamkit_b200.so for the op-level entry points (see include/slamkit_b200.h), plus the
// error / device-info plumbing.  The handle-level entry points live in lm_step.cu and hubert_step.cu.
#include <stdlib.h>
#include "kernels.h"
#include "../../include/slamkit_b200.h"
#include <atomic>
#include <stdarg.h>
#include <stdio.h>
#include <string.h>
#include <vector>

namespace {
thread_local char g_err[1024] = "";
std::atomic<long long> g_launches{0};
}  // namespace

void sk_set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
bool sk_pdl_enabled() {
  static const bool on = [] { const char* e = getenv("SK_PDL"); return e ? atoi(e) != 0 : true; }();
  return on;
}
void sk_count_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }

// ---- optional per-category device timing (bench.py's roofline leg): CUDA events recorded around the launches of one
// category on the launching stream.  Off by default; never active inside bench.py's timed region.
namespace {
constexpr int PROF_CATS = 4;
constexpr int PROF_MAX = 8192;
bool g_prof_on = false;
std::vector<cudaEvent_t> g_prof_ev;
std::vector<int> g_prof_cat;
int g_prof_used = 0;
}  // namespace
void sk_prof_begin(int cat, cudaStream_t s) {
  if (!g_prof_on || g_prof_used + 2 > PROF_MAX) return;
  cudaEventRecord(g_prof_ev[g_prof_used], s);
  g_prof_cat[g_prof_used / 2] = cat;
  g_prof_used += 1;
}
void sk_prof_end(cudaStream_t s) {
  if (!g_prof_on || (g_prof_used & 1) == 0) return;
  cudaEventRecord(g_prof_ev[g_prof_used], s);
  g_prof_used += 1;
}

int sk_num_sms() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess ||
        cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0)
      n = 132;   // H100 SXM
  }
  return n;
}

#define S(x) ((cudaStream_t)(x))
#define BF(x) (reinterpret_cast<bf16*>(x))
#define CBF(x) (reinterpret_cast<const bf16*>(x))

extern "C" {

const char* sk_last_error(void) { return g_err; }
int sk_version(void) { return 1; }
int sk_device_sm_count(void) { return sk_num_sms(); }
int sk_device_cc(void) {
  int dev = 0, ma = 0, mi = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return -2;
  cudaDeviceGetAttribute(&ma, cudaDevAttrComputeCapabilityMajor, dev);
  cudaDeviceGetAttribute(&mi, cudaDevAttrComputeCapabilityMinor, dev);
  return 10 * ma + mi;
}
int64_t sk_launch_count(void) { return (int64_t)g_launches.load(); }

int sk_prof_enable(int on) {
  if (on && g_prof_ev.empty()) {
    g_prof_ev.resize(PROF_MAX);
    g_prof_cat.resize(PROF_MAX / 2);
    for (int i = 0; i < PROF_MAX; ++i) SK_CUDA_CHECK(cudaEventCreate(&g_prof_ev[i]));
  }
  g_prof_on = on != 0;
  g_prof_used = 0;
  return 0;
}
int sk_prof_collect(double* ms_by_cat, int64_t* count_by_cat) {
  SK_CUDA_CHECK(cudaDeviceSynchronize());
  for (int c = 0; c < PROF_CATS; ++c) { ms_by_cat[c] = 0.0; count_by_cat[c] = 0; }
  for (int i = 0; i + 1 < g_prof_used; i += 2) {
    float ms = 0.f;
    SK_CUDA_CHECK(cudaEventElapsedTime(&ms, g_prof_ev[i], g_prof_ev[i + 1]));
    const int c = g_prof_cat[i / 2];
    if (c >= 0 && c < PROF_CATS) { ms_by_cat[c] += ms; count_by_cat[c] += 1; }
  }
  g_prof_used = 0;
  return 0;
}

int sk_gemm_bf16(int M, int N, int K, const void* A, int lda, int a_mn, const void* B, int ldb, int b_mn, void* C,
                 int ldc, int out_f32, const void* bias, const void* residual, int ldr, int round_before_res, int act,
                 int force_bn, void* stream) {
  SK_REQUIRE(A && B && C, "sk_gemm_bf16: null operand");
  return sk_gemm_ex_launch(sk_gemm_desc(M, N, K, A, lda, a_mn, B, ldb, b_mn, C, ldc, out_f32, bias, residual, ldr,
                                        round_before_res, act, force_bn, nullptr, 0),
                           S(stream));
}
int sk_linear_swiglu_fwd(int M, int F, int K, const void* x, const void* w_gu, void* gu, void* act, void* stream) {
  SK_REQUIRE(x && w_gu && gu && act, "sk_linear_swiglu_fwd: null operand");
  return sk_gemm_ex_launch(sk_gemm_swiglu_fwd(M, F, K, x, w_gu, gu, act), S(stream));
}
int sk_linear_swiglu_bwd(int M, int N, int F, const void* dy, const void* w_down, const void* gu, void* dgu, void* stream) {
  SK_REQUIRE(dy && w_down && gu && dgu, "sk_linear_swiglu_bwd: null operand");
  return sk_gemm_ex_launch(sk_gemm_swiglu_bwd(M, N, F, dy, w_down, gu, dgu), S(stream));
}
int sk_linear_rope(int M, int N, int K, const void* x, const void* w, const void* bias, void* out, const void* cos_t,
                   const void* sin_t, const int32_t* pos_ids, int T, int rope_cols, int max_positions, void* stream) {
  SK_REQUIRE(x && w && out && cos_t && sin_t, "sk_linear_rope: null operand");
  return sk_gemm_ex_launch(sk_gemm_rope(M, N, K, x, w, bias, out, cos_t, sin_t, pos_ids, T, rope_cols, max_positions, 0),
                           S(stream));
}
int sk_linear_rope_partial(int M, int N, int K, const void* x, const void* w, const void* bias, void* out, const void* cos_t,
                           const void* sin_t, const int32_t* pos_ids, int T, int rope_cols, int max_positions, int rot_dims,
                           void* stream) {
  SK_REQUIRE(x && w && out && cos_t && sin_t, "sk_linear_rope_partial: null operand");
  SK_REQUIRE(rot_dims == 16 || rot_dims == 32 || rot_dims == 64,
             "sk_linear_rope_partial: rot_dims=%d is not supported (16, 32 or 64)", rot_dims);
  return sk_gemm_ex_launch(sk_gemm_rope(M, N, K, x, w, bias, out, cos_t, sin_t, pos_ids, T, rope_cols, max_positions, rot_dims),
                           S(stream));
}
int sk_linear_gelu_fwd(int M, int F, int K, const void* x, const void* w1, const void* b1, void* pre, void* act, void* stream) {
  SK_REQUIRE(x && w1 && pre && act, "sk_linear_gelu_fwd: null operand");
  return sk_gemm_ex_launch(sk_gemm_gelu_fwd(M, F, K, x, w1, b1, pre, act), S(stream));
}
int sk_linear_gelu_bwd(int M, int N, int F, const void* dy, const void* w2, const void* pre, void* dpre, void* stream) {
  SK_REQUIRE(dy && w2 && pre && dpre, "sk_linear_gelu_bwd: null operand");
  return sk_gemm_ex_launch(sk_gemm_gelu_bwd(M, N, F, dy, w2, pre, dpre), S(stream));
}
int sk_linear_res2(int M, int N, int K, const void* x, const void* w, const void* bias, const void* res2, const void* res,
                   void* out, void* ws, int64_t ws_bytes, void* stream) {
  SK_REQUIRE(x && w && res2 && res && out, "sk_linear_res2: null operand");
  return sk_gemm_ex_launch(sk_gemm_res2(M, N, K, x, w, bias, res2, res, out, ws, (size_t)ws_bytes), S(stream));
}
int sk_neox_gemm_plan(int kind, int M, int N, int K, int with_ws, SkGemmPlan* plan) {
  SK_REQUIRE(plan && kind >= 0 && kind <= 6, "sk_neox_gemm_plan: kind must be 0..6");
  // the descriptor each fused linear launches, on stand-in operands: 256-byte aligned, never dereferenced by the planner
  void* p = reinterpret_cast<void*>((uintptr_t)1 << 20);
  SkGemmEx g;
  switch (kind) {
    case 0:   // sk_linear_rope_partial on the fused q|k|v projection: q and k heads rotate
      g = sk_gemm_rope(M, N, K, p, p, p, p, p, p, nullptr, 1, N / 3 * 2, 1, 16);
      break;
    case 1: g = sk_gemm_gelu_fwd(M, N, K, p, p, p, p, p); break;
    case 2: g = sk_gemm_gelu_bwd(M, K, N, p, p, p, p); break;       // the builder takes dy's width K and F = N
    case 3: g = sk_gemm_res2(M, N, K, p, p, p, p, p, p, with_ws ? p : nullptr, with_ws ? sk_gemm_ws_min_bytes() : 0); break;
    case 4: g = sk_gemm_swiglu_fwd(M, N / 2, K, p, p, p, p); break;   // N = 2F gate|up columns
    case 5: g = sk_gemm_swiglu_bwd(M, K, N, p, p, p, p); break;       // likewise; d_gu [M, 2F] from the saved gu [M, 2F]
    default:
      // sk_linear_rope, the Qwen2 q|k|v projection: full-rotary 64-column heads; the plan does not depend on how many of
      // them rotate
      g = sk_gemm_rope(M, N, K, p, p, p, p, p, p, nullptr, 1, N, 1, 0);
  }
  return sk_gemm_plan_ex(g, plan);
}
int sk_gemm_bf16_splitk(int M, int N, int K, const void* A, int lda, int a_mn, const void* B, int ldb, int b_mn, void* C,
                        int ldc, int accumulate, void* splitk_ws, int64_t splitk_ws_bytes, void* stream) {
  SK_REQUIRE(A && B && C, "sk_gemm_bf16_splitk: null operand");
  return sk_gemm_ex_launch(sk_gemm_desc(M, N, K, A, lda, a_mn, B, ldb, b_mn, C, ldc, 0, nullptr, accumulate ? C : nullptr, ldc,
                                        1, SK_ACT_NONE, 0, splitk_ws, (size_t)splitk_ws_bytes),
                           S(stream));
}
int sk_gemm_bf16_ws(int M, int N, int K, const void* A, int lda, int a_mn, const void* B, int ldb, int b_mn, void* C,
                    int ldc, int out_f32, const void* bias, const void* residual, int ldr, int round_before_res, int act,
                    int force_bn, void* ws, int64_t ws_bytes, void* stream) {
  SK_REQUIRE(A && B && C, "sk_gemm_bf16_ws: null operand");
  SK_REQUIRE(ws == nullptr || (((uintptr_t)ws & 15) == 0 && ws_bytes % 16 == 0), "sk_gemm_bf16_ws: scratch must be 16-byte aligned");
  return sk_gemm_ex_launch(sk_gemm_desc(M, N, K, A, lda, a_mn, B, ldb, b_mn, C, ldc, out_f32, bias, residual, ldr,
                                        round_before_res, act, force_bn, ws, (size_t)ws_bytes),
                           S(stream));
}
int64_t sk_gemm_ws_bytes(void) { return (int64_t)sk_gemm_ws_min_bytes(); }
int sk_gemm_plan(int M, int N, int K, const void* A, int lda, int a_mn, const void* B, int ldb, int b_mn, const void* C,
                 int ldc, int out_f32, const void* bias, const void* residual, int ldr, int round_before_res, int act,
                 int force_bn, const void* ws, int64_t ws_bytes, SkGemmPlan* plan) {
  SK_REQUIRE(plan, "sk_gemm_plan: null plan");
  return sk_gemm_plan_ex(sk_gemm_desc(M, N, K, A, lda, a_mn, B, ldb, b_mn, const_cast<void*>(C), ldc, out_f32, bias, residual,
                                      ldr, round_before_res, act, force_bn, const_cast<void*>(ws), (size_t)ws_bytes),
                         plan);
}
}  // extern "C"

namespace {
SkGemmEx split_desc_to_ex(const SkGemmSplitDesc& d) {
  SkGemmEx g = sk_gemm_base(d.M, d.N, d.K);
  g.batch = d.batch; g.a_mode = d.a_mode; g.passes = d.passes;
  g.A = d.A; g.A_lo = d.A_lo; g.lda = d.lda; g.a_mn = d.a_mn;
  g.a_inner = (long)d.a_inner; g.a_rows = (long)d.a_rows; g.a_row_stride = (long)d.a_row_stride;
  g.a_batch_stride = (long)d.a_batch_stride;
  g.B = d.B; g.B_lo = d.B_lo; g.ldb = d.ldb;
  g.C = d.C; g.C_lo = d.C_lo; g.ldc = d.ldc; g.out_f32 = d.out_f32;
  g.bias = d.bias; g.bias_f32 = d.bias_f32;
  g.residual = d.residual; g.residual_lo = d.residual_lo; g.ldr = d.ldr;
  g.act = d.act;
  g.col_gin = d.col_gin; g.col_gout = d.col_gout;
  g.force_bn = d.force_bn;
  return g;
}
}  // namespace

extern "C" {

int sk_gemm_split(const SkGemmSplitDesc* desc, void* stream) {
  SK_REQUIRE(desc && desc->A && desc->B && desc->C, "sk_gemm_split: null argument");
  return sk_gemm_ex_launch(split_desc_to_ex(*desc), S(stream));
}
int sk_gemm_split_plan(const SkGemmSplitDesc* desc, SkGemmPlan* plan) {
  SK_REQUIRE(desc && plan, "sk_gemm_split_plan: null argument");
  return sk_gemm_plan_ex(split_desc_to_ex(*desc), plan);
}
int sk_embed_fwd(const int64_t* ids, const void* table, void* out, int M, int D, int V, void* stream) {
  return sk_embed_fwd_launch(ids, CBF(table), BF(out), M, D, V, S(stream));
}
int sk_embed_bwd(const int64_t* ids, const void* dx, float* scratch, void* dtable, int M, int D, int V, int Vpad,
                 int accumulate, void* stream) {
  return sk_embed_bwd_launch(ids, CBF(dx), scratch, BF(dtable), M, D, V, Vpad, accumulate, S(stream));
}
int sk_rmsnorm_fwd(const void* x, const void* w, void* y, float* rstd, int M, int D, float eps, void* stream) {
  return sk_rmsnorm_fwd_launch(CBF(x), CBF(w), BF(y), rstd, M, D, eps, S(stream));
}
int sk_rmsnorm_bwd(const void* dy, const void* x, const void* w, const float* rstd, const void* dres, void* dx,
                   void* dw, float* dw_partial, int M, int D, int accumulate_dw, void* stream) {
  return sk_rmsnorm_bwd_launch(CBF(dy), CBF(x), CBF(w), rstd, CBF(dres), BF(dx), BF(dw), dw_partial, M, D,
                               accumulate_dw, S(stream));
}
int sk_layernorm_fwd(const void* x, const void* w, const void* b, void* y, float* mean, float* rstd, int M, int D, float eps,
                     void* stream) {
  return sk_layernorm_fwd_launch(CBF(x), CBF(w), CBF(b), BF(y), mean, rstd, M, D, eps, S(stream));
}
int sk_layernorm_bwd(const void* dy, const void* x, const void* w, const float* mean, const float* rstd, const void* dres,
                     void* dx, void* dw, void* db, float* dw_partial, float* db_partial, int M, int D, int accumulate,
                     void* stream) {
  return sk_layernorm_bwd_launch(CBF(dy), CBF(x), CBF(w), mean, rstd, CBF(dres), BF(dx), BF(dw), BF(db), dw_partial, db_partial,
                                 M, D, accumulate, S(stream));
}
int sk_layernorm2_fwd(const void* x, const void* w1, const void* b1, const void* w2, const void* b2, void* y1, void* y2,
                      float* mean, float* rstd, int M, int D, float eps, void* stream) {
  SK_REQUIRE(x && w1 && b1 && w2 && b2 && y1 && y2, "sk_layernorm2_fwd: null argument");
  return sk_layernorm2_fwd_launch(CBF(x), CBF(w1), CBF(b1), CBF(w2), CBF(b2), BF(y1), BF(y2), mean, rstd, M, D, eps, S(stream));
}
int sk_layernorm2_bwd(const void* dy1, const void* dy2, const void* x, const void* w1, const void* w2, const float* mean,
                      const float* rstd, const void* dres, void* dx, void* dw1, void* db1, void* dw2, void* db2,
                      float* partial, int M, int D, int accumulate, void* stream) {
  SK_REQUIRE(dy1 && dy2 && x && w1 && w2 && mean && rstd && dx && dw1 && db1 && dw2 && db2 && partial,
             "sk_layernorm2_bwd: null argument");
  return sk_layernorm2_bwd_launch(CBF(dy1), CBF(dy2), CBF(x), CBF(w1), CBF(w2), mean, rstd, CBF(dres), BF(dx), BF(dw1), BF(db1),
                                  BF(dw2), BF(db2), partial, M, D, accumulate, S(stream));
}
int sk_rope_partial(void* qkv, const void* cos_t, const void* sin_t, const int32_t* pos_ids, int M, int T, int ld,
                    int n_rot_heads, int head_dim, int rot_dims, int inverse, int max_positions, void* stream) {
  SK_REQUIRE(rot_dims > 0, "sk_rope_partial: rot_dims must be positive");
  return sk_rope_launch(BF(qkv), CBF(cos_t), CBF(sin_t), pos_ids, M, T, ld, n_rot_heads, head_dim, inverse, max_positions,
                        S(stream), rot_dims);
}
int sk_colsum(const void* x, void* out, float* partial, int M, int N, int ld, int accumulate, void* stream) {
  return sk_colsum_launch(CBF(x), BF(out), partial, M, N, ld, accumulate, S(stream));
}
int sk_rope(void* qkv, const void* cos_t, const void* sin_t, const int32_t* pos_ids, int M, int T, int ld,
            int n_rot_heads, int head_dim, int inverse, int max_positions, void* stream) {
  return sk_rope_launch(BF(qkv), CBF(cos_t), CBF(sin_t), pos_ids, M, T, ld, n_rot_heads, head_dim, inverse, max_positions,
                        S(stream));
}
int sk_swiglu_fwd(const void* gu, void* act, int M, int F, void* stream) {
  return sk_swiglu_fwd_launch(CBF(gu), BF(act), M, F, S(stream));
}
int sk_swiglu_bwd(const void* gu, const void* dact, void* dgu, int M, int F, void* stream) {
  return sk_swiglu_bwd_launch(CBF(gu), CBF(dact), BF(dgu), M, F, S(stream));
}
int sk_ce_fwd_bwd(const void* logits, const int64_t* labels, void* dlogits, float* partial, float* row_nll,
                  float* stats, int M, int T, int V, int ldl, float num_items, float dloss, void* stream) {
  return sk_ce_launch(CBF(logits), labels, BF(dlogits), partial, row_nll, stats, M, T, V, ldl, num_items, dloss,
                      S(stream));
}
int sk_ce_fwd_bwd_weighted(const void* logits, const int64_t* labels, void* dlogits, float* partial, float* row_nll,
                           const float* row_weight, float* stats, int M, int T, int V, int ldl, float num_items, float dloss,
                           void* stream) {
  SK_REQUIRE(logits && labels && partial && row_weight && stats && M > 0 && T > 0, "sk_ce_fwd_bwd_weighted: bad arguments");
  return sk_ce_launch(CBF(logits), labels, BF(dlogits), partial, row_nll, stats, M, T, V, ldl, num_items, dloss, S(stream),
                      row_weight);
}
int sk_ce_chunk(const void* logits_chunk, const int64_t* labels, void* dlogits_chunk, float* partial, int row0, int rows,
                int M, int T, int V, int ldl, float grad_scale, void* stream) {
  SK_REQUIRE(logits_chunk && labels && partial && T > 0, "sk_ce_chunk: bad arguments");
  return sk_ce_chunk_launch(CBF(logits_chunk), labels, BF(dlogits_chunk), partial, row0, rows, M, T, V, ldl, grad_scale,
                            S(stream));
}
int sk_ce_finalize(const float* partial, int M, float num_items, float* stats, void* stream) {
  SK_REQUIRE(partial && stats && M > 0, "sk_ce_finalize: bad arguments");
  return sk_ce_finalize_launch(partial, M, num_items, stats, S(stream));
}
int sk_opt_pos_bwd(const int32_t* pos_ids, const void* dx, float* scratch, void* dP, int M, int T, int D, int n_pos,
                   int accumulate, void* stream) {
  SK_REQUIRE(dx && scratch && dP && M > 0, "sk_opt_pos_bwd: bad arguments");
  return sk_opt_pos_bwd_launch(pos_ids, CBF(dx), scratch, BF(dP), M, T, D, n_pos, accumulate, S(stream));
}
int sk_relu_bwd(void* g, const void* a, int64_t n, void* stream) {
  SK_REQUIRE(g && a && n > 0, "sk_relu_bwd: bad arguments");
  return sk_relu_bwd_launch(BF(g), CBF(a), (long)n, S(stream));
}
int sk_attn_fwd(const void* q, const void* k, const void* v, void* o, float* lse, int B, int T, int H, int KVH, int ld,
                int ldo, int causal, float scale, void* stream) {
  return sk_attn_fwd_launch(CBF(q), CBF(k), CBF(v), BF(o), lse, B, T, H, KVH, ld, ldo, causal, scale, S(stream));
}
int sk_attn_tc_fwd(const void* qkv, void* o, float* lse, int B, int T, int H, int KVH, int ld, int ldo, int causal,
                   float scale, const int32_t* seg_start, void* stream) {
  SK_REQUIRE(qkv && o, "sk_attn_tc_fwd: null argument");
  return sk_attn_tc_fwd_launch(CBF(qkv), BF(o), lse, B, T, H, KVH, ld, ldo, causal, scale, S(stream), seg_start);
}
int sk_seg_bounds(const int32_t* pos_ids, int32_t* seg_start, int32_t* seg_end, int B, int T, void* stream) {
  return sk_seg_bounds_launch(pos_ids, seg_start, seg_end, B, T, S(stream));
}
int sk_attn_tc_bwd(const void* qkv, const void* o, const void* d_o, const float* lse, float* delta, float* partial,
                   void* dqkv, int B, int T, int H, int KVH, int ld, int ldo, int ldg, int causal, float scale,
                   const int32_t* seg_start, const int32_t* seg_end, void* stream) {
  SK_REQUIRE(qkv && o && d_o && lse && delta && dqkv, "sk_attn_tc_bwd: null argument");
  return sk_attn_tc_bwd_launch(CBF(qkv), CBF(o), CBF(d_o), lse, delta, partial, BF(dqkv), B, T, H, KVH, ld, ldo, ldg, causal,
                               scale, S(stream), seg_start, seg_end);
}
int sk_attn_tc_fwd_split(const void* qkv_hi, const void* qkv_lo, void* o_hi, void* o_lo, int B, int T, int H, int ld,
                         int ldo, float scale, void* stream) {
  SK_REQUIRE(qkv_hi && qkv_lo && o_hi && o_lo, "sk_attn_tc_fwd_split: null argument");
  return sk_attn_tc_fwd_split_launch(CBF(qkv_hi), CBF(qkv_lo), BF(o_hi), BF(o_lo), B, T, H, ld, ldo, scale, S(stream));
}
int sk_attn_tc_fwd_split_causal(const void* qkv_hi, const void* qkv_lo, void* o_hi, void* o_lo, int B, int T, int H, int ld,
                                int ldo, float scale, void* stream) {
  SK_REQUIRE(qkv_hi && qkv_lo && o_hi && o_lo, "sk_attn_tc_fwd_split_causal: null argument");
  return sk_attn_tc_fwd_split_launch(CBF(qkv_hi), CBF(qkv_lo), BF(o_hi), BF(o_lo), B, T, H, ld, ldo, scale, S(stream), 1);
}
int sk_attn_bwd(const void* q, const void* k, const void* v, const void* o, const void* d_o, const float* lse,
                float* delta, void* dq, void* dk, void* dv, int B, int T, int H, int KVH, int ld, int ldo, int ldg,
                int causal, float scale, void* stream) {
  return sk_attn_bwd_launch(CBF(q), CBF(k), CBF(v), CBF(o), CBF(d_o), lse, delta, BF(dq), BF(dk), BF(dv), B, T, H, KVH,
                            ld, ldo, ldg, causal, scale, S(stream));
}
int sk_grad_norm(const void* grads, const int64_t* chunk_start, const int32_t* chunk_len, int n_chunks,
                 const int32_t* tensor_chunk_begin, int n_tensors, float* partial, float max_norm, int emulate_bf16,
                 float* stats, void* stream) {
  return sk_gradnorm_launch(CBF(grads), reinterpret_cast<const long*>(chunk_start), chunk_len, n_chunks,
                            tensor_chunk_begin, n_tensors, partial, max_norm, emulate_bf16, stats, S(stream));
}
int sk_add_layernorm_f32(const float* x, const void* y, const float* w, const float* b, float* xo, void* h, float* mean, float* rstd,
                        int M, int D, float eps, void* stream) {
  SK_REQUIRE(x && w && b && h, "sk_add_layernorm_f32: null argument");
  return sk_add_layernorm_f32_launch(x, CBF(y), w, b, xo, BF(h), mean, rstd, M, D, eps, S(stream));
}
int sk_layernorm_bwd_f32(const void* dy, const float* x, const float* w, const float* mean, const float* rstd, const float* dres_in,
                         float* dres_out, void* dres16, float* dw, float* db, float* partial, int M, int D, int accumulate,
                         void* stream) {
  SK_REQUIRE(dy && x && w && mean && rstd && dres_out && dres16 && dw && db && partial, "sk_layernorm_bwd_f32: null argument");
  return sk_layernorm_bwd_f32_launch(CBF(dy), x, w, mean, rstd, dres_in, dres_out, BF(dres16), dw, db, partial, M, D, accumulate,
                                     S(stream));
}
int sk_grad_norm_f32(const float* grads, const int64_t* chunk_start, const int32_t* chunk_len, int n_chunks,
                     const int32_t* tensor_chunk_begin, int n_tensors, float* partial, float max_norm, float* stats, void* stream) {
  return sk_gradnorm_f32_launch(grads, reinterpret_cast<const long*>(chunk_start), chunk_len, n_chunks, tensor_chunk_begin,
                                n_tensors, partial, max_norm, stats, S(stream));
}
int sk_table_bwd_f32(const int64_t* ids, const int32_t* pos_ids, const float* dx, float* scratch, float* dtable, const void* head,
                     int M, int T, int D, int n_rows, int n_rows_padded, int keep, void* stream) {
  SK_REQUIRE(dx && scratch && dtable && M > 0 && n_rows_padded >= n_rows && (n_rows_padded * (int64_t)D) % 4 == 0,
             "sk_table_bwd_f32: bad arguments");
  SK_REQUIRE(ids || !head, "sk_table_bwd_f32: the tied head gradient belongs to the token table (ids given)");
  return sk_table_bwd_f32_launch(ids, pos_ids, dx, scratch, dtable, CBF(head), M, T, D, n_rows, n_rows_padded, keep, S(stream));
}
int sk_widen_grads(const void* g16, float* g32, const int64_t* chunk_start, const int32_t* chunk_len, int n_chunks, int keep,
                   void* stream) {
  SK_REQUIRE(g16 && g32 && chunk_start && chunk_len && n_chunks >= 0, "sk_widen_grads: bad arguments");
  return sk_widen_grads_launch(CBF(g16), g32, reinterpret_cast<const long*>(chunk_start), chunk_len, n_chunks, keep, S(stream));
}
int sk_adamw_master_step(float* params, void* shadow, const float* grads, float* exp_avg, float* exp_avg_sq, int64_t n, float lr,
                         float beta1, float beta2, float eps, float weight_decay, int step, const float* clip_stats, void* stream) {
  return sk_adamw_master_launch(params, BF(shadow), grads, exp_avg, exp_avg_sq, (long)n, lr, beta1, beta2, eps, weight_decay, step,
                                clip_stats, S(stream));
}
int sk_adamw_step(void* params, const void* grads, void* exp_avg, void* exp_avg_sq, int64_t n, float lr, float beta1,
                  float beta2, float eps, float weight_decay, int step, const float* clip_stats, void* stream) {
  return sk_adamw_launch(BF(params), CBF(grads), BF(exp_avg), BF(exp_avg_sq), (long)n, lr, beta1, beta2, eps,
                         weight_decay, step, clip_stats, S(stream));
}

}  // extern "C"

// ---- peer-memory gradient all-reduce (p2p_comm.cu) ------------------------------------------------------------------
int64_t sk_p2p_flag_bytes(void) { return (int64_t)sk_p2p_flag_bytes_impl(); }
int sk_p2p_set_trace(void* buf) { return sk_p2p_set_trace_impl(buf); }
int sk_p2p_debug_hog(int ctas, int64_t ns, void* started_u32, void* stream) {
  return sk_p2p_hog_launch(ctas, (long long)ns, reinterpret_cast<unsigned*>(started_u32), S(stream));
}
int sk_p2p_alloc(int64_t bytes, void** out) { return sk_p2p_alloc_impl((size_t)bytes, out); }
int sk_p2p_free(void* p) { return sk_p2p_free_impl(p); }
int sk_p2p_export(const void* ptr, void* handle64, int64_t* offset) {
  size_t off = 0;
  const int rc = sk_p2p_export_impl(ptr, handle64, &off);
  if (offset) *offset = (int64_t)off;
  return rc;
}
int sk_p2p_open(const void* handle64, void** base) { return sk_p2p_open_impl(handle64, base); }
int sk_p2p_close(void* base) { return sk_p2p_close_impl(base); }
int sk_p2p_signal(void* const* flags, int rank, int world, int slot, uint32_t epoch, void* stream) {
  return sk_p2p_signal_launch(flags, rank, world, slot, epoch, S(stream));
}
int sk_p2p_wait(void* const* flags, int rank, int world, int slot_lo, int n_slots, uint32_t epoch, int* err_flag, void* stream) {
  return sk_p2p_wait_launch(flags, rank, world, slot_lo, n_slots, epoch, err_flag, S(stream));
}
int sk_p2p_allreduce_bf16(void* const* bufs, void* const* flags, int rank, int world, int64_t offset_elems, int64_t n_elems,
                          int slot, uint32_t epoch, int ctas, int* err_flag, void* stream) {
  SK_REQUIRE(offset_elems >= 0 && n_elems > 0, "p2p_allreduce: bad range");
  return sk_p2p_allreduce_launch(bufs, flags, rank, world, (size_t)offset_elems, (size_t)n_elems, slot, epoch, ctas, err_flag,
                                 S(stream));
}
