// Causal-LM train step orchestration (host C++): parameter layout, workspace layout, forward, backward and the
// optimiser step of a Qwen2-shaped decoder, composed from the kernels in gemm_tcgen05.cu / attention.cu /
// lm_kernels.cu.  This replaces, for hot path (ii), UnitLM.forward + compute_loss + torch autograd
// (slamkit/model/unit_lm.py:13-29,135-182 -> HF:models/qwen2/modeling_qwen2.py:332-487) and the clip + AdamW part of
// HF Trainer's inner step.  No tensor library is involved below the C ABI: raw device pointers in, kernels out.
#include "kernels.h"
#include "../../include/slamkit_b200.h"
#include <algorithm>
#include <string>
#include <vector>
#include <math.h>
#include <string.h>
#include <stdlib.h>

namespace {
constexpr int64_t ALIGN_ELEMS = 64;  // 128-byte alignment of every tensor in the flat buffers
constexpr int GN_CHUNK = 16384;

struct TensorDesc {
  std::string name;
  int64_t off;
  int rows, cols;
};
struct LayerOff {
  int64_t ln1, wqkv, bqkv, wo, ln2, wgu, wd;
};
// byte offsets into the workspace for one (B,T)
struct WsLayout {
  int64_t X, h1, rstd1, qkv, ao, lse, xmid, h2, rstd2, gu, act;  // per-layer strides below
  int64_t sX, sh, srstd, sqkv, slse, sgu, sact;
  int64_t hf, rstdf, logits, dlogits, dxA, dxB, dh, dao, dqkv, dgu, delta;
  int64_t dw_partial, colsum_partial, ce_partial, embed_scratch, splitk, splitk_bytes, seg_start, seg_end, total;
};
}  // namespace

struct SkLm {
  SkLmConfig cfg;
  int d, F, H, KVH, hd, L, V, Vp, qkv_dim;
  std::vector<TensorDesc> tensors;
  std::vector<LayerOff> lo;
  int64_t off_final_norm = 0, off_embed = 0, off_head = 0, n_params = 0;
  bf16* params = nullptr;
  bf16* grads = nullptr;
  const bf16* rope_cos = nullptr;
  const bf16* rope_sin = nullptr;
  uint8_t* ws = nullptr;
  int64_t ws_bytes = 0;
  // gradient-norm chunk tables (device)
  long* d_chunk_start = nullptr;
  int* d_chunk_len = nullptr;
  int* d_tensor_chunk_begin = nullptr;
  float* d_chunk_partial = nullptr;
  int n_chunks = 0, n_norm_groups = 0;
  int last_B = 0, last_T = 0;
  int head_chunk = 0;   // > 0: rows per chunk of the chunked lm_head + CE (large vocabularies), 0: one pass
  // optional: events recorded on the compute stream as soon as a layer's gradients are final (index = layer; index
  // n_layers = lm_head / final-norm part), so the host can start that bucket's all-reduce while backward continues
  std::vector<cudaEvent_t> bwd_events;
};

namespace {

int64_t align_up(int64_t v, int64_t a) { return (v + a - 1) / a * a; }

int64_t add_tensor(SkLm* lm, const std::string& name, int rows, int cols) {
  const int64_t off = lm->n_params;
  lm->tensors.push_back({name, off, rows, cols});
  lm->n_params = align_up(off + (int64_t)rows * cols, ALIGN_ELEMS);
  return off;
}

WsLayout make_layout(const SkLm* lm, int B, int T) {
  WsLayout w;
  const int64_t M = (int64_t)B * T;
  int64_t cur = 0;
  auto take = [&](int64_t bytes) {
    const int64_t o = cur;
    cur = align_up(cur + bytes, 256);
    return o;
  };
  const int L = lm->L;
  w.sX = align_up(M * lm->d * 2, 256);
  w.sh = w.sX;
  w.srstd = align_up(M * 4, 256);
  w.sqkv = align_up(M * lm->qkv_dim * 2, 256);
  w.slse = align_up((int64_t)B * lm->H * T * 4, 256);
  w.sgu = align_up(M * 2 * lm->F * 2, 256);
  w.sact = align_up(M * lm->F * 2, 256);
  // GEMM scratch first: its offset (and the stream-K flag words in its last 4 KB, zeroed by sk_lm_bind) must not move
  // with (B, T).  Sized for 8 fp32 slabs of the largest split-K wgrad and for the stream-K partial tiles.
  w.splitk_bytes = align_up(std::max<int64_t>((int64_t)8 * lm->qkv_dim * lm->d * 4, (int64_t)sk_gemm_ws_min_bytes()) + 4096, 256);
  w.splitk = take(w.splitk_bytes);
  w.X = take(w.sX * (L + 1));
  w.h1 = take(w.sh * L);
  w.rstd1 = take(w.srstd * L);
  w.qkv = take(w.sqkv * L);
  w.ao = take(w.sX * L);
  w.lse = take(w.slse * L);
  w.xmid = take(w.sX * L);
  w.h2 = take(w.sh * L);
  w.rstd2 = take(w.srstd * L);
  w.gu = take(w.sgu * L);
  w.act = take(w.sact * L);
  w.hf = take(w.sX);
  w.rstdf = take(w.srstd);
  w.logits = take(M * lm->Vp * 2);
  // large vocabularies run the lm_head + CE in row chunks with the gradient written in place (head_chunked below): no
  // second [M, Vp] buffer
  w.dlogits = lm->head_chunk > 0 ? w.logits : take(M * lm->Vp * 2);
  w.dxA = take(w.sX);
  w.dxB = take(w.sX);
  w.dh = take(w.sX);
  w.dao = take(w.sX);
  w.dqkv = take(w.sqkv);
  w.dgu = take(w.sgu);
  w.delta = take(w.slse);
  w.dw_partial = take((int64_t)sk_rmsnorm_bwd_blocks() * lm->d * 4);
  w.colsum_partial = take((int64_t)sk_colsum_splits() * lm->qkv_dim * 4);
  w.ce_partial = take((int64_t)sk_ce_blocks((int)M) * 2 * 4);
  w.embed_scratch = take((int64_t)lm->Vp * lm->d * 8);   // 64-bit fixed-point accumulators of the embedding gradient
  w.seg_start = take(M * 4);   // document bounds of packed batches (position_ids given), int32 per token
  w.seg_end = take(M * 4);
  w.total = cur;
  return w;
}

template <typename T>
T* wsp(const SkLm* lm, int64_t off) {
  return reinterpret_cast<T*>(lm->ws + off);
}

#define SK_TRY(expr)        \
  do {                      \
    int _rc = (expr);       \
    if (_rc) return _rc;    \
  } while (0)

// y[M,N] = x[M,K] * W[N,K]^T (+bias) (+residual)
// (forward and dgrad GEMMs get no scratch: whole-tile scheduling keeps every output row's fp32 summation order
//  independent of the batch it sits in -- logits of a sequence are bit-identical alone or inside a batch)
int linear_fwd(int M, int N, int K, const bf16* x, const bf16* W, bf16* y, const bf16* bias, const bf16* res,
               cudaStream_t s) {
  return sk_gemm_launch(M, N, K, x, K, 0, W, K, 0, y, N, 0, bias, res, N, res ? 1 : 0, 0, 0, s);
}
// dx[M,K] = dy[M,N] * W[N,K]
int linear_dgrad(int M, int N, int K, const bf16* dy, const bf16* W, bf16* dx, cudaStream_t s) {
  return sk_gemm_launch(M, K, N, dy, N, 0, W, K, 1, dx, K, 0, nullptr, nullptr, 0, 0, 0, 0, s);
}
// dW[N,K] (+)= dy[M,N]^T * x[M,K]   (scratch: split-K for the small wgrads, stream-K balancing for the large ones)
int linear_wgrad(int M, int N, int K, const bf16* dy, const bf16* x, bf16* dW, int accumulate, cudaStream_t s,
                 void* splitk_ws, size_t splitk_bytes) {
  return sk_gemm_launch(N, K, M, dy, N, 1, x, K, 1, dW, K, 0, nullptr, accumulate ? dW : nullptr, K, 1, 0, 0, s,
                        splitk_ws, splitk_bytes);
}

int linear_qkv_rope(const SkLm* lm, int M, int T, const bf16* x, const bf16* W, const bf16* bias, bf16* qkv,
                    const int32_t* pos_ids, cudaStream_t s) {
  return sk_linear_rope_launch(M, lm->qkv_dim, lm->d, x, W, bias, qkv, lm->rope_cos, lm->rope_sin, pos_ids, T,
                               (lm->H + lm->KVH) * lm->hd, lm->cfg.max_positions, s);
}

int check_bound(const SkLm* lm, int B, int T, const WsLayout& w, const int32_t* pos_ids) {
  SK_REQUIRE(lm->params && lm->ws, "sk_lm: sk_lm_bind has not been called");
  // a packed row (position_ids given) may be longer than the RoPE tables: positions restart per document
  SK_REQUIRE(B > 0 && T > 0 && (T <= lm->cfg.max_positions || pos_ids != nullptr),
             "sk_lm: bad batch shape B=%d T=%d (max_positions=%d; longer rows need position_ids)", B, T, lm->cfg.max_positions);
  SK_REQUIRE(w.total <= lm->ws_bytes, "sk_lm: workspace too small: need %lld bytes, bound %lld", (long long)w.total,
             (long long)lm->ws_bytes);
  return 0;
}

int forward_impl(SkLm* lm, const int64_t* ids, const int64_t* labels, const int32_t* pos_ids, int B, int T,
                 float num_items, float dloss, bool want_dlogits, float* stats, const WsLayout& w, cudaStream_t s,
                 float* row_nll = nullptr, bool with_head = true) {
  const int M = B * T, d = lm->d, F = lm->F, L = lm->L;
  const bf16* P = lm->params;
  bf16* X0 = wsp<bf16>(lm, w.X);
  SK_TRY(sk_embed_fwd_launch(ids, P + lm->off_embed, X0, M, d, lm->V, s));
  const float scale = 1.0f / sqrtf((float)lm->hd);
  // packed batch (position_ids given): document bounds -> block-diagonal causal attention, as the reference's varlen
  // flash-attention path does (slamkit/data/hf_dataset.py:61-62 + HF prepare_fa_kwargs_from_position_ids)
  const int* seg_start = nullptr;
  if (pos_ids) {
    SK_TRY(sk_seg_bounds_launch(pos_ids, wsp<int32_t>(lm, w.seg_start), wsp<int32_t>(lm, w.seg_end), B, T, s));
    seg_start = wsp<int32_t>(lm, w.seg_start);
  }
  for (int l = 0; l < L; ++l) {
    const LayerOff& o = lm->lo[l];
    bf16* x = wsp<bf16>(lm, w.X + w.sX * l);
    bf16* xn = wsp<bf16>(lm, w.X + w.sX * (l + 1));
    bf16* h1 = wsp<bf16>(lm, w.h1 + w.sh * l);
    float* r1 = wsp<float>(lm, w.rstd1 + w.srstd * l);
    bf16* qkv = wsp<bf16>(lm, w.qkv + w.sqkv * l);
    bf16* ao = wsp<bf16>(lm, w.ao + w.sX * l);
    float* lse = wsp<float>(lm, w.lse + w.slse * l);
    bf16* xmid = wsp<bf16>(lm, w.xmid + w.sX * l);
    bf16* h2 = wsp<bf16>(lm, w.h2 + w.sh * l);
    float* r2 = wsp<float>(lm, w.rstd2 + w.srstd * l);
    bf16* gu = wsp<bf16>(lm, w.gu + w.sgu * l);
    bf16* act = wsp<bf16>(lm, w.act + w.sact * l);

    SK_TRY(sk_rmsnorm_fwd_launch(x, P + o.ln1, h1, r1, M, d, lm->cfg.rms_eps, s));
    SK_TRY(linear_qkv_rope(lm, M, T, h1, P + o.wqkv, lm->cfg.qkv_bias ? P + o.bqkv : nullptr, qkv, pos_ids, s));
    SK_TRY(sk_attn_tc_fwd_launch(qkv, ao, lse, B, T, lm->H, lm->KVH, lm->qkv_dim, d, 1, scale, s, seg_start));
    SK_TRY(linear_fwd(M, d, d, ao, P + o.wo, xmid, nullptr, x, s));
    SK_TRY(sk_rmsnorm_fwd_launch(xmid, P + o.ln2, h2, r2, M, d, lm->cfg.rms_eps, s));
    SK_TRY(sk_linear_swiglu_fwd_launch(M, F, d, h2, P + o.wgu, gu, act, s));
    SK_TRY(linear_fwd(M, d, F, act, P + o.wd, xn, nullptr, xmid, s));
  }
  bf16* xL = wsp<bf16>(lm, w.X + w.sX * L);
  bf16* hf = wsp<bf16>(lm, w.hf);
  SK_TRY(sk_rmsnorm_fwd_launch(xL, P + lm->off_final_norm, hf, wsp<float>(lm, w.rstdf), M, d, lm->cfg.rms_eps, s));
  lm->last_B = B;
  lm->last_T = T;
  if (!with_head) return 0;
  bf16* logits = wsp<bf16>(lm, w.logits);
  SK_TRY(linear_fwd(M, lm->Vp, d, hf, P + lm->off_head, logits, nullptr, nullptr, s));
  if (labels) {
    SK_TRY(sk_ce_launch(logits, labels, want_dlogits ? wsp<bf16>(lm, w.dlogits) : nullptr, wsp<float>(lm, w.ce_partial),
                        row_nll, stats, M, T, lm->V, lm->Vp, num_items, dloss, s));
  }
  return 0;
}

// lm_head + compute_loss + their backward for text+unit vocabularies (~152 k columns; BASELINE cfg-4), in row chunks:
//   logits_c = hf_c * E^T  ->  CE on the chunk, gradient written over the logits  ->  dh_c = dlogits_c * E,  dE += dlogits_c^T hf_c
// Only [chunk, Vp] logits ever exist (0.6 GB at 2048 rows instead of 2 x 2.5 GB at [8192, 152 k]) and every element
// moves through HBM as in the one-pass form; the price is one read-modify-write of dE per extra chunk.  (A fully fused
// "flash" CE would recompute the logits GEMM in the backward pass -- 2.2 TFLOP at this shape, more time than the 7.5 GB
// of logits traffic it removes.)  The sums per row meet in `ce_partial`, finalised once.
int head_chunked(SkLm* lm, const int64_t* labels, int B, int T, float num_items, float dloss, int accumulate, float* stats,
                 const WsLayout& w, cudaStream_t s) {
  const int M = B * T, d = lm->d;
  SK_REQUIRE(num_items > 0.f, "sk_lm: training with a large vocabulary needs num_items_in_batch (the 'sum / num_items' loss of "
                              "slamkit/model/unit_lm.py:26-28): the gradient scale must be known before the first chunk");
  const bf16* P = lm->params;
  bf16* G = lm->grads;
  bf16* hf = wsp<bf16>(lm, w.hf);
  bf16* dh = wsp<bf16>(lm, w.dh);
  bf16* chunk = wsp<bf16>(lm, w.logits);
  float* partial = wsp<float>(lm, w.ce_partial);
  const float gs = dloss / num_items;
  for (int r0 = 0; r0 < M; r0 += lm->head_chunk) {
    const int rows = std::min(lm->head_chunk, M - r0);
    SK_TRY(linear_fwd(rows, lm->Vp, d, hf + (size_t)r0 * d, P + lm->off_head, chunk, nullptr, nullptr, s));
    SK_TRY(sk_ce_chunk_launch(chunk, labels, chunk, partial, r0, rows, M, T, lm->V, lm->Vp, gs, s));
    SK_TRY(linear_dgrad(rows, lm->Vp, d, chunk, P + lm->off_head, dh + (size_t)r0 * d, s));
    SK_TRY(linear_wgrad(rows, lm->Vp, d, chunk, hf + (size_t)r0 * d, G + lm->off_head, (accumulate || r0 > 0) ? 1 : 0, s,
                        lm->ws + w.splitk, (size_t)w.splitk_bytes));
  }
  return sk_ce_finalize_launch(partial, M, num_items, stats, s);
}

int backward_impl(SkLm* lm, const int64_t* ids, const int32_t* pos_ids, int B, int T, int accumulate,
                  const WsLayout& w, cudaStream_t s, bool with_head = true) {
  const int M = B * T, d = lm->d, F = lm->F, L = lm->L, Q = lm->qkv_dim;
  const bf16* P = lm->params;
  bf16* G = lm->grads;
  float* dwp = wsp<float>(lm, w.dw_partial);
  bf16* dxA = wsp<bf16>(lm, w.dxA);
  bf16* dxB = wsp<bf16>(lm, w.dxB);
  bf16* dh = wsp<bf16>(lm, w.dh);
  bf16* dao = wsp<bf16>(lm, w.dao);
  bf16* dqkv = wsp<bf16>(lm, w.dqkv);
  bf16* dgu = wsp<bf16>(lm, w.dgu);
  bf16* dlogits = wsp<bf16>(lm, w.dlogits);
  bf16* hf = wsp<bf16>(lm, w.hf);
  const float scale = 1.0f / sqrtf((float)lm->hd);

  // lm_head (already done chunk by chunk for large vocabularies)
  if (with_head) {
    SK_TRY(linear_dgrad(M, lm->Vp, d, dlogits, P + lm->off_head, dh, s));
    SK_TRY(linear_wgrad(M, lm->Vp, d, dlogits, hf, G + lm->off_head, accumulate, s, lm->ws + w.splitk, (size_t)w.splitk_bytes));
  }
  SK_TRY(sk_rmsnorm_bwd_launch(dh, wsp<bf16>(lm, w.X + w.sX * L), P + lm->off_final_norm, wsp<float>(lm, w.rstdf),
                               nullptr, dxA, G + lm->off_final_norm, dwp, M, d, accumulate, s));
  if (!lm->bwd_events.empty()) SK_CUDA_CHECK(cudaEventRecord(lm->bwd_events[L], s));
  for (int l = L - 1; l >= 0; --l) {
    const LayerOff& o = lm->lo[l];
    bf16* x = wsp<bf16>(lm, w.X + w.sX * l);
    bf16* h1 = wsp<bf16>(lm, w.h1 + w.sh * l);
    float* r1 = wsp<float>(lm, w.rstd1 + w.srstd * l);
    bf16* qkv = wsp<bf16>(lm, w.qkv + w.sqkv * l);
    bf16* ao = wsp<bf16>(lm, w.ao + w.sX * l);
    float* lse = wsp<float>(lm, w.lse + w.slse * l);
    bf16* xmid = wsp<bf16>(lm, w.xmid + w.sX * l);
    bf16* h2 = wsp<bf16>(lm, w.h2 + w.sh * l);
    float* r2 = wsp<float>(lm, w.rstd2 + w.srstd * l);
    bf16* gu = wsp<bf16>(lm, w.gu + w.sgu * l);
    bf16* act = wsp<bf16>(lm, w.act + w.sact * l);

    // MLP
    SK_TRY(sk_linear_swiglu_bwd_launch(M, d, F, dxA, P + o.wd, gu, dgu, s));
    SK_TRY(linear_wgrad(M, d, F, dxA, act, G + o.wd, accumulate, s, lm->ws + w.splitk, (size_t)w.splitk_bytes));
    SK_TRY(linear_dgrad(M, 2 * F, d, dgu, P + o.wgu, dh, s));
    SK_TRY(linear_wgrad(M, 2 * F, d, dgu, h2, G + o.wgu, accumulate, s, lm->ws + w.splitk, (size_t)w.splitk_bytes));
    SK_TRY(sk_rmsnorm_bwd_launch(dh, xmid, P + o.ln2, r2, dxA, dxB, G + o.ln2, dwp, M, d, accumulate, s));
    // attention
    SK_TRY(linear_dgrad(M, d, d, dxB, P + o.wo, dao, s));
    SK_TRY(linear_wgrad(M, d, d, dxB, ao, G + o.wo, accumulate, s, lm->ws + w.splitk, (size_t)w.splitk_bytes));
    SK_TRY(sk_attn_tc_bwd_launch(qkv, ao, dao, lse, wsp<float>(lm, w.delta), nullptr, dqkv, B, T,
                                 lm->H, lm->KVH, Q, d, Q, 1, scale, s, pos_ids ? wsp<int32_t>(lm, w.seg_start) : nullptr,
                                 pos_ids ? wsp<int32_t>(lm, w.seg_end) : nullptr, lm->rope_cos, lm->rope_sin, pos_ids,
                                 lm->cfg.max_positions));   // inverse RoPE on dq / dk applied after the attention backward
    if (lm->cfg.qkv_bias)
      SK_TRY(sk_colsum_launch(dqkv, G + o.bqkv, wsp<float>(lm, w.colsum_partial), M, Q, Q, accumulate, s));
    SK_TRY(linear_dgrad(M, Q, d, dqkv, P + o.wqkv, dh, s));
    SK_TRY(linear_wgrad(M, Q, d, dqkv, h1, G + o.wqkv, accumulate, s, lm->ws + w.splitk, (size_t)w.splitk_bytes));
    SK_TRY(sk_rmsnorm_bwd_launch(dh, x, P + o.ln1, r1, dxB, dxA, G + o.ln1, dwp, M, d, accumulate, s));
    if (!lm->bwd_events.empty()) SK_CUDA_CHECK(cudaEventRecord(lm->bwd_events[l], s));
  }
  // embedding: tied -> add on top of the lm_head gradient just written; untied -> honour `accumulate`
  SK_TRY(sk_embed_bwd_launch(ids, dxA, wsp<float>(lm, w.embed_scratch), G + lm->off_embed, M, d, lm->V, lm->Vp,
                             lm->cfg.tie_embeddings ? 1 : accumulate, s));
  return 0;
}

// byte offsets into the decode workspace for (B, T_cache): one token per row
struct DecLayout {
  int64_t gemm, gemm_bytes, x0, x1, h, qkv, ao, gu, act, lens, partial, total;
};

DecLayout make_dec_layout(const SkLm* lm, int B, int T_cache) {
  DecLayout w;
  int64_t cur = 0;
  auto take = [&](int64_t bytes) {
    const int64_t o = cur;
    cur = align_up(cur + bytes, 256);
    return o;
  };
  // GEMM scratch: split-K slabs of the down projection and stream-K partial tiles, flag words in its last 4 KB
  w.gemm_bytes = align_up((int64_t)sk_gemm_ws_min_bytes(), 256);
  w.gemm = take(w.gemm_bytes);
  w.x0 = take((int64_t)B * lm->d * 2);
  w.x1 = take((int64_t)B * lm->d * 2);
  w.h = take((int64_t)B * lm->d * 2);
  w.qkv = take((int64_t)B * lm->qkv_dim * 2);
  w.ao = take((int64_t)B * lm->d * 2);
  w.gu = take((int64_t)B * 2 * lm->F * 2);
  w.act = take((int64_t)B * lm->F * 2);
  w.lens = take((int64_t)B * 4);
  w.partial = take(sk_attn_decode_partial_bytes(B, lm->H, T_cache));
  w.total = cur;
  return w;
}

int check_decode(const SkLm* lm, int B, int T_cache, int ldl, const void* kv_cache, const void* logits, const void* ws,
                 int64_t ws_bytes, const DecLayout& w) {
  SK_REQUIRE(lm->params && lm->ws, "sk_lm: sk_lm_bind has not been called");
  SK_REQUIRE(kv_cache && logits && ws, "sk_lm decode: null argument");
  SK_REQUIRE(B > 0 && T_cache > 0 && T_cache <= lm->cfg.max_positions, "sk_lm decode: bad shape B=%d T_cache=%d (max_positions=%d)",
             B, T_cache, lm->cfg.max_positions);
  SK_REQUIRE(ldl >= lm->Vp && ldl % 8 == 0, "sk_lm decode: ldl must be >= %d and a multiple of 8 (got %d)", lm->Vp, ldl);
  SK_REQUIRE(((uintptr_t)ws & 255) == 0 && ((uintptr_t)kv_cache & 15) == 0 && ((uintptr_t)logits & 15) == 0,
             "sk_lm decode: decode workspace must be 256-byte, cache and logits 16-byte aligned");
  SK_REQUIRE(ws_bytes >= w.total, "sk_lm decode: decode workspace too small: need %lld bytes, got %lld", (long long)w.total,
             (long long)ws_bytes);
  return 0;
}

}  // namespace

extern "C" {

int64_t sk_lm_kv_cache_bytes(const SkLm* lm, int B, int T_cache) {
  if (!lm || B <= 0 || T_cache <= 0) return 0;
  return (int64_t)lm->L * 2 * B * lm->KVH * T_cache * lm->hd * 2;
}

int64_t sk_lm_decode_workspace_bytes(const SkLm* lm, int B, int T_cache) {
  if (!lm || B <= 0 || T_cache <= 0) return 0;
  return make_dec_layout(lm, B, T_cache).total;
}

int sk_lm_prefill(SkLm* lm, const int64_t* ids, const int32_t* lens, int B, int T, void* kv_cache, int T_cache,
                  void* logits, int ldl, void* decode_ws, int64_t decode_ws_bytes, void* stream) {
  SK_REQUIRE(lm && ids && lens, "sk_lm_prefill: null argument");
  const DecLayout dl = make_dec_layout(lm, B, T_cache);
  SK_TRY(check_decode(lm, B, T_cache, ldl, kv_cache, logits, decode_ws, decode_ws_bytes, dl));
  SK_REQUIRE(T > 0 && T <= T_cache, "sk_lm_prefill: prompt width T=%d must be in [1, T_cache=%d]", T, T_cache);
  const WsLayout w = make_layout(lm, B, T);
  SK_TRY(check_bound(lm, B, T, w, nullptr));
  cudaStream_t s = (cudaStream_t)stream;
  uint8_t* dws = reinterpret_cast<uint8_t*>(decode_ws);
  SK_CUDA_CHECK(cudaMemsetAsync(dws + dl.gemm + dl.gemm_bytes - 4096, 0, 4096, s));
  SK_TRY(forward_impl(lm, ids, nullptr, nullptr, B, T, 0.f, 1.f, false, nullptr, w, s, nullptr, false));
  SK_TRY(sk_kv_prefill_launch(wsp<bf16>(lm, w.qkv), w.sqkv / 2, lm->qkv_dim, reinterpret_cast<bf16*>(kv_cache), lens, lm->L, B,
                              T, lm->H, lm->KVH, T_cache, s));
  bf16* hl = reinterpret_cast<bf16*>(dws + dl.h);
  SK_TRY(sk_gather_last_launch(wsp<bf16>(lm, w.hf), lens, hl, B, T, lm->d, s));
  return sk_gemm_launch(B, lm->Vp, lm->d, hl, lm->d, 0, lm->params + lm->off_head, lm->d, 0, logits, ldl, 0, nullptr, nullptr,
                        0, 0, 0, 0, s);
}

int sk_lm_decode_step(SkLm* lm, const int64_t* tokens, const int32_t* pos, int B, void* kv_cache, int T_cache,
                      void* logits, int ldl, void* decode_ws, int64_t decode_ws_bytes, void* stream) {
  SK_REQUIRE(lm && tokens && pos, "sk_lm_decode_step: null argument");
  const DecLayout dl = make_dec_layout(lm, B, T_cache);
  SK_TRY(check_decode(lm, B, T_cache, ldl, kv_cache, logits, decode_ws, decode_ws_bytes, dl));
  cudaStream_t s = (cudaStream_t)stream;
  const int d = lm->d, F = lm->F, Q = lm->qkv_dim;
  const bf16* P = lm->params;
  uint8_t* dws = reinterpret_cast<uint8_t*>(decode_ws);
  bf16* x = reinterpret_cast<bf16*>(dws + dl.x0);
  bf16* xm = reinterpret_cast<bf16*>(dws + dl.x1);
  bf16* h = reinterpret_cast<bf16*>(dws + dl.h);
  bf16* qkv = reinterpret_cast<bf16*>(dws + dl.qkv);
  bf16* ao = reinterpret_cast<bf16*>(dws + dl.ao);
  bf16* gu = reinterpret_cast<bf16*>(dws + dl.gu);
  bf16* act = reinterpret_cast<bf16*>(dws + dl.act);
  int32_t* lens = reinterpret_cast<int32_t*>(dws + dl.lens);
  float* partial = reinterpret_cast<float*>(dws + dl.partial);
  void* gemm_ws = dws + dl.gemm;
  const size_t plane = (size_t)B * lm->KVH * T_cache * lm->hd;
  const float scale = 1.0f / sqrtf((float)lm->hd);
  SK_TRY(sk_embed_fwd_launch(tokens, P + lm->off_embed, x, B, d, lm->V, s));
  for (int l = 0; l < lm->L; ++l) {
    const LayerOff& o = lm->lo[l];
    bf16* kc = reinterpret_cast<bf16*>(kv_cache) + (size_t)l * 2 * plane;
    bf16* vc = kc + plane;
    SK_TRY(sk_rmsnorm_fwd_launch(x, P + o.ln1, h, nullptr, B, d, lm->cfg.rms_eps, s));
    SK_TRY(sk_linear_rope_launch(B, Q, d, h, P + o.wqkv, lm->cfg.qkv_bias ? P + o.bqkv : nullptr, qkv, lm->rope_cos,
                                 lm->rope_sin, pos, 1, (lm->H + lm->KVH) * lm->hd, lm->cfg.max_positions, s));
    SK_TRY(sk_kv_append_launch(qkv, Q, kc, vc, pos, lens, B, lm->H, lm->KVH, T_cache, s));
    SK_TRY(sk_attn_decode_launch(qkv, Q, kc, vc, lens, ao, d, partial, B, lm->H, lm->KVH, T_cache, scale, s));
    SK_TRY(linear_fwd(B, d, d, ao, P + o.wo, xm, nullptr, x, s));
    SK_TRY(sk_rmsnorm_fwd_launch(xm, P + o.ln2, h, nullptr, B, d, lm->cfg.rms_eps, s));
    SK_TRY(sk_linear_swiglu_fwd_launch(B, F, d, h, P + o.wgu, gu, act, s));
    // down projection added in place (residual == output): with M = B there is a single row of output tiles, so the
    // scratch lets the GEMM split its long K loop over idle SMs (fixed-order reduction)
    SK_TRY(sk_gemm_launch(B, d, F, act, F, 0, P + o.wd, F, 0, xm, d, 0, nullptr, xm, d, 0, 0, 0, s, gemm_ws,
                          (size_t)dl.gemm_bytes));
    std::swap(x, xm);
  }
  SK_TRY(sk_rmsnorm_fwd_launch(x, P + lm->off_final_norm, h, nullptr, B, d, lm->cfg.rms_eps, s));
  return sk_gemm_launch(B, lm->Vp, d, h, d, 0, P + lm->off_head, d, 0, logits, ldl, 0, nullptr, nullptr, 0, 0, 0, 0, s);
}

int sk_lm_create(const SkLmConfig* cfg, SkLm** out) {
  SK_REQUIRE(cfg && out, "sk_lm_create: null argument");
  SK_REQUIRE(cfg->head_dim == 64, "sk_lm_create: only head_dim 64 is supported (got %d)", cfg->head_dim);
  SK_REQUIRE(cfg->hidden % 8 == 0 && cfg->hidden <= 1024, "sk_lm_create: hidden must be a multiple of 8 and <= 1024");
  SK_REQUIRE(cfg->ffn % 128 == 0, "sk_lm_create: ffn must be a multiple of 128 (gate/up rows are stored in 128-row blocks)");
  SK_REQUIRE(cfg->n_heads % cfg->n_kv_heads == 0, "sk_lm_create: n_heads must be a multiple of n_kv_heads");
  SK_REQUIRE(cfg->vocab_size > 0 && cfg->vocab_size <= (1 << 20),
             "sk_lm_create: vocab_size must be in [1, 2^20] (unit vocabularies are ~502, interleaved text+unit ones ~152 k)");
  SkLm* lm = new SkLm();
  lm->cfg = *cfg;
  lm->d = cfg->hidden;
  lm->F = cfg->ffn;
  lm->H = cfg->n_heads;
  lm->KVH = cfg->n_kv_heads;
  lm->hd = cfg->head_dim;
  lm->L = cfg->n_layers;
  lm->V = cfg->vocab_size;
  lm->Vp = (cfg->vocab_size + 63) / 64 * 64;
  lm->qkv_dim = (lm->H + 2 * lm->KVH) * lm->hd;
  // text+unit vocabularies: chunked lm_head + CE (SK_HEAD_CHUNK=rows overrides, 0 turns it off)
  lm->head_chunk = lm->Vp > 8192 ? 2048 : 0;
  if (const char* e = getenv("SK_HEAD_CHUNK")) lm->head_chunk = (atoi(e) / 128) * 128;
  lm->lo.resize(lm->L);
  for (int l = 0; l < lm->L; ++l) {
    const std::string p = "layers." + std::to_string(l) + ".";
    LayerOff& o = lm->lo[l];
    o.ln1 = add_tensor(lm, p + "ln1", 1, lm->d);
    o.wqkv = add_tensor(lm, p + "wqkv", lm->qkv_dim, lm->d);
    o.bqkv = add_tensor(lm, p + "bqkv", 1, lm->qkv_dim);
    o.wo = add_tensor(lm, p + "wo", lm->d, lm->H * lm->hd);
    o.ln2 = add_tensor(lm, p + "ln2", 1, lm->d);
    o.wgu = add_tensor(lm, p + "wgu", 2 * lm->F, lm->d);
    o.wd = add_tensor(lm, p + "wd", lm->d, lm->F);
  }
  lm->off_final_norm = add_tensor(lm, "final_norm", 1, lm->d);
  lm->off_embed = add_tensor(lm, "embed", lm->Vp, lm->d);
  lm->off_head = cfg->tie_embeddings ? lm->off_embed : add_tensor(lm, "lm_head", lm->Vp, lm->d);
  SK_REQUIRE(lm->H * lm->hd == lm->d, "sk_lm_create: n_heads*head_dim must equal hidden");

  // gradient-norm chunk tables.  torch.nn.utils.clip_grad_norm_ takes one norm per PARAMETER (rounded to bf16 on bf16
  // gradients), and HF keeps q/k/v and gate/up as separate parameters: a norm group here is one HF parameter, i.e. a
  // list of element ranges of the flat buffer (q, k, v are row ranges of wqkv / bqkv; gate and up alternate in 128-row
  // blocks of wgu).  Chunks are listed group by group, so a group is a contiguous run of the chunk table.
  std::vector<long> cs;
  std::vector<int> cl, tb;
  auto add_range = [&](int64_t off, int64_t n) {
    for (int64_t o = 0; o < n; o += GN_CHUNK) {
      cs.push_back((long)(off + o));
      cl.push_back((int)((n - o) < GN_CHUNK ? (n - o) : GN_CHUNK));
    }
  };
  auto begin_group = [&]() { tb.push_back((int)cs.size()); };
  const int64_t qd = (int64_t)lm->H * lm->hd, kvd = (int64_t)lm->KVH * lm->hd;
  for (int l = 0; l < lm->L; ++l) {
    const LayerOff& o = lm->lo[l];
    begin_group(); add_range(o.ln1, lm->d);
    begin_group(); add_range(o.wqkv, qd * lm->d);
    begin_group(); add_range(o.wqkv + qd * lm->d, kvd * lm->d);
    begin_group(); add_range(o.wqkv + (qd + kvd) * lm->d, kvd * lm->d);
    if (cfg->qkv_bias) {
      begin_group(); add_range(o.bqkv, qd);
      begin_group(); add_range(o.bqkv + qd, kvd);
      begin_group(); add_range(o.bqkv + qd + kvd, kvd);
    }
    begin_group(); add_range(o.wo, (int64_t)lm->d * lm->d);
    begin_group(); add_range(o.ln2, lm->d);
    for (int half = 0; half < 2; ++half) {   // gate, then up
      begin_group();
      for (int b = 0; b < lm->F / 128; ++b) add_range(o.wgu + ((int64_t)b * 256 + half * 128) * lm->d, (int64_t)128 * lm->d);
    }
    begin_group(); add_range(o.wd, (int64_t)lm->d * lm->F);
  }
  begin_group(); add_range(lm->off_final_norm, lm->d);
  begin_group(); add_range(lm->off_embed, (int64_t)lm->Vp * lm->d);
  if (!cfg->tie_embeddings) { begin_group(); add_range(lm->off_head, (int64_t)lm->Vp * lm->d); }
  lm->n_norm_groups = (int)tb.size();
  tb.push_back((int)cs.size());
  lm->n_chunks = (int)cs.size();
  SK_CUDA_CHECK(cudaMalloc(&lm->d_chunk_start, cs.size() * sizeof(long)));
  SK_CUDA_CHECK(cudaMalloc(&lm->d_chunk_len, cl.size() * sizeof(int)));
  SK_CUDA_CHECK(cudaMalloc(&lm->d_tensor_chunk_begin, tb.size() * sizeof(int)));
  SK_CUDA_CHECK(cudaMalloc(&lm->d_chunk_partial, cs.size() * sizeof(float)));
  SK_CUDA_CHECK(cudaMemcpy(lm->d_chunk_start, cs.data(), cs.size() * sizeof(long), cudaMemcpyHostToDevice));
  SK_CUDA_CHECK(cudaMemcpy(lm->d_chunk_len, cl.data(), cl.size() * sizeof(int), cudaMemcpyHostToDevice));
  SK_CUDA_CHECK(cudaMemcpy(lm->d_tensor_chunk_begin, tb.data(), tb.size() * sizeof(int), cudaMemcpyHostToDevice));
  *out = lm;
  return 0;
}

void sk_lm_destroy(SkLm* lm) {
  if (!lm) return;
  cudaFree(lm->d_chunk_start);
  cudaFree(lm->d_chunk_len);
  cudaFree(lm->d_tensor_chunk_begin);
  cudaFree(lm->d_chunk_partial);
  delete lm;
}

int64_t sk_lm_param_count(const SkLm* lm) { return lm ? lm->n_params : 0; }

int sk_lm_tensor_info(const SkLm* lm, int idx, char* name_buf, int name_cap, int64_t* offset, int32_t* rows,
                      int32_t* cols) {
  SK_REQUIRE(lm, "sk_lm_tensor_info: null handle");
  if (idx < 0) return (int)lm->tensors.size();
  SK_REQUIRE(idx < (int)lm->tensors.size(), "sk_lm_tensor_info: index %d out of range", idx);
  const TensorDesc& t = lm->tensors[idx];
  if (name_buf && name_cap > 0) {
    strncpy(name_buf, t.name.c_str(), name_cap - 1);
    name_buf[name_cap - 1] = 0;
  }
  if (offset) *offset = t.off;
  if (rows) *rows = t.rows;
  if (cols) *cols = t.cols;
  return 0;
}

int64_t sk_lm_workspace_bytes(const SkLm* lm, int B, int T) {
  if (!lm || B <= 0 || T <= 0) return 0;
  return make_layout(lm, B, T).total;
}

int sk_lm_bind(SkLm* lm, void* params, void* grads, const void* rope_cos, const void* rope_sin, void* workspace,
               int64_t workspace_bytes) {
  SK_REQUIRE(lm && params && rope_cos && rope_sin && workspace, "sk_lm_bind: null argument");
  SK_REQUIRE(((uintptr_t)params & 127) == 0 && (grads == nullptr || ((uintptr_t)grads & 127) == 0) &&
                 ((uintptr_t)workspace & 255) == 0,
             "sk_lm_bind: params/grads must be 128-byte and workspace 256-byte aligned");
  lm->params = reinterpret_cast<bf16*>(params);
  lm->grads = reinterpret_cast<bf16*>(grads);
  lm->rope_cos = reinterpret_cast<const bf16*>(rope_cos);
  lm->rope_sin = reinterpret_cast<const bf16*>(rope_sin);
  lm->ws = reinterpret_cast<uint8_t*>(workspace);
  lm->ws_bytes = workspace_bytes;
  // stream-K publish flags (last 4 KB of the GEMM scratch, which sits at a fixed offset) start out zero; the GEMM
  // re-arms them itself after every launch
  const WsLayout w = make_layout(lm, 1, 1);
  SK_REQUIRE(workspace_bytes >= w.splitk + w.splitk_bytes, "sk_lm_bind: workspace smaller than the GEMM scratch");
  SK_CUDA_CHECK(cudaMemset(lm->ws + w.splitk + w.splitk_bytes - 4096, 0, 4096));
  SK_CUDA_CHECK(cudaDeviceSynchronize());
  return 0;
}

int sk_lm_forward(SkLm* lm, const int64_t* ids, const int64_t* labels, const int32_t* pos_ids, int B, int T,
                  float num_items, float* stats, void* stream) {
  SK_REQUIRE(lm && ids, "sk_lm_forward: null argument");
  SK_REQUIRE(labels == nullptr || stats != nullptr, "sk_lm_forward: stats is required when labels are given");
  const WsLayout w = make_layout(lm, B, T);
  SK_TRY(check_bound(lm, B, T, w, pos_ids));
  return forward_impl(lm, ids, labels, pos_ids, B, T, num_items, 1.0f, false, stats, w, (cudaStream_t)stream);
}

int sk_lm_forward_backward(SkLm* lm, const int64_t* ids, const int64_t* labels, const int32_t* pos_ids, int B, int T,
                           float num_items, float dloss, int accumulate, float* stats, void* stream) {
  SK_REQUIRE(lm && ids && labels && stats, "sk_lm_forward_backward: null argument");
  SK_REQUIRE(lm->grads, "sk_lm_forward_backward: no gradient buffer bound");
  const WsLayout w = make_layout(lm, B, T);
  SK_TRY(check_bound(lm, B, T, w, pos_ids));
  if (lm->head_chunk > 0) {
    SK_TRY(forward_impl(lm, ids, labels, pos_ids, B, T, num_items, dloss, true, stats, w, (cudaStream_t)stream, nullptr, false));
    SK_TRY(head_chunked(lm, labels, B, T, num_items, dloss, accumulate, stats, w, (cudaStream_t)stream));
    return backward_impl(lm, ids, pos_ids, B, T, accumulate, w, (cudaStream_t)stream, false);
  }
  SK_TRY(forward_impl(lm, ids, labels, pos_ids, B, T, num_items, dloss, true, stats, w, (cudaStream_t)stream));
  return backward_impl(lm, ids, pos_ids, B, T, accumulate, w, (cudaStream_t)stream);
}

int sk_lm_set_backward_events(SkLm* lm, void* const* events, int n) {
  SK_REQUIRE(lm, "sk_lm_set_backward_events: null handle");
  if (events == nullptr || n == 0) {
    lm->bwd_events.clear();
    return 0;
  }
  SK_REQUIRE(n == lm->L + 1, "sk_lm_set_backward_events: expected n_layers+1 = %d events, got %d", lm->L + 1, n);
  lm->bwd_events.assign(n, nullptr);
  for (int i = 0; i < n; ++i) lm->bwd_events[i] = (cudaEvent_t)events[i];
  return 0;
}

int sk_lm_forward_rows(SkLm* lm, const int64_t* ids, const int64_t* labels, const int32_t* pos_ids, int B, int T,
                       float* row_nll, float* stats, void* stream) {
  SK_REQUIRE(lm && ids && labels && row_nll && stats, "sk_lm_forward_rows: null argument");
  const WsLayout w = make_layout(lm, B, T);
  SK_TRY(check_bound(lm, B, T, w, pos_ids));
  return forward_impl(lm, ids, labels, pos_ids, B, T, 1.0f, 1.0f, false, stats, w, (cudaStream_t)stream, row_nll);
}

int sk_lm_backward_weighted(SkLm* lm, const int64_t* ids, const int64_t* labels, const int32_t* pos_ids, int B, int T,
                            const float* row_weight, int accumulate, float* stats, void* stream) {
  SK_REQUIRE(lm && ids && labels && row_weight && stats, "sk_lm_backward_weighted: null argument");
  SK_REQUIRE(lm->grads, "sk_lm_backward_weighted: no gradient buffer bound");
  SK_REQUIRE(lm->last_B == B && lm->last_T == T, "sk_lm_backward_weighted: call sk_lm_forward_rows on the same batch first");
  const WsLayout w = make_layout(lm, B, T);
  SK_TRY(check_bound(lm, B, T, w, pos_ids));
  cudaStream_t s = (cudaStream_t)stream;
  // d loss / d logits[row] = row_weight[row] * (softmax - onehot): recomputed from the logits the forward pass left in
  // the workspace (num_items = 1, dloss = 1: the caller's weights carry every scale factor)
  SK_TRY(sk_ce_launch(wsp<bf16>(lm, w.logits), labels, wsp<bf16>(lm, w.dlogits), wsp<float>(lm, w.ce_partial), nullptr,
                      stats, B * T, T, lm->V, lm->Vp, 1.0f, 1.0f, s, row_weight));
  return backward_impl(lm, ids, pos_ids, B, T, accumulate, w, s);
}

const void* sk_lm_logits(const SkLm* lm) {
  if (!lm || !lm->ws || lm->last_B == 0) return nullptr;
  return lm->ws + make_layout(lm, lm->last_B, lm->last_T).logits;
}
int sk_lm_logits_ld(const SkLm* lm) { return lm ? lm->Vp : 0; }

int sk_lm_optimizer_step(SkLm* lm, void* exp_avg, void* exp_avg_sq, float lr, float beta1, float beta2, float eps,
                         float weight_decay, int step, float max_grad_norm, int emulate_bf16_norm, float* stats,
                         void* stream) {
  SK_REQUIRE(lm && exp_avg && exp_avg_sq && stats, "sk_lm_optimizer_step: null argument");
  SK_REQUIRE(lm->params && lm->grads, "sk_lm_optimizer_step: params/grads not bound");
  cudaStream_t s = (cudaStream_t)stream;
  sk_prof_begin(2, s);
  SK_TRY(sk_gradnorm_launch(lm->grads, lm->d_chunk_start, lm->d_chunk_len, lm->n_chunks, lm->d_tensor_chunk_begin,
                            lm->n_norm_groups, lm->d_chunk_partial, max_grad_norm, emulate_bf16_norm, stats, s));
  int rc = 0;
  if (weight_decay == 0.0f) {
    rc = sk_adamw_launch(lm->params, lm->grads, reinterpret_cast<bf16*>(exp_avg), reinterpret_cast<bf16*>(exp_avg_sq),
                         lm->n_params, lr, beta1, beta2, eps, 0.0f, step, stats, s);
  } else {
    // HF Trainer's decay groups (HF:trainer.py get_decay_parameter_names): biases and norm weights are NOT decayed.
    // Non-default configuration (config/training_args/default.yaml has no weight_decay): one launch per tensor.
    for (const TensorDesc& t : lm->tensors) {
      const bool no_decay = t.rows == 1;   // ln1 / ln2 / final_norm / bqkv are the [1, n] tensors of the layout
      const int64_t n = (((int64_t)t.rows * t.cols + ALIGN_ELEMS - 1) / ALIGN_ELEMS) * ALIGN_ELEMS;
      rc = sk_adamw_launch(lm->params + t.off, lm->grads + t.off, reinterpret_cast<bf16*>(exp_avg) + t.off,
                           reinterpret_cast<bf16*>(exp_avg_sq) + t.off, n, lr, beta1, beta2, eps,
                           no_decay ? 0.0f : weight_decay, step, stats, s);
      if (rc) break;
    }
  }
  sk_prof_end(s);
  return rc;
}

}  // extern "C"
