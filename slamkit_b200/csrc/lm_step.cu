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
// LayerNorm decoder layer: OPT (HF OPTDecoderLayer) and GPT-NeoX (HF GPTNeoXLayer, use_parallel_residual = True).  Two
// affine LayerNorms and biased linears, q|k|v fused as in Qwen2; each architecture registers them in its own order.
struct LnLayerOff {
  int64_t ln1w, ln1b, ln2w, ln2b, wqkv, bqkv, wo, bo, w1, b1, w2, b2;
};
enum { SK_ARCH_QWEN2 = 0, SK_ARCH_OPT = 1, SK_ARCH_NEOX = 2 };
// byte offsets into the workspace for one (B,T)
struct WsLayout {
  int64_t X, h1, rstd1, qkv, ao, lse, xmid, h2, rstd2, gu, act;  // per-layer strides below
  int64_t sX, sh, srstd, sqkv, slse, sgu, sact;
  int64_t hf, rstdf, logits, dlogits, dxA, dxB, dh, dao, dqkv, dgu, delta;
  int64_t dw_partial, colsum_partial, ce_partial, embed_scratch, splitk, splitk_bytes, seg_start, seg_end, total;
  int64_t sR = 0, dres32 = 0;   // OPT: residual-stream slab stride (X, xmid); fp32 residual gradient (master weights)
  int64_t pe = 0;               // post-LN OPT with projections: the token rows e [M, proj_dim] that project_in reads
};
}  // namespace

struct SkLm {
  int arch = SK_ARCH_QWEN2;
  int d, F, H, KVH, hd, L, V, Vp, qkv_dim;
  int max_pos;                    // rows of the RoPE tables (Qwen2, GPT-NeoX) or OPT's max_position_embeddings
  float eps;                      // RMSNorm (Qwen2) or LayerNorm eps
  bool tie, qkv_bias;             // lm_head shares the token table; q|k|v projection has a bias
  std::vector<TensorDesc> tensors;
  std::vector<LayerOff> lo;       // Qwen2 layers
  std::vector<LnLayerOff> lnl;    // OPT and GPT-NeoX layers
  int rot = 64;                   // GPT-NeoX: rotated columns per q / k head (rotary_ndims)
  int64_t off_final_norm_b = 0, off_pos = 0;
  int n_pos = 0;                  // OPT: rows of the learned position table (max_positions + 2)
  // post-LayerNorm OPT (opt-350m): no final LayerNorm; with `proj`, the token table and the tied head are pw = proj_dim
  // wide and proj_in [d, pw] / proj_out [pw, d] map between them and the residual stream.  pw = d otherwise.
  bool post_ln = false, proj = false;
  int pw = 0;
  int64_t off_pin = 0, off_pout = 0;
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
  // OPT with fp32 master weights (sk_lm_set_master): `params` is then the bf16 shadow of params32 that the GEMMs read,
  // `grads` the bf16 scratch of the linear gradients, widened into grads32 over the widen_* chunks once per micro-batch
  bool master = false;
  float* params32 = nullptr;
  float* grads32 = nullptr;
  long* d_widen_start = nullptr;
  int* d_widen_len = nullptr;
  int n_widen = 0;
  // OPT fp32 inference (sk_lm_set_fp32): params32 holds the model, w_hi / w_lo its split-bf16 (hi, lo) copy that the
  // GEMMs read; forward only
  bool fp32 = false;
  bf16* w_hi = nullptr;
  bf16* w_lo = nullptr;
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

// Workspace plan of the bf16 and master-weight paths, one set of per-layer slabs per saved activation.  Qwen2: rstd
// slabs hold the RMSNorm rstd, `gu` gate|up [M, 2F] and `act` the SwiGLU output.  OPT: rstd slabs hold the LayerNorm
// mean then rstd (fp32 [2][M]), `gu` the ReLU output a = relu(fc1) [M, F] that fc2 and the ReLU backward read, `dgu`
// its gradient; `act` is unused.  GPT-NeoX: rstd1 slabs hold the shared mean then rstd of the two LayerNorms, h1 / h2
// their outputs, `gu` the pre-activation of dense_h_to_4h [M, F] and `act` its GELU; `xmid` is one [M, d] slab for the
// attention branch's output (read once, by the same layer's dense_4h_to_h epilogue); rstd2 is unused.  Unused slots
// take 0 bytes.
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
  const bool qwen2 = lm->arch == SK_ARCH_QWEN2, opt = lm->arch == SK_ARCH_OPT, neox = lm->arch == SK_ARCH_NEOX;
  w.sX = align_up(M * lm->d * 2, 256);
  w.sh = w.sX;
  w.srstd = align_up(M * (qwen2 ? 4 : 8), 256);
  w.sqkv = align_up(M * lm->qkv_dim * 2, 256);
  w.slse = align_up((int64_t)B * lm->H * T * 4, 256);
  w.sgu = align_up(M * (qwen2 ? 2 : 1) * lm->F * 2, 256);
  w.sact = opt ? 0 : align_up(M * lm->F * 2, 256);
  w.sR = lm->master ? align_up(M * lm->d * 4, 256) : w.sX;   // master weights: the residual stream is fp32
  // GEMM scratch first: its offset (and the stream-K flag words in its last 4 KB, zeroed by sk_lm_bind) must not move
  // with (B, T).  Sized for 8 fp32 slabs of the largest split-K wgrad and for the stream-K partial tiles.
  w.splitk_bytes = align_up(std::max<int64_t>((int64_t)8 * lm->qkv_dim * lm->d * 4, (int64_t)sk_gemm_ws_min_bytes()) + 4096, 256);
  w.splitk = take(w.splitk_bytes);
  w.X = take(w.sR * (L + 1));
  w.h1 = take(w.sh * L);
  w.rstd1 = take(w.srstd * L);
  w.qkv = take(w.sqkv * L);
  w.ao = take(w.sX * L);
  w.lse = take(w.slse * L);
  w.xmid = take(neox ? w.sX : w.sR * L);
  w.h2 = take(w.sh * L);
  w.rstd2 = take(neox ? 0 : w.srstd * L);
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
  // RMSNorm weight partials; LayerNorm weight and bias partials (OPT), the dual LayerNorm's four (GPT-NeoX)
  w.dw_partial = take(qwen2 ? (int64_t)sk_rmsnorm_bwd_blocks() * lm->d * 4
                            : (int64_t)(opt ? 2 : 4) * sk_layernorm_bwd_blocks() * lm->d * 4);
  w.colsum_partial = take((int64_t)sk_colsum_splits() * (qwen2 ? lm->qkv_dim : std::max(lm->qkv_dim, lm->F)) * 4);
  w.ce_partial = take((int64_t)sk_ce_blocks((int)M) * 2 * 4);
  // 64-bit fixed-point accumulators of the embedding gradient; OPT's token and position tables share them, their
  // gradients are formed one after the other
  w.embed_scratch = take((int64_t)std::max(lm->Vp, lm->n_pos) * lm->d * 8);
  w.seg_start = take(M * 4);   // document bounds of packed batches (position_ids given), int32 per token
  w.seg_end = take(M * 4);
  if (lm->master) w.dres32 = take(w.sR);
  if (lm->proj) w.pe = take(M * lm->pw * 2);
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

// width of the lm_head's input: proj_dim for a post-LN OPT with project_out, else hidden
int head_k(const SkLm* lm) { return lm->proj ? lm->pw : lm->d; }
// the lm_head's input rows [M, head_k]: the final LayerNorm's output, or for post-LN OPT (no final LayerNorm) the last
// layer's output or its project_out image
bf16* head_in(const SkLm* lm, const WsLayout& w) {
  if (lm->post_ln && !lm->proj) return wsp<bf16>(lm, w.X + w.sX * lm->L);
  return wsp<bf16>(lm, w.hf);
}

// y[M,N] = act(x[M,K] * W[N,K]^T + bias) (+ res)
// (forward and dgrad GEMMs get no scratch: whole-tile scheduling keeps every output row's fp32 summation order
//  independent of the batch it sits in -- logits of a sequence are bit-identical alone or inside a batch; only the
//  decode steps' down-projections, one row of output tiles, take scratch)
int linear_fwd(int M, int N, int K, const bf16* x, const bf16* W, bf16* y, const bf16* bias, const bf16* res,
               cudaStream_t s, int act = SK_ACT_NONE, void* splitk_ws = nullptr, size_t splitk_bytes = 0) {
  return sk_gemm_ex_launch(sk_gemm_linear(M, N, K, x, W, y, N, bias, res, act, splitk_ws, splitk_bytes), s);
}
// dx[M,K] = dy[M,N] * W[N,K] (+ res)
int linear_dgrad(int M, int N, int K, const bf16* dy, const bf16* W, bf16* dx, cudaStream_t s, const bf16* res = nullptr) {
  return sk_gemm_ex_launch(sk_gemm_dgrad(M, N, K, dy, W, dx, res), s);
}
// dW[N,K] (+)= dy[M,N]^T * x[M,K]   (scratch: split-K for the small wgrads, stream-K balancing for the large ones)
int linear_wgrad(int M, int N, int K, const bf16* dy, const bf16* x, bf16* dW, bool accumulate, cudaStream_t s,
                 void* splitk_ws, size_t splitk_bytes) {
  return sk_gemm_ex_launch(sk_gemm_wgrad(M, N, K, dy, x, dW, accumulate, splitk_ws, splitk_bytes), s);
}
// logits [M, Vp] at pitch ldl: the lm_head on the rows h [M, K]
int head_logits(const SkLm* lm, int M, int K, const bf16* h, void* logits, int ldl, cudaStream_t s) {
  return sk_gemm_ex_launch(
      sk_gemm_linear(M, lm->Vp, K, h, lm->params + lm->off_head, logits, ldl, nullptr, nullptr, SK_ACT_NONE), s);
}

int linear_qkv_rope(const SkLm* lm, int M, int T, const bf16* x, const bf16* W, const bf16* bias, bf16* qkv,
                    const int32_t* pos_ids, cudaStream_t s) {
  return sk_gemm_ex_launch(sk_gemm_rope(M, lm->qkv_dim, lm->d, x, W, bias, qkv, lm->rope_cos, lm->rope_sin, pos_ids, T,
                                        (lm->H + lm->KVH) * lm->hd, lm->max_pos, 0),
                           s);
}

int check_bound(const SkLm* lm, int B, int T, const WsLayout& w, const int32_t* pos_ids) {
  SK_REQUIRE(lm->params && lm->ws, "sk_lm: sk_lm_bind has not been called");
  // a packed row (position_ids given) may be longer than the RoPE tables: positions restart per document
  SK_REQUIRE(B > 0 && T > 0 && (T <= lm->max_pos || pos_ids != nullptr),
             "sk_lm: bad batch shape B=%d T=%d (max_positions=%d; longer rows need position_ids)", B, T, lm->max_pos);
  SK_REQUIRE(w.total <= lm->ws_bytes, "sk_lm: workspace too small: need %lld bytes, bound %lld", (long long)w.total,
             (long long)lm->ws_bytes);
  return 0;
}

// One pass over a batch: what the forward computes and, for the backward, which batch it differentiates
struct FwdArgs {
  const int64_t* ids;
  const int64_t* labels;      // nullptr: logits only
  const int32_t* pos_ids;     // packed batch, or nullptr
  int B, T;
  float num_items = 0.f, dloss = 1.f;
  bool want_dlogits = false;  // the CE writes the logit gradient for the backward pass
  float* stats = nullptr;
  float* row_nll = nullptr;
  bool with_head = true;      // false: stop at the lm_head's input (chunked head, prefill)
  // fp32 prefill: the fp32 cache of T_cache positions that receives the K / V of positions < lens[b]
  float* kv = nullptr;
  const int32_t* lens = nullptr;
  int T_cache = 0;
};

// packed batch (position_ids given): document bounds -> block-diagonal causal attention, as the reference's varlen
// flash-attention path does (slamkit/data/hf_dataset.py:61-62 + HF prepare_fa_kwargs_from_position_ids)
int seg_bounds(const SkLm* lm, const FwdArgs& a, const WsLayout& w, cudaStream_t s) {
  if (!a.pos_ids) return 0;
  return sk_seg_bounds_launch(a.pos_ids, wsp<int32_t>(lm, w.seg_start), wsp<int32_t>(lm, w.seg_end), a.B, a.T, s);
}
const int* seg_ptr(const SkLm* lm, const FwdArgs& a, int64_t off) { return a.pos_ids ? wsp<int32_t>(lm, off) : nullptr; }

// lm_head on the rows hin [M, K] and, with labels, compute_loss; records the batch shape for the logits and backward
int head_forward(SkLm* lm, const WsLayout& w, const FwdArgs& a, const bf16* hin, int K, cudaStream_t s) {
  lm->last_B = a.B;
  lm->last_T = a.T;
  if (!a.with_head) return 0;
  const int M = a.B * a.T;
  bf16* logits = wsp<bf16>(lm, w.logits);
  SK_TRY(head_logits(lm, M, K, hin, logits, lm->Vp, s));
  if (!a.labels) return 0;
  return sk_ce_launch(logits, a.labels, a.want_dlogits ? wsp<bf16>(lm, w.dlogits) : nullptr, wsp<float>(lm, w.ce_partial),
                      a.row_nll, a.stats, M, a.T, lm->V, lm->Vp, a.num_items, a.dloss, s);
}

// the lm_head's backward from dlogits: its input gradient into dst [M, K], its weight gradient (+)= into the head
int head_backward(SkLm* lm, const WsLayout& w, int M, bf16* dst, const bf16* hin, int K, int accumulate, cudaStream_t s) {
  const bf16* dlogits = wsp<bf16>(lm, w.dlogits);
  SK_TRY(linear_dgrad(M, lm->Vp, K, dlogits, lm->params + lm->off_head, dst, s));
  return linear_wgrad(M, lm->Vp, K, dlogits, hin, lm->grads + lm->off_head, accumulate, s, lm->ws + w.splitk,
                      (size_t)w.splitk_bytes);
}

int qwen2_forward(SkLm* lm, const FwdArgs& a, const WsLayout& w, cudaStream_t s) {
  const int B = a.B, T = a.T, M = B * T, d = lm->d, F = lm->F, L = lm->L;
  const int32_t* pos_ids = a.pos_ids;
  const bf16* P = lm->params;
  bf16* X0 = wsp<bf16>(lm, w.X);
  SK_TRY(sk_embed_fwd_launch(a.ids, P + lm->off_embed, X0, M, d, lm->V, s));
  const float scale = 1.0f / sqrtf((float)lm->hd);
  SK_TRY(seg_bounds(lm, a, w, s));
  const int* seg_start = seg_ptr(lm, a, w.seg_start);
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

    SK_TRY(sk_rmsnorm_fwd_launch(x, P + o.ln1, h1, r1, M, d, lm->eps, s));
    SK_TRY(linear_qkv_rope(lm, M, T, h1, P + o.wqkv, lm->qkv_bias ? P + o.bqkv : nullptr, qkv, pos_ids, s));
    SK_TRY(sk_attn_tc_fwd_launch(qkv, ao, lse, B, T, lm->H, lm->KVH, lm->qkv_dim, d, 1, scale, s, seg_start));
    SK_TRY(linear_fwd(M, d, d, ao, P + o.wo, xmid, nullptr, x, s));
    SK_TRY(sk_rmsnorm_fwd_launch(xmid, P + o.ln2, h2, r2, M, d, lm->eps, s));
    SK_TRY(sk_gemm_ex_launch(sk_gemm_swiglu_fwd(M, F, d, h2, P + o.wgu, gu, act), s));
    SK_TRY(linear_fwd(M, d, F, act, P + o.wd, xn, nullptr, xmid, s));
  }
  bf16* xL = wsp<bf16>(lm, w.X + w.sX * L);
  bf16* hf = wsp<bf16>(lm, w.hf);
  SK_TRY(sk_rmsnorm_fwd_launch(xL, P + lm->off_final_norm, hf, wsp<float>(lm, w.rstdf), M, d, lm->eps, s));
  return head_forward(lm, w, a, hf, d, s);
}

// lm_head + compute_loss + their backward for text+unit vocabularies (~152 k columns; BASELINE cfg-4), in row chunks:
//   logits_c = hf_c * E^T  ->  CE on the chunk, gradient written over the logits  ->  dh_c = dlogits_c * E,  dE += dlogits_c^T hf_c
// Only [chunk, Vp] logits ever exist (0.6 GB at 2048 rows instead of 2 x 2.5 GB at [8192, 152 k]) and every element
// moves through HBM as in the one-pass form; the price is one read-modify-write of dE per extra chunk.  (A fully fused
// "flash" CE would recompute the logits GEMM in the backward pass -- 2.2 TFLOP at this shape, more time than the 7.5 GB
// of logits traffic it removes.)  The sums per row meet in `ce_partial`, finalised once.
int head_chunked(SkLm* lm, const FwdArgs& a, int accumulate, const WsLayout& w, cudaStream_t s) {
  const int M = a.B * a.T, d = head_k(lm);
  SK_REQUIRE(a.num_items > 0.f, "sk_lm: training with a large vocabulary needs num_items_in_batch (the 'sum / num_items' loss of "
                              "slamkit/model/unit_lm.py:26-28): the gradient scale must be known before the first chunk");
  const bf16* P = lm->params;
  bf16* G = lm->grads;
  bf16* hf = head_in(lm, w);
  // post-LN OPT without projections: the head's input gradient is the residual-stream gradient that the layers read
  bf16* dh = wsp<bf16>(lm, lm->post_ln && !lm->proj ? w.dxA : w.dh);
  bf16* chunk = wsp<bf16>(lm, w.logits);
  float* partial = wsp<float>(lm, w.ce_partial);
  const float gs = a.dloss / a.num_items;
  for (int r0 = 0; r0 < M; r0 += lm->head_chunk) {
    const int rows = std::min(lm->head_chunk, M - r0);
    SK_TRY(linear_fwd(rows, lm->Vp, d, hf + (size_t)r0 * d, P + lm->off_head, chunk, nullptr, nullptr, s));
    SK_TRY(sk_ce_chunk_launch(chunk, a.labels, chunk, partial, r0, rows, M, a.T, lm->V, lm->Vp, gs, s));
    SK_TRY(linear_dgrad(rows, lm->Vp, d, chunk, P + lm->off_head, dh + (size_t)r0 * d, s));
    SK_TRY(linear_wgrad(rows, lm->Vp, d, chunk, hf + (size_t)r0 * d, G + lm->off_head, (accumulate || r0 > 0) ? 1 : 0, s,
                        lm->ws + w.splitk, (size_t)w.splitk_bytes));
  }
  return sk_ce_finalize_launch(partial, M, a.num_items, a.stats, s);
}

int qwen2_backward(SkLm* lm, const FwdArgs& a, int accumulate, const WsLayout& w, cudaStream_t s) {
  const int B = a.B, T = a.T, M = B * T, d = lm->d, F = lm->F, L = lm->L, Q = lm->qkv_dim;
  const int32_t* pos_ids = a.pos_ids;
  const bf16* P = lm->params;
  bf16* G = lm->grads;
  float* dwp = wsp<float>(lm, w.dw_partial);
  bf16* dxA = wsp<bf16>(lm, w.dxA);
  bf16* dxB = wsp<bf16>(lm, w.dxB);
  bf16* dh = wsp<bf16>(lm, w.dh);
  bf16* dao = wsp<bf16>(lm, w.dao);
  bf16* dqkv = wsp<bf16>(lm, w.dqkv);
  bf16* dgu = wsp<bf16>(lm, w.dgu);
  const float scale = 1.0f / sqrtf((float)lm->hd);

  // lm_head (already done chunk by chunk for large vocabularies)
  if (a.with_head) SK_TRY(head_backward(lm, w, M, dh, wsp<bf16>(lm, w.hf), d, accumulate, s));
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
    SK_TRY(sk_gemm_ex_launch(sk_gemm_swiglu_bwd(M, d, F, dxA, P + o.wd, gu, dgu), s));
    SK_TRY(linear_wgrad(M, d, F, dxA, act, G + o.wd, accumulate, s, lm->ws + w.splitk, (size_t)w.splitk_bytes));
    SK_TRY(linear_dgrad(M, 2 * F, d, dgu, P + o.wgu, dh, s));
    SK_TRY(linear_wgrad(M, 2 * F, d, dgu, h2, G + o.wgu, accumulate, s, lm->ws + w.splitk, (size_t)w.splitk_bytes));
    SK_TRY(sk_rmsnorm_bwd_launch(dh, xmid, P + o.ln2, r2, dxA, dxB, G + o.ln2, dwp, M, d, accumulate, s));
    // attention
    SK_TRY(linear_dgrad(M, d, d, dxB, P + o.wo, dao, s));
    SK_TRY(linear_wgrad(M, d, d, dxB, ao, G + o.wo, accumulate, s, lm->ws + w.splitk, (size_t)w.splitk_bytes));
    SK_TRY(sk_attn_tc_bwd_launch(qkv, ao, dao, lse, wsp<float>(lm, w.delta), nullptr, dqkv, B, T,
                                 lm->H, lm->KVH, Q, d, Q, 1, scale, s, seg_ptr(lm, a, w.seg_start), seg_ptr(lm, a, w.seg_end),
                                 lm->rope_cos, lm->rope_sin, pos_ids,
                                 lm->max_pos));   // inverse RoPE on dq / dk applied after the attention backward
    if (lm->qkv_bias)
      SK_TRY(sk_colsum_launch(dqkv, G + o.bqkv, wsp<float>(lm, w.colsum_partial), M, Q, Q, accumulate, s));
    SK_TRY(linear_dgrad(M, Q, d, dqkv, P + o.wqkv, dh, s));
    SK_TRY(linear_wgrad(M, Q, d, dqkv, h1, G + o.wqkv, accumulate, s, lm->ws + w.splitk, (size_t)w.splitk_bytes));
    SK_TRY(sk_rmsnorm_bwd_launch(dh, x, P + o.ln1, r1, dxB, dxA, G + o.ln1, dwp, M, d, accumulate, s));
    if (!lm->bwd_events.empty()) SK_CUDA_CHECK(cudaEventRecord(lm->bwd_events[l], s));
  }
  // embedding: tied -> add on top of the lm_head gradient just written; untied -> honour `accumulate`
  return sk_embed_bwd_launch(a.ids, dxA, wsp<float>(lm, w.embed_scratch), G + lm->off_embed, M, d, lm->V, lm->Vp,
                             lm->tie ? 1 : accumulate, s);
}

// byte offsets into the decode workspace for (B, T_cache): one token per row
struct DecLayout {
  int64_t gemm, gemm_bytes, x0, x1, h, qkv, ao, gu, act, lens, partial, total;
  int64_t e32 = 0;   // fp32 inference: the fp32 embedding sum [B, d]
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
  // fp32 inference: the activations are (hi, lo) pairs, lo right after hi
  const int64_t pf = lm->fp32 ? 2 : 1;
  w.gemm_bytes = align_up((int64_t)sk_gemm_ws_min_bytes(), 256);
  w.gemm = take(w.gemm_bytes);
  w.x0 = take((int64_t)B * lm->d * 2 * pf);
  w.x1 = take((int64_t)B * lm->d * 2 * pf);
  w.h = take((int64_t)B * lm->d * 2 * pf);
  w.qkv = take((int64_t)B * lm->qkv_dim * 2 * pf);
  w.ao = take((int64_t)B * lm->d * 2 * pf);
  // Qwen2: gate|up [B, 2F]; GPT-NeoX: pre-activation [B, F] followed by ln2's output [B, d]
  w.gu = take((int64_t)B * std::max(2 * lm->F, lm->F + lm->d) * 2 * pf);
  w.act = take((int64_t)B * lm->F * 2);
  w.lens = take((int64_t)B * 4);
  w.partial = take(sk_attn_decode_partial_bytes(B, lm->H, T_cache));
  if (lm->fp32) w.e32 = take((int64_t)B * lm->d * 4);
  w.total = cur;
  return w;
}

// n_cols: the logits columns the head writes (Vp, or the compact head's rows)
int check_decode(const SkLm* lm, int B, int T_cache, int ldl, int n_cols, const void* kv_cache, const void* logits,
                 const void* ws, int64_t ws_bytes, const DecLayout& w) {
  SK_REQUIRE(lm->params && lm->ws, "sk_lm: sk_lm_bind has not been called");
  SK_REQUIRE(kv_cache && logits && ws, "sk_lm decode: null argument");
  SK_REQUIRE(B > 0 && T_cache > 0 && T_cache <= lm->max_pos, "sk_lm decode: bad shape B=%d T_cache=%d (max_positions=%d)",
             B, T_cache, lm->max_pos);
  SK_REQUIRE(ldl >= n_cols && ldl % 8 == 0, "sk_lm decode: ldl must be >= %d and a multiple of 8 (got %d)", n_cols, ldl);
  SK_REQUIRE(((uintptr_t)ws & 255) == 0 && ((uintptr_t)kv_cache & 15) == 0 && ((uintptr_t)logits & 15) == 0,
             "sk_lm decode: decode workspace must be 256-byte, cache and logits 16-byte aligned");
  SK_REQUIRE(ws_bytes >= w.total, "sk_lm decode: decode workspace too small: need %lld bytes, got %lld", (long long)w.total,
             (long long)ws_bytes);
  return 0;
}

// the decode workspace's slots as typed pointers (fp32 inference: each hi half, its lo half right after it)
struct DecBufs {
  bf16 *x0, *x1, *h, *qkv, *ao, *gu, *act;
  int32_t* lens;
  float* partial;
  float* e32;
  void* gemm;
  size_t gemm_bytes;
  // compact head of sk_lm_prefill_sub / sk_lm_decode_step_sub: rows [head_n, head_k] (nullptr: the model's head)
  const bf16* head = nullptr;
  int head_n = 0;
};

DecBufs dec_bufs(void* ws, const DecLayout& dl) {
  uint8_t* p = reinterpret_cast<uint8_t*>(ws);
  auto b16 = [&](int64_t off) { return reinterpret_cast<bf16*>(p + off); };
  return DecBufs{b16(dl.x0), b16(dl.x1), b16(dl.h), b16(dl.qkv), b16(dl.ao), b16(dl.gu), b16(dl.act),
                 reinterpret_cast<int32_t*>(p + dl.lens), reinterpret_cast<float*>(p + dl.partial),
                 reinterpret_cast<float*>(p + dl.e32), p + dl.gemm, (size_t)dl.gemm_bytes};
}

// logits [B, ldl] of a bf16 decode step or prefill from the head input h [B, K]: the model's head, or the compact head.
// The compact GEMM is the same whole-tile plan as the full head (no scratch: no split-K, no stream-K), so every logit
// is the same K-ordered fp32 sum as the column of its id in the full step, only the tile width follows N.
int dec_head(const SkLm* lm, const DecBufs& b, int B, int K, const bf16* h, void* logits, int ldl, cudaStream_t s) {
  if (!b.head) return head_logits(lm, B, K, h, logits, ldl, s);
  return sk_gemm_ex_launch(sk_gemm_linear(B, b.head_n, K, h, b.head, logits, ldl, nullptr, nullptr, SK_ACT_NONE), s);
}

// ---- OPT decoder (HF:models/opt/modeling_opt.py:45-70 positions, :100-182 attention, :185-260 decoder layer,
// :480-560 decoder).  Separate functions from the Qwen2 ones above; forward / backward / decode_step pick one.

// OPT fp32 inference (forward only): every activation is a (hi, lo) bf16 pair [M, cols], lo at hi + the slab stride
// (sX, sqkv, sgu); no per-layer copies.  X / xmid are the residual stream before / after the attention branch, h1 the
// LayerNorm outputs (the final one included), gu relu(fc1); embed_scratch the fp32 embedding sum; logits fp32 [M, Vp].
WsLayout make_opt_fp32_layout(const SkLm* lm, int B, int T) {
  WsLayout w{};
  const int64_t M = (int64_t)B * T;
  int64_t cur = 0;
  auto take = [&](int64_t bytes) {
    const int64_t o = cur;
    cur = align_up(cur + bytes, 256);
    return o;
  };
  w.sX = w.sh = align_up(M * lm->d * 2, 256);
  w.sqkv = align_up(M * lm->qkv_dim * 2, 256);
  w.sgu = align_up(M * lm->F * 2, 256);
  // the split GEMMs take no scratch: only the 4 KB of flag words that sk_lm_bind clears at the fixed offset
  w.splitk_bytes = 4096;
  w.splitk = take(w.splitk_bytes);
  w.X = take(2 * w.sX);
  w.xmid = take(2 * w.sX);
  w.h1 = take(2 * w.sX);
  w.qkv = take(2 * w.sqkv);
  w.ao = take(2 * w.sX);
  w.gu = take(2 * w.sgu);
  w.embed_scratch = take(M * lm->d * 4);
  w.logits = take(M * lm->Vp * 4);
  w.total = cur;
  return w;
}

WsLayout layout_of(const SkLm* lm, int B, int T) {
  return lm->fp32 ? make_opt_fp32_layout(lm, B, T) : make_layout(lm, B, T);
}

// ---- GPT-NeoX decoder (HF:models/gpt_neox/modeling_gpt_neox.py: GPTNeoXAttention, GPTNeoXMLP, GPTNeoXLayer with
// use_parallel_residual = True, GPTNeoXModel, GPTNeoXForCausalLM).  Separate functions, picked as above.
//   h1 = LN1(x), h2 = LN2(x)              one dual-LayerNorm launch, shared mean / rstd
//   qkv = h1 Wqkv + b, partial RoPE       the RoPE epilogue with rot columns per head (weights in [Q;K;V] row order)
//   attn = attention(qkv) Wo + bo
//   pre = h2 W1 + b1, act = gelu(pre)     one epilogue, two outputs
//   x' = bf16(bf16(act W2 + b2 + attn) + x)   the two-residual epilogue, HF's order `mlp + attn + hidden_states`
int neox_forward(SkLm* lm, const FwdArgs& a, const WsLayout& w, cudaStream_t s) {
  const int B = a.B, T = a.T, M = B * T, d = lm->d, F = lm->F, L = lm->L, Q = lm->qkv_dim;
  const int32_t* pos_ids = a.pos_ids;
  const float eps = lm->eps;
  const bf16* P = lm->params;
  SK_TRY(sk_embed_fwd_launch(a.ids, P + lm->off_embed, wsp<bf16>(lm, w.X), M, d, lm->V, s));
  const float scale = 1.0f / sqrtf((float)lm->hd);
  SK_TRY(seg_bounds(lm, a, w, s));
  const int* seg_start = seg_ptr(lm, a, w.seg_start);
  bf16* attn = wsp<bf16>(lm, w.xmid);
  for (int l = 0; l < L; ++l) {
    const LnLayerOff& o = lm->lnl[l];
    bf16* x = wsp<bf16>(lm, w.X + w.sX * l);
    bf16* xn = wsp<bf16>(lm, w.X + w.sX * (l + 1));
    bf16* h1 = wsp<bf16>(lm, w.h1 + w.sh * l);
    bf16* h2 = wsp<bf16>(lm, w.h2 + w.sh * l);
    float* st = wsp<float>(lm, w.rstd1 + w.srstd * l);
    bf16* qkv = wsp<bf16>(lm, w.qkv + w.sqkv * l);
    bf16* ao = wsp<bf16>(lm, w.ao + w.sX * l);
    float* lse = wsp<float>(lm, w.lse + w.slse * l);
    bf16* pre = wsp<bf16>(lm, w.gu + w.sgu * l);
    bf16* act = wsp<bf16>(lm, w.act + w.sact * l);

    SK_TRY(sk_layernorm2_fwd_launch(x, P + o.ln1w, P + o.ln1b, P + o.ln2w, P + o.ln2b, h1, h2, st, st + M, M, d, eps, s));
    SK_TRY(sk_gemm_ex_launch(sk_gemm_rope(M, Q, d, h1, P + o.wqkv, P + o.bqkv, qkv, lm->rope_cos, lm->rope_sin, pos_ids, T,
                                          2 * d, lm->max_pos, lm->rot),
                             s));
    SK_TRY(sk_attn_tc_fwd_launch(qkv, ao, lse, B, T, lm->H, lm->H, Q, d, 1, scale, s, seg_start));
    SK_TRY(linear_fwd(M, d, d, ao, P + o.wo, attn, P + o.bo, nullptr, s));
    SK_TRY(sk_gemm_ex_launch(sk_gemm_gelu_fwd(M, F, d, h2, P + o.w1, P + o.b1, pre, act), s));
    SK_TRY(sk_gemm_ex_launch(sk_gemm_res2(M, d, F, act, P + o.w2, P + o.b2, attn, x, xn), s));
  }
  float* stf = wsp<float>(lm, w.rstdf);
  SK_TRY(sk_layernorm_fwd_launch(wsp<bf16>(lm, w.X + w.sX * L), P + lm->off_final_norm, P + lm->off_final_norm_b,
                                 wsp<bf16>(lm, w.hf), stf, stf + M, M, d, eps, s));
  return head_forward(lm, w, a, wsp<bf16>(lm, w.hf), d, s);
}

// The layer output's gradient dy reaches the MLP, the attention branch and the residual unchanged.  dense and
// dense_4h_to_h both take dy; their bias gradients are the same column sums, formed once per bias as HF does.  The input
// gradient dx = dy + LN1'(dh1) + LN2'(dh2) is summed in fp32 inside the dual-LayerNorm backward.
int neox_backward(SkLm* lm, const FwdArgs& a, int accumulate, const WsLayout& w, cudaStream_t s) {
  const int B = a.B, T = a.T, M = B * T, d = lm->d, F = lm->F, L = lm->L, Q = lm->qkv_dim;
  const int32_t* pos_ids = a.pos_ids;
  const bf16* P = lm->params;
  bf16* G = lm->grads;
  float* lnp = wsp<float>(lm, w.dw_partial);
  float* csp = wsp<float>(lm, w.colsum_partial);
  bf16* dy = wsp<bf16>(lm, w.dxA);
  bf16* dnext = wsp<bf16>(lm, w.dxB);
  bf16* dh = wsp<bf16>(lm, w.dh);
  bf16* dao = wsp<bf16>(lm, w.dao);
  bf16* dqkv = wsp<bf16>(lm, w.dqkv);
  bf16* dpre = wsp<bf16>(lm, w.dgu);
  void* sws = lm->ws + w.splitk;
  const size_t swb = (size_t)w.splitk_bytes;
  const float scale = 1.0f / sqrtf((float)lm->hd);
  const int* seg_start = seg_ptr(lm, a, w.seg_start);
  const int* seg_end = seg_ptr(lm, a, w.seg_end);

  if (a.with_head) SK_TRY(head_backward(lm, w, M, dh, wsp<bf16>(lm, w.hf), d, accumulate, s));
  const float* stf = wsp<float>(lm, w.rstdf);
  SK_TRY(sk_layernorm_bwd_launch(dh, wsp<bf16>(lm, w.X + w.sX * L), P + lm->off_final_norm, stf, stf + M, nullptr, dy,
                                 G + lm->off_final_norm, G + lm->off_final_norm_b, lnp,
                                 lnp + (size_t)sk_layernorm_bwd_blocks() * d, M, d, accumulate, s));
  if (!lm->bwd_events.empty()) SK_CUDA_CHECK(cudaEventRecord(lm->bwd_events[L], s));
  for (int l = L - 1; l >= 0; --l) {
    const LnLayerOff& o = lm->lnl[l];
    const bf16* x = wsp<bf16>(lm, w.X + w.sX * l);
    const bf16* h1 = wsp<bf16>(lm, w.h1 + w.sh * l);
    const bf16* h2 = wsp<bf16>(lm, w.h2 + w.sh * l);
    const float* st = wsp<float>(lm, w.rstd1 + w.srstd * l);
    const bf16* qkv = wsp<bf16>(lm, w.qkv + w.sqkv * l);
    const bf16* ao = wsp<bf16>(lm, w.ao + w.sX * l);
    const float* lse = wsp<float>(lm, w.lse + w.slse * l);
    const bf16* pre = wsp<bf16>(lm, w.gu + w.sgu * l);
    const bf16* act = wsp<bf16>(lm, w.act + w.sact * l);

    // MLP: d_pre = bf16(bf16(dy W2) * gelu'(pre)) from the GEMM epilogue; dh2 -> dh
    SK_TRY(sk_gemm_ex_launch(sk_gemm_gelu_bwd(M, d, F, dy, P + o.w2, pre, dpre), s));
    SK_TRY(linear_wgrad(M, d, F, dy, act, G + o.w2, accumulate, s, sws, swb));
    SK_TRY(sk_colsum_launch(dy, G + o.b2, csp, M, d, d, accumulate, s));
    SK_TRY(linear_dgrad(M, F, d, dpre, P + o.w1, dh, s));
    SK_TRY(linear_wgrad(M, F, d, dpre, h2, G + o.w1, accumulate, s, sws, swb));
    SK_TRY(sk_colsum_launch(dpre, G + o.b1, csp, M, F, F, accumulate, s));
    // attention: the same dy; inverse partial RoPE on dq / dk after the attention backward; dh1 -> dao
    SK_TRY(linear_dgrad(M, d, d, dy, P + o.wo, dao, s));
    SK_TRY(linear_wgrad(M, d, d, dy, ao, G + o.wo, accumulate, s, sws, swb));
    SK_TRY(sk_colsum_launch(dy, G + o.bo, csp, M, d, d, accumulate, s));
    SK_TRY(sk_attn_tc_bwd_launch(qkv, ao, dao, lse, wsp<float>(lm, w.delta), nullptr, dqkv, B, T, lm->H, lm->H, Q, d, Q, 1,
                                 scale, s, seg_start, seg_end));
    SK_TRY(sk_rope_launch(dqkv, lm->rope_cos, lm->rope_sin, pos_ids, M, T, Q, 2 * lm->H, lm->hd, 1, lm->max_pos, s,
                          lm->rot));
    SK_TRY(sk_colsum_launch(dqkv, G + o.bqkv, csp, M, Q, Q, accumulate, s));
    SK_TRY(linear_dgrad(M, Q, d, dqkv, P + o.wqkv, dao, s));
    SK_TRY(linear_wgrad(M, Q, d, dqkv, h1, G + o.wqkv, accumulate, s, sws, swb));
    SK_TRY(sk_layernorm2_bwd_launch(dao, dh, x, P + o.ln1w, P + o.ln2w, st, st + M, dy, dnext, G + o.ln1w, G + o.ln1b,
                                    G + o.ln2w, G + o.ln2b, lnp, M, d, accumulate, s));
    std::swap(dy, dnext);
    if (!lm->bwd_events.empty()) SK_CUDA_CHECK(cudaEventRecord(lm->bwd_events[l], s));
  }
  return sk_embed_bwd_launch(a.ids, dy, wsp<float>(lm, w.embed_scratch), G + lm->off_embed, M, d, lm->V, lm->Vp, accumulate, s);
}

// One token per row at position pos[b] (read on the device: the step is graph-capturable).  Decode workspace: h = ln1,
// `gu` = [pre (B x F) | ln2 (B x d)], `act` = the GELU, x1 = the attention branch's output; the layer output is written
// over x in place by the two-residual epilogue.
int neox_decode_step(SkLm* lm, const int64_t* tokens, const int32_t* pos, int B, void* kv_cache, int T_cache, void* logits,
                     int ldl, const DecBufs& b, cudaStream_t s) {
  const int d = lm->d, F = lm->F, Q = lm->qkv_dim;
  const float eps = lm->eps;
  const bf16* P = lm->params;
  bf16* x = b.x0;
  bf16* attn = b.x1;
  bf16* h = b.h;
  bf16* qkv = b.qkv;
  bf16* ao = b.ao;
  bf16* pre = b.gu;
  bf16* h2 = pre + (size_t)B * F;
  bf16* act = b.act;
  const size_t plane = (size_t)B * lm->H * T_cache * lm->hd;
  const float scale = 1.0f / sqrtf((float)lm->hd);
  SK_TRY(sk_embed_fwd_launch(tokens, P + lm->off_embed, x, B, d, lm->V, s));
  for (int l = 0; l < lm->L; ++l) {
    const LnLayerOff& o = lm->lnl[l];
    bf16* kc = reinterpret_cast<bf16*>(kv_cache) + (size_t)l * 2 * plane;
    bf16* vc = kc + plane;
    SK_TRY(sk_layernorm2_fwd_launch(x, P + o.ln1w, P + o.ln1b, P + o.ln2w, P + o.ln2b, h, h2, nullptr, nullptr, B, d, eps, s));
    SK_TRY(sk_gemm_ex_launch(
        sk_gemm_rope(B, Q, d, h, P + o.wqkv, P + o.bqkv, qkv, lm->rope_cos, lm->rope_sin, pos, 1, 2 * d, lm->max_pos, lm->rot),
        s));
    SK_TRY(sk_kv_append_launch(qkv, Q, kc, vc, pos, b.lens, B, lm->H, lm->H, T_cache, s));
    SK_TRY(sk_attn_decode_launch(qkv, Q, kc, vc, b.lens, ao, d, b.partial, B, lm->H, lm->H, T_cache, scale, s));
    SK_TRY(linear_fwd(B, d, d, ao, P + o.wo, attn, P + o.bo, nullptr, s));
    SK_TRY(sk_gemm_ex_launch(sk_gemm_gelu_fwd(B, F, d, h2, P + o.w1, P + o.b1, pre, act), s));
    // with M = B the scratch lets stream-K spread dense_4h_to_h's long K loop over idle SMs
    SK_TRY(sk_gemm_ex_launch(sk_gemm_res2(B, d, F, act, P + o.w2, P + o.b2, attn, x, x, b.gemm, b.gemm_bytes), s));
  }
  SK_TRY(sk_layernorm_fwd_launch(x, P + lm->off_final_norm, P + lm->off_final_norm_b, h, nullptr, nullptr, B, d, eps, s));
  return dec_head(lm, b, B, d, h, logits, ldl, s);
}

// ---- OPT with fp32 master weights (sk_lm_set_master): HF OPTForCausalLM with fp32 parameters under
// torch.autocast(bfloat16).  The residual stream X / xmid is fp32 and never rounded; every LayerNorm reads it with fp32
// gamma / beta and hands the next linear one bf16 rounding; every linear is the bf16 path's GEMM on the bf16 shadow
// weights with a bf16 output, which is autocast's linear.  Each branch output's residual add is fused into the next
// LayerNorm (the last fc2's into the final norm); the bf16 branch output waits in the dxB slab, unused until backward.
int opt_master_forward(SkLm* lm, const FwdArgs& a, const WsLayout& w, cudaStream_t s) {
  const int B = a.B, T = a.T, M = B * T, d = lm->d, F = lm->F, L = lm->L, Q = lm->qkv_dim;
  const float eps = lm->eps;
  const bf16* P = lm->params;
  const float* P32 = lm->params32;
  bf16* y = wsp<bf16>(lm, w.dxB);
  SK_TRY(sk_opt_embed_fwd_f32_launch(a.ids, a.pos_ids, P32 + lm->off_embed, P32 + lm->off_pos, wsp<float>(lm, w.X), M, T, d,
                                     lm->V, lm->n_pos, s));
  const float scale = 1.0f / sqrtf((float)lm->hd);
  SK_TRY(seg_bounds(lm, a, w, s));
  const int* seg_start = seg_ptr(lm, a, w.seg_start);
  for (int l = 0; l < L; ++l) {
    const LnLayerOff& o = lm->lnl[l];
    float* x = wsp<float>(lm, w.X + w.sR * l);
    float* xmid = wsp<float>(lm, w.xmid + w.sR * l);
    bf16* h1 = wsp<bf16>(lm, w.h1 + w.sh * l);
    float* st1 = wsp<float>(lm, w.rstd1 + w.srstd * l);
    bf16* qkv = wsp<bf16>(lm, w.qkv + w.sqkv * l);
    bf16* ao = wsp<bf16>(lm, w.ao + w.sX * l);
    float* lse = wsp<float>(lm, w.lse + w.slse * l);
    bf16* h2 = wsp<bf16>(lm, w.h2 + w.sh * l);
    float* st2 = wsp<float>(lm, w.rstd2 + w.srstd * l);
    bf16* a = wsp<bf16>(lm, w.gu + w.sgu * l);

    // x = xmid[l-1] + fc2 output of layer l-1 (layer 0: the embedding sum as it is)
    const float* xin = l == 0 ? x : wsp<float>(lm, w.xmid + w.sR * (l - 1));
    SK_TRY(sk_add_layernorm_f32_launch(xin, l == 0 ? nullptr : y, P32 + o.ln1w, P32 + o.ln1b, l == 0 ? nullptr : x, h1, st1,
                                       st1 + M, M, d, eps, s));
    SK_TRY(linear_fwd(M, Q, d, h1, P + o.wqkv, qkv, P + o.bqkv, nullptr, s));
    SK_TRY(sk_attn_tc_fwd_launch(qkv, ao, lse, B, T, lm->H, lm->H, Q, d, 1, scale, s, seg_start));
    SK_TRY(linear_fwd(M, d, d, ao, P + o.wo, y, P + o.bo, nullptr, s));
    SK_TRY(sk_add_layernorm_f32_launch(x, y, P32 + o.ln2w, P32 + o.ln2b, xmid, h2, st2, st2 + M, M, d, eps, s));
    SK_TRY(linear_fwd(M, F, d, h2, P + o.w1, a, P + o.b1, nullptr, s, SK_ACT_RELU));   // relu(fc1)
    SK_TRY(linear_fwd(M, d, F, a, P + o.w2, y, P + o.b2, nullptr, s));
  }
  float* stf = wsp<float>(lm, w.rstdf);
  SK_TRY(sk_add_layernorm_f32_launch(wsp<float>(lm, w.xmid + w.sR * (L - 1)), y, P32 + lm->off_final_norm,
                                     P32 + lm->off_final_norm_b, wsp<float>(lm, w.X + w.sR * L), wsp<bf16>(lm, w.hf), stf,
                                     stf + M, M, d, eps, s));
  return head_forward(lm, w, a, wsp<bf16>(lm, w.hf), d, s);
}

// The residual gradient dres is fp32 (dres32); each branch's GEMMs and bias column sums read its bf16 copy (dxA), and
// each LayerNorm backward adds its input gradient to dres in fp32.  Linear weight and bias gradients land in the bf16
// buffer (never accumulated there) and are widened into grads32 at the end; LayerNorm and table gradients go straight
// into grads32.  `accumulate` = a later micro-batch: add to grads32 instead of overwriting it.
int opt_master_backward(SkLm* lm, const FwdArgs& a, int accumulate, const WsLayout& w, cudaStream_t s) {
  const int B = a.B, T = a.T, M = B * T, d = lm->d, F = lm->F, L = lm->L, Q = lm->qkv_dim;
  const bf16* P = lm->params;
  const float* P32 = lm->params32;
  bf16* G = lm->grads;
  float* G32 = lm->grads32;
  float* lnp = wsp<float>(lm, w.dw_partial);
  float* csp = wsp<float>(lm, w.colsum_partial);
  float* dres = wsp<float>(lm, w.dres32);
  bf16* dr16 = wsp<bf16>(lm, w.dxA);
  bf16* dh = wsp<bf16>(lm, w.dh);
  bf16* dao = wsp<bf16>(lm, w.dao);
  bf16* dqkv = wsp<bf16>(lm, w.dqkv);
  bf16* da = wsp<bf16>(lm, w.dgu);
  void* sws = lm->ws + w.splitk;
  const size_t swb = (size_t)w.splitk_bytes;
  const float scale = 1.0f / sqrtf((float)lm->hd);
  const int* seg_start = seg_ptr(lm, a, w.seg_start);
  const int* seg_end = seg_ptr(lm, a, w.seg_end);

  // the bf16 gradient buffer holds one micro-batch (grads32 accumulates)
  if (a.with_head) SK_TRY(head_backward(lm, w, M, dh, wsp<bf16>(lm, w.hf), d, 0, s));
  const float* stf = wsp<float>(lm, w.rstdf);
  SK_TRY(sk_layernorm_bwd_f32_launch(dh, wsp<float>(lm, w.X + w.sR * L), P32 + lm->off_final_norm, stf, stf + M, nullptr, dres,
                                     dr16, G32 + lm->off_final_norm, G32 + lm->off_final_norm_b, lnp, M, d, accumulate, s));
  if (!lm->bwd_events.empty()) SK_CUDA_CHECK(cudaEventRecord(lm->bwd_events[L], s));
  for (int l = L - 1; l >= 0; --l) {
    const LnLayerOff& o = lm->lnl[l];
    const float* x = wsp<float>(lm, w.X + w.sR * l);
    const float* xmid = wsp<float>(lm, w.xmid + w.sR * l);
    const bf16* h1 = wsp<bf16>(lm, w.h1 + w.sh * l);
    const float* st1 = wsp<float>(lm, w.rstd1 + w.srstd * l);
    const bf16* qkv = wsp<bf16>(lm, w.qkv + w.sqkv * l);
    const bf16* ao = wsp<bf16>(lm, w.ao + w.sX * l);
    const float* lse = wsp<float>(lm, w.lse + w.slse * l);
    const bf16* h2 = wsp<bf16>(lm, w.h2 + w.sh * l);
    const float* st2 = wsp<float>(lm, w.rstd2 + w.srstd * l);
    const bf16* a = wsp<bf16>(lm, w.gu + w.sgu * l);

    // MLP on bf16(dres)
    SK_TRY(linear_dgrad(M, d, F, dr16, P + o.w2, da, s));
    SK_TRY(sk_relu_bwd_launch(da, a, (long)M * F, s));
    SK_TRY(linear_wgrad(M, d, F, dr16, a, G + o.w2, false, s, sws, swb));
    SK_TRY(sk_colsum_launch(dr16, G + o.b2, csp, M, d, d, 0, s));
    SK_TRY(linear_dgrad(M, F, d, da, P + o.w1, dh, s));
    SK_TRY(linear_wgrad(M, F, d, da, h2, G + o.w1, false, s, sws, swb));
    SK_TRY(sk_colsum_launch(da, G + o.b1, csp, M, F, F, 0, s));
    SK_TRY(sk_layernorm_bwd_f32_launch(dh, xmid, P32 + o.ln2w, st2, st2 + M, dres, dres, dr16, G32 + o.ln2w, G32 + o.ln2b, lnp, M,
                                       d, accumulate, s));
    // attention on bf16(dres)
    SK_TRY(linear_dgrad(M, d, d, dr16, P + o.wo, dao, s));
    SK_TRY(linear_wgrad(M, d, d, dr16, ao, G + o.wo, false, s, sws, swb));
    SK_TRY(sk_colsum_launch(dr16, G + o.bo, csp, M, d, d, 0, s));
    SK_TRY(sk_attn_tc_bwd_launch(qkv, ao, dao, lse, wsp<float>(lm, w.delta), nullptr, dqkv, B, T, lm->H, lm->H, Q, d, Q, 1,
                                 scale, s, seg_start, seg_end));
    SK_TRY(sk_colsum_launch(dqkv, G + o.bqkv, csp, M, Q, Q, 0, s));
    SK_TRY(linear_dgrad(M, Q, d, dqkv, P + o.wqkv, dh, s));
    SK_TRY(linear_wgrad(M, Q, d, dqkv, h1, G + o.wqkv, false, s, sws, swb));
    SK_TRY(sk_layernorm_bwd_f32_launch(dh, x, P32 + o.ln1w, st1, st1 + M, dres, dres, dr16, G32 + o.ln1w, G32 + o.ln1b, lnp, M, d,
                                       accumulate, s));
    if (!lm->bwd_events.empty()) SK_CUDA_CHECK(cudaEventRecord(lm->bwd_events[l], s));
  }
  float* scratch = wsp<float>(lm, w.embed_scratch);
  SK_TRY(sk_table_bwd_f32_launch(a.ids, nullptr, dres, scratch, G32 + lm->off_embed,
                                 lm->tie ? G + lm->off_head : nullptr, M, T, d, lm->V, lm->Vp, accumulate, s));
  SK_TRY(sk_table_bwd_f32_launch(nullptr, a.pos_ids, dres, scratch, G32 + lm->off_pos, nullptr, M, T, d, lm->n_pos, lm->n_pos,
                                 accumulate, s));
  return sk_widen_grads_launch(G, G32, lm->d_widen_start, lm->d_widen_len, lm->n_widen, accumulate, s);
}

// ---- post-LayerNorm OPT (HF OPTDecoderLayer with do_layer_norm_before = False, and OPTDecoder's bias-free
// project_in / project_out; facebook/opt-350m).  No new per-layer memory: X[l] holds the layer input, xmid
// s1 = bf16(bf16(attn W_o + b_o) + x), h1 y1 = LN1(s1), h2 s2 = bf16(bf16(relu(y1 W_1 + b_1) W_2 + b_2) + y1),
// X[l+1] = LN2(s2); rstd1 / rstd2 the two LayerNorms' mean / rstd, gu relu(fc1).  With projections, `pe` holds the token
// rows e [M, proj_dim] and hf the head input h = bf16(x_L W_out^T) [M, proj_dim].
int opt_postln_forward(SkLm* lm, const FwdArgs& a, const WsLayout& w, cudaStream_t s) {
  const int B = a.B, T = a.T, M = B * T, d = lm->d, F = lm->F, L = lm->L, Q = lm->qkv_dim, K = head_k(lm);
  const int64_t* ids = a.ids;
  const int32_t* pos_ids = a.pos_ids;
  const float eps = lm->eps;
  const bf16* P = lm->params;
  bf16* X0 = wsp<bf16>(lm, w.X);
  if (lm->proj) {
    // x0 = bf16(bf16(e W_in^T) + pos[p + 2]): the position rows, gathered into dxB (unused until the backward pass), are
    // the GEMM's residual, added after the projection is rounded
    bf16* e = wsp<bf16>(lm, w.pe);
    bf16* prow = wsp<bf16>(lm, w.dxB);
    SK_TRY(sk_embed_fwd_launch(ids, P + lm->off_embed, e, M, K, lm->V, s));
    SK_TRY(sk_opt_embed_fwd_launch(ids, pos_ids, nullptr, P + lm->off_pos, prow, M, T, d, lm->V, lm->n_pos, s));
    SK_TRY(linear_fwd(M, d, K, e, P + lm->off_pin, X0, nullptr, prow, s));
  } else {
    SK_TRY(sk_opt_embed_fwd_launch(ids, pos_ids, P + lm->off_embed, P + lm->off_pos, X0, M, T, d, lm->V, lm->n_pos, s));
  }
  const float scale = 1.0f / sqrtf((float)lm->hd);
  SK_TRY(seg_bounds(lm, a, w, s));
  const int* seg_start = seg_ptr(lm, a, w.seg_start);
  for (int l = 0; l < L; ++l) {
    const LnLayerOff& o = lm->lnl[l];
    bf16* x = wsp<bf16>(lm, w.X + w.sX * l);
    bf16* xn = wsp<bf16>(lm, w.X + w.sX * (l + 1));
    bf16* y1 = wsp<bf16>(lm, w.h1 + w.sh * l);
    float* st1 = wsp<float>(lm, w.rstd1 + w.srstd * l);
    bf16* qkv = wsp<bf16>(lm, w.qkv + w.sqkv * l);
    bf16* ao = wsp<bf16>(lm, w.ao + w.sX * l);
    float* lse = wsp<float>(lm, w.lse + w.slse * l);
    bf16* s1 = wsp<bf16>(lm, w.xmid + w.sX * l);
    bf16* s2 = wsp<bf16>(lm, w.h2 + w.sh * l);
    float* st2 = wsp<float>(lm, w.rstd2 + w.srstd * l);
    bf16* a = wsp<bf16>(lm, w.gu + w.sgu * l);

    SK_TRY(linear_fwd(M, Q, d, x, P + o.wqkv, qkv, P + o.bqkv, nullptr, s));
    SK_TRY(sk_attn_tc_fwd_launch(qkv, ao, lse, B, T, lm->H, lm->H, Q, d, 1, scale, s, seg_start));
    SK_TRY(linear_fwd(M, d, d, ao, P + o.wo, s1, P + o.bo, x, s));
    SK_TRY(sk_layernorm_fwd_launch(s1, P + o.ln1w, P + o.ln1b, y1, st1, st1 + M, M, d, eps, s));
    SK_TRY(linear_fwd(M, F, d, y1, P + o.w1, a, P + o.b1, nullptr, s, SK_ACT_RELU));   // relu(fc1)
    SK_TRY(linear_fwd(M, d, F, a, P + o.w2, s2, P + o.b2, y1, s));
    SK_TRY(sk_layernorm_fwd_launch(s2, P + o.ln2w, P + o.ln2b, xn, st2, st2 + M, M, d, eps, s));
  }
  if (lm->proj)
    SK_TRY(linear_fwd(M, K, d, wsp<bf16>(lm, w.X + w.sX * L), P + lm->off_pout, wsp<bf16>(lm, w.hf), nullptr, nullptr, s));
  return head_forward(lm, w, a, head_in(lm, w), K, s);
}

// The residual stream is the LayerNorm output, so each LayerNorm backward reads the sum of its output's two gradients:
// the fc1 and q|k|v dgrad GEMMs add the skip path's gradient in their epilogue, bf16(ds + bf16(dgrad)) as autograd
// rounds it.  Every reduction is the deterministic one of the pre-LN path.
int opt_postln_backward(SkLm* lm, const FwdArgs& a, int accumulate, const WsLayout& w, cudaStream_t s) {
  const int B = a.B, T = a.T, M = B * T, d = lm->d, F = lm->F, L = lm->L, Q = lm->qkv_dim, K = head_k(lm);
  const bf16* P = lm->params;
  bf16* G = lm->grads;
  float* dwp = wsp<float>(lm, w.dw_partial);
  float* dbp = dwp + (size_t)sk_layernorm_bwd_blocks() * d;
  float* csp = wsp<float>(lm, w.colsum_partial);
  bf16* dxA = wsp<bf16>(lm, w.dxA);
  bf16* dxB = wsp<bf16>(lm, w.dxB);
  bf16* dh = wsp<bf16>(lm, w.dh);   // [M, proj_dim]: the gradient of h, later of e
  bf16* dao = wsp<bf16>(lm, w.dao);
  bf16* dqkv = wsp<bf16>(lm, w.dqkv);
  bf16* da = wsp<bf16>(lm, w.dgu);
  bf16* xL = wsp<bf16>(lm, w.X + w.sX * L);
  void* sws = lm->ws + w.splitk;
  const size_t swb = (size_t)w.splitk_bytes;
  const float scale = 1.0f / sqrtf((float)lm->hd);
  const int* seg_start = seg_ptr(lm, a, w.seg_start);
  const int* seg_end = seg_ptr(lm, a, w.seg_end);

  // tied head at K = proj_dim (already done chunk by chunk for large vocabularies)
  if (a.with_head) SK_TRY(head_backward(lm, w, M, lm->proj ? dh : dxA, head_in(lm, w), K, accumulate, s));
  if (lm->proj) {
    SK_TRY(linear_dgrad(M, K, d, dh, P + lm->off_pout, dxA, s));
    SK_TRY(linear_wgrad(M, K, d, dh, xL, G + lm->off_pout, accumulate, s, sws, swb));
  }
  if (!lm->bwd_events.empty()) SK_CUDA_CHECK(cudaEventRecord(lm->bwd_events[L], s));
  for (int l = L - 1; l >= 0; --l) {   // dxA: the gradient of the layer's output LN2(s2)
    const LnLayerOff& o = lm->lnl[l];
    const bf16* x = wsp<bf16>(lm, w.X + w.sX * l);
    const bf16* y1 = wsp<bf16>(lm, w.h1 + w.sh * l);
    const float* st1 = wsp<float>(lm, w.rstd1 + w.srstd * l);
    const bf16* qkv = wsp<bf16>(lm, w.qkv + w.sqkv * l);
    const bf16* ao = wsp<bf16>(lm, w.ao + w.sX * l);
    const float* lse = wsp<float>(lm, w.lse + w.slse * l);
    const bf16* s1 = wsp<bf16>(lm, w.xmid + w.sX * l);
    const bf16* s2 = wsp<bf16>(lm, w.h2 + w.sh * l);
    const float* st2 = wsp<float>(lm, w.rstd2 + w.srstd * l);
    const bf16* a = wsp<bf16>(lm, w.gu + w.sgu * l);

    // LN2 backward from s2: ds2 -> dxB
    SK_TRY(sk_layernorm_bwd_launch(dxA, s2, P + o.ln2w, st2, st2 + M, nullptr, dxB, G + o.ln2w, G + o.ln2b, dwp, dbp, M, d,
                                   accumulate, s));
    // MLP: dy = ds2; ReLU backward masked by the saved a = relu(fc1) > 0
    SK_TRY(linear_dgrad(M, d, F, dxB, P + o.w2, da, s));
    SK_TRY(sk_relu_bwd_launch(da, a, (long)M * F, s));
    SK_TRY(linear_wgrad(M, d, F, dxB, a, G + o.w2, accumulate, s, sws, swb));
    SK_TRY(sk_colsum_launch(dxB, G + o.b2, csp, M, d, d, accumulate, s));
    // dy1 = bf16(ds2 + bf16(da W_1)) -> dxA: fc1's dgrad with the skip path's gradient as its residual
    SK_TRY(linear_dgrad(M, F, d, da, P + o.w1, dxA, s, dxB));
    SK_TRY(linear_wgrad(M, F, d, da, y1, G + o.w1, accumulate, s, sws, swb));
    SK_TRY(sk_colsum_launch(da, G + o.b1, csp, M, F, F, accumulate, s));
    // LN1 backward from s1: ds1 -> dxB
    SK_TRY(sk_layernorm_bwd_launch(dxA, s1, P + o.ln1w, st1, st1 + M, nullptr, dxB, G + o.ln1w, G + o.ln1b, dwp, dbp, M, d,
                                   accumulate, s));
    // attention: dy = ds1
    SK_TRY(linear_dgrad(M, d, d, dxB, P + o.wo, dao, s));
    SK_TRY(linear_wgrad(M, d, d, dxB, ao, G + o.wo, accumulate, s, sws, swb));
    SK_TRY(sk_colsum_launch(dxB, G + o.bo, csp, M, d, d, accumulate, s));
    SK_TRY(sk_attn_tc_bwd_launch(qkv, ao, dao, lse, wsp<float>(lm, w.delta), nullptr, dqkv, B, T, lm->H, lm->H, Q, d, Q, 1,
                                 scale, s, seg_start, seg_end));
    SK_TRY(sk_colsum_launch(dqkv, G + o.bqkv, csp, M, Q, Q, accumulate, s));
    // dx = bf16(ds1 + bf16(dqkv W_qkv)) -> dxA
    SK_TRY(linear_dgrad(M, Q, d, dqkv, P + o.wqkv, dxA, s, dxB));
    SK_TRY(linear_wgrad(M, Q, d, dqkv, x, G + o.wqkv, accumulate, s, sws, swb));
    if (!lm->bwd_events.empty()) SK_CUDA_CHECK(cudaEventRecord(lm->bwd_events[l], s));
  }
  // dxA = the gradient of x0: the position table, then project_in, then the (tied) token table
  float* scratch = wsp<float>(lm, w.embed_scratch);
  SK_TRY(sk_opt_pos_bwd_launch(a.pos_ids, dxA, scratch, G + lm->off_pos, M, T, d, lm->n_pos, accumulate, s));
  const bf16* de = dxA;
  if (lm->proj) {
    SK_TRY(linear_wgrad(M, d, K, dxA, wsp<bf16>(lm, w.pe), G + lm->off_pin, accumulate, s, sws, swb));
    SK_TRY(linear_dgrad(M, d, K, dxA, P + lm->off_pin, dh, s));
    de = dh;
  }
  return sk_embed_bwd_launch(a.ids, de, scratch, G + lm->off_embed, M, K, lm->V, lm->Vp, lm->tie ? 1 : accumulate, s);
}

int opt_forward(SkLm* lm, const FwdArgs& a, const WsLayout& w, cudaStream_t s) {
  const int B = a.B, T = a.T, M = B * T, d = lm->d, F = lm->F, L = lm->L, Q = lm->qkv_dim;
  const float eps = lm->eps;
  const bf16* P = lm->params;
  SK_TRY(sk_opt_embed_fwd_launch(a.ids, a.pos_ids, P + lm->off_embed, P + lm->off_pos, wsp<bf16>(lm, w.X), M, T, d, lm->V,
                                 lm->n_pos, s));
  // q is multiplied by head_dim^-0.5 = 1/8 after q_proj (HF:modeling_opt.py:146); a power of two, so the same value as
  // scaling the scores inside attention
  const float scale = 1.0f / sqrtf((float)lm->hd);
  SK_TRY(seg_bounds(lm, a, w, s));
  const int* seg_start = seg_ptr(lm, a, w.seg_start);
  for (int l = 0; l < L; ++l) {
    const LnLayerOff& o = lm->lnl[l];
    bf16* x = wsp<bf16>(lm, w.X + w.sX * l);
    bf16* xn = wsp<bf16>(lm, w.X + w.sX * (l + 1));
    bf16* h1 = wsp<bf16>(lm, w.h1 + w.sh * l);
    float* st1 = wsp<float>(lm, w.rstd1 + w.srstd * l);
    bf16* qkv = wsp<bf16>(lm, w.qkv + w.sqkv * l);
    bf16* ao = wsp<bf16>(lm, w.ao + w.sX * l);
    float* lse = wsp<float>(lm, w.lse + w.slse * l);
    bf16* xmid = wsp<bf16>(lm, w.xmid + w.sX * l);
    bf16* h2 = wsp<bf16>(lm, w.h2 + w.sh * l);
    float* st2 = wsp<float>(lm, w.rstd2 + w.srstd * l);
    bf16* a = wsp<bf16>(lm, w.gu + w.sgu * l);

    SK_TRY(sk_layernorm_fwd_launch(x, P + o.ln1w, P + o.ln1b, h1, st1, st1 + M, M, d, eps, s));
    SK_TRY(linear_fwd(M, Q, d, h1, P + o.wqkv, qkv, P + o.bqkv, nullptr, s));
    SK_TRY(sk_attn_tc_fwd_launch(qkv, ao, lse, B, T, lm->H, lm->H, Q, d, 1, scale, s, seg_start));
    SK_TRY(linear_fwd(M, d, d, ao, P + o.wo, xmid, P + o.bo, x, s));
    SK_TRY(sk_layernorm_fwd_launch(xmid, P + o.ln2w, P + o.ln2b, h2, st2, st2 + M, M, d, eps, s));
    SK_TRY(linear_fwd(M, F, d, h2, P + o.w1, a, P + o.b1, nullptr, s, SK_ACT_RELU));   // relu(fc1)
    SK_TRY(linear_fwd(M, d, F, a, P + o.w2, xn, P + o.b2, xmid, s));
  }
  float* stf = wsp<float>(lm, w.rstdf);
  SK_TRY(sk_layernorm_fwd_launch(wsp<bf16>(lm, w.X + w.sX * L), P + lm->off_final_norm, P + lm->off_final_norm_b,
                                 wsp<bf16>(lm, w.hf), stf, stf + M, M, d, eps, s));
  return head_forward(lm, w, a, wsp<bf16>(lm, w.hf), d, s);
}

// The embedding table's pad row gets the gradient of every token equal to pad_token_id.  HF's nn.Embedding(padding_idx)
// drops that row's gradient instead; in right-padded and packed batches the two agree exactly, because the gradient
// reaching a pad position is zero (pad targets carry no loss and only later pad positions attend to a pad key).
int opt_backward(SkLm* lm, const FwdArgs& a, int accumulate, const WsLayout& w, cudaStream_t s) {
  const int B = a.B, T = a.T, M = B * T, d = lm->d, F = lm->F, L = lm->L, Q = lm->qkv_dim;
  const bf16* P = lm->params;
  bf16* G = lm->grads;
  float* dwp = wsp<float>(lm, w.dw_partial);
  float* dbp = dwp + (size_t)sk_layernorm_bwd_blocks() * d;
  float* csp = wsp<float>(lm, w.colsum_partial);
  bf16* dxA = wsp<bf16>(lm, w.dxA);
  bf16* dxB = wsp<bf16>(lm, w.dxB);
  bf16* dh = wsp<bf16>(lm, w.dh);
  bf16* dao = wsp<bf16>(lm, w.dao);
  bf16* dqkv = wsp<bf16>(lm, w.dqkv);
  bf16* da = wsp<bf16>(lm, w.dgu);
  void* sws = lm->ws + w.splitk;
  const size_t swb = (size_t)w.splitk_bytes;
  const float scale = 1.0f / sqrtf((float)lm->hd);
  const int* seg_start = seg_ptr(lm, a, w.seg_start);
  const int* seg_end = seg_ptr(lm, a, w.seg_end);

  if (a.with_head) SK_TRY(head_backward(lm, w, M, dh, wsp<bf16>(lm, w.hf), d, accumulate, s));
  const float* stf = wsp<float>(lm, w.rstdf);
  SK_TRY(sk_layernorm_bwd_launch(dh, wsp<bf16>(lm, w.X + w.sX * L), P + lm->off_final_norm, stf, stf + M, nullptr, dxA,
                                 G + lm->off_final_norm, G + lm->off_final_norm_b, dwp, dbp, M, d, accumulate, s));
  if (!lm->bwd_events.empty()) SK_CUDA_CHECK(cudaEventRecord(lm->bwd_events[L], s));
  for (int l = L - 1; l >= 0; --l) {
    const LnLayerOff& o = lm->lnl[l];
    const bf16* x = wsp<bf16>(lm, w.X + w.sX * l);
    const bf16* h1 = wsp<bf16>(lm, w.h1 + w.sh * l);
    const float* st1 = wsp<float>(lm, w.rstd1 + w.srstd * l);
    const bf16* qkv = wsp<bf16>(lm, w.qkv + w.sqkv * l);
    const bf16* ao = wsp<bf16>(lm, w.ao + w.sX * l);
    const float* lse = wsp<float>(lm, w.lse + w.slse * l);
    const bf16* xmid = wsp<bf16>(lm, w.xmid + w.sX * l);
    const bf16* h2 = wsp<bf16>(lm, w.h2 + w.sh * l);
    const float* st2 = wsp<float>(lm, w.rstd2 + w.srstd * l);
    const bf16* a = wsp<bf16>(lm, w.gu + w.sgu * l);

    // MLP: dy = dxA.  ReLU backward as one element-wise pass over fc2's dgrad, masked by the saved a = relu(fc1) > 0
    SK_TRY(linear_dgrad(M, d, F, dxA, P + o.w2, da, s));
    SK_TRY(sk_relu_bwd_launch(da, a, (long)M * F, s));
    SK_TRY(linear_wgrad(M, d, F, dxA, a, G + o.w2, accumulate, s, sws, swb));
    SK_TRY(sk_colsum_launch(dxA, G + o.b2, csp, M, d, d, accumulate, s));
    SK_TRY(linear_dgrad(M, F, d, da, P + o.w1, dh, s));
    SK_TRY(linear_wgrad(M, F, d, da, h2, G + o.w1, accumulate, s, sws, swb));
    SK_TRY(sk_colsum_launch(da, G + o.b1, csp, M, F, F, accumulate, s));
    SK_TRY(sk_layernorm_bwd_launch(dh, xmid, P + o.ln2w, st2, st2 + M, dxA, dxB, G + o.ln2w, G + o.ln2b, dwp, dbp, M, d,
                                   accumulate, s));
    // attention: dy = dxB
    SK_TRY(linear_dgrad(M, d, d, dxB, P + o.wo, dao, s));
    SK_TRY(linear_wgrad(M, d, d, dxB, ao, G + o.wo, accumulate, s, sws, swb));
    SK_TRY(sk_colsum_launch(dxB, G + o.bo, csp, M, d, d, accumulate, s));
    SK_TRY(sk_attn_tc_bwd_launch(qkv, ao, dao, lse, wsp<float>(lm, w.delta), nullptr, dqkv, B, T, lm->H, lm->H, Q, d, Q, 1,
                                 scale, s, seg_start, seg_end));
    SK_TRY(sk_colsum_launch(dqkv, G + o.bqkv, csp, M, Q, Q, accumulate, s));
    SK_TRY(linear_dgrad(M, Q, d, dqkv, P + o.wqkv, dh, s));
    SK_TRY(linear_wgrad(M, Q, d, dqkv, h1, G + o.wqkv, accumulate, s, sws, swb));
    SK_TRY(sk_layernorm_bwd_launch(dh, x, P + o.ln1w, st1, st1 + M, dxB, dxA, G + o.ln1w, G + o.ln1b, dwp, dbp, M, d,
                                   accumulate, s));
    if (!lm->bwd_events.empty()) SK_CUDA_CHECK(cudaEventRecord(lm->bwd_events[l], s));
  }
  SK_TRY(sk_embed_bwd_launch(a.ids, dxA, wsp<float>(lm, w.embed_scratch), G + lm->off_embed, M, d, lm->V, lm->Vp,
                             lm->tie ? 1 : accumulate, s));
  return sk_opt_pos_bwd_launch(a.pos_ids, dxA, wsp<float>(lm, w.embed_scratch), G + lm->off_pos, M, T, d, lm->n_pos, accumulate, s);
}

// Post-LN decode step (the formulas of opt_postln_forward at M = B).  With projections the h slot holds e [B, proj_dim]
// at the start and the head input bf16(x_L W_out^T) at the end; x1 the position rows, then s1 and s2.
int opt_postln_decode_step(SkLm* lm, const int64_t* tokens, const int32_t* pos, int B, void* kv_cache, int T_cache,
                           void* logits, int ldl, const DecBufs& b, cudaStream_t s) {
  const int d = lm->d, F = lm->F, Q = lm->qkv_dim, K = head_k(lm);
  const float eps = lm->eps;
  const bf16* P = lm->params;
  bf16* x = b.x0;
  bf16* xm = b.x1;
  bf16* h = b.h;
  bf16* qkv = b.qkv;
  bf16* ao = b.ao;
  bf16* a = b.gu;
  const size_t plane = (size_t)B * lm->H * T_cache * lm->hd;
  const float scale = 1.0f / sqrtf((float)lm->hd);
  if (lm->proj) {
    SK_TRY(sk_embed_fwd_launch(tokens, P + lm->off_embed, h, B, K, lm->V, s));
    SK_TRY(sk_opt_embed_fwd_launch(tokens, pos, nullptr, P + lm->off_pos, xm, B, 1, d, lm->V, lm->n_pos, s));
    SK_TRY(linear_fwd(B, d, K, h, P + lm->off_pin, x, nullptr, xm, s));
  } else {
    SK_TRY(sk_opt_embed_fwd_launch(tokens, pos, P + lm->off_embed, P + lm->off_pos, x, B, 1, d, lm->V, lm->n_pos, s));
  }
  for (int l = 0; l < lm->L; ++l) {
    const LnLayerOff& o = lm->lnl[l];
    bf16* kc = reinterpret_cast<bf16*>(kv_cache) + (size_t)l * 2 * plane;
    bf16* vc = kc + plane;
    SK_TRY(linear_fwd(B, Q, d, x, P + o.wqkv, qkv, P + o.bqkv, nullptr, s));
    SK_TRY(sk_kv_append_launch(qkv, Q, kc, vc, pos, b.lens, B, lm->H, lm->H, T_cache, s));
    SK_TRY(sk_attn_decode_launch(qkv, Q, kc, vc, b.lens, ao, d, b.partial, B, lm->H, lm->H, T_cache, scale, s));
    SK_TRY(linear_fwd(B, d, d, ao, P + o.wo, xm, P + o.bo, x, s));
    SK_TRY(sk_layernorm_fwd_launch(xm, P + o.ln1w, P + o.ln1b, h, nullptr, nullptr, B, d, eps, s));
    SK_TRY(linear_fwd(B, F, d, h, P + o.w1, a, P + o.b1, nullptr, s, SK_ACT_RELU));
    SK_TRY(linear_fwd(B, d, F, a, P + o.w2, xm, P + o.b2, h, s, SK_ACT_NONE, b.gemm, b.gemm_bytes));
    SK_TRY(sk_layernorm_fwd_launch(xm, P + o.ln2w, P + o.ln2b, x, nullptr, nullptr, B, d, eps, s));
  }
  const bf16* hin = x;
  if (lm->proj) {
    SK_TRY(linear_fwd(B, K, d, x, P + lm->off_pout, h, nullptr, nullptr, s));
    hin = h;
  }
  return dec_head(lm, b, B, K, hin, logits, ldl, s);
}

// One token per row at position pos[b] (read on the device: the step is graph-capturable).  The KV cache layout is the
// Qwen2 one with KVH = H.
int opt_decode_step(SkLm* lm, const int64_t* tokens, const int32_t* pos, int B, void* kv_cache, int T_cache, void* logits,
                    int ldl, const DecBufs& b, cudaStream_t s) {
  const int d = lm->d, F = lm->F, Q = lm->qkv_dim;
  const float eps = lm->eps;
  const bf16* P = lm->params;
  bf16* x = b.x0;
  bf16* xm = b.x1;
  bf16* h = b.h;
  bf16* qkv = b.qkv;
  bf16* ao = b.ao;
  bf16* a = b.gu;
  const size_t plane = (size_t)B * lm->H * T_cache * lm->hd;
  const float scale = 1.0f / sqrtf((float)lm->hd);
  SK_TRY(sk_opt_embed_fwd_launch(tokens, pos, P + lm->off_embed, P + lm->off_pos, x, B, 1, d, lm->V, lm->n_pos, s));
  for (int l = 0; l < lm->L; ++l) {
    const LnLayerOff& o = lm->lnl[l];
    bf16* kc = reinterpret_cast<bf16*>(kv_cache) + (size_t)l * 2 * plane;
    bf16* vc = kc + plane;
    SK_TRY(sk_layernorm_fwd_launch(x, P + o.ln1w, P + o.ln1b, h, nullptr, nullptr, B, d, eps, s));
    SK_TRY(linear_fwd(B, Q, d, h, P + o.wqkv, qkv, P + o.bqkv, nullptr, s));
    SK_TRY(sk_kv_append_launch(qkv, Q, kc, vc, pos, b.lens, B, lm->H, lm->H, T_cache, s));
    SK_TRY(sk_attn_decode_launch(qkv, Q, kc, vc, b.lens, ao, d, b.partial, B, lm->H, lm->H, T_cache, scale, s));
    SK_TRY(linear_fwd(B, d, d, ao, P + o.wo, xm, P + o.bo, x, s));
    SK_TRY(sk_layernorm_fwd_launch(xm, P + o.ln2w, P + o.ln2b, h, nullptr, nullptr, B, d, eps, s));
    SK_TRY(linear_fwd(B, F, d, h, P + o.w1, a, P + o.b1, nullptr, s, SK_ACT_RELU));
    // fc2 + bias + residual into x (not in place): with M = B the scratch lets stream-K spread the long K loop over idle
    // SMs; rounded before the residual add like the forward pass
    SK_TRY(linear_fwd(B, d, F, a, P + o.w2, x, P + o.b2, xm, s, SK_ACT_NONE, b.gemm, b.gemm_bytes));
  }
  SK_TRY(sk_layernorm_fwd_launch(x, P + lm->off_final_norm, P + lm->off_final_norm_b, h, nullptr, nullptr, B, d, eps, s));
  return dec_head(lm, b, B, d, h, logits, ldl, s);
}

// ---- OPT fp32 inference (sk_lm_set_fp32): HF OPTForCausalLM in fp32, as the reference scores and generates a float32
// checkpoint.  Every linear is the split-bf16 three-product GEMM (hi*hi + hi*lo + lo*hi, fp32 accumulation) on the
// (hi, lo) weight copy with the fp32 bias; activations and the residual stream are (hi, lo) pairs; LayerNorms read the
// pair (plus an optional second one) with fp32 gamma / beta; attention is the causal split-bf16 kernel; the lm_head
// writes fp32 logits.
struct Pair {
  bf16* hi;
  bf16* lo;
};

// sk_gemm_linear_split on the split weights at w_off (bias fp32 at b_off >= 0)
int linear_split(const SkLm* lm, int M, int N, int K, Pair x, int64_t w_off, int64_t b_off, int act, const Pair* res, Pair y,
                 float* y32, int ldy, cudaStream_t s) {
  return sk_gemm_ex_launch(sk_gemm_linear_split(M, N, K, x.hi, x.lo, lm->w_hi + w_off, lm->w_lo + w_off,
                                                b_off >= 0 ? lm->params32 + b_off : nullptr, act, res ? res->hi : nullptr,
                                                res ? res->lo : nullptr, y.hi, y.lo, y32, ldy),
                           s);
}

// the lm_head's input rows [M, head_k] of fp32 inference: the final LayerNorm's output in h1, or for post-LN OPT the last
// layer's output in X or its project_out image in h1
Pair head_in_fp32(const SkLm* lm, const WsLayout& w) {
  const int64_t off = lm->post_ln && !lm->proj ? w.X : w.h1;
  return Pair{wsp<bf16>(lm, off), wsp<bf16>(lm, off + w.sX)};
}

// Post-LN fp32 inference.  The slabs: X the layer input x, xmid s1 then s2, h1 y1 (and, with projections, e at the start
// and the head input h = x_L W_out^T at the end); embed_scratch the fp32 rows before they are split.
int opt_postln_forward_fp32(SkLm* lm, const FwdArgs& fa, const WsLayout& w, cudaStream_t s) {
  const int B = fa.B, T = fa.T, M = B * T, d = lm->d, F = lm->F, L = lm->L, Q = lm->qkv_dim, K = head_k(lm);
  const int64_t* ids = fa.ids;
  const float eps = lm->eps;
  const float* P32 = lm->params32;
  auto pair = [&](int64_t off, int64_t stride) { return Pair{wsp<bf16>(lm, off), wsp<bf16>(lm, off + stride)}; };
  const Pair x = pair(w.X, w.sX), xm = pair(w.xmid, w.sX), h = pair(w.h1, w.sX), qkv = pair(w.qkv, w.sqkv),
             ao = pair(w.ao, w.sX), a = pair(w.gu, w.sgu);
  float* e32 = wsp<float>(lm, w.embed_scratch);
  if (lm->proj) {   // x0 = e W_in^T + pos[p + 2], the position rows as the split GEMM's residual
    SK_TRY(sk_opt_embed_fwd_f32_launch(ids, nullptr, nullptr, P32 + lm->off_pos, e32, M, T, d, lm->V, lm->n_pos, s));
    SK_TRY(sk_split_f32_launch(e32, xm.hi, xm.lo, (long)M * d, s));
    SK_TRY(sk_opt_embed_fwd_f32_launch(ids, nullptr, P32 + lm->off_embed, nullptr, e32, M, T, K, lm->V, lm->n_pos, s));
    SK_TRY(sk_split_f32_launch(e32, h.hi, h.lo, (long)M * K, s));
    SK_TRY(linear_split(lm, M, d, K, h, lm->off_pin, -1, SK_ACT_NONE, &xm, x, nullptr, d, s));
  } else {
    SK_TRY(sk_opt_embed_fwd_f32_launch(ids, nullptr, P32 + lm->off_embed, P32 + lm->off_pos, e32, M, T, d, lm->V, lm->n_pos, s));
    SK_TRY(sk_split_f32_launch(e32, x.hi, x.lo, (long)M * d, s));
  }
  const float scale = 1.0f / sqrtf((float)lm->hd);
  const size_t plane = (size_t)B * lm->H * fa.T_cache * lm->hd;
  for (int l = 0; l < L; ++l) {
    const LnLayerOff& o = lm->lnl[l];
    SK_TRY(linear_split(lm, M, Q, d, x, o.wqkv, o.bqkv, SK_ACT_NONE, nullptr, qkv, nullptr, Q, s));
    if (fa.kv)
      SK_TRY(sk_kv_prefill_f32_launch(qkv.hi, qkv.lo, Q, fa.kv + (size_t)l * 2 * plane, fa.lens, B, T, lm->H, fa.T_cache, s));
    SK_TRY(sk_attn_tc_fwd_split_launch(qkv.hi, qkv.lo, ao.hi, ao.lo, B, T, lm->H, Q, d, scale, s, 1));
    SK_TRY(linear_split(lm, M, d, d, ao, o.wo, o.bo, SK_ACT_NONE, &x, xm, nullptr, d, s));
    SK_TRY(sk_layernorm_hilo_launch(xm.hi, xm.lo, nullptr, nullptr, P32 + o.ln1w, P32 + o.ln1b, h.hi, h.lo, nullptr, M, d, eps, s));
    SK_TRY(linear_split(lm, M, F, d, h, o.w1, o.b1, SK_ACT_RELU, nullptr, a, nullptr, F, s));   // relu(fc1)
    SK_TRY(linear_split(lm, M, d, F, a, o.w2, o.b2, SK_ACT_NONE, &h, xm, nullptr, d, s));
    SK_TRY(sk_layernorm_hilo_launch(xm.hi, xm.lo, nullptr, nullptr, P32 + o.ln2w, P32 + o.ln2b, x.hi, x.lo, nullptr, M, d, eps, s));
  }
  if (lm->proj) SK_TRY(linear_split(lm, M, K, d, x, lm->off_pout, -1, SK_ACT_NONE, nullptr, h, nullptr, K, s));
  lm->last_B = B;
  lm->last_T = T;
  if (!fa.with_head) return 0;
  return linear_split(lm, M, lm->Vp, K, head_in_fp32(lm, w), lm->off_head, -1, SK_ACT_NONE, nullptr, Pair{nullptr, nullptr},
                      wsp<float>(lm, w.logits), lm->Vp, s);
}

// Post-LN fp32 decode step: the slots of opt_decode_step_fp32, with h holding e at the start and the head input at the end
int opt_postln_decode_step_fp32(SkLm* lm, const int64_t* tokens, const int32_t* pos, int B, float* kv, int T_cache,
                                float* logits, int ldl, const DecBufs& b, cudaStream_t s) {
  const int d = lm->d, F = lm->F, Q = lm->qkv_dim, K = head_k(lm);
  const float eps = lm->eps;
  const float* P32 = lm->params32;
  auto pair = [&](bf16* hi, int64_t n) { return Pair{hi, hi + n}; };
  const Pair x = pair(b.x0, (int64_t)B * d), xm = pair(b.x1, (int64_t)B * d), h = pair(b.h, (int64_t)B * d),
             qkv = pair(b.qkv, (int64_t)B * Q), ao = pair(b.ao, (int64_t)B * d), a = pair(b.gu, (int64_t)B * F);
  const size_t plane = (size_t)B * lm->H * T_cache * lm->hd;
  const float scale = 1.0f / sqrtf((float)lm->hd);
  if (lm->proj) {
    SK_TRY(sk_opt_embed_fwd_f32_launch(tokens, pos, nullptr, P32 + lm->off_pos, b.e32, B, 1, d, lm->V, lm->n_pos, s));
    SK_TRY(sk_split_f32_launch(b.e32, xm.hi, xm.lo, (long)B * d, s));
    SK_TRY(sk_opt_embed_fwd_f32_launch(tokens, pos, P32 + lm->off_embed, nullptr, b.e32, B, 1, K, lm->V, lm->n_pos, s));
    SK_TRY(sk_split_f32_launch(b.e32, h.hi, h.lo, (long)B * K, s));
    SK_TRY(linear_split(lm, B, d, K, h, lm->off_pin, -1, SK_ACT_NONE, &xm, x, nullptr, d, s));
  } else {
    SK_TRY(sk_opt_embed_fwd_f32_launch(tokens, pos, P32 + lm->off_embed, P32 + lm->off_pos, b.e32, B, 1, d, lm->V, lm->n_pos, s));
    SK_TRY(sk_split_f32_launch(b.e32, x.hi, x.lo, (long)B * d, s));
  }
  for (int l = 0; l < lm->L; ++l) {
    const LnLayerOff& o = lm->lnl[l];
    float* kc = kv + (size_t)l * 2 * plane;
    float* vc = kc + plane;
    SK_TRY(linear_split(lm, B, Q, d, x, o.wqkv, o.bqkv, SK_ACT_NONE, nullptr, qkv, nullptr, Q, s));
    SK_TRY(sk_kv_append_f32_launch(qkv.hi, qkv.lo, Q, kc, vc, pos, b.lens, B, lm->H, T_cache, s));
    SK_TRY(sk_attn_decode_f32_launch(qkv.hi, qkv.lo, Q, kc, vc, b.lens, ao.hi, ao.lo, d, b.partial, B, lm->H, T_cache, scale, s));
    SK_TRY(linear_split(lm, B, d, d, ao, o.wo, o.bo, SK_ACT_NONE, &x, xm, nullptr, d, s));
    SK_TRY(sk_layernorm_hilo_launch(xm.hi, xm.lo, nullptr, nullptr, P32 + o.ln1w, P32 + o.ln1b, h.hi, h.lo, nullptr, B, d, eps, s));
    SK_TRY(linear_split(lm, B, F, d, h, o.w1, o.b1, SK_ACT_RELU, nullptr, a, nullptr, F, s));
    SK_TRY(linear_split(lm, B, d, F, a, o.w2, o.b2, SK_ACT_NONE, &h, xm, nullptr, d, s));
    SK_TRY(sk_layernorm_hilo_launch(xm.hi, xm.lo, nullptr, nullptr, P32 + o.ln2w, P32 + o.ln2b, x.hi, x.lo, nullptr, B, d, eps, s));
  }
  Pair hin = x;
  if (lm->proj) {
    SK_TRY(linear_split(lm, B, K, d, x, lm->off_pout, -1, SK_ACT_NONE, nullptr, h, nullptr, K, s));
    hin = h;
  }
  return linear_split(lm, B, lm->Vp, K, hin, lm->off_head, -1, SK_ACT_NONE, nullptr, Pair{nullptr, nullptr}, logits, ldl, s);
}

int opt_forward_fp32(SkLm* lm, const FwdArgs& fa, const WsLayout& w, cudaStream_t s) {
  const int B = fa.B, T = fa.T, M = B * T, d = lm->d, F = lm->F, L = lm->L, Q = lm->qkv_dim;
  const int64_t* ids = fa.ids;
  const float eps = lm->eps;
  const float* P32 = lm->params32;
  auto pair = [&](int64_t off, int64_t stride) { return Pair{wsp<bf16>(lm, off), wsp<bf16>(lm, off + stride)}; };
  const Pair x = pair(w.X, w.sX), xm = pair(w.xmid, w.sX), h = pair(w.h1, w.sX), qkv = pair(w.qkv, w.sqkv),
             ao = pair(w.ao, w.sX), a = pair(w.gu, w.sgu);
  float* e32 = wsp<float>(lm, w.embed_scratch);
  SK_TRY(sk_opt_embed_fwd_f32_launch(ids, nullptr, P32 + lm->off_embed, P32 + lm->off_pos, e32, M, T, d, lm->V, lm->n_pos, s));
  SK_TRY(sk_split_f32_launch(e32, x.hi, x.lo, (long)M * d, s));
  // q * head_dim^-0.5 = q / 8 (HF:modeling_opt.py:146): a power of two, folded into the softmax scale exactly
  const float scale = 1.0f / sqrtf((float)lm->hd);
  const size_t plane = (size_t)B * lm->H * fa.T_cache * lm->hd;
  for (int l = 0; l < L; ++l) {
    const LnLayerOff& o = lm->lnl[l];
    SK_TRY(sk_layernorm_hilo_launch(x.hi, x.lo, nullptr, nullptr, P32 + o.ln1w, P32 + o.ln1b, h.hi, h.lo, nullptr, M, d, eps, s));
    SK_TRY(linear_split(lm, M, Q, d, h, o.wqkv, o.bqkv, SK_ACT_NONE, nullptr, qkv, nullptr, Q, s));
    if (fa.kv)
      SK_TRY(sk_kv_prefill_f32_launch(qkv.hi, qkv.lo, Q, fa.kv + (size_t)l * 2 * plane, fa.lens, B, T, lm->H, fa.T_cache, s));
    SK_TRY(sk_attn_tc_fwd_split_launch(qkv.hi, qkv.lo, ao.hi, ao.lo, B, T, lm->H, Q, d, scale, s, 1));
    SK_TRY(linear_split(lm, M, d, d, ao, o.wo, o.bo, SK_ACT_NONE, &x, xm, nullptr, d, s));
    SK_TRY(sk_layernorm_hilo_launch(xm.hi, xm.lo, nullptr, nullptr, P32 + o.ln2w, P32 + o.ln2b, h.hi, h.lo, nullptr, M, d, eps, s));
    SK_TRY(linear_split(lm, M, F, d, h, o.w1, o.b1, SK_ACT_RELU, nullptr, a, nullptr, F, s));   // relu(fc1)
    SK_TRY(linear_split(lm, M, d, F, a, o.w2, o.b2, SK_ACT_NONE, &xm, x, nullptr, d, s));
  }
  SK_TRY(sk_layernorm_hilo_launch(x.hi, x.lo, nullptr, nullptr, P32 + lm->off_final_norm, P32 + lm->off_final_norm_b, h.hi,
                                  h.lo, nullptr, M, d, eps, s));
  lm->last_B = B;
  lm->last_T = T;
  if (!fa.with_head) return 0;
  return linear_split(lm, M, lm->Vp, d, h, lm->off_head, -1, SK_ACT_NONE, nullptr, Pair{nullptr, nullptr},
                      wsp<float>(lm, w.logits), lm->Vp, s);
}

// One token per row at position pos[b] on the fp32 cache ([K|V][B][H][T_cache][64] fp32 per layer); fp32 logits [B, ldl]
int opt_decode_step_fp32(SkLm* lm, const int64_t* tokens, const int32_t* pos, int B, float* kv, int T_cache, float* logits,
                         int ldl, const DecBufs& b, cudaStream_t s) {
  const int d = lm->d, F = lm->F, Q = lm->qkv_dim;
  const float eps = lm->eps;
  const float* P32 = lm->params32;
  auto pair = [&](bf16* hi, int64_t n) { return Pair{hi, hi + n}; };
  const Pair x = pair(b.x0, (int64_t)B * d), xm = pair(b.x1, (int64_t)B * d), h = pair(b.h, (int64_t)B * d),
             qkv = pair(b.qkv, (int64_t)B * Q), ao = pair(b.ao, (int64_t)B * d), a = pair(b.gu, (int64_t)B * F);
  const size_t plane = (size_t)B * lm->H * T_cache * lm->hd;
  const float scale = 1.0f / sqrtf((float)lm->hd);
  SK_TRY(sk_opt_embed_fwd_f32_launch(tokens, pos, P32 + lm->off_embed, P32 + lm->off_pos, b.e32, B, 1, d, lm->V, lm->n_pos, s));
  SK_TRY(sk_split_f32_launch(b.e32, x.hi, x.lo, (long)B * d, s));
  for (int l = 0; l < lm->L; ++l) {
    const LnLayerOff& o = lm->lnl[l];
    float* kc = kv + (size_t)l * 2 * plane;
    float* vc = kc + plane;
    SK_TRY(sk_layernorm_hilo_launch(x.hi, x.lo, nullptr, nullptr, P32 + o.ln1w, P32 + o.ln1b, h.hi, h.lo, nullptr, B, d, eps, s));
    SK_TRY(linear_split(lm, B, Q, d, h, o.wqkv, o.bqkv, SK_ACT_NONE, nullptr, qkv, nullptr, Q, s));
    SK_TRY(sk_kv_append_f32_launch(qkv.hi, qkv.lo, Q, kc, vc, pos, b.lens, B, lm->H, T_cache, s));
    SK_TRY(sk_attn_decode_f32_launch(qkv.hi, qkv.lo, Q, kc, vc, b.lens, ao.hi, ao.lo, d, b.partial, B, lm->H, T_cache, scale, s));
    SK_TRY(linear_split(lm, B, d, d, ao, o.wo, o.bo, SK_ACT_NONE, &x, xm, nullptr, d, s));
    SK_TRY(sk_layernorm_hilo_launch(xm.hi, xm.lo, nullptr, nullptr, P32 + o.ln2w, P32 + o.ln2b, h.hi, h.lo, nullptr, B, d, eps, s));
    SK_TRY(linear_split(lm, B, F, d, h, o.w1, o.b1, SK_ACT_RELU, nullptr, a, nullptr, F, s));
    SK_TRY(linear_split(lm, B, d, F, a, o.w2, o.b2, SK_ACT_NONE, &xm, x, nullptr, d, s));
  }
  SK_TRY(sk_layernorm_hilo_launch(x.hi, x.lo, nullptr, nullptr, P32 + lm->off_final_norm, P32 + lm->off_final_norm_b, h.hi,
                                  h.lo, nullptr, B, d, eps, s));
  return linear_split(lm, B, lm->Vp, d, h, lm->off_head, -1, SK_ACT_NONE, nullptr, Pair{nullptr, nullptr}, logits, ldl, s);
}

#define SK_REFUSE_FP32(lm, who)                                                                                          \
  SK_REQUIRE(!(lm)->fp32, who ": this handle runs fp32 inference (sk_lm_set_fp32), which is forward only; train with a " \
                          "bf16 or master-weights handle")

// gradient-norm groups and their device chunk tables.  A group is one HF parameter, a list of (offset, n) element ranges
// of the flat buffer; chunks are listed group by group, so a group is a contiguous run of the chunk table.
using NormGroups = std::vector<std::vector<std::pair<int64_t, int64_t>>>;
int upload_norm_groups(SkLm* lm, const NormGroups& groups) {
  std::vector<long> cs;
  std::vector<int> cl, tb;
  for (const auto& g : groups) {
    tb.push_back((int)cs.size());
    for (const auto& r : g)
      for (int64_t o = 0; o < r.second; o += GN_CHUNK) {
        cs.push_back((long)(r.first + o));
        cl.push_back((int)((r.second - o) < GN_CHUNK ? (r.second - o) : GN_CHUNK));
      }
  }
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
  return 0;
}

// A handle with the shape fields every decoder shares (head_dim 64); the caller has checked the shapes
SkLm* new_lm(int arch, int V, int d, int L, int H, int KVH, int F, int max_pos, float eps, bool tie, bool qkv_bias) {
  SkLm* lm = new SkLm();
  lm->arch = arch;
  lm->d = d;
  lm->F = F;
  lm->H = H;
  lm->KVH = KVH;
  lm->hd = 64;
  lm->L = L;
  lm->V = V;
  lm->Vp = (V + 63) / 64 * 64;
  lm->qkv_dim = (H + 2 * KVH) * lm->hd;
  lm->max_pos = max_pos;
  lm->eps = eps;
  lm->tie = tie;
  lm->qkv_bias = qkv_bias;
  // text+unit vocabularies: chunked lm_head + CE (SK_HEAD_CHUNK=rows overrides, 0 turns it off)
  lm->head_chunk = lm->Vp > 8192 ? 2048 : 0;
  if (const char* e = getenv("SK_HEAD_CHUNK")) lm->head_chunk = (atoi(e) / 128) * 128;
  return lm;
}

// upload the norm groups and hand the handle out, or free it
int publish(SkLm* lm, const NormGroups& groups, SkLm** out) {
  const int rc = upload_norm_groups(lm, groups);
  if (rc) {
    sk_lm_destroy(lm);
    return rc;
  }
  *out = lm;
  return 0;
}

// One token per row at position pos[b] (read on the device: the step is graph-capturable)
int qwen2_decode_step(SkLm* lm, const int64_t* tokens, const int32_t* pos, int B, void* kv_cache, int T_cache, void* logits,
                      int ldl, const DecBufs& b, cudaStream_t s) {
  const int d = lm->d, F = lm->F, Q = lm->qkv_dim;
  const bf16* P = lm->params;
  bf16* x = b.x0;
  bf16* xm = b.x1;
  bf16* h = b.h;
  bf16* qkv = b.qkv;
  bf16* ao = b.ao;
  bf16* gu = b.gu;
  bf16* act = b.act;
  const size_t plane = (size_t)B * lm->KVH * T_cache * lm->hd;
  const float scale = 1.0f / sqrtf((float)lm->hd);
  SK_TRY(sk_embed_fwd_launch(tokens, P + lm->off_embed, x, B, d, lm->V, s));
  for (int l = 0; l < lm->L; ++l) {
    const LayerOff& o = lm->lo[l];
    bf16* kc = reinterpret_cast<bf16*>(kv_cache) + (size_t)l * 2 * plane;
    bf16* vc = kc + plane;
    SK_TRY(sk_rmsnorm_fwd_launch(x, P + o.ln1, h, nullptr, B, d, lm->eps, s));
    SK_TRY(linear_qkv_rope(lm, B, 1, h, P + o.wqkv, lm->qkv_bias ? P + o.bqkv : nullptr, qkv, pos, s));
    SK_TRY(sk_kv_append_launch(qkv, Q, kc, vc, pos, b.lens, B, lm->H, lm->KVH, T_cache, s));
    SK_TRY(sk_attn_decode_launch(qkv, Q, kc, vc, b.lens, ao, d, b.partial, B, lm->H, lm->KVH, T_cache, scale, s));
    SK_TRY(linear_fwd(B, d, d, ao, P + o.wo, xm, nullptr, x, s));
    SK_TRY(sk_rmsnorm_fwd_launch(xm, P + o.ln2, h, nullptr, B, d, lm->eps, s));
    SK_TRY(sk_gemm_ex_launch(sk_gemm_swiglu_fwd(B, F, d, h, P + o.wgu, gu, act), s));
    // down projection added in place (residual == output): with M = B there is a single row of output tiles, so the
    // scratch lets the GEMM split its long K loop over idle SMs (fixed-order reduction); rounded before the residual
    // add like the forward pass's down projection
    SK_TRY(linear_fwd(B, d, F, act, P + o.wd, xm, nullptr, xm, s, SK_ACT_NONE, b.gemm, b.gemm_bytes));
    std::swap(x, xm);
  }
  SK_TRY(sk_rmsnorm_fwd_launch(x, P + lm->off_final_norm, h, nullptr, B, d, lm->eps, s));
  return dec_head(lm, b, B, d, h, logits, ldl, s);
}

// ---- the decoder variant: (fp32 inference) -> architecture -> (post-LN) -> (master weights), the only place that picks
// one.  Master weights are never post-LN, fp32 inference is OPT forward only, and master handles do not decode.
int forward(SkLm* lm, const FwdArgs& a, const WsLayout& w, cudaStream_t s) {
  if (lm->fp32) return lm->post_ln ? opt_postln_forward_fp32(lm, a, w, s) : opt_forward_fp32(lm, a, w, s);
  if (lm->arch == SK_ARCH_QWEN2) return qwen2_forward(lm, a, w, s);
  if (lm->arch == SK_ARCH_NEOX) return neox_forward(lm, a, w, s);
  if (lm->post_ln) return opt_postln_forward(lm, a, w, s);
  if (lm->master) return opt_master_forward(lm, a, w, s);
  return opt_forward(lm, a, w, s);
}

int backward(SkLm* lm, const FwdArgs& a, int accumulate, const WsLayout& w, cudaStream_t s) {
  if (lm->arch == SK_ARCH_QWEN2) return qwen2_backward(lm, a, accumulate, w, s);
  if (lm->arch == SK_ARCH_NEOX) return neox_backward(lm, a, accumulate, w, s);
  if (lm->post_ln) return opt_postln_backward(lm, a, accumulate, w, s);
  if (lm->master) return opt_master_backward(lm, a, accumulate, w, s);
  return opt_backward(lm, a, accumulate, w, s);
}

int decode_step(SkLm* lm, const int64_t* tokens, const int32_t* pos, int B, void* kv_cache, int T_cache, void* logits, int ldl,
                const DecBufs& b, cudaStream_t s) {
  if (lm->fp32) {
    float* kv = reinterpret_cast<float*>(kv_cache);
    float* lg = reinterpret_cast<float*>(logits);
    return lm->post_ln ? opt_postln_decode_step_fp32(lm, tokens, pos, B, kv, T_cache, lg, ldl, b, s)
                       : opt_decode_step_fp32(lm, tokens, pos, B, kv, T_cache, lg, ldl, b, s);
  }
  if (lm->arch == SK_ARCH_QWEN2) return qwen2_decode_step(lm, tokens, pos, B, kv_cache, T_cache, logits, ldl, b, s);
  if (lm->arch == SK_ARCH_NEOX) return neox_decode_step(lm, tokens, pos, B, kv_cache, T_cache, logits, ldl, b, s);
  if (lm->post_ln) return opt_postln_decode_step(lm, tokens, pos, B, kv_cache, T_cache, logits, ldl, b, s);
  return opt_decode_step(lm, tokens, pos, B, kv_cache, T_cache, logits, ldl, b, s);
}

// sk_lm_prefill, or with head != nullptr sk_lm_prefill_sub (its caller has checked the compact head)
int prefill(const char* who, SkLm* lm, const int64_t* ids, const int32_t* lens, int B, int T, void* kv_cache, int T_cache,
            const bf16* head, int head_n, void* logits, int ldl, void* decode_ws, int64_t decode_ws_bytes, void* stream) {
  SK_REQUIRE(lm && ids && lens, "%s: null argument", who);
  SK_REQUIRE(!lm->master, "%s: this handle trains fp32 master weights (sk_lm_set_master); generate from its saved "
                          "checkpoint with a handle that has no master weights", who);
  const DecLayout dl = make_dec_layout(lm, B, T_cache);
  SK_TRY(check_decode(lm, B, T_cache, ldl, head ? head_n : lm->Vp, kv_cache, logits, decode_ws, decode_ws_bytes, dl));
  SK_REQUIRE(T > 0 && T <= T_cache, "%s: prompt width T=%d must be in [1, T_cache=%d]", who, T, T_cache);
  const WsLayout w = layout_of(lm, B, T);
  SK_TRY(check_bound(lm, B, T, w, nullptr));
  cudaStream_t s = (cudaStream_t)stream;
  DecBufs b = dec_bufs(decode_ws, dl);
  b.head = head;
  b.head_n = head_n;
  SK_CUDA_CHECK(cudaMemsetAsync(reinterpret_cast<uint8_t*>(b.gemm) + b.gemm_bytes - 4096, 0, 4096, s));
  FwdArgs a{ids, nullptr, nullptr, B, T};
  a.with_head = false;
  if (lm->fp32) {
    a.kv = reinterpret_cast<float*>(kv_cache);
    a.lens = lens;
    a.T_cache = T_cache;
  }
  SK_TRY(forward(lm, a, w, s));
  const int K = head_k(lm);
  if (lm->fp32) {
    const Pair hf = head_in_fp32(lm, w);
    const Pair hl{b.h, b.h + (int64_t)B * lm->d};
    SK_TRY(sk_gather_last_launch(hf.hi, lens, hl.hi, B, T, K, s));
    SK_TRY(sk_gather_last_launch(hf.lo, lens, hl.lo, B, T, K, s));
    return linear_split(lm, B, lm->Vp, K, hl, lm->off_head, -1, SK_ACT_NONE, nullptr, Pair{nullptr, nullptr},
                        reinterpret_cast<float*>(logits), ldl, s);
  }
  SK_TRY(sk_kv_prefill_launch(wsp<bf16>(lm, w.qkv), w.sqkv / 2, lm->qkv_dim, reinterpret_cast<bf16*>(kv_cache), lens, lm->L, B,
                              T, lm->H, lm->KVH, T_cache, s));
  SK_TRY(sk_gather_last_launch(head_in(lm, w), lens, b.h, B, T, K, s));
  return dec_head(lm, b, B, K, b.h, logits, ldl, s);
}

// sk_lm_decode_step, or with head != nullptr sk_lm_decode_step_sub
int decode(const char* who, SkLm* lm, const int64_t* tokens, const int32_t* pos, int B, void* kv_cache, int T_cache,
           const bf16* head, int head_n, void* logits, int ldl, void* decode_ws, int64_t decode_ws_bytes, void* stream) {
  SK_REQUIRE(lm && tokens && pos, "%s: null argument", who);
  SK_REQUIRE(!lm->master, "%s: this handle trains fp32 master weights (sk_lm_set_master); generate from its "
                          "saved checkpoint with a handle that has no master weights", who);
  const DecLayout dl = make_dec_layout(lm, B, T_cache);
  SK_TRY(check_decode(lm, B, T_cache, ldl, head ? head_n : lm->Vp, kv_cache, logits, decode_ws, decode_ws_bytes, dl));
  DecBufs b = dec_bufs(decode_ws, dl);
  b.head = head;
  b.head_n = head_n;
  return decode_step(lm, tokens, pos, B, kv_cache, T_cache, logits, ldl, b, (cudaStream_t)stream);
}

// the compact head of the _sub entry points: n_pad rows of head_k(lm) bf16 (sk_lm_gather_head), bf16 handles only
int check_sub_head(const char* who, const SkLm* lm, const void* head, int n_pad) {
  SK_REQUIRE(lm, "%s: null argument", who);
  SK_REQUIRE(!lm->fp32, "%s: fp32 inference handles decode with the full head (sk_lm_decode_step)", who);
  SK_REQUIRE(head && ((uintptr_t)head & 15) == 0, "%s: the compact head must be a 16-byte aligned device buffer", who);
  SK_REQUIRE(n_pad > 0 && n_pad % 64 == 0 && n_pad <= lm->Vp, "%s: n_pad=%d must be a positive multiple of 64, at most %d",
             who, n_pad, lm->Vp);
  return 0;
}

}  // namespace

extern "C" {

int64_t sk_lm_kv_cache_bytes(const SkLm* lm, int B, int T_cache) {
  if (!lm || B <= 0 || T_cache <= 0) return 0;
  return (int64_t)lm->L * 2 * B * lm->KVH * T_cache * lm->hd * (lm->fp32 ? 4 : 2);
}

int64_t sk_lm_decode_workspace_bytes(const SkLm* lm, int B, int T_cache) {
  if (!lm || B <= 0 || T_cache <= 0) return 0;
  return make_dec_layout(lm, B, T_cache).total;
}

int sk_lm_prefill(SkLm* lm, const int64_t* ids, const int32_t* lens, int B, int T, void* kv_cache, int T_cache,
                  void* logits, int ldl, void* decode_ws, int64_t decode_ws_bytes, void* stream) {
  return prefill("sk_lm_prefill", lm, ids, lens, B, T, kv_cache, T_cache, nullptr, 0, logits, ldl, decode_ws,
                 decode_ws_bytes, stream);
}

int sk_lm_prefill_sub(SkLm* lm, const int64_t* ids, const int32_t* lens, int B, int T, void* kv_cache, int T_cache,
                      const void* head, int n_pad, void* logits, int ld_sub, void* decode_ws, int64_t decode_ws_bytes,
                      void* stream) {
  SK_TRY(check_sub_head("sk_lm_prefill_sub", lm, head, n_pad));
  return prefill("sk_lm_prefill_sub", lm, ids, lens, B, T, kv_cache, T_cache, reinterpret_cast<const bf16*>(head), n_pad,
                 logits, ld_sub, decode_ws, decode_ws_bytes, stream);
}

int sk_lm_decode_step(SkLm* lm, const int64_t* tokens, const int32_t* pos, int B, void* kv_cache, int T_cache,
                      void* logits, int ldl, void* decode_ws, int64_t decode_ws_bytes, void* stream) {
  return decode("sk_lm_decode_step", lm, tokens, pos, B, kv_cache, T_cache, nullptr, 0, logits, ldl, decode_ws,
                decode_ws_bytes, stream);
}

int sk_lm_decode_step_sub(SkLm* lm, const int64_t* tokens, const int32_t* pos, int B, void* kv_cache, int T_cache,
                          const void* head, int n_pad, void* logits, int ld_sub, void* decode_ws, int64_t decode_ws_bytes,
                          void* stream) {
  SK_TRY(check_sub_head("sk_lm_decode_step_sub", lm, head, n_pad));
  return decode("sk_lm_decode_step_sub", lm, tokens, pos, B, kv_cache, T_cache, reinterpret_cast<const bf16*>(head), n_pad,
                logits, ld_sub, decode_ws, decode_ws_bytes, stream);
}

int sk_lm_gather_head(const SkLm* lm, const int32_t* ids, int n, int n_pad, void* head, void* stream) {
  SK_TRY(check_sub_head("sk_lm_gather_head", lm, head, n_pad));
  SK_REQUIRE(ids && n > 0 && n <= n_pad, "sk_lm_gather_head: need 1 <= n=%d <= n_pad=%d ids", n, n_pad);
  SK_REQUIRE(lm->params, "sk_lm: sk_lm_bind has not been called");
  return sk_gather_rows_launch(lm->params + lm->off_head, ids, n, n_pad, lm->V, head_k(lm), reinterpret_cast<bf16*>(head),
                               (cudaStream_t)stream);
}

int sk_lm_kv_fanout(const SkLm* lm, const void* src_cache, int B, int k, void* dst_cache, int T_cache, const int32_t* lens,
                    void* stream) {
  SK_REQUIRE(lm && src_cache && dst_cache && lens, "sk_lm_kv_fanout: null argument");
  return sk_kv_fanout_launch(src_cache, dst_cache, lens, lm->L, B, k, lm->KVH, T_cache, lm->hd * (lm->fp32 ? 4 : 2),
                             (cudaStream_t)stream);
}

int sk_lm_create(const SkLmConfig* cfg, SkLm** out) {
  SK_REQUIRE(cfg && out, "sk_lm_create: null argument");
  SK_REQUIRE(cfg->head_dim == 64, "sk_lm_create: only head_dim 64 is supported (got %d)", cfg->head_dim);
  SK_REQUIRE(cfg->hidden % 8 == 0 && cfg->hidden <= 1024, "sk_lm_create: hidden must be a multiple of 8 and <= 1024");
  SK_REQUIRE(cfg->ffn % 128 == 0, "sk_lm_create: ffn must be a multiple of 128 (gate/up rows are stored in 128-row blocks)");
  SK_REQUIRE(cfg->n_heads % cfg->n_kv_heads == 0, "sk_lm_create: n_heads must be a multiple of n_kv_heads");
  SK_REQUIRE(cfg->vocab_size > 0 && cfg->vocab_size <= (1 << 20),
             "sk_lm_create: vocab_size must be in [1, 2^20] (unit vocabularies are ~502, interleaved text+unit ones ~152 k)");
  SK_REQUIRE(cfg->n_heads * cfg->head_dim == cfg->hidden, "sk_lm_create: n_heads*head_dim must equal hidden");
  SkLm* lm = new_lm(SK_ARCH_QWEN2, cfg->vocab_size, cfg->hidden, cfg->n_layers, cfg->n_heads, cfg->n_kv_heads, cfg->ffn,
                    cfg->max_positions, cfg->rms_eps, cfg->tie_embeddings != 0, cfg->qkv_bias != 0);
  const int d = lm->d, F = lm->F;
  lm->lo.resize(lm->L);
  for (int l = 0; l < lm->L; ++l) {
    const std::string p = "layers." + std::to_string(l) + ".";
    LayerOff& o = lm->lo[l];
    o.ln1 = add_tensor(lm, p + "ln1", 1, d);
    o.wqkv = add_tensor(lm, p + "wqkv", lm->qkv_dim, d);
    o.bqkv = add_tensor(lm, p + "bqkv", 1, lm->qkv_dim);
    o.wo = add_tensor(lm, p + "wo", d, lm->H * lm->hd);
    o.ln2 = add_tensor(lm, p + "ln2", 1, d);
    o.wgu = add_tensor(lm, p + "wgu", 2 * F, d);
    o.wd = add_tensor(lm, p + "wd", d, F);
  }
  lm->off_final_norm = add_tensor(lm, "final_norm", 1, d);
  lm->off_embed = add_tensor(lm, "embed", lm->Vp, d);
  lm->off_head = lm->tie ? lm->off_embed : add_tensor(lm, "lm_head", lm->Vp, d);

  // torch.nn.utils.clip_grad_norm_ takes one norm per PARAMETER (rounded to bf16 on bf16 gradients), and HF keeps q/k/v
  // and gate/up as separate parameters: q, k, v are row ranges of wqkv / bqkv; gate and up alternate in 128-row blocks
  // of wgu
  NormGroups groups;
  auto one = [&](int64_t off, int64_t n) { groups.push_back({{off, n}}); };
  const int64_t qd = (int64_t)lm->H * lm->hd, kvd = (int64_t)lm->KVH * lm->hd;
  for (int l = 0; l < lm->L; ++l) {
    const LayerOff& o = lm->lo[l];
    one(o.ln1, d);
    one(o.wqkv, qd * d);
    one(o.wqkv + qd * d, kvd * d);
    one(o.wqkv + (qd + kvd) * d, kvd * d);
    if (lm->qkv_bias) {
      one(o.bqkv, qd);
      one(o.bqkv + qd, kvd);
      one(o.bqkv + qd + kvd, kvd);
    }
    one(o.wo, (int64_t)d * d);
    one(o.ln2, d);
    for (int half = 0; half < 2; ++half) {   // gate, then up
      groups.emplace_back();
      for (int b = 0; b < F / 128; ++b) groups.back().push_back({o.wgu + ((int64_t)b * 256 + half * 128) * d, (int64_t)128 * d});
    }
    one(o.wd, (int64_t)d * F);
  }
  one(lm->off_final_norm, d);
  one(lm->off_embed, (int64_t)lm->Vp * d);
  if (!lm->tie) one(lm->off_head, (int64_t)lm->Vp * d);
  return publish(lm, groups, out);
}

int sk_lm_create_opt(const SkOptConfig* cfg, SkLm** out) {
  SK_REQUIRE(cfg && out, "sk_lm_create_opt: null argument");
  SK_REQUIRE(cfg->n_heads > 0 && cfg->hidden == 64 * cfg->n_heads, "sk_lm_create_opt: only head_dim 64 is supported (hidden %d, %d heads)",
             cfg->hidden, cfg->n_heads);
  SK_REQUIRE(cfg->hidden <= 2048, "sk_lm_create_opt: hidden must be <= 2048 (got %d)", cfg->hidden);
  SK_REQUIRE(cfg->ffn > 0 && cfg->ffn % 8 == 0, "sk_lm_create_opt: ffn must be a positive multiple of 8 (got %d)", cfg->ffn);
  SK_REQUIRE(cfg->n_layers > 0 && cfg->max_positions > 0, "sk_lm_create_opt: n_layers and max_positions must be positive");
  SK_REQUIRE(cfg->vocab_size > 0 && cfg->vocab_size <= (1 << 20), "sk_lm_create_opt: vocab_size must be in [1, 2^20]");
  SK_REQUIRE(cfg->post_ln == 0 || cfg->post_ln == 1, "sk_lm_create_opt: post_ln must be 0 or 1 (got %d)", cfg->post_ln);
  const bool proj = cfg->proj_dim != 0 && cfg->proj_dim != cfg->hidden;
  SK_REQUIRE(!proj || cfg->post_ln, "sk_lm_create_opt: proj_dim=%d != hidden=%d (project_in / project_out) is implemented for "
                                    "the post-LayerNorm decoder only (post_ln = 1)", cfg->proj_dim, cfg->hidden);
  SK_REQUIRE(!proj || (cfg->proj_dim > 0 && cfg->proj_dim % 64 == 0 && cfg->proj_dim < cfg->hidden),
             "sk_lm_create_opt: proj_dim must be a positive multiple of 64 below hidden (got %d)", cfg->proj_dim);
  SkLm* lm = new_lm(SK_ARCH_OPT, cfg->vocab_size, cfg->hidden, cfg->n_layers, cfg->n_heads, cfg->n_heads, cfg->ffn,
                    cfg->max_positions, cfg->ln_eps, cfg->tie_embeddings != 0, true);
  lm->post_ln = cfg->post_ln != 0;
  lm->proj = proj;
  lm->pw = proj ? cfg->proj_dim : cfg->hidden;
  lm->n_pos = cfg->max_positions + 2;   // OPTLearnedPositionalEmbedding: offset 2
  const int d = lm->d, F = lm->F, pw = lm->pw;
  lm->lnl.resize(lm->L);
  for (int l = 0; l < lm->L; ++l) {
    const std::string p = "layers." + std::to_string(l) + ".";
    LnLayerOff& o = lm->lnl[l];
    o.ln1w = add_tensor(lm, p + "ln1", 1, d);
    o.ln1b = add_tensor(lm, p + "ln1_b", 1, d);
    o.wqkv = add_tensor(lm, p + "wqkv", 3 * d, d);
    o.bqkv = add_tensor(lm, p + "bqkv", 1, 3 * d);
    o.wo = add_tensor(lm, p + "wo", d, d);
    o.bo = add_tensor(lm, p + "bo", 1, d);
    o.ln2w = add_tensor(lm, p + "ln2", 1, d);
    o.ln2b = add_tensor(lm, p + "ln2_b", 1, d);
    o.w1 = add_tensor(lm, p + "w1", F, d);
    o.b1 = add_tensor(lm, p + "b1", 1, F);
    o.w2 = add_tensor(lm, p + "w2", d, F);
    o.b2 = add_tensor(lm, p + "b2", 1, d);
  }
  if (!lm->post_ln) {   // post-LN OPT has no decoder-level final LayerNorm
    lm->off_final_norm = add_tensor(lm, "final_norm", 1, d);
    lm->off_final_norm_b = add_tensor(lm, "final_norm_b", 1, d);
  }
  lm->off_embed = add_tensor(lm, "embed", lm->Vp, pw);
  lm->off_pos = add_tensor(lm, "pos_embed", lm->n_pos, d);
  if (proj) {
    lm->off_pin = add_tensor(lm, "proj_in", d, pw);
    lm->off_pout = add_tensor(lm, "proj_out", pw, d);
  }
  lm->off_head = lm->tie ? lm->off_embed : add_tensor(lm, "lm_head", lm->Vp, pw);
  // one gradient-norm group per HF parameter, weights and biases apart (torch clip_grad_norm_ over OPTForCausalLM, whose
  // decoder lists embed_tokens, embed_positions, project_out, project_in, then the layers)
  NormGroups groups;
  auto one = [&](int64_t off, int64_t n) { groups.push_back({{off, n}}); };
  const int64_t dd = (int64_t)d * d;
  one(lm->off_embed, (int64_t)lm->Vp * pw);
  one(lm->off_pos, (int64_t)lm->n_pos * d);
  if (proj) {
    one(lm->off_pout, (int64_t)pw * d);
    one(lm->off_pin, (int64_t)d * pw);
  }
  for (int l = 0; l < lm->L; ++l) {
    const LnLayerOff& o = lm->lnl[l];
    for (int j = 0; j < 3; ++j) {   // q, k, v
      one(o.wqkv + j * dd, dd);
      one(o.bqkv + (int64_t)j * d, d);
    }
    one(o.wo, dd); one(o.bo, d);
    one(o.ln1w, d); one(o.ln1b, d);
    one(o.w1, (int64_t)F * d); one(o.b1, F);
    one(o.w2, (int64_t)d * F); one(o.b2, d);
    one(o.ln2w, d); one(o.ln2b, d);
  }
  if (!lm->post_ln) {
    one(lm->off_final_norm, d);
    one(lm->off_final_norm_b, d);
  }
  if (!lm->tie) one(lm->off_head, (int64_t)lm->Vp * pw);
  return publish(lm, groups, out);
}

int sk_lm_create_neox(const SkNeoxConfig* cfg, SkLm** out) {
  SK_REQUIRE(cfg && out, "sk_lm_create_neox: null argument");
  SK_REQUIRE(cfg->n_heads > 0 && cfg->hidden == 64 * cfg->n_heads,
             "sk_lm_create_neox: only head_dim 64 is supported (hidden %d, %d heads)", cfg->hidden, cfg->n_heads);
  SK_REQUIRE(cfg->hidden <= 2048, "sk_lm_create_neox: hidden must be <= 2048 (got %d)", cfg->hidden);
  SK_REQUIRE(cfg->ffn > 0 && cfg->ffn % 64 == 0, "sk_lm_create_neox: ffn must be a positive multiple of 64 (got %d)", cfg->ffn);
  SK_REQUIRE(cfg->rot_dims == 16 || cfg->rot_dims == 32 || cfg->rot_dims == 64,
             "sk_lm_create_neox: rot_dims (rotary_ndims) must be 16, 32 or 64 (got %d)", cfg->rot_dims);
  SK_REQUIRE(cfg->n_layers > 0 && cfg->max_positions > 0, "sk_lm_create_neox: n_layers and max_positions must be positive");
  SK_REQUIRE(cfg->vocab_size > 0 && cfg->vocab_size <= (1 << 20), "sk_lm_create_neox: vocab_size must be in [1, 2^20]");
  SkLm* lm = new_lm(SK_ARCH_NEOX, cfg->vocab_size, cfg->hidden, cfg->n_layers, cfg->n_heads, cfg->n_heads, cfg->ffn,
                    cfg->max_positions, cfg->ln_eps, false, true);
  lm->rot = cfg->rot_dims;
  const int d = lm->d, F = lm->F;
  lm->lnl.resize(lm->L);
  for (int l = 0; l < lm->L; ++l) {
    const std::string p = "layers." + std::to_string(l) + ".";
    LnLayerOff& o = lm->lnl[l];
    o.ln1w = add_tensor(lm, p + "ln1", 1, d);
    o.ln1b = add_tensor(lm, p + "ln1_b", 1, d);
    o.ln2w = add_tensor(lm, p + "ln2", 1, d);
    o.ln2b = add_tensor(lm, p + "ln2_b", 1, d);
    o.wqkv = add_tensor(lm, p + "wqkv", 3 * d, d);
    o.bqkv = add_tensor(lm, p + "bqkv", 1, 3 * d);
    o.wo = add_tensor(lm, p + "wo", d, d);
    o.bo = add_tensor(lm, p + "bo", 1, d);
    o.w1 = add_tensor(lm, p + "w1", F, d);
    o.b1 = add_tensor(lm, p + "b1", 1, F);
    o.w2 = add_tensor(lm, p + "w2", d, F);
    o.b2 = add_tensor(lm, p + "b2", 1, d);
  }
  lm->off_final_norm = add_tensor(lm, "final_norm", 1, d);
  lm->off_final_norm_b = add_tensor(lm, "final_norm_b", 1, d);
  lm->off_embed = add_tensor(lm, "embed", lm->Vp, d);
  lm->off_head = add_tensor(lm, "lm_head", lm->Vp, d);
  // one gradient-norm group per HF parameter, in GPTNeoXForCausalLM.parameters() order (query_key_value is one tensor)
  NormGroups groups;
  auto one = [&](int64_t off, int64_t n) { groups.push_back({{off, n}}); };
  const int64_t dd = (int64_t)d * d;
  one(lm->off_embed, (int64_t)lm->Vp * d);
  for (int l = 0; l < lm->L; ++l) {
    const LnLayerOff& o = lm->lnl[l];
    one(o.ln1w, d); one(o.ln1b, d);
    one(o.ln2w, d); one(o.ln2b, d);
    one(o.wqkv, 3 * dd); one(o.bqkv, 3 * d);
    one(o.wo, dd); one(o.bo, d);
    one(o.w1, (int64_t)F * d); one(o.b1, F);
    one(o.w2, (int64_t)d * F); one(o.b2, d);
  }
  one(lm->off_final_norm, d);
  one(lm->off_final_norm_b, d);
  one(lm->off_head, (int64_t)lm->Vp * d);
  return publish(lm, groups, out);
}

void sk_lm_destroy(SkLm* lm) {
  if (!lm) return;
  cudaFree(lm->d_chunk_start);
  cudaFree(lm->d_chunk_len);
  cudaFree(lm->d_tensor_chunk_begin);
  cudaFree(lm->d_chunk_partial);
  cudaFree(lm->d_widen_start);
  cudaFree(lm->d_widen_len);
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
  return layout_of(lm, B, T).total;
}

int sk_lm_bind(SkLm* lm, void* params, void* grads, const void* rope_cos, const void* rope_sin, void* workspace,
               int64_t workspace_bytes) {
  SK_REQUIRE(lm && params && workspace, "sk_lm_bind: null argument");
  SK_REQUIRE((rope_cos && rope_sin) || lm->arch == SK_ARCH_OPT, "sk_lm_bind: a Qwen2 or GPT-NeoX handle needs the RoPE tables");
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
  const WsLayout w = layout_of(lm, 1, 1);
  SK_REQUIRE(workspace_bytes >= w.splitk + w.splitk_bytes, "sk_lm_bind: workspace smaller than the GEMM scratch");
  SK_CUDA_CHECK(cudaMemset(lm->ws + w.splitk + w.splitk_bytes - 4096, 0, 4096));
  SK_CUDA_CHECK(cudaDeviceSynchronize());
  return 0;
}

int sk_lm_set_master(SkLm* lm, float* params32, float* grads32) {
  SK_REQUIRE(lm && params32, "sk_lm_set_master: null argument");
  SK_REQUIRE(lm->arch == SK_ARCH_OPT, "sk_lm_set_master: fp32 master weights are implemented for the OPT decoder only (the "
                                      "Qwen2 and GPT-NeoX recipes train bf16 parameters)");
  SK_REQUIRE(!lm->post_ln, "sk_lm_set_master: fp32 master weights are implemented for the pre-LayerNorm OPT decoder only; "
                           "this handle is post-LayerNorm (post_ln = 1): train it with bf16 parameters");
  SK_REQUIRE(lm->params && lm->ws, "sk_lm_set_master: call sk_lm_bind first");
  SK_REQUIRE(!lm->fp32, "sk_lm_set_master: this handle runs fp32 inference (sk_lm_set_fp32); master weights are a training "
                        "mode, create a separate handle");
  SK_REQUIRE(((uintptr_t)params32 & 127) == 0 && ((uintptr_t)grads32 & 127) == 0,
             "sk_lm_set_master: params32 / grads32 must be 128-byte aligned");
  if (!lm->d_widen_start) {
    // linear weights and biases, whose bf16 gradients are widened: per layer [wqkv .. bo] and [w1 .. b2] (contiguous in
    // the layout), plus an untied lm_head; the tied lm_head's gradient is folded into the embedding's
    std::vector<std::pair<int64_t, int64_t>> ranges;
    for (int l = 0; l < lm->L; ++l) {
      const LnLayerOff& o = lm->lnl[l];
      ranges.push_back({o.wqkv, o.ln2w - o.wqkv});
      const int64_t end = l + 1 < lm->L ? lm->lnl[l + 1].ln1w : lm->off_final_norm;
      ranges.push_back({o.w1, end - o.w1});
    }
    if (!lm->tie) ranges.push_back({lm->off_head, lm->n_params - lm->off_head});
    std::vector<long> cs;
    std::vector<int> cl;
    for (const auto& r : ranges)
      for (int64_t o = 0; o < r.second; o += GN_CHUNK) {
        cs.push_back((long)(r.first + o));
        cl.push_back((int)std::min<int64_t>(GN_CHUNK, r.second - o));
      }
    SK_CUDA_CHECK(cudaMalloc(&lm->d_widen_start, cs.size() * sizeof(long)));
    SK_CUDA_CHECK(cudaMalloc(&lm->d_widen_len, cl.size() * sizeof(int)));
    SK_CUDA_CHECK(cudaMemcpy(lm->d_widen_start, cs.data(), cs.size() * sizeof(long), cudaMemcpyHostToDevice));
    SK_CUDA_CHECK(cudaMemcpy(lm->d_widen_len, cl.data(), cl.size() * sizeof(int), cudaMemcpyHostToDevice));
    lm->n_widen = (int)cs.size();
  }
  lm->params32 = params32;
  lm->grads32 = grads32;
  lm->master = true;
  return 0;
}

int sk_lm_widen_chunks(const SkLm* lm, int64_t* chunk_start, int32_t* chunk_len, int cap) {
  SK_REQUIRE(lm && chunk_start && chunk_len, "sk_lm_widen_chunks: null argument");
  SK_REQUIRE(lm->d_widen_start, "sk_lm_widen_chunks: the handle has no master weights (sk_lm_set_master)");
  SK_REQUIRE(cap >= lm->n_widen, "sk_lm_widen_chunks: %d chunks do not fit in %d", lm->n_widen, cap);
  std::vector<long> cs(lm->n_widen);
  SK_CUDA_CHECK(cudaMemcpy(cs.data(), lm->d_widen_start, cs.size() * sizeof(long), cudaMemcpyDeviceToHost));
  SK_CUDA_CHECK(cudaMemcpy(chunk_len, lm->d_widen_len, (size_t)lm->n_widen * sizeof(int), cudaMemcpyDeviceToHost));
  for (int i = 0; i < lm->n_widen; ++i) chunk_start[i] = (int64_t)cs[i];
  return lm->n_widen;
}

int64_t sk_lm_fp32_prepared_bytes(const SkLm* lm) { return lm ? 2 * align_up(lm->n_params * 2, 256) : 0; }

int sk_lm_set_fp32(SkLm* lm, const float* params32, void* prepared, int64_t prepared_bytes, void* stream) {
  SK_REQUIRE(lm && params32 && prepared, "sk_lm_set_fp32: null argument");
  SK_REQUIRE(lm->arch == SK_ARCH_OPT, "sk_lm_set_fp32: fp32 inference is implemented for the OPT decoder only (the Qwen2 and "
                                      "GPT-NeoX recipes are bf16)");
  SK_REQUIRE(lm->params && lm->ws, "sk_lm_set_fp32: call sk_lm_bind first");
  SK_REQUIRE(!lm->master, "sk_lm_set_fp32: this handle trains fp32 master weights (sk_lm_set_master); score its saved "
                          "checkpoint with a separate handle");
  SK_REQUIRE(lm->d <= 1024, "sk_lm_set_fp32: hidden must be <= 1024 (got %d)", lm->d);
  SK_REQUIRE(prepared_bytes >= sk_lm_fp32_prepared_bytes(lm), "sk_lm_set_fp32: prepared buffer too small: need %lld bytes",
             (long long)sk_lm_fp32_prepared_bytes(lm));
  SK_REQUIRE(((uintptr_t)params32 & 127) == 0 && ((uintptr_t)prepared & 255) == 0,
             "sk_lm_set_fp32: params32 must be 128-byte and prepared 256-byte aligned");
  uint8_t* p = reinterpret_cast<uint8_t*>(prepared);
  lm->params32 = const_cast<float*>(params32);
  lm->w_hi = reinterpret_cast<bf16*>(p);
  lm->w_lo = reinterpret_cast<bf16*>(p + align_up(lm->n_params * 2, 256));
  SK_TRY(sk_split_f32_launch(params32, lm->w_hi, lm->w_lo, (long)lm->n_params, (cudaStream_t)stream));
  lm->fp32 = true;
  return 0;
}

int sk_lm_forward(SkLm* lm, const int64_t* ids, const int64_t* labels, const int32_t* pos_ids, int B, int T,
                  float num_items, float* stats, void* stream) {
  SK_REQUIRE(lm && ids, "sk_lm_forward: null argument");
  SK_REQUIRE(labels == nullptr || stats != nullptr, "sk_lm_forward: stats is required when labels are given");
  SK_REQUIRE(!lm->fp32 || (labels == nullptr && pos_ids == nullptr), "sk_lm_forward: an fp32 inference handle (sk_lm_set_fp32) "
                                                                     "takes neither labels (score with sk_seq_loglik_f32) nor "
                                                                     "position_ids");
  const WsLayout w = layout_of(lm, B, T);
  SK_TRY(check_bound(lm, B, T, w, pos_ids));
  FwdArgs a{ids, labels, pos_ids, B, T};
  a.num_items = num_items;
  a.stats = stats;
  return forward(lm, a, w, (cudaStream_t)stream);
}

int sk_lm_forward_backward(SkLm* lm, const int64_t* ids, const int64_t* labels, const int32_t* pos_ids, int B, int T,
                           float num_items, float dloss, int accumulate, float* stats, void* stream) {
  SK_REQUIRE(lm && ids && labels && stats, "sk_lm_forward_backward: null argument");
  SK_REFUSE_FP32(lm, "sk_lm_forward_backward");
  SK_REQUIRE(lm->grads, "sk_lm_forward_backward: no gradient buffer bound");
  SK_REQUIRE(!lm->master || lm->grads32, "sk_lm_forward_backward: no fp32 gradient buffer given to sk_lm_set_master");
  const WsLayout w = layout_of(lm, B, T);
  SK_TRY(check_bound(lm, B, T, w, pos_ids));
  cudaStream_t s = (cudaStream_t)stream;
  FwdArgs a{ids, labels, pos_ids, B, T, num_items, dloss, true, stats};
  a.with_head = lm->head_chunk == 0;
  SK_TRY(forward(lm, a, w, s));
  // master weights: the bf16 gradient buffer holds one micro-batch (grads32 accumulates)
  if (!a.with_head) SK_TRY(head_chunked(lm, a, lm->master ? 0 : accumulate, w, s));
  return backward(lm, a, accumulate, w, s);
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
  SK_REFUSE_FP32(lm, "sk_lm_forward_rows");
  const WsLayout w = layout_of(lm, B, T);
  SK_TRY(check_bound(lm, B, T, w, pos_ids));
  FwdArgs a{ids, labels, pos_ids, B, T, 1.0f, 1.0f, false, stats, row_nll};
  return forward(lm, a, w, (cudaStream_t)stream);
}

int sk_lm_backward_weighted(SkLm* lm, const int64_t* ids, const int64_t* labels, const int32_t* pos_ids, int B, int T,
                            const float* row_weight, int accumulate, float* stats, void* stream) {
  SK_REQUIRE(lm && ids && labels && row_weight && stats, "sk_lm_backward_weighted: null argument");
  SK_REFUSE_FP32(lm, "sk_lm_backward_weighted");
  SK_REQUIRE(lm->grads, "sk_lm_backward_weighted: no gradient buffer bound");
  SK_REQUIRE(!lm->master || lm->grads32, "sk_lm_backward_weighted: no fp32 gradient buffer given to sk_lm_set_master");
  SK_REQUIRE(lm->last_B == B && lm->last_T == T, "sk_lm_backward_weighted: call sk_lm_forward_rows on the same batch first");
  const WsLayout w = layout_of(lm, B, T);
  SK_TRY(check_bound(lm, B, T, w, pos_ids));
  cudaStream_t s = (cudaStream_t)stream;
  // d loss / d logits[row] = row_weight[row] * (softmax - onehot): recomputed from the logits the forward pass left in
  // the workspace (num_items = 1, dloss = 1: the caller's weights carry every scale factor)
  SK_TRY(sk_ce_launch(wsp<bf16>(lm, w.logits), labels, wsp<bf16>(lm, w.dlogits), wsp<float>(lm, w.ce_partial), nullptr,
                      stats, B * T, T, lm->V, lm->Vp, 1.0f, 1.0f, s, row_weight));
  return backward(lm, FwdArgs{ids, labels, pos_ids, B, T}, accumulate, w, s);
}

const void* sk_lm_logits(const SkLm* lm) {
  if (!lm || !lm->ws || lm->last_B == 0 || lm->fp32) return nullptr;
  return lm->ws + layout_of(lm, lm->last_B, lm->last_T).logits;
}
const float* sk_lm_logits_f32(const SkLm* lm) {
  if (!lm || !lm->ws || lm->last_B == 0 || !lm->fp32) return nullptr;
  return reinterpret_cast<const float*>(lm->ws + layout_of(lm, lm->last_B, lm->last_T).logits);
}
int sk_lm_logits_ld(const SkLm* lm) { return lm ? lm->Vp : 0; }

int sk_lm_optimizer_step(SkLm* lm, void* exp_avg, void* exp_avg_sq, float lr, float beta1, float beta2, float eps,
                         float weight_decay, int step, float max_grad_norm, int emulate_bf16_norm, float* stats,
                         void* stream) {
  SK_REQUIRE(lm && exp_avg && exp_avg_sq && stats, "sk_lm_optimizer_step: null argument");
  SK_REFUSE_FP32(lm, "sk_lm_optimizer_step");
  SK_REQUIRE(lm->params && lm->grads, "sk_lm_optimizer_step: params/grads not bound");
  cudaStream_t s = (cudaStream_t)stream;
  if (lm->master) {
    // fp32 master weights: exp_avg / exp_avg_sq are fp32; clip_grad_norm_ and AdamW over the fp32 gradients, the bf16
    // shadow rewritten from the new masters (emulate_bf16_norm does not apply to fp32 gradients)
    SK_REQUIRE(lm->grads32, "sk_lm_optimizer_step: no fp32 gradient buffer given to sk_lm_set_master");
    float* m = reinterpret_cast<float*>(exp_avg);
    float* v = reinterpret_cast<float*>(exp_avg_sq);
    sk_prof_begin(2, s);
    SK_TRY(sk_gradnorm_f32_launch(lm->grads32, lm->d_chunk_start, lm->d_chunk_len, lm->n_chunks, lm->d_tensor_chunk_begin,
                                  lm->n_norm_groups, lm->d_chunk_partial, max_grad_norm, stats, s));
    int rc = 0;
    if (weight_decay == 0.0f) {
      rc = sk_adamw_master_launch(lm->params32, lm->params, lm->grads32, m, v, lm->n_params, lr, beta1, beta2, eps, 0.0f, step,
                                  stats, s);
    } else {
      for (const TensorDesc& t : lm->tensors) {   // decay groups as below
        const int64_t n = (((int64_t)t.rows * t.cols + ALIGN_ELEMS - 1) / ALIGN_ELEMS) * ALIGN_ELEMS;
        rc = sk_adamw_master_launch(lm->params32 + t.off, lm->params + t.off, lm->grads32 + t.off, m + t.off, v + t.off, n, lr,
                                    beta1, beta2, eps, t.rows == 1 ? 0.0f : weight_decay, step, stats, s);
        if (rc) break;
      }
    }
    sk_prof_end(s);
    return rc;
  }
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
