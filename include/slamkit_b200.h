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
 *   act: 0 none, 1 GELU(erf) on (acc+bias).  round_before_res: round (acc+bias) to bf16 before adding the residual
 *   (bit-matches an unfused bf16 linear followed by a bf16 add).  force_bn: 0 auto, else 64/128/256.
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
  int32_t bn;                /* tile width: 64, 128 or 256 (tiles are 128 rows) */
  int32_t epi_warps;         /* 4, or 8 (two per 32-row quadrant) */
  int32_t splits;            /* > 1: split-K into this many K ranges, fp32 slabs summed by a second kernel */
  int32_t sk_units;          /* > 0: stream-K over the last sk_units units (rows of tiles, or columns: sk_colunits) */
  int32_t sk_groups;         /* CTA groups that share the stream-K iteration space (cut into equal K ranges) */
  int32_t sk_G;              /* tiles per unit = CTAs per group */
  int32_t sk_colunits;       /* 1: a stream-K unit is a column of tiles (selected by SK_STREAMK=2) */
  int32_t tma_store;         /* 1: bf16 output through TMA stores; 0: direct stores (fp32 output, split-K slabs) */
  int32_t grid;              /* CTAs of the GEMM kernel */
} SkGemmPlan;
int sk_gemm_plan(int M, int N, int K, const void* A, int lda, int a_mn, const void* B, int ldb, int b_mn, const void* C,
                 int ldc, int out_f32, const void* bias, const void* residual, int ldr, int round_before_res, int act,
                 int force_bn, const void* ws, int64_t ws_bytes, SkGemmPlan* plan);

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
/* Column sums of a bf16 matrix (bias gradient). partial: fp32 [sk_colsum_splits()*N]. */
int sk_colsum_splits(void);
int sk_colsum(const void* x, void* out, float* partial, int M, int N, int ld, int accumulate, void* stream);
/* Rotary embedding (rotate_half form) in place on the first n_rot_heads heads of each row,
 * HF:models/qwen2/modeling_qwen2.py:102-146 (apply_rotary_pos_emb). cos/sin: bf16 [maxpos, head_dim/2].
 * pos_ids: int32 [M] or NULL (position = row % T), clamped to [0, max_positions) = the rows of the tables.
 * inverse=1 applies the transposed rotation (backward). */
int sk_rope(void* qkv, const void* cos_t, const void* sin_t, const int32_t* pos_ids, int M, int T, int ld,
            int n_rot_heads, int head_dim, int inverse, int max_positions, void* stream);
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
/* Stand-alone decode attention: o[b, h*64 .. h*64+63] (pitch ldo) = softmax(q k^T * scale) v over keys [0, lens[b]) of
 * row b; q [B, H*64] pitch ldq; k_cache / v_cache [B][KVH][T_cache][64] bf16.  Flash-decoding over fixed 64-key splits
 * (one CTA per row, kv head and split serves the H/KVH <= 16 query heads of its group) and a combine pass in split
 * order: bit-identical run to run, and no key at or past lens[b] is read.  partial: sk_attn_decode_partial_bytes. */
int64_t sk_attn_decode_partial_bytes(int B, int H, int T_cache);
int sk_attn_decode(const void* q, int ldq, const void* k_cache, const void* v_cache, const int32_t* lens, void* o, int ldo,
                   float* partial, int B, int H, int KVH, int T_cache, float scale, void* stream);
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
/* UnitTokeniser.tokenise on the device (slamkit/tokeniser/unit_tokeniser.py:40-73 with its `<S> $0 <S>` template): sk_rle's
 * units int32 [B, T_units] and counts int32 [B] -> right-padded ids int64 [B, T_out] = [bos, units + offset..., eos, pad...].
 * T_out = max(counts) + 2 gives the batch tokenise() builds. */
int sk_units_to_tokens(const int32_t* units, const int32_t* counts, int B, int T_units, int offset, int bos, int eos, int pad,
                       int64_t* ids, int T_out, void* stream);
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
 * [B*T_i, conv_dim]; 200 = projection [B*T, hidden]; 201 = positional conv; 0..n_layers = hidden_states[stage]. */
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
 * gradient buffer and a small flag array with CUDA IPC, and one small-footprint kernel per bucket (64-thread CTAs, no
 * shared memory: they co-reside with the GEMM / attention CTAs of the backward pass) reduce-scatters and all-gathers in
 * one pass -- rank r sums the W copies of its 1/W of the bucket in rank order (fp32, one rounding: bit-identical on all
 * ranks) and stores the result into all W buffers.  Protocol per bucket (all on one side stream):
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
/* Test hook: `ctas` CTAs with the reduce kernel's footprint (64 threads, <= 64 registers, no shared memory) that hold their
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
