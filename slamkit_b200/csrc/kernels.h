// Internal C++ launcher declarations shared by api.cu / lm_step.cu / hubert_step.cu.
// (The public, C-ABI surface is include/slamkit_b200.h.)
#pragma once
#include "common.cuh"

// gemm_tcgen05.cu
int sk_make_tmap_2d(CUtensorMap* out, const void* ptr, int elem_bytes, uint64_t inner, uint64_t outer, uint64_t ld,
                    uint32_t box_inner, uint32_t box_outer);
int sk_make_tmap_3d(CUtensorMap* out, const void* ptr, uint64_t inner, uint64_t rows, uint64_t batch, uint64_t row_stride,
                    uint64_t batch_stride, uint32_t box_rows);
int sk_pick_bn(int M, int N, int force_bn);
size_t sk_gemm_ws_min_bytes(void);   // scratch size that enables stream-K (last 4 KB = flag words, zero on first use)
// Extended GEMM description (HuBERT path): batched / strided-window A operands (convolutions as GEMMs without an
// im2col copy), split-bf16 3-pass accumulation, fp32 bias, hi/lo residual and outputs, grouped column compaction.
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
  // Fused epilogues of the LM step (0 = none):
  //   1 SwiGLU forward : B = gate/up weight in [128 gate rows | 128 up rows] blocks, N = 2F; C = gu [M,2F] (same block
  //                      layout) and aux_out = act [M,F] = bf16(bf16(silu(gate)) * up)
  //   2 SwiGLU backward: N = F, acc = d_act; aux = gu [M,2F]; C = d_gu [M,2F] (ldc = its pitch)
  //   3 bias + RoPE    : 64-column heads with column < rope_cols are rotated with cos/sin[pos] (pos = rope_pos[row] or
  //                      row % rope_T, clamped to [0, rope_maxpos))
  int epi;
  const void* aux;
  int ld_aux;
  void* aux_out;
  int ld_aux_out;
  const void *rope_cos, *rope_sin;
  const int* rope_pos;
  int rope_T, rope_cols, rope_maxpos;
};
int sk_gemm_ex_launch(const SkGemmEx& g, cudaStream_t stream);
int sk_gemm_launch(int M, int N, int K, const void* A, int lda, int a_mn, const void* B, int ldb, int b_mn, void* C,
                   int ldc, int out_f32, const void* bias, const void* residual, int ldr, int round_before_res, int act,
                   int force_bn, cudaStream_t stream, void* splitk_ws = nullptr, size_t splitk_ws_bytes = 0);
int sk_linear_swiglu_fwd_launch(int M, int F, int K, const void* x, const void* Wgu, void* gu, void* act, cudaStream_t s);
int sk_linear_swiglu_bwd_launch(int M, int N, int F, const void* dy, const void* Wd, const void* gu, void* dgu, cudaStream_t s);
int sk_linear_rope_launch(int M, int N, int K, const void* x, const void* W, const void* bias, void* out, const void* cos_t,
                          const void* sin_t, const int32_t* pos_ids, int T, int rope_cols, int max_positions, cudaStream_t s);

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
int sk_rope_launch(bf16* qkv, const bf16* cos_t, const bf16* sin_t, const int* pos_ids, int M, int T, int ld,
                   int n_rot_heads, int head_dim, int inverse, int max_positions, cudaStream_t s);
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

// attention.cu
int sk_attn_fwd_launch(const bf16* q, const bf16* k, const bf16* v, bf16* o, float* lse, int B, int T, int H, int KVH,
                       int ld, int ldo, int causal, float scale, cudaStream_t s, const int* seg_start = nullptr);
int sk_attn_bwd_launch(const bf16* q, const bf16* k, const bf16* v, const bf16* o, const bf16* d_o, const float* lse,
                       float* delta, bf16* dq, bf16* dk, bf16* dv, int B, int T, int H, int KVH, int ld, int ldo,
                       int ldg, int causal, float scale, cudaStream_t s, const int* seg_start = nullptr);
int sk_attn_fwd_split_launch(const bf16* q_hi, const bf16* q_lo, const bf16* k_hi, const bf16* k_lo, const bf16* v_hi,
                             const bf16* v_lo, bf16* o_hi, bf16* o_lo, int B, int T, int H, int ld, int ldo, float scale,
                             cudaStream_t s);

// attention.cu: entry points on the fused q|k|v projection (LM step, HuBERT encoder)
int sk_attn_tc_fwd_split_launch(const bf16* qkv_hi, const bf16* qkv_lo, bf16* o_hi, bf16* o_lo, int B, int T, int H, int ld,
                                int ldo, float scale, cudaStream_t s);
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
int sk_attn_decode_splits(int T_cache);
int sk_attn_decode_launch(const bf16* q, int ldq, const bf16* kc, const bf16* vc, const int32_t* lens, bf16* o, int ldo,
                          float* partial, int B, int H, int KVH, int T_cache, float scale, cudaStream_t s);
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
