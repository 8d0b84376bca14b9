// Flash-style attention for the causal-LM path (GQA, head_dim 64; HF:models/qwen2/modeling_qwen2.py:187-246) and the
// bidirectional HuBERT encoder (HF:models/hubert/modeling_hubert.py:262-345), forward and backward.
//
// Tiled online-softmax kernels on the sm_90a warpgroup tensor cores: every 64-row block of scores and every product
// with P / dS is one wgmma.mma_async chain (m64n64k16 bf16, fp32 accumulate).  Operand tiles are staged by cp.async
// (double-buffered) into 1024-byte-aligned [rows][64] bf16 tiles in the 128B-swizzled layout wgmma reads directly;
// P and dS stay in registers and feed the next product as the register A operand.  S/P never touch HBM; the backward
// has two deterministic parts (dK/dV per key tile looping over the GQA group, dQ per query tile) so no atomics are
// needed; they share one launch, so dQ tiles fill the SMs while the long dK/dV tiles run.
//
// Packed batches: with seg_start (int32 [B*T], in-row index of the first token of each token's document) the causal
// kernels mask keys before the query's document start -- block-diagonal causal attention.
//
// Layout: q/k/v are column slices of the fused projection output [B*T, ld] (q: H*64 cols, k/v: KVH*64 cols);
// o is [B*T, H*64]; lse is [B, H, T] fp32 (natural log of the scaled-score softmax denominator); delta likewise.
#include "kernels.h"

namespace {

constexpr int HD = 64;  // head dim

// [rows][64] bf16 tile, 128-byte rows, 16-byte chunks XOR-swizzled by row % 8: with a 1024-byte-aligned base this is the
// SWIZZLE_128B K-major layout wgmma descriptors describe
SK_DEVINL uint32_t tile_addr(uint32_t base, int r, int chunk) { return base + r * 128 + ((chunk ^ (r & 7)) << 4); }
// 1024-byte-aligned start of the dynamic shared memory (launches request 1 KB extra)
SK_DEVINL uint32_t smem_base_1k(const void* p) { return (smem_u32(p) + 1023u) & ~1023u; }

SK_DEVINL void cp_async16(uint32_t saddr, const void* g, bool pred) {
  const int sz = pred ? 16 : 0;
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(saddr), "l"(g), "r"(sz) : "memory");
}
SK_DEVINL void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
SK_DEVINL void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}

// m64n64k16 with the A operand in registers (a[4]: the mma.sync m16n8k16 A fragment of this warp's 16 rows)
SK_DEVINL void wgmma_m64n64_rs(float (&d)[32], const uint32_t (&a)[4], uint64_t db) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.eq.u32 p, 1, 1;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,"
      "%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, {%32,%33,%34,%35}, %36, p, 1, 1, 1;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
        "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
        "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
        "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db));
}

// rows x 64 bf16 tile, global (row pitch ld) -> swizzled smem; rows >= limit are zero-filled
template <int ROWS, int NT>
SK_DEVINL void load_tile(uint32_t sbase, const bf16* g, int ld, int row0, int limit) {
  for (int i = threadIdx.x; i < ROWS * 8; i += NT) {
    const int r = i >> 3, c = i & 7;
    const int gr = row0 + r;
    const bool ok = gr < limit;
    cp_async16(tile_addr(sbase, r, c), g + (size_t)(ok ? gr : 0) * ld + c * 8, ok);
  }
}

// Per warpgroup, acc = this warp's 16 rows x 64 columns of a 64 x 64 fp32 tile in the mma.sync C layout (acc[nt][e]:
// rows lane/4 (+8 for e >= 2), columns 8 nt + 2 (lane % 4) + (e & 1)), which is also the wgmma m64n64 accumulator layout.
// All four warps of the warpgroup call these together.

// acc += A * B^T: A = [64 rows][64 k] smem tile (this warpgroup's rows), B = [64 n-rows][64 k] smem tile; both K-major.
// Used for S = Q K^T, S^T = K Q^T, dP = dO V^T, dP^T = V dO^T.
SK_DEVINL void wg_a_bT(float (&acc)[8][4], uint32_t sA, uint32_t sB) {
  float(&d)[32] = reinterpret_cast<float(&)[32]>(acc);
  wgmma_fence();
#pragma unroll
  for (int ks = 0; ks < 4; ++ks)
    wgmma_m64n64<0, 0>(d, gmma_desc_sw128(sA + ks * 32, 16, 1024), gmma_desc_sw128(sB + ks * 32, 16, 1024));
  wgmma_commit();
  wgmma_wait<0>();
}

// acc += P * B: P = this warp's 16 x 64 bf16 A fragments p[kk][4] (registers), B = [64 k-rows][64 n] smem tile (the n
// index contiguous: MN-major, 16 k-rows = 2048 bytes per step).  Used for O = P V, dV = P^T dO, dK = dS^T Q, dQ = dS K.
SK_DEVINL void wg_p_b(float (&acc)[8][4], const uint32_t (&p)[4][4], uint32_t sB) {
  float(&d)[32] = reinterpret_cast<float(&)[32]>(acc);
  wgmma_fence();
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) wgmma_m64n64_rs(d, p[kk], gmma_desc_sw128(sB + kk * 2048, 8192, 1024));
  wgmma_commit();
  wgmma_wait<0>();
}

// Two independent products issued back to back and waited on once; each accumulator sees its MMAs in the order two
// separate calls would issue them, so the results are those of wg_a_bT / wg_p_b.
SK_DEVINL void wg_a_bT2(float (&acc1)[8][4], uint32_t sA1, uint32_t sB1, float (&acc2)[8][4], uint32_t sA2, uint32_t sB2) {
  float(&d1)[32] = reinterpret_cast<float(&)[32]>(acc1);
  float(&d2)[32] = reinterpret_cast<float(&)[32]>(acc2);
  wgmma_fence();
#pragma unroll
  for (int ks = 0; ks < 4; ++ks)
    wgmma_m64n64<0, 0>(d1, gmma_desc_sw128(sA1 + ks * 32, 16, 1024), gmma_desc_sw128(sB1 + ks * 32, 16, 1024));
#pragma unroll
  for (int ks = 0; ks < 4; ++ks)
    wgmma_m64n64<0, 0>(d2, gmma_desc_sw128(sA2 + ks * 32, 16, 1024), gmma_desc_sw128(sB2 + ks * 32, 16, 1024));
  wgmma_commit();
  wgmma_wait<0>();
}
SK_DEVINL void wg_p_b2(float (&acc1)[8][4], const uint32_t (&p1)[4][4], uint32_t sB1, float (&acc2)[8][4],
                       const uint32_t (&p2)[4][4], uint32_t sB2) {
  float(&d1)[32] = reinterpret_cast<float(&)[32]>(acc1);
  float(&d2)[32] = reinterpret_cast<float(&)[32]>(acc2);
  wgmma_fence();
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) wgmma_m64n64_rs(d1, p1[kk], gmma_desc_sw128(sB1 + kk * 2048, 8192, 1024));
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) wgmma_m64n64_rs(d2, p2[kk], gmma_desc_sw128(sB2 + kk * 2048, 8192, 1024));
  wgmma_commit();
  wgmma_wait<0>();
}

// accumulator tile (16 x 64, fp32) -> bf16 A fragments for the next matmul
SK_DEVINL void acc_to_a(const float (&s)[8][4], uint32_t (&p)[4][4]) {
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) {
    p[kk][0] = pack_bf16(s[2 * kk][0], s[2 * kk][1]);
    p[kk][1] = pack_bf16(s[2 * kk][2], s[2 * kk][3]);
    p[kk][2] = pack_bf16(s[2 * kk + 1][0], s[2 * kk + 1][1]);
    p[kk][3] = pack_bf16(s[2 * kk + 1][2], s[2 * kk + 1][3]);
  }
}

SK_DEVINL void zero_acc(float (&a)[8][4]) {
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) a[i][j] = 0.f;
}

// ------------------------------------------------------------------------------------------------
// forward: BR = 128 query rows per CTA (8 warps x 16 rows), BC = 64 keys per step
// ------------------------------------------------------------------------------------------------
template <bool CAUSAL>
__global__ void __launch_bounds__(256, 2)
attn_fwd_kernel(const bf16* __restrict__ q, const bf16* __restrict__ k, const bf16* __restrict__ v, bf16* __restrict__ o,
                float* __restrict__ lse, int T, int ld, int ldo, int H, int group, float scale,
                const int* __restrict__ seg_start) {
  extern __shared__ __align__(128) uint8_t smem_attn[];
  const uint32_t sQ = smem_base_1k(smem_attn);
  const uint32_t sK = sQ + 128 * 128;
  const uint32_t sV = sK + 2 * 64 * 128;
  const int b = blockIdx.z, h = blockIdx.y;
  const int qt = gridDim.x - 1 - blockIdx.x;  // heaviest (last) query tiles first
  const int q0 = qt * 128;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const bf16* qp = q + (size_t)b * T * ld + h * HD;
  const bf16* kp = k + (size_t)b * T * ld + (h / group) * HD;
  const bf16* vp = v + (size_t)b * T * ld + (h / group) * HD;
  const float sl2 = scale * 1.4426950408889634f;

  int n_kv = (T + 63) / 64;
  if (CAUSAL) {
    const int last = min(T - 1, q0 + 127);
    n_kv = last / 64 + 1;
  }
  load_tile<128, 256>(sQ, qp, ld, q0, T);
  load_tile<64, 256>(sK, kp, ld, 0, T);
  load_tile<64, 256>(sV, vp, ld, 0, T);
  cp_async_commit();

  const uint32_t sQw = sQ + (uint32_t)(warp >> 2) * 8192u;   // this warpgroup's 64 query rows
  float oacc[8][4];
  zero_acc(oacc);
  float m_i[2] = {-INFINITY, -INFINITY}, l_i[2] = {0.f, 0.f};
  const int row_a = q0 + warp * 16 + (lane >> 2);  // this thread's rows: row_a, row_a + 8
  int seg_r[2] = {0, 0};                            // first key of each row's document
#pragma unroll
  for (int r = 0; r < 2; ++r)
    if (seg_start && row_a + 8 * r < T) seg_r[r] = seg_start[(size_t)b * T + row_a + 8 * r];

  for (int j = 0; j < n_kv; ++j) {
    const int st = j & 1;
    if (j + 1 < n_kv) {
      load_tile<64, 256>(sK + (st ^ 1) * 8192, kp, ld, (j + 1) * 64, T);
      load_tile<64, 256>(sV + (st ^ 1) * 8192, vp, ld, (j + 1) * 64, T);
      cp_async_commit();
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();

    float s[8][4];
    zero_acc(s);
    wg_a_bT(s, sQw, sK + st * 8192);

    const int k0 = j * 64;
    const bool need_mask = (CAUSAL && (k0 + 63 > q0 + warp * 16)) || (k0 + 64 > T) || seg_start;
    if (need_mask) {
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int key = k0 + nt * 8 + (lane & 3) * 2 + (e & 1);
          const int row = row_a + ((e >> 1) << 3);
          if (key >= T || (CAUSAL && key > row) || key < seg_r[e >> 1]) s[nt][e] = -INFINITY;
        }
      }
    }
    // online softmax
    float mx[2] = {m_i[0], m_i[1]};
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      mx[0] = fmaxf(mx[0], fmaxf(s[nt][0], s[nt][1]));
      mx[1] = fmaxf(mx[1], fmaxf(s[nt][2], s[nt][3]));
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
    }
    float corr[2], rs[2] = {0.f, 0.f};
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      corr[r] = (m_i[r] == -INFINITY) ? 0.f : exp2f((m_i[r] - mx[r]) * sl2);
      m_i[r] = mx[r];
    }
    const float mb0 = (mx[0] == -INFINITY) ? 0.f : mx[0] * sl2;
    const float mb1 = (mx[1] == -INFINITY) ? 0.f : mx[1] * sl2;
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      s[nt][0] = exp2f(s[nt][0] * sl2 - mb0);
      s[nt][1] = exp2f(s[nt][1] * sl2 - mb0);
      s[nt][2] = exp2f(s[nt][2] * sl2 - mb1);
      s[nt][3] = exp2f(s[nt][3] * sl2 - mb1);
      rs[0] += s[nt][0] + s[nt][1];
      rs[1] += s[nt][2] + s[nt][3];
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) l_i[r] = l_i[r] * corr[r] + rs[r];
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      oacc[nt][0] *= corr[0];
      oacc[nt][1] *= corr[0];
      oacc[nt][2] *= corr[1];
      oacc[nt][3] *= corr[1];
    }
    uint32_t pa[4][4];
    acc_to_a(s, pa);
    wg_p_b(oacc, pa, sV + st * 8192);
    __syncthreads();
  }
  // finalize
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    l_i[r] += __shfl_xor_sync(0xffffffffu, l_i[r], 1);
    l_i[r] += __shfl_xor_sync(0xffffffffu, l_i[r], 2);
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int row = row_a + 8 * r;
    if (row < T) {
      const float inv = l_i[r] > 0.f ? 1.0f / l_i[r] : 0.f;
      bf16* op = o + ((size_t)b * T + row) * ldo + h * HD;
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
        const uint32_t pk = pack_bf16(oacc[nt][2 * r] * inv, oacc[nt][2 * r + 1] * inv);
        *reinterpret_cast<uint32_t*>(op + nt * 8 + (lane & 3) * 2) = pk;
      }
      if (lse && (lane & 3) == 0) lse[((size_t)b * H + h) * T + row] = m_i[r] * scale + logf(l_i[r]);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// forward, split-bf16 precision (HuBERT encoder, fp32 OPT inference): q/k/v/o are (hi, lo) bf16 pairs representing
// fp32-grade values; S = Qh Kh^T + Qh Kl^T + Ql Kh^T and O = Ph Vh + Ph Vl + Pl Vh, all accumulated in fp32.  Forward
// only.  Bidirectional for HuBERT (the reference passes no mask, hubert_feature_extractor.py:42); the causal instance
// (OPT) reads no key tile past the diagonal and masks keys > query inside it, heaviest query tiles first.
// ------------------------------------------------------------------------------------------------
SK_DEVINL void acc_to_a_split(const float (&s)[8][4], uint32_t (&ph)[4][4], uint32_t (&pl)[4][4]) {
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
    for (int half = 0; half < 2; ++half) {
      const float (&t)[4] = s[2 * kk + half];
      const float h0 = bf16_round(t[0]), h1 = bf16_round(t[1]), h2 = bf16_round(t[2]), h3 = bf16_round(t[3]);
      ph[kk][2 * half] = pack_bf16(h0, h1);
      ph[kk][2 * half + 1] = pack_bf16(h2, h3);
      pl[kk][2 * half] = pack_bf16(t[0] - h0, t[1] - h1);
      pl[kk][2 * half + 1] = pack_bf16(t[2] - h2, t[3] - h3);
    }
  }
}

template <bool CAUSAL>
__global__ void __launch_bounds__(256)
attn_fwd_split_kernel(const bf16* __restrict__ q_hi, const bf16* __restrict__ q_lo, const bf16* __restrict__ k_hi,
                      const bf16* __restrict__ k_lo, const bf16* __restrict__ v_hi, const bf16* __restrict__ v_lo,
                      bf16* __restrict__ o_hi, bf16* __restrict__ o_lo, int T, int ld, int ldo, float scale) {
  extern __shared__ __align__(128) uint8_t smem_attn[];
  const uint32_t sQh = smem_base_1k(smem_attn);
  const uint32_t sQl = sQh + 128 * 128;
  const uint32_t sKV = sQl + 128 * 128;  // per stage: Kh, Kl, Vh, Vl (4 x 8 KB)
  const int b = blockIdx.z, h = blockIdx.y;
  const int q0 = (CAUSAL ? gridDim.x - 1 - blockIdx.x : blockIdx.x) * 128;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const size_t base = (size_t)b * T * ld + h * HD;
  const float sl2 = scale * 1.4426950408889634f;
  const int n_kv = CAUSAL ? min(T - 1, q0 + 127) / 64 + 1 : (T + 63) / 64;

  auto load_kv = [&](int j, int st) {
    const uint32_t sb = sKV + st * 4 * 8192;
    load_tile<64, 256>(sb, k_hi + base, ld, j * 64, T);
    load_tile<64, 256>(sb + 8192, k_lo + base, ld, j * 64, T);
    load_tile<64, 256>(sb + 2 * 8192, v_hi + base, ld, j * 64, T);
    load_tile<64, 256>(sb + 3 * 8192, v_lo + base, ld, j * 64, T);
  };
  load_tile<128, 256>(sQh, q_hi + base, ld, q0, T);
  load_tile<128, 256>(sQl, q_lo + base, ld, q0, T);
  load_kv(0, 0);
  cp_async_commit();

  const uint32_t qh = sQh + (uint32_t)(warp >> 2) * 8192u, ql = sQl + (uint32_t)(warp >> 2) * 8192u;   // this warpgroup's rows
  float oacc[8][4];
  zero_acc(oacc);
  float m_i[2] = {-INFINITY, -INFINITY}, l_i[2] = {0.f, 0.f};
  const int row_a = q0 + warp * 16 + (lane >> 2);

  for (int j = 0; j < n_kv; ++j) {
    const int st = j & 1;
    if (j + 1 < n_kv) {
      load_kv(j + 1, st ^ 1);
      cp_async_commit();
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
    const uint32_t sb = sKV + st * 4 * 8192;
    float s[8][4];
    zero_acc(s);
    wg_a_bT(s, ql, sb);          // Ql Kh^T (small terms first)
    wg_a_bT(s, qh, sb + 8192);   // Qh Kl^T
    wg_a_bT(s, qh, sb);          // Qh Kh^T
    const int k0 = j * 64;
    if (k0 + 64 > T || (CAUSAL && k0 + 63 > q0 + warp * 16)) {
#pragma unroll
      for (int nt = 0; nt < 8; ++nt)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int key = k0 + nt * 8 + (lane & 3) * 2 + (e & 1);
          if (key >= T || (CAUSAL && key > row_a + ((e >> 1) << 3))) s[nt][e] = -INFINITY;
        }
    }
    float mx[2] = {m_i[0], m_i[1]};
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      mx[0] = fmaxf(mx[0], fmaxf(s[nt][0], s[nt][1]));
      mx[1] = fmaxf(mx[1], fmaxf(s[nt][2], s[nt][3]));
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
    }
    float corr[2], rs[2] = {0.f, 0.f};
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      corr[r] = (m_i[r] == -INFINITY) ? 0.f : exp2f((m_i[r] - mx[r]) * sl2);
      m_i[r] = mx[r];
    }
    const float mb0 = mx[0] * sl2, mb1 = mx[1] * sl2;
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      s[nt][0] = exp2f(s[nt][0] * sl2 - mb0);
      s[nt][1] = exp2f(s[nt][1] * sl2 - mb0);
      s[nt][2] = exp2f(s[nt][2] * sl2 - mb1);
      s[nt][3] = exp2f(s[nt][3] * sl2 - mb1);
      rs[0] += s[nt][0] + s[nt][1];
      rs[1] += s[nt][2] + s[nt][3];
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) l_i[r] = l_i[r] * corr[r] + rs[r];
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      oacc[nt][0] *= corr[0];
      oacc[nt][1] *= corr[0];
      oacc[nt][2] *= corr[1];
      oacc[nt][3] *= corr[1];
    }
    uint32_t ph[4][4], pl[4][4];
    acc_to_a_split(s, ph, pl);
    wg_p_b(oacc, pl, sb + 2 * 8192);  // Pl Vh
    wg_p_b(oacc, ph, sb + 3 * 8192);  // Ph Vl
    wg_p_b(oacc, ph, sb + 2 * 8192);  // Ph Vh
    __syncthreads();
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    l_i[r] += __shfl_xor_sync(0xffffffffu, l_i[r], 1);
    l_i[r] += __shfl_xor_sync(0xffffffffu, l_i[r], 2);
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int row = row_a + 8 * r;
    if (row < T) {
      const float inv = 1.0f / l_i[r];
      const size_t off = ((size_t)b * T + row) * ldo + h * HD;
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
        const float v0 = oacc[nt][2 * r] * inv, v1 = oacc[nt][2 * r + 1] * inv;
        const float h0 = bf16_round(v0), h1 = bf16_round(v1);
        *reinterpret_cast<uint32_t*>(o_hi + off + nt * 8 + (lane & 3) * 2) = pack_bf16(h0, h1);
        *reinterpret_cast<uint32_t*>(o_lo + off + nt * 8 + (lane & 3) * 2) = pack_bf16(v0 - h0, v1 - h1);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// backward preprocess: delta[b,h,t] = sum_d dO*O
// ------------------------------------------------------------------------------------------------
__global__ void attn_delta_kernel(const bf16* __restrict__ o, const bf16* __restrict__ d_o, float* __restrict__ delta,
                                  int B, int T, int H, int ldo) {
  griddep_launch();
  griddep_wait();
  const long total = (long)B * T * H * 8;  // 8 threads per (row, head)
  const long i = blockIdx.x * (long)blockDim.x + threadIdx.x;
  const bool ok = i < total;
  float acc = 0.f;
  long rh = 0;
  if (ok) {
    const int part = (int)(i & 7);
    rh = i >> 3;
    const int h = (int)(rh % H);
    const long m = rh / H;
    const uint4 a = ldg128_stream(o + m * ldo + h * HD + part * 8);
    const uint4 g = ldg128_stream(d_o + m * ldo + h * HD + part * 8);
    const uint32_t au[4] = {a.x, a.y, a.z, a.w}, gu[4] = {g.x, g.y, g.z, g.w};
#pragma unroll
    for (int kq = 0; kq < 4; ++kq) {
      const float2 x = unpack_bf16(au[kq]), y = unpack_bf16(gu[kq]);
      acc += x.x * y.x + x.y * y.y;
    }
  }
  acc += __shfl_xor_sync(0xffffffffu, acc, 1);
  acc += __shfl_xor_sync(0xffffffffu, acc, 2);
  acc += __shfl_xor_sync(0xffffffffu, acc, 4);
  if (ok && (i & 7) == 0) {
    const int h = (int)(rh % H);
    const long m = rh / H;
    const long bb = m / T, t = m % T;
    delta[(bb * H + h) * T + t] = acc;
  }
}

// ------------------------------------------------------------------------------------------------
// backward dK/dV: one CTA per (64-key tile kt, kv head g, batch b); 4 warps x 16 keys; loops over the GQA group's query
// heads and their query tiles.  Works on transposed score tiles S^T = K Q^T so P^T/dS^T are directly A operands.
// ------------------------------------------------------------------------------------------------
template <bool CAUSAL>
SK_DEVINL void attn_bwd_dkdv_tile(const bf16* __restrict__ q, const bf16* __restrict__ k, const bf16* __restrict__ v,
                                  const bf16* __restrict__ d_o, const float* __restrict__ lse,
                                  const float* __restrict__ delta, bf16* __restrict__ dk, bf16* __restrict__ dv, int T,
                                  int ld, int ldo, int ldg, int H, int group, float scale,
                                  const int* __restrict__ seg_start, int kt, int g, int b) {
  extern __shared__ __align__(128) uint8_t smem_attn[];
  const uint32_t sKV = smem_base_1k(smem_attn);        // K tile then V tile (each 8 KB)
  const uint32_t sQ = sKV + 2 * 8192;                  // 2 stages
  const uint32_t sdO = sQ + 2 * 8192;                  // 2 stages
  float* sStat = reinterpret_cast<float*>(smem_attn + (sKV - smem_u32(smem_attn)) + 6 * 8192);  // [2 stages][2 (lse, delta)][64]
  int* sSeg = reinterpret_cast<int*>(sStat + 2 * 2 * 64);          // [2 stages][64] document start of each query row
  const int k0 = kt * 64;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const float sl2 = scale * 1.4426950408889634f;
  const bf16* kp = k + (size_t)b * T * ld + g * HD;
  const bf16* vp = v + (size_t)b * T * ld + g * HD;

  load_tile<64, 128>(sKV, kp, ld, k0, T);
  load_tile<64, 128>(sKV + 8192, vp, ld, k0, T);
  cp_async_commit();

  const int n_qt = (T + 63) / 64;
  const int qt_begin = CAUSAL ? kt : 0;
  const int per_head = n_qt - qt_begin;
  const int n_iter = per_head * group;

  auto issue = [&](int it, int st) {
    const int h = g * group + it / per_head;
    const int qt = qt_begin + it % per_head;
    const bf16* qp = q + (size_t)b * T * ld + h * HD;
    const bf16* dop = d_o + (size_t)b * T * ldo + h * HD;
    load_tile<64, 128>(sQ + st * 8192, qp, ld, qt * 64, T);
    load_tile<64, 128>(sdO + st * 8192, dop, ldo, qt * 64, T);
    if (threadIdx.x < 64) {
      const int row = qt * 64 + threadIdx.x;
      const size_t off = ((size_t)b * H + h) * T + (row < T ? row : 0);
      sStat[(st * 2 + 0) * 64 + threadIdx.x] = row < T ? lse[off] : 0.f;
      sStat[(st * 2 + 1) * 64 + threadIdx.x] = row < T ? delta[off] : 0.f;
      sSeg[st * 64 + threadIdx.x] = (seg_start && row < T) ? seg_start[(size_t)b * T + row] : 0;
    }
    cp_async_commit();
  };
  if (n_iter > 0) issue(0, 0);

  float dkacc[8][4], dvacc[8][4];
  zero_acc(dkacc);
  zero_acc(dvacc);
  const int key_a = k0 + warp * 16 + (lane >> 2);  // this thread's keys: key_a, key_a + 8

  for (int it = 0; it < n_iter; ++it) {
    const int st = it & 1;
    if (it + 1 < n_iter) {
      issue(it + 1, st ^ 1);
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
    const int qt = qt_begin + it % per_head;
    const int q0 = qt * 64;
    const float* s_lse = sStat + (st * 2 + 0) * 64;
    const float* s_del = sStat + (st * 2 + 1) * 64;

    float st_acc[8][4];  // S^T tile: rows = keys (this warp's 16), cols = 64 query rows
    float dp[8][4];      // dP^T = V dO^T
    zero_acc(st_acc);
    zero_acc(dp);
    wg_a_bT2(st_acc, sKV, sQ + st * 8192, dp, sKV + 8192, sdO + st * 8192);
    const int* s_seg = sSeg + st * 64;
    const bool need_mask = (CAUSAL && (q0 < k0 + 64)) || (q0 + 64 > T) || (k0 + 64 > T) || seg_start;
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int qi = nt * 8 + (lane & 3) * 2 + (e & 1);
        const int key = key_a + ((e >> 1) << 3);
        float pv = exp2f(st_acc[nt][e] * sl2 - s_lse[qi] * 1.4426950408889634f);
        if (need_mask) {
          const int qrow = q0 + qi;
          if (qrow >= T || key >= T || (CAUSAL && key > qrow) || key < s_seg[qi]) pv = 0.f;
        }
        st_acc[nt][e] = pv;
        dp[nt][e] = pv * (dp[nt][e] - s_del[qi]) * scale;  // dS^T
      }
    }
    uint32_t pa[4][4], dsa[4][4];
    acc_to_a(st_acc, pa);
    acc_to_a(dp, dsa);
    wg_p_b2(dvacc, pa, sdO + st * 8192, dkacc, dsa, sQ + st * 8192);  // dV += P^T dO, dK += dS^T Q
    __syncthreads();
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int key = key_a + 8 * r;
    if (key < T) {
      bf16* dkp = dk + ((size_t)b * T + key) * ldg + g * HD;
      bf16* dvp = dv + ((size_t)b * T + key) * ldg + g * HD;
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
        *reinterpret_cast<uint32_t*>(dkp + nt * 8 + (lane & 3) * 2) = pack_bf16(dkacc[nt][2 * r], dkacc[nt][2 * r + 1]);
        *reinterpret_cast<uint32_t*>(dvp + nt * 8 + (lane & 3) * 2) = pack_bf16(dvacc[nt][2 * r], dvacc[nt][2 * r + 1]);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// backward dQ: one CTA per (64-row query tile qt, head h, batch b); loops over key tiles up to the diagonal
// ------------------------------------------------------------------------------------------------
template <bool CAUSAL>
SK_DEVINL void attn_bwd_dq_tile(const bf16* __restrict__ q, const bf16* __restrict__ k, const bf16* __restrict__ v,
                                const bf16* __restrict__ d_o, const float* __restrict__ lse,
                                const float* __restrict__ delta, bf16* __restrict__ dq, int T, int ld, int ldo, int ldg,
                                int H, int group, float scale, const int* __restrict__ seg_start, int qt, int h, int b) {
  extern __shared__ __align__(128) uint8_t smem_attn[];
  const uint32_t sQdO = smem_base_1k(smem_attn);  // Q tile, dO tile
  const uint32_t sK = sQdO + 2 * 8192;        // 2 stages
  const uint32_t sV = sK + 2 * 8192;          // 2 stages
  const int q0 = qt * 64;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const float sl2 = scale * 1.4426950408889634f;
  const bf16* qp = q + (size_t)b * T * ld + h * HD;
  const bf16* dop = d_o + (size_t)b * T * ldo + h * HD;
  const bf16* kp = k + (size_t)b * T * ld + (h / group) * HD;
  const bf16* vp = v + (size_t)b * T * ld + (h / group) * HD;

  int n_kv = (T + 63) / 64;
  if (CAUSAL) n_kv = min(T - 1, q0 + 63) / 64 + 1;
  load_tile<64, 128>(sQdO, qp, ld, q0, T);
  load_tile<64, 128>(sQdO + 8192, dop, ldo, q0, T);
  load_tile<64, 128>(sK, kp, ld, 0, T);
  load_tile<64, 128>(sV, vp, ld, 0, T);
  cp_async_commit();

  const int row_a = q0 + warp * 16 + (lane >> 2);
  float lse_r[2], del_r[2];
  int seg_r[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int row = row_a + 8 * r;
    const size_t off = ((size_t)b * H + h) * T + (row < T ? row : 0);
    lse_r[r] = row < T ? lse[off] * 1.4426950408889634f : 0.f;
    del_r[r] = row < T ? delta[off] : 0.f;
    seg_r[r] = (seg_start && row < T) ? seg_start[(size_t)b * T + row] : 0;
  }
  float dqacc[8][4];
  zero_acc(dqacc);

  for (int j = 0; j < n_kv; ++j) {
    const int st = j & 1;
    if (j + 1 < n_kv) {
      load_tile<64, 128>(sK + (st ^ 1) * 8192, kp, ld, (j + 1) * 64, T);
      load_tile<64, 128>(sV + (st ^ 1) * 8192, vp, ld, (j + 1) * 64, T);
      cp_async_commit();
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
    const int k0 = j * 64;
    float s[8][4];
    zero_acc(s);
    wg_a_bT(s, sQdO, sK + st * 8192);
    const bool need_mask = (CAUSAL && (k0 + 63 > q0 + warp * 16)) || (k0 + 64 > T) || (q0 + 64 > T) || seg_start;
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        float pv = exp2f(s[nt][e] * sl2 - lse_r[e >> 1]);
        if (need_mask) {
          const int key = k0 + nt * 8 + (lane & 3) * 2 + (e & 1);
          const int row = row_a + ((e >> 1) << 3);
          if (row >= T || key >= T || (CAUSAL && key > row) || key < seg_r[e >> 1]) pv = 0.f;
        }
        s[nt][e] = pv;
      }
    }
    float dp[8][4];
    zero_acc(dp);
    wg_a_bT(dp, sQdO + 8192, sV + st * 8192);  // dP = dO V^T
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
#pragma unroll
      for (int e = 0; e < 4; ++e) dp[nt][e] = s[nt][e] * (dp[nt][e] - del_r[e >> 1]) * scale;
    }
    uint32_t pa[4][4];
    acc_to_a(dp, pa);
    wg_p_b(dqacc, pa, sK + st * 8192);  // dQ += dS K
    __syncthreads();
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int row = row_a + 8 * r;
    if (row < T) {
      bf16* dqp = dq + ((size_t)b * T + row) * ldg + h * HD;
#pragma unroll
      for (int nt = 0; nt < 8; ++nt)
        *reinterpret_cast<uint32_t*>(dqp + nt * 8 + (lane & 3) * 2) = pack_bf16(dqacc[nt][2 * r], dqacc[nt][2 * r + 1]);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// backward: the dK/dV tiles (blocks [0, n_dkdv)) and the dQ tiles (the rest) in one grid.  Under the causal mask key
// tile 0 loops over every query tile of the group, a chain far longer than the others; in one launch the dQ tiles run
// beside it instead of after it.  Both parts go heaviest first: key tiles ascending, then query tiles descending.
// Each output element is computed exactly as by two separate kernels.
// ------------------------------------------------------------------------------------------------
template <bool CAUSAL>
__global__ void __launch_bounds__(128, 3)
attn_bwd_kernel(const bf16* __restrict__ q, const bf16* __restrict__ k, const bf16* __restrict__ v,
                const bf16* __restrict__ d_o, const float* __restrict__ lse, const float* __restrict__ delta,
                bf16* __restrict__ dq, bf16* __restrict__ dk, bf16* __restrict__ dv, int B, int T, int ld, int ldo,
                int ldg, int H, int KVH, float scale, const int* __restrict__ seg_start) {
  const int group = H / KVH;
  const int n_dkdv = (T + 63) / 64 * KVH * B;
  int i = blockIdx.x;
  if (i < n_dkdv) {
    attn_bwd_dkdv_tile<CAUSAL>(q, k, v, d_o, lse, delta, dk, dv, T, ld, ldo, ldg, H, group, scale, seg_start,
                               i / (KVH * B), i % KVH, i / KVH % B);
  } else {
    i -= n_dkdv;
    const int n_qt = (T + 63) / 64;
    attn_bwd_dq_tile<CAUSAL>(q, k, v, d_o, lse, delta, dq, T, ld, ldo, ldg, H, group, scale, seg_start,
                             n_qt - 1 - i / (H * B), i % H, i / H % B);
  }
}

// +1024: the tiles start at the first 1024-byte boundary of the dynamic shared memory
constexpr int FWD_SMEM = 128 * 128 + 4 * 8192 + 1024;        // 48 KB
constexpr int DKDV_SMEM = 6 * 8192 + 2 * 2 * 64 * 4 + 2 * 64 * 4 + 1024;  // 48 KB + stats + document starts
constexpr int DQ_SMEM = 6 * 8192 + 1024;
constexpr int BWD_SMEM = DKDV_SMEM > DQ_SMEM ? DKDV_SMEM : DQ_SMEM;
constexpr int FWD_SPLIT_SMEM = 2 * 128 * 128 + 8 * 8192 + 1024;  // 96 KB

template <typename K>
int set_smem(K kernel, int bytes) {
  SK_CUDA_CHECK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
  return 0;
}

}  // namespace

int sk_attn_fwd_launch(const bf16* q, const bf16* k, const bf16* v, bf16* o, float* lse, int B, int T, int H, int KVH,
                       int ld, int ldo, int causal, float scale, cudaStream_t s, const int* seg_start) {
  SK_REQUIRE(seg_start == nullptr || causal, "attention: document segments need the causal kernel");
  SK_REQUIRE(B > 0 && T > 0 && H > 0 && KVH > 0, "attention: bad shape B=%d T=%d H=%d KVH=%d", B, T, H, KVH);
  SK_REQUIRE(H % KVH == 0, "attention: H must be a multiple of KVH");
  SK_REQUIRE(ld % 8 == 0 && ldo % 8 == 0, "attention: leading dims must be multiples of 8");
  static bool init = false;
  if (!init) {
    if (set_smem(attn_fwd_kernel<true>, FWD_SMEM)) return -2;
    if (set_smem(attn_fwd_kernel<false>, FWD_SMEM)) return -2;
    init = true;
  }
  dim3 grid((T + 127) / 128, H, B);
  sk_prof_begin(1, s);
  if (causal) attn_fwd_kernel<true><<<grid, 256, FWD_SMEM, s>>>(q, k, v, o, lse, T, ld, ldo, H, H / KVH, scale, seg_start);
  else attn_fwd_kernel<false><<<grid, 256, FWD_SMEM, s>>>(q, k, v, o, lse, T, ld, ldo, H, H / KVH, scale, nullptr);
  sk_prof_end(s);
  SK_LAUNCH_CHECK();
  return 0;
}

// dq/dk/dv are column slices of one gradient buffer with row pitch ldg (same layout as the fused qkv activation)
int sk_attn_bwd_launch(const bf16* q, const bf16* k, const bf16* v, const bf16* o, const bf16* d_o, const float* lse,
                       float* delta, bf16* dq, bf16* dk, bf16* dv, int B, int T, int H, int KVH, int ld, int ldo,
                       int ldg, int causal, float scale, cudaStream_t s, const int* seg_start) {
  SK_REQUIRE(seg_start == nullptr || causal, "attention: document segments need the causal kernels");
  SK_REQUIRE(B > 0 && T > 0 && H > 0 && KVH > 0, "attention: bad shape B=%d T=%d H=%d KVH=%d", B, T, H, KVH);
  SK_REQUIRE(H % KVH == 0, "attention: H must be a multiple of KVH");
  // q/k/v/o/d_o are read 16 bytes at a time (cp.async, ldg128); dq/dk/dv are written as bf16 pairs
  SK_REQUIRE(ld % 8 == 0 && ldo % 8 == 0 && ldg % 2 == 0, "attention: ld and ldo must be multiples of 8 and ldg even");
  static bool init = false;
  if (!init) {
    if (set_smem(attn_bwd_kernel<true>, BWD_SMEM)) return -2;
    if (set_smem(attn_bwd_kernel<false>, BWD_SMEM)) return -2;
    init = true;
  }
  const long n_blocks = (long)(T + 63) / 64 * (KVH + H) * B;   // dK/dV tiles, then dQ tiles
  SK_REQUIRE(n_blocks <= 0x7fffffffL, "attention: grid of %ld blocks too large", n_blocks);
  const long total = (long)B * T * H * 8;
  sk_prof_begin(1, s);
  SK_CUDA_CHECK(sk_launch_pdl(attn_delta_kernel, dim3((int)((total + 255) / 256)), dim3(256), (size_t)(0), s, o, d_o, delta, B, T, H, ldo));
  SK_LAUNCH_CHECK();
  if (causal)
    attn_bwd_kernel<true><<<(unsigned)n_blocks, 128, BWD_SMEM, s>>>(q, k, v, d_o, lse, delta, dq, dk, dv, B, T, ld, ldo, ldg,
                                                                    H, KVH, scale, seg_start);
  else
    attn_bwd_kernel<false><<<(unsigned)n_blocks, 128, BWD_SMEM, s>>>(q, k, v, d_o, lse, delta, dq, dk, dv, B, T, ld, ldo,
                                                                     ldg, H, KVH, scale, nullptr);
  sk_prof_end(s);
  SK_LAUNCH_CHECK();
  return 0;
}

// split-bf16 (hi, lo) forward: bidirectional for the HuBERT encoder, causal for fp32 OPT inference; all six inputs share
// the row pitch ld
int sk_attn_fwd_split_launch(const bf16* q_hi, const bf16* q_lo, const bf16* k_hi, const bf16* k_lo, const bf16* v_hi,
                             const bf16* v_lo, bf16* o_hi, bf16* o_lo, int B, int T, int H, int ld, int ldo, float scale,
                             cudaStream_t s, int causal) {
  SK_REQUIRE(B > 0 && T > 0 && H > 0, "attention: bad shape B=%d T=%d H=%d", B, T, H);
  SK_REQUIRE(ld % 8 == 0 && ldo % 8 == 0, "attention: leading dims must be multiples of 8");
  static bool init[2] = {false, false};
  if (!init[causal ? 1 : 0]) {
    if (set_smem(causal ? attn_fwd_split_kernel<true> : attn_fwd_split_kernel<false>, FWD_SPLIT_SMEM)) return -2;
    init[causal ? 1 : 0] = true;
  }
  dim3 grid((T + 127) / 128, H, B);
  sk_prof_begin(1, s);
  if (causal)
    attn_fwd_split_kernel<true><<<grid, 256, FWD_SPLIT_SMEM, s>>>(q_hi, q_lo, k_hi, k_lo, v_hi, v_lo, o_hi, o_lo, T, ld, ldo,
                                                                  scale);
  else
    attn_fwd_split_kernel<false><<<grid, 256, FWD_SPLIT_SMEM, s>>>(q_hi, q_lo, k_hi, k_lo, v_hi, v_lo, o_hi, o_lo, T, ld, ldo,
                                                                   scale);
  sk_prof_end(s);
  SK_LAUNCH_CHECK();
  return 0;
}

int sk_attn_delta_launch(const bf16* o, const bf16* d_o, float* delta, int B, int T, int H, int ldo, cudaStream_t s) {
  const long total = (long)B * T * H * 8;
  sk_prof_begin(1, s);
  SK_CUDA_CHECK(sk_launch_pdl(attn_delta_kernel, dim3((int)((total + 255) / 256)), dim3(256), (size_t)(0), s, o, d_o, delta, B, T, H, ldo));
  sk_prof_end(s);
  SK_LAUNCH_CHECK();
  return 0;
}

// ---- fused-projection entry points of the LM step ---------------------------------------------------------------
// q/k/v: column slices of one [B*T, ld] bf16 buffer starting at `qkv` (q heads first, then KVH k heads, then KVH v heads)
int sk_attn_tc_fwd_launch(const bf16* qkv, bf16* o, float* lse, int B, int T, int H, int KVH, int ld, int ldo, int causal,
                          float scale, cudaStream_t s, const int* seg_start) {
  return sk_attn_fwd_launch(qkv, qkv + H * HD, qkv + (H + KVH) * HD, o, lse, B, T, H, KVH, ld, ldo, causal, scale, s,
                            seg_start);
}

// dqkv: same column layout as qkv (row pitch ldg).  seg_end is accepted with seg_start (a packed batch); the masks are
// fully determined by seg_start.  With rope tables, the inverse rotary embedding is applied to dq / dk afterwards
// (rope_kernel's inverse mode: the backward of the forward RoPE, same bf16 rounding points).  `partial` is unused here.
int sk_attn_tc_bwd_launch(const bf16* qkv, const bf16* o, const bf16* d_o, const float* lse, float* delta, float* partial,
                          bf16* dqkv, int B, int T, int H, int KVH, int ld, int ldo, int ldg, int causal, float scale,
                          cudaStream_t s, const int* seg_start, const int* seg_end, const bf16* rope_cos,
                          const bf16* rope_sin, const int* pos_ids, int max_pos) {
  (void)partial;
  SK_REQUIRE((seg_start == nullptr) == (seg_end == nullptr), "attn_tc_bwd: seg_start and seg_end go together");
  SK_REQUIRE((rope_cos == nullptr) == (rope_sin == nullptr) && (rope_cos == nullptr || max_pos > 0), "attn_tc_bwd: rope tables go together");
  int rc = sk_attn_bwd_launch(qkv, qkv + H * HD, qkv + (H + KVH) * HD, o, d_o, lse, delta, dqkv, dqkv + H * HD,
                              dqkv + (H + KVH) * HD, B, T, H, KVH, ld, ldo, ldg, causal, scale, s, seg_start);
  if (rc) return rc;
  if (rope_cos) return sk_rope_launch(dqkv, rope_cos, rope_sin, pos_ids, B * T, T, ldg, H + KVH, HD, 1, max_pos, s);
  return 0;
}

// qkv_hi / qkv_lo: [B*T, ld] with H q-heads, H k-heads, H v-heads (64 columns each); o_hi / o_lo: [B*T, ldo]
int sk_attn_tc_fwd_split_launch(const bf16* qkv_hi, const bf16* qkv_lo, bf16* o_hi, bf16* o_lo, int B, int T, int H, int ld,
                                int ldo, float scale, cudaStream_t s, int causal) {
  return sk_attn_fwd_split_launch(qkv_hi, qkv_lo, qkv_hi + H * HD, qkv_lo + H * HD, qkv_hi + 2 * H * HD, qkv_lo + 2 * H * HD,
                                  o_hi, o_lo, B, T, H, ld, ldo, scale, s, causal);
}
