// wgmma GEMM for sm_90a:  C[M,N] = A[M,K] * B[N,K]^T (+bias[N]) (+residual[M,N]),  bf16 in, fp32 accumulate,
// bf16 (or fp32) out.
//
// One persistent CTA per SM, 9 warps:
//   warps 0..7  two consumer warpgroups: warpgroup g issues wgmma.mma_async m64 x BN x 16 on rows [64g, 64g + 64) of
//               the 128-row tile, accumulating in registers; each warp releases a ring slot once the MMAs that read
//               it have retired.  After a tile's K loop the fp32 accumulator is parked in the (then idle) stage ring
//               as a [128][BN] row-major tile, and the epilogue warps read it back one ROW per thread (32 columns at a
//               time): bias / residual / fused element-wise op -> swizzled smem -> TMA store.  EW = 4 epilogue
//               warps (one per 32-row quadrant) or EW = 8 (two per quadrant, each owning half of the columns).
//               Register epilogue (GemmParams::reg_epi: one-pass TMA-store tiles with the plain convert or SwiGLU-forward
//               epilogue, 4-epilogue-warp kernels): the accumulator is not parked; each of the 8 consumer warps packs its
//               16 rows from the wgmma fragments, stmatrix -> swizzled 16-row staging box -> TMA store.
//   warp 8      TMA producer (cp.async.bulk.tensor -> 128B-swizzled smem ring, mbarrier complete_tx); it starts the
//               next tile's loads once the parked accumulator has been consumed, or at once under the register epilogue.
//
// Operand majors.  "K-major" = the contraction index is contiguous in memory (A row-major [M,K], B row-major [N,K]).
// "MN-major" = the M (or N) index is contiguous (A stored as [K,M], B stored as [K,N]).  MN-major operands let the
// backward GEMMs (dgrad: dX = dY * W ; wgrad: dW = dY^T * X) read activations and weights in place, with no
// transposed copies in HBM (wgmma's transpose bits).  Layouts are the canonical GMMA SW128 forms:
//    K-major : ((8,m),(T,2)) : ((8T,SBO),(1,T))          rows of 128 B, 8-row groups SBO=1024 B apart
//    MN-major: ((T,8,m),(8,k)) : ((1,T,LBO),(8T,SBO))    64-element MN atoms, LBO apart; 8-k-row groups SBO apart
#include "common.cuh"
#include <cudaTypedefs.h>
#include <stdio.h>
#include <mutex>
#include <type_traits>
#include <string.h>
#include <stdlib.h>
#include "kernels.h"
#include "../../include/slamkit_b200.h"

namespace {

constexpr int BM = 128;
constexpr int BK = 64;
constexpr int MMA_K = 16;
constexpr int GEMM_THREADS = 288;   // 2 consumer warpgroups + 1 producer warp


struct GemmParams {
  int M, N, K;          // M = rows per batch item when batch > 1
  int batch;            // > 1: A is a 3-D tensor map (k, m, b) and C rows are b*M + m (conv layers, positional conv)
  int a_mode;           // 0: A tile at (kb*64, m0[, b]);  1: shifted window (n_blk*64, m0 + kb, b) (grouped pos-conv)
  int passes;           // 1, or 3 = split-bf16 (A_hi*B_hi + A_hi*B_lo + A_lo*B_hi per k-block): fp32-grade products on bf16 pipes
  void* C;
  void* C_lo;           // non-null: write (hi, lo) bf16 pair, lo = bf16(v - hi)
  int ldc;
  const void* bias;
  int bias_f32;         // bias is float (HuBERT path) instead of bf16
  const bf16* residual;
  const bf16* residual_lo;
  int ldr;
  int tiles_m, tiles_n;
  int out_f32;          // 1: C is float
  int round_before_res; // 1: out = bf16(bf16(acc+bias) + res)  (matches an unfused bf16 linear followed by an add)
  int act;              // 0 none, 1 GELU(erf), 2 ReLU, applied to acc+bias
  int col_gin, col_gout;  // > 0: output column c -> (c / col_gin) * col_gout + c % col_gin, dropped if c % col_gin >= col_gout
  int splits;           // > 1: split-K; work item = (tile, split), fp32 partial tiles go to splitk_ws[split][M][N]
  float* splitk_ws;
  int tma_store;        // 1: bf16 output leaves through swizzled smem staging + cp.async.bulk.tensor stores (tmC)
  int reg_epi;          // 1: register epilogue (one-pass TMA-store tiles, plain convert or SwiGLU forward; see the kernel)
  int pdl;              // host-only: launch attribute
  int sk_units;         // > 0: stream-K over the first sk_units tile groups ("units", see WorkIter)
  int sk_groups;        // CTA groups that share the stream-K iteration space (each unit is cut into <= ~4 ranges)
  int sk_G;             // tiles per unit = CTAs per group (they run the same k-blocks in lockstep)
  int sk_colunits;      // 0: a unit is one row of tiles (same A rows);  1: one column of tiles (same B rows)
  int sk_carry;         // 1: carry-in stream-K (see WorkIter): a split tile's second range starts from the first's accumulator
  int units, n_groups;  // total units, CTA groups in the grid
  float* sk_ws;         // stream-K partial tiles, one 128 x 256 fp32 slot per CTA
  uint32_t* sk_flags;   // [grid][4] publish flags (per epilogue warp), zero between launches
  // Fused epilogues of the LM step (TMA-store path only; see SkGemmEx::epi):
  //   1 SwiGLU forward : N = 2F laid out in [128 gate | 128 up] column blocks; writes gu through tmC AND act[M,F] =
  //                      bf16(bf16(silu(gate)) * up) through tmAux -- the unfused swiglu_fwd_kernel's rounding points
  //   2 SwiGLU backward: the accumulator is d_act[M,F]; reads gu (same block layout) and writes d_gu[M,2F] through tmC
  //   3 RoPE           : after bias + bf16 rounding, every 64-column head below rope_cols is rotated (rotate_half form);
  //                      rope_rot < 64: only its first rope_rot columns (GPT-NeoX partial rotary)
  //   4 GELU forward   : C = pre = bf16(acc + bias) through tmC and bf16(gelu(pre)) through tmAux
  //   5 GELU backward  : the accumulator is d_act; reads the saved pre (aux) and writes bf16(bf16(d_act) * gelu'(pre))
  //   6 two residuals  : bf16(bf16(bf16(acc + bias) + aux) + residual), in epi_residual (every output path)
  int epi;
  const bf16* aux;      // epi 2: gu; epi 5: pre; epi 6: the residual added first
  int ld_aux;
  const bf16* rope_cos; // epi 3: bf16 [rope_maxpos, rope_rot / 2]
  const bf16* rope_sin;
  const int* rope_pos;  // int32 [M] or null (position = row % rope_T)
  int rope_T, rope_cols, rope_maxpos, rope_rot;
};

template <int BN, int EW = 4>
struct GemmCfg {
  static constexpr int A_BYTES = BM * BK * 2;
  static constexpr int B_ATOMS = (BN + 63) / 64;            // MN-major B is fetched in 64-column atoms
  static constexpr int B_BYTES = B_ATOMS * 64 * BK * 2;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int STAGES = (BN > 128) ? 4 : (BN > 64 ? 6 : 8);
  // TMA-store buffers: parked epilogue 2 x (32 rows x 128 B) per epilogue warp (EW = 4) or 1 (EW = 8); register epilogue
  // 2 x (16 rows x 128 B) per consumer warp
  static constexpr int STAGING_BYTES = 4 * 2 * 4096;
  static constexpr int BAR_BYTES = 256;
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + STAGING_BYTES + BAR_BYTES + 1024;  // +1024: manual alignment
  static_assert(BN % 64 == 0 || (BN == 224 && EW == 4), "a 32-column tail chunk only on the 224-wide tile");
  static_assert(STAGES * STAGE_BYTES >= BM * BN * 4, "the parked fp32 accumulator must fit in the stage ring");
  static_assert(SMEM_BYTES <= 227 * 1024, "sm_90 allows 227 KB of shared memory per block");
};

// Parked accumulator: fp32 [BM][BN] row-major at `base`, 16-byte chunks XOR-swizzled by (row & 7) so that both the
// fragment-order stores and the row-per-thread loads spread over all banks.
template <int BN>
SK_DEVINL uint32_t acc_chunk_addr(uint32_t base, int row, int chunk) {
  return base + (uint32_t)row * (BN * 4) + (uint32_t)((chunk ^ (row & 7)) << 4);
}
// one warpgroup's m64 x BN wgmma accumulator (rows [64 wg, 64 wg + 64)) -> parked tile
template <int BN>
SK_DEVINL void acc_park(uint32_t base, const float (&d)[BN / 2], int wg, int warp_in_wg, int lane) {
  const int r0 = 64 * wg + 16 * warp_in_wg + (lane >> 2);
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
    const int chunk = 2 * j + ((lane & 3) >> 1);
    const uint32_t off = (uint32_t)(lane & 1) * 8u;
    asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(acc_chunk_addr<BN>(base, r0, chunk) + off), "f"(d[4 * j]),
                 "f"(d[4 * j + 1]) : "memory");
    asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(acc_chunk_addr<BN>(base, r0 + 8, chunk) + off), "f"(d[4 * j + 2]),
                 "f"(d[4 * j + 3]) : "memory");
  }
}
// row (ta >> 16) + lane, columns [ta & 0xffff, +32) of the parked tile -> r[32]
template <int BN>
SK_DEVINL void acc_ld_32x32(uint32_t base, uint32_t ta, uint32_t (&r)[32]) {
  const int row = (int)(ta >> 16) + (int)(threadIdx.x & 31);
  const int c0 = (int)(ta & 0xffffu) >> 2;
#pragma unroll
  for (int i = 0; i < 8; ++i)
    asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];"
                 : "=r"(r[4 * i]), "=r"(r[4 * i + 1]), "=r"(r[4 * i + 2]), "=r"(r[4 * i + 3])
                 : "r"(acc_chunk_addr<BN>(base, row, c0 + i)) : "memory");
}

// TMA-store staging address of 16-byte piece j of this lane's row.  A 64-column chunk has 128-byte rows in the 128B
// swizzle (map tmC); the 32-column tail chunk of a 224-wide tile has 64-byte rows in the 64B swizzle and leaves through
// a 32-column box (map tmAux), so a tile never writes its neighbour's columns.
SK_DEVINL uint32_t staging_addr(uint32_t sbuf, int lane, int j, bool tail) {
  return tail ? sbuf + (uint32_t)lane * 64u + (uint32_t)((j ^ ((lane >> 1) & 3)) << 4)
              : sbuf + (uint32_t)lane * 128u + (uint32_t)((j ^ (lane & 7)) << 4);
}

// GELU(erf) for the fused epilogue (HuBERT conv layers and FFN): branch-free Abramowitz-Stegun 7.1.26 erf, folded as
//   gelu(y) = relu(y) - |y| * (P(t)/2) * exp(-y^2/2),  t = 1/(1 + p|y|/sqrt2)
// |error| <= 1.5e-7 * |y|/2 absolute -- below the 2^-17 relative grid of the hi/lo bf16 outputs it feeds -- at a third of
// the instructions of libdevice's two-branch erff (same form as hubert_kernels.cu's conv0 front).
SK_DEVINL float gelu_erf(float y) {
  const float a = fabsf(y);
  float t;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(fmaf(0.3275911f * 0.70710678118654752440f, a, 1.0f)));
  float s = fmaf(0.5f * 1.061405429f, t, 0.5f * -1.453152027f);
  s = fmaf(s, t, 0.5f * 1.421413741f);
  s = fmaf(s, t, 0.5f * -0.284496736f);
  s = fmaf(s, t, 0.5f * 0.254829592f);
  const float e = ex2_approx((y * y) * -0.72134752044448170368f);
  return fmaf(-a, (s * t) * e, fmaxf(y, 0.0f));
}

// GELU(erf) of the GPT-NeoX MLP (epi 4 / 5): the expressions of torch's CUDA gelu / gelu_backward kernels in fp32 with
// the accurate erff / expf, so that the bf16 results track torch.nn.functional.gelu and its autograd to the ulp
SK_DEVINL float gelu_exact(float x) { return x * 0.5f * (1.0f + erff(x * 0.70710678118654752440f)); }
SK_DEVINL float gelu_exact_grad(float x) {
  const float cdf = 0.5f * (1.0f + erff(x * 0.70710678118654752440f));
  const float pdf = expf(-0.5f * x * x) * 0.39894228040143267794f;   // M_2_SQRTPI * M_SQRT1_2 * 0.5
  return cdf + x * pdf;
}

SK_DEVINL void stmatrix_x4(uint32_t addr, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
  asm volatile("stmatrix.sync.aligned.m8n8.x4.shared.b16 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(a), "r"(b), "r"(c),
               "r"(d) : "memory");
}

// Work scheduler shared by the three warp roles.
//
// Plain mode (p.sk_units == 0): work item i = blockIdx.x + k * gridDim.x is a whole tile (or a legacy split-K slice).
//
// Stream-K mode: tiles are grouped into "units" of G tiles that read the same rows of the large operand (a row of
// output tiles shares A, a column shares B) and CTAs into groups of G; member j of a group always works on tile j of
// the group's unit, so the G CTAs walk the same k-blocks together and the shared operand is fetched from HBM once
// (what whole-tile scheduling gets for free from running adjacent tiles in the same wave).  The units that would form
// the last, partial wave have their K loops laid end to end and cut into p.sk_groups equal ranges; a range touches at
// most two units.  role 1 = the range starts inside a unit: the fp32 partial tile goes to the CTA's scratch slot;
// role 2 = the range holds the unit's first k-block but not its last: this CTA finishes the tile and adds the partials
// of the same member of the following groups in a fixed order (deterministic); role 0 = whole tile.  The remaining
// units are processed whole, after the stream-K ranges, so the fix-up of a tile overlaps the next tile's MMAs.
//
// Carry-in mode (p.sk_carry, every range at least one unit long): a unit is cut into at most two ranges, and each group
// runs its range's pieces last unit first.  role 1 = the unit's first k-blocks: the fp32 accumulator goes to the CTA's
// scratch slot (published before this CTA's later pieces start); role 3 = the unit's remaining k-blocks: this CTA loads
// that accumulator from the same member of the previous group into its registers and continues the K loop, so every
// element sees the same MMAs in the same order as a whole tile (results bit-identical to whole-tile scheduling).
template <bool SK>
struct WorkIter {
  int num_kb, splits, kb_per_split, total_items, tiles_n;
  // stream-K
  int G, colunits, carry, units, n_groups, sk_groups, grp, mem;
  long sk_total, sk_cur, sk_end;
  int next_unit, next_item;
  // current item
  int tile, split, kb_begin, kb_end, role;
  long unit_end_it;
  SK_DEVINL WorkIter(const GemmParams& p, int num_kb_, int kb_per_split_, int total_items_) {
    num_kb = num_kb_;
    splits = p.splits;
    kb_per_split = kb_per_split_;
    total_items = total_items_;
    tiles_n = p.tiles_n;
    G = p.sk_G;
    colunits = p.sk_colunits;
    carry = p.sk_carry;
    units = p.units;
    n_groups = p.n_groups;
    sk_groups = p.sk_groups;
    tile = split = kb_begin = kb_end = role = 0;
    unit_end_it = 0;
    sk_total = sk_cur = sk_end = 0;
    next_item = (int)blockIdx.x;
    next_unit = 0;
    grp = mem = 0;
    if (SK && p.sk_units > 0) {
      grp = (int)blockIdx.x / G;
      mem = (int)blockIdx.x - grp * G;
      next_item = total_items;                               // plain mode off
      next_unit = grp < n_groups ? p.sk_units + grp : units; // CTAs past the last full group stay idle
      if (grp < sk_groups) {
        sk_total = (long)p.sk_units * num_kb;
        sk_cur = sk_total * grp / sk_groups;
        sk_end = sk_total * (grp + 1) / sk_groups;
      }
    }
  }
  SK_DEVINL int tile_of(int unit) const { return colunits ? mem * tiles_n + unit : unit * G + mem; }
  SK_DEVINL bool next() {
    if (SK && sk_cur < sk_end && carry) {   // last piece of the range first
      const int unit = (int)((sk_end - 1) / num_kb);
      const long ustart = (long)unit * num_kb;
      const long b = sk_cur > ustart ? sk_cur : ustart;
      kb_begin = (int)(b - ustart);
      kb_end = (int)(sk_end - ustart);
      unit_end_it = ustart + num_kb;
      tile = tile_of(unit);
      split = 0;
      role = kb_begin != 0 ? 3 : (kb_end < num_kb ? 1 : 0);
      sk_end = b;
      return true;
    }
    if (SK && sk_cur < sk_end) {
      const int unit = (int)(sk_cur / num_kb);
      kb_begin = (int)(sk_cur - (long)unit * num_kb);
      unit_end_it = (long)(unit + 1) * num_kb;
      const long e = sk_end < unit_end_it ? sk_end : unit_end_it;
      kb_end = kb_begin + (int)(e - sk_cur);
      tile = tile_of(unit);
      split = 0;
      role = kb_begin != 0 ? 1 : (e < unit_end_it ? 2 : 0);
      sk_cur = e;
      return true;
    }
    if (SK && next_unit < units) {
      tile = tile_of(next_unit);
      split = 0;
      kb_begin = 0;
      kb_end = num_kb;
      role = 0;
      next_unit += n_groups;
      return true;
    }
    if (next_item < total_items) {
      split = next_item % splits;
      tile = next_item / splits;
      kb_begin = split * kb_per_split;
      kb_end = min(num_kb, kb_begin + kb_per_split);
      role = 0;
      next_item += (int)gridDim.x;
      return true;
    }
    return false;
  }
  // number of following groups whose range starts inside the current unit (the owner's contributors)
  SK_DEVINL int n_contrib() const {
    int n = 0;
    for (int g = grp + 1; g < sk_groups && sk_total * g / sk_groups < unit_end_it; ++g) ++n;
    return n;
  }
};

SK_DEVINL uint32_t ld_acquire_u32(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
SK_DEVINL void st_release_u32(uint32_t* p, uint32_t v) {
  asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

// bias (+ activation) on 8 consecutive accumulator columns starting at `col`
SK_DEVINL void epi_bias_act(float (&v)[8], const GemmParams& p, int col) {
  if (p.bias) {
    if (p.bias_f32) {
      const float* bp = reinterpret_cast<const float*>(p.bias) + col;
      const float4 b0 = __ldg(reinterpret_cast<const float4*>(bp));
      const float4 b1 = __ldg(reinterpret_cast<const float4*>(bp + 4));
      v[0] += b0.x; v[1] += b0.y; v[2] += b0.z; v[3] += b0.w;
      v[4] += b1.x; v[5] += b1.y; v[6] += b1.z; v[7] += b1.w;
    } else {
      const uint4 bv = ldg128(reinterpret_cast<const bf16*>(p.bias) + col);
      const uint32_t bw[4] = {bv.x, bv.y, bv.z, bv.w};
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float2 f = unpack_bf16(bw[i]);
        v[2 * i] += f.x;
        v[2 * i + 1] += f.y;
      }
    }
  }
  if (p.act == 1) {
#pragma unroll
    for (int i = 0; i < 8; ++i) v[i] = gelu_erf(v[i]);
  } else if (p.act == 2) {   // ReLU commutes with the bf16 rounding that follows: bf16(relu(v)) == relu(bf16(v))
#pragma unroll
    for (int i = 0; i < 8; ++i) v[i] = fmaxf(v[i], 0.0f);
  }
}

// residual (hi, and lo when present) read at output column `ocol` of row `row`
SK_DEVINL void epi_residual(float (&v)[8], const GemmParams& p, size_t row, int ocol) {
  if (p.epi == SK_EPI_RES2) {   // mlp + attn first, rounded (then + x below with round_before_res)
    const uint4 av = *reinterpret_cast<const uint4*>(p.aux + row * p.ld_aux + ocol);
    const uint32_t aw[4] = {av.x, av.y, av.z, av.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 f = unpack_bf16(aw[i]);
      v[2 * i] = bf16_round(bf16_round(v[2 * i]) + f.x);
      v[2 * i + 1] = bf16_round(bf16_round(v[2 * i + 1]) + f.y);
    }
  }
  if (!p.residual) return;
  const uint4 rv = *reinterpret_cast<const uint4*>(p.residual + row * p.ldr + ocol);
  const uint32_t rw[4] = {rv.x, rv.y, rv.z, rv.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 f = unpack_bf16(rw[i]);
    if (p.round_before_res) {
      v[2 * i] = bf16_round(v[2 * i]) + f.x;
      v[2 * i + 1] = bf16_round(v[2 * i + 1]) + f.y;
    } else {
      v[2 * i] += f.x;
      v[2 * i + 1] += f.y;
    }
  }
  if (p.residual_lo) {
    const uint4 lv = *reinterpret_cast<const uint4*>(p.residual_lo + row * p.ldr + ocol);
    const uint32_t lw[4] = {lv.x, lv.y, lv.z, lv.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 f = unpack_bf16(lw[i]);
      v[2 * i] += f.x;
      v[2 * i + 1] += f.y;
    }
  }
}

// Stream-K partial tiles live in p.sk_ws, one 128 x 256 fp32 slot per CTA, laid out [32-col chunk][float4 j][row][4]
// so that a warp (32 consecutive rows) stores and loads 512 contiguous bytes per access.
constexpr int SK_SLOT_FLOATS = BM * 256;
SK_DEVINL size_t sk_slot_off(int chunk, int j4, int row_in_tile) { return ((size_t)(chunk * 8 + j4) * BM + row_in_tile) * 4; }

// add the partial tiles of n following groups (CTA first_cta, first_cta + G, ...) to the 32 accumulator columns in r, in
// group order (deterministic).  One partial (8 x float4 per thread) is in flight at a time: with 8 epilogue warps a thread
// has 168 registers, and the two-deep version spilled.
SK_DEVINL void sk_fixup_add(uint32_t (&r)[32], const float* ws, int chunk, int row_in_tile, int first_cta, int G, int n) {
  for (int c0 = 0; c0 < n; ++c0) {
    const float* slot = ws + (size_t)(first_cta + c0 * G) * SK_SLOT_FLOATS;
    float4 a[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) a[j] = __ldcg(reinterpret_cast<const float4*>(slot + sk_slot_off(chunk, j, row_in_tile)));
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      r[4 * j + 0] = __float_as_uint(__uint_as_float(r[4 * j + 0]) + a[j].x);
      r[4 * j + 1] = __float_as_uint(__uint_as_float(r[4 * j + 1]) + a[j].y);
      r[4 * j + 2] = __float_as_uint(__uint_as_float(r[4 * j + 2]) + a[j].z);
      r[4 * j + 3] = __float_as_uint(__uint_as_float(r[4 * j + 3]) + a[j].w);
    }
  }
}

template <int BN, bool A_MN, bool B_MN, bool SK, int EW>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                  const __grid_constant__ CUtensorMap tmA_lo, const __grid_constant__ CUtensorMap tmB_lo,
                  const __grid_constant__ CUtensorMap tmC, const __grid_constant__ CUtensorMap tmAux, GemmParams p) {
  using Cfg = GemmCfg<BN, EW>;
  static_assert(EW == 4 || (EW == 8 && BN == 256 && !SK), "8 epilogue warps: plain 256-wide tiles only");
  constexpr int CS = EW / 4;          // column split: epilogue warps per 32-row quadrant
  constexpr int NC64 = BN / 64;       // whole 64-column chunks of a tile
  constexpr bool TAIL = BN % 64 != 0; // BN = 224: a last 32-column chunk, stored through tmAux
  griddep_launch();                 // the next kernel on the stream may start its own prologue now
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t staging_base = smem_base + Cfg::STAGES * Cfg::STAGE_BYTES;   // 1024-byte aligned
  const uint32_t bar_base = staging_base + Cfg::STAGING_BYTES;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (Cfg::STAGES + s); };
  const uint32_t acc_free = bar_base + 8u * (2 * Cfg::STAGES);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int tiles_per_batch = p.tiles_m * p.tiles_n;
  const int total_items = tiles_per_batch * p.batch * p.splits;
  const int num_kb_total = (p.K + BK - 1) / BK;
  const int kb_per_split = (num_kb_total + p.splits - 1) / p.splits;
  // bytes one stage receives: A tile + B tile (a K-major B box is exactly BN rows; MN-major B comes in 64-column atoms)
  constexpr uint32_t STAGE_TX = Cfg::A_BYTES + (B_MN ? Cfg::B_ATOMS * 64 * BK * 2 : BN * BK * 2);

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int s = 0; s < Cfg::STAGES; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), 8);   // one arrival per consumer warp
    }
    mbar_init(acc_free, 1);
    fence_mbar_init();
  }
  __syncthreads();
  griddep_wait();                   // prologue done; inputs of this GEMM are complete and visible from here on

  if (warp == 8) {
    // ===== TMA producer =====
    // Split-bf16 mode (passes == 3) pairs two ring slots per k-block: [A_hi | B_hi] [A_lo | B_lo] are fetched once and
    // feed all three products (hi*hi, hi*lo, lo*hi) -- 4 tile loads per k-block instead of the 6 that three separate
    // passes over K would issue.
    if (lane == 0) {
      const bool split = p.passes == 3;
      const int n_stage = split ? Cfg::STAGES / 2 : Cfg::STAGES;
      const uint32_t stage_bytes = split ? 2u * Cfg::STAGE_BYTES : (uint32_t)Cfg::STAGE_BYTES;
      int stage = 0;
      uint32_t phase = 0;
      uint32_t acc_phase = 0;
      bool first = true;
      WorkIter<SK> w(p, num_kb_total, kb_per_split, total_items);
      while (w.next()) {
        if (!first && !p.reg_epi) {   // the previous tile's accumulator is parked in the ring until its epilogue is done
          mbar_wait_nocall(acc_free, acc_phase);
          acc_phase ^= 1u;
        }
        first = false;
        const int bidx = w.tile / tiles_per_batch;
        const int r = w.tile - bidx * tiles_per_batch;
        const int m0 = (r / p.tiles_n) * BM;
        const int n_blk = r % p.tiles_n;
        const int n0 = n_blk * BN;
        for (int kb = w.kb_begin; kb < w.kb_end; ++kb) {
          mbar_wait_nocall(empty_bar(stage), phase ^ 1u);
          const uint32_t fb = full_bar(stage);
          mbar_arrive_expect_tx(fb, split ? 2u * STAGE_TX : STAGE_TX);
          for (int part = 0; part < (split ? 2 : 1); ++part) {
            const CUtensorMap* mapA = part ? &tmA_lo : &tmA;
            const CUtensorMap* mapB = part ? &tmB_lo : &tmB;
            const uint32_t sA = smem_base + stage * stage_bytes + part * Cfg::STAGE_BYTES;
            const uint32_t sB = sA + Cfg::A_BYTES;
            if (!A_MN) {
              if (p.a_mode & 2) {
                if (p.a_mode & 1) tma_load_3d(sA, mapA, fb, n_blk * 64, m0 + kb, bidx);
                else tma_load_3d(sA, mapA, fb, kb * BK, m0, bidx);
              } else {
                tma_load_2d(sA, mapA, fb, kb * BK, m0);
              }
            } else {
#pragma unroll
              for (int j = 0; j < BM / 64; ++j) tma_load_2d(sA + j * (BK * 128), mapA, fb, m0 + 64 * j, kb * BK);
            }
            if (!B_MN) {
              tma_load_2d(sB, mapB, fb, kb * BK, n0);
            } else {
#pragma unroll
              for (int j = 0; j < Cfg::B_ATOMS; ++j) tma_load_2d(sB + j * (BK * 128), mapB, fb, n0 + 64 * j, kb * BK);
            }
          }
          if (++stage == n_stage) { stage = 0; phase ^= 1u; }
        }
      }
    }
  } else {
    // ===== consumer warpgroups (MMA) and epilogue warps 0..EW-1 =====
    const int wg = warp >> 2;
    const int q = warp & 3;            // 32-row quadrant of the tile this warp's epilogue owns
    const int chalf = warp >> 2;       // column half (EW == 8)
    const bool epi_warp = warp < EW;
    auto acc_ld = [&](uint32_t ta, uint32_t (&r)[32]) { acc_ld_32x32<BN>(smem_base, ta, r); };
    const bool split = p.passes == 3;
    const int n_stage = split ? Cfg::STAGES / 2 : Cfg::STAGES;
    const uint32_t stage_bytes = split ? 2u * Cfg::STAGE_BYTES : (uint32_t)Cfg::STAGE_BYTES;
    int stage = 0;
    uint32_t phase = 0;
    uint32_t store_cnt = 0;
    // the parked accumulator has been read: the ring may be refilled (async-proxy writes after generic accesses)
    auto release_acc = [&] {
      fence_proxy_async();
      named_bar_sync(1, 256);
      if (threadIdx.x == 0) mbar_arrive(acc_free);
    };
    WorkIter<SK> w(p, num_kb_total, kb_per_split, total_items);
    while (w.next()) {
      {
        // ---- K loop: this warpgroup's 64 rows x BN columns accumulate in registers ----
        // A tile that continues from a carried-in accumulator and one that starts from zero run separate copies of the
        // K loop: with one copy the two definitions merge ahead of the loop and ptxas serialises its wgmma pipeline.
        // Register epilogue (p.reg_epi): each consumer warp converts its 16 rows of the tile straight from the wgmma
        // fragments -- thread (lane) holds rows r and r + 8 (r = 16 * warp + lane / 4 of the tile), columns 8j + 2(lane % 4)
        // + {0, 1} as acc[4j + 2h], acc[4j + 2h + 1] -- packs a 64-column chunk to bf16 pairs pk[2jj + h], writes them to
        // one of the warp's two 16 x 64 staging boxes with stmatrix (128B swizzle; the 32-column tail chunk of a 224-wide
        // tile: 64B swizzle) and stores the box by TMA.  The ring never holds the accumulator, so the producer loads the
        // next tile's k-blocks while this runs, and a staging box is waited on only before it is rewritten.
        auto reg_epilogue = [&](const float (&acc)[BN / 2]) {
          const int rr = w.tile;   // (batch == 1 on this path)
          const int m0 = (rr / p.tiles_n) * BM, n0 = (rr % p.tiles_n) * BN;
          const int row0 = m0 + 16 * warp;   // this warp's first output row
          const uint32_t stg = staging_base + (uint32_t)warp * 4096u;
          auto emit = [&](const uint32_t (&pk)[16], const CUtensorMap* map, int col, bool tail) {
            const uint32_t sbuf = stg + (store_cnt & 1u) * 2048u;
            if (lane == 0) tma_store_wait_read<1>();
            __syncwarp();
            const int srow = (lane & 7) + (lane & 8);   // stmatrix: lanes 8i..8i+7 address the rows of matrix i
#pragma unroll
            for (int jj = 0; jj < (tail ? 4 : 8); jj += 2) {
              const int ch = jj + (lane >> 4);
              const uint32_t addr = tail ? sbuf + (uint32_t)srow * 64u + (uint32_t)((ch ^ ((srow >> 1) & 3)) << 4)
                                         : sbuf + (uint32_t)srow * 128u + (uint32_t)((ch ^ (srow & 7)) << 4);
              stmatrix_x4(addr, pk[2 * jj], pk[2 * jj + 1], pk[2 * jj + 2], pk[2 * jj + 3]);
            }
            fence_proxy_async();
            __syncwarp();
            if (lane == 0) {
              tma_store_2d(map, sbuf, col, row0);
              tma_store_commit();
            }
            ++store_cnt;
          };
          auto pair_bf16 = [&](int j, int h) { return pack_bf16(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]); };
          if (p.epi == SK_EPI_SWIGLU_FWD) {
            // SwiGLU forward: tile columns [0,128) = gate, [128,256) = up of the same 128 hidden units; gate, up and
            // act = bf16(bf16(silu(gate)) * up) -- the unfused swiglu_fwd_kernel's rounding points
            if constexpr (BN == 256) {
#pragma unroll
              for (int i = 0; i < 2; ++i) {
                uint32_t pk[16];
#pragma unroll
                for (int t = 0; t < 16; ++t) pk[t] = pair_bf16(8 * i + (t >> 1), t & 1);
                emit(pk, &tmC, n0 + 64 * i, false);
#pragma unroll
                for (int t = 0; t < 16; ++t) pk[t] = pair_bf16(16 + 8 * i + (t >> 1), t & 1);
                emit(pk, &tmC, n0 + 128 + 64 * i, false);
#pragma unroll
                for (int t = 0; t < 16; ++t) {
                  const float2 gf = unpack_bf16(pair_bf16(8 * i + (t >> 1), t & 1));
                  const float2 uf = unpack_bf16(pair_bf16(16 + 8 * i + (t >> 1), t & 1));
                  const float2 sb = unpack_bf16(pack_bf16(silu_f(gf.x), silu_f(gf.y)));   // bf16(silu(g))
                  pk[t] = pack_bf16(sb.x * uf.x, sb.y * uf.y);
                }
                emit(pk, &tmAux, (n0 >> 1) + 64 * i, false);
              }
            }
          } else {
            // plain convert; the 32-column tail chunk of a 224-wide tile leaves through tmAux
#pragma unroll
            for (int c2 = 0; c2 < (BN + 63) / 64; ++c2) {
              const bool tail = BN % 64 != 0 && c2 == BN / 64;
              if (n0 + 64 * c2 >= p.N) continue;
              uint32_t pk[16];
#pragma unroll
              for (int t = 0; t < (tail ? 8 : 16); ++t) pk[t] = pair_bf16(8 * c2 + (t >> 1), t & 1);
              emit(pk, tail ? &tmAux : &tmC, n0 + 64 * c2, tail);
            }
          }
        };
        auto mainloop_park = [&](float (&acc)[BN / 2]) {
          const int k_iters = max(0, w.kb_end - w.kb_begin);
          int prev = -1;
          for (int kb = 0; kb < k_iters; ++kb) {
            mbar_wait_nocall(full_bar(stage), phase);
            wgmma_fence();
            const uint32_t s_hi = smem_base + stage * stage_bytes;
            // products per k-block: hi*hi, then (split mode) hi*lo and lo*hi
            for (int g = 0; g < (split ? 3 : 1); ++g) {
              // this warpgroup's rows: 64 K-major rows of 128 B, or the g-th 64-row MN atom -- 8 KB in both layouts
              const uint32_t sA = s_hi + (g == 2 ? Cfg::STAGE_BYTES : 0) + (uint32_t)wg * 8192u;
              const uint32_t sB = s_hi + Cfg::A_BYTES + (g == 1 ? Cfg::STAGE_BYTES : 0);
#pragma unroll
              for (int k = 0; k < BK / MMA_K; ++k) {
                const uint64_t adesc = A_MN ? gmma_desc_sw128(sA + k * (MMA_K * 128), BK * 128, 1024)
                                            : gmma_desc_sw128(sA + k * (MMA_K * 2), 16, 1024);
                const uint64_t bdesc = B_MN ? gmma_desc_sw128(sB + k * (MMA_K * 128), BK * 128, 1024)
                                            : gmma_desc_sw128(sB + k * (MMA_K * 2), 16, 1024);
                wgmma_bf16<BN, A_MN ? 1 : 0, B_MN ? 1 : 0>(acc, adesc, bdesc);
              }
            }
            wgmma_commit();
            wgmma_wait<1>();            // the previous k-block's MMAs have retired: its slot can be refilled
            if (prev >= 0 && lane == 0) mbar_arrive(empty_bar(prev));
            prev = stage;
            if (++stage == n_stage) { stage = 0; phase ^= 1u; }
          }
          wgmma_wait<0>();
          if (prev >= 0 && lane == 0) mbar_arrive(empty_bar(prev));
          if constexpr (!SK && EW == 4) {
            if (p.reg_epi) {
              reg_epilogue(acc);
              return;
            }
          }
          // every k-block of this tile has been consumed and the producer waits for acc_free: the ring is idle
          named_bar_sync(1, 256);
          acc_park<BN>(smem_base, acc, wg, warp & 3, lane);
          named_bar_sync(1, 256);
        };
        if (SK && w.role == 3) {
          float acc[BN / 2];
          // carry-in: continue from the fp32 accumulator of the tile's first k-blocks (same member, previous group)
          const int src = (int)blockIdx.x - w.G;
          if (threadIdx.x == 0) {
            for (int qq = 0; qq < 4; ++qq) {
              const uint32_t* f = p.sk_flags + src * 4 + qq;
              const uint64_t t0 = globaltimer_ns();
              while (ld_acquire_u32(f) == 0u) {
                __nanosleep(64);
                if (globaltimer_ns() - t0 > 8000000000ull) __trap();
              }
            }
            for (int qq = 0; qq < 4; ++qq) p.sk_flags[src * 4 + qq] = 0u;   // re-armed for the next launch
          }
          named_bar_sync(1, 256);
          const float* slot = p.sk_ws + (size_t)src * SK_SLOT_FLOATS;
          const int r0 = 64 * wg + 16 * (warp & 3) + (lane >> 2);
#pragma unroll
          for (int j = 0; j < BN / 8; ++j) {
            const int col = 8 * j + 2 * (lane & 3);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const float2 v = __ldcg(reinterpret_cast<const float2*>(slot + sk_slot_off(col >> 5, (col & 31) >> 2, r0 + 8 * h) +
                                                                      (col & 3)));
              acc[4 * j + 2 * h] = v.x;
              acc[4 * j + 2 * h + 1] = v.y;
            }
          }
          mainloop_park(acc);
        } else {
          float acc[BN / 2];
#pragma unroll
          for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
          mainloop_park(acc);
        }
      }
      if (!SK && p.reg_epi) continue;
      if (!epi_warp) {
        release_acc();
        continue;
      }
      const int split_idx = w.split;
      const int bidx = w.tile / tiles_per_batch;
      const int rr = w.tile - bidx * tiles_per_batch;
      const int m0 = (rr / p.tiles_n) * BM;
      const int n0 = (rr % p.tiles_n) * BN;
      if (!SK && p.tma_store && p.epi == SK_EPI_SWIGLU_BWD) {
        // ===== SwiGLU backward epilogue: acc = d_act; d_gate = bf16(bf16(d_act*u) * silu'(g)), d_up = bf16(d_act * bf16(silu(g)))
        // The accumulator arrives one ROW per thread, but gu / d_gu must move with coalesced accesses (a thread walking
        // its own row issues 32 scattered 16-byte requests per instruction: measured slower than the unfused kernels).
        // So bf16(d_act) goes through the warp's swizzled staging buffer and is re-read in a (4 rows x 8 pieces of
        // 16 bytes) arrangement -- lane = (row % 4, piece) -- in which every global load / store instruction covers
        // four full 128-byte row segments.  The gu registers are refilled in place for the NEXT chunk of the tile as
        // soon as they have been consumed, so a whole chunk of math hides the DRAM latency.  Products of two bf16 values
        // rounded to bf16 are single packed HMUL2.BF16 (exact product, one rounding: the same value as rounding the fp32 product).
        const int lpiece = lane & 7, lrsub = lane >> 3;
        const uint32_t sX = staging_base + (uint32_t)warp * (EW == 4 ? 8192u : 4096u);
        constexpr int NCH = BN / 64 / CS;           // 64-column chunks per warp and tile
        const int c_lo = chalf * NCH;
        // byte offset of this lane's gate piece for (tile origin m0/n0, chunk c2, k = 0); rows advance by 4 per k
        auto piece_off = [&](int bidx, int m0, int n0, int c2, size_t ld) -> size_t {
          const int acol = n0 + c2 * 64;
          const int gcol = (acol >> 7) * 256 + (acol & 127) + lpiece * 8;
          return (((size_t)bidx * p.M + m0 + q * 32 + lrsub) * ld + gcol) * sizeof(bf16);
        };
        const size_t row4_in = (size_t)4 * p.ld_aux * sizeof(bf16), row4_out = (size_t)4 * p.ldc * sizeof(bf16);
        uint4 gv[8], uv[8];
        auto gu_load_k = [&](int k, const uint8_t* base, int m0, int n0, int c2) {
          const int rin = m0 + q * 32 + 4 * k + lrsub;
          if (rin < p.M && n0 + c2 * 64 < p.N) {
            gv[k] = ldg128(base + k * row4_in);
            uv[k] = ldg128(base + k * row4_in + 256);
          } else {
            gv[k] = make_uint4(0u, 0u, 0u, 0u);
            uv[k] = make_uint4(0u, 0u, 0u, 0u);
          }
        };
        {
          const uint8_t* base = reinterpret_cast<const uint8_t*>(p.aux) + piece_off(bidx, m0, n0, c_lo, (size_t)p.ld_aux);
#pragma unroll
          for (int k = 0; k < 8; ++k) gu_load_k(k, base, m0, n0, c_lo);
        }
        const uint32_t taddr = (uint32_t)(q * 32) << 16;
#pragma unroll 1
        for (int c2 = c_lo; c2 < c_lo + NCH; ++c2) {
          const bool col_ok = n0 + c2 * 64 < p.N;
          {
            uint32_t r0[32], r1[32];
            acc_ld(taddr + c2 * 64, r0);
            acc_ld(taddr + c2 * 64 + 32, r1);
#pragma unroll
            for (int j = 0; j < 8; ++j) {
              const uint32_t* r = j < 4 ? r0 + 8 * j : r1 + 8 * (j - 4);
              const uint32_t dst = sX + (uint32_t)lane * 128u + (uint32_t)((j ^ (lane & 7)) << 4);
              asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(dst),
                           "r"(pack_bf16(__uint_as_float(r[0]), __uint_as_float(r[1]))),
                           "r"(pack_bf16(__uint_as_float(r[2]), __uint_as_float(r[3]))),
                           "r"(pack_bf16(__uint_as_float(r[4]), __uint_as_float(r[5]))),
                           "r"(pack_bf16(__uint_as_float(r[6]), __uint_as_float(r[7])))
                           : "memory");
            }
          }
          __syncwarp();
          // the registers freed below are refilled from the next chunk of this tile
          const bool refill = c2 + 1 < c_lo + NCH;
          const int fm0 = m0, fn0 = n0, fc2 = c2 + 1;
          const uint8_t* fbase = reinterpret_cast<const uint8_t*>(p.aux) + piece_off(bidx, fm0, fn0, fc2, (size_t)p.ld_aux);
          uint8_t* obase = reinterpret_cast<uint8_t*>(p.C) + piece_off(bidx, m0, n0, c2, (size_t)p.ldc);
#pragma unroll
          for (int k = 0; k < 8; ++k) {
            const int rr2 = 4 * k + lrsub;
            const uint32_t off = (uint32_t)rr2 * 128u + (uint32_t)((lpiece ^ (rr2 & 7)) << 4);
            uint32_t dw[4];
            asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(dw[0]), "=r"(dw[1]), "=r"(dw[2]), "=r"(dw[3]) : "r"(sX + off));
            const uint32_t gw[4] = {gv[k].x, gv[k].y, gv[k].z, gv[k].w}, uw[4] = {uv[k].x, uv[k].y, uv[k].z, uv[k].w};
            if (refill) gu_load_k(k, fbase, fm0, fn0, fc2);
            uint32_t og[4], ou[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
              const float2 gf = unpack_bf16(gw[e]);
              const float s0 = sigmoid_f(gf.x), s1 = sigmoid_f(gf.y);
              const uint32_t sil2 = pack_bf16(gf.x * s0, gf.y * s1);                       // bf16(silu(g))
              const float ds0 = s0 * (1.0f + gf.x * (1.0f - s0)), ds1 = s1 * (1.0f + gf.y * (1.0f - s1));
              const bf162 d2 = *reinterpret_cast<const bf162*>(&dw[e]);
              bf162 du2 = __hmul2(d2, *reinterpret_cast<const bf162*>(&uw[e]));             // bf16(d_act * u)
              bf162 o2 = __hmul2(d2, *reinterpret_cast<const bf162*>(&sil2));              // d_up
              const float2 duf = __bfloat1622float2(du2);
              og[e] = pack_bf16(duf.x * ds0, duf.y * ds1);
              ou[e] = *reinterpret_cast<uint32_t*>(&o2);
            }
            if (col_ok && m0 + q * 32 + rr2 < p.M) {
              stg128(obase + k * row4_out, make_uint4(og[0], og[1], og[2], og[3]));
              stg128(obase + k * row4_out + 256, make_uint4(ou[0], ou[1], ou[2], ou[3]));
            }
          }
          __syncwarp();                              // all lanes are done reading sX before the next chunk overwrites it
        }
        release_acc();
        continue;
      }
      const int row_in_tile = q * 32 + lane;
      const int row_in = m0 + row_in_tile;
      const bool row_ok = row_in < p.M;
      const size_t row = (size_t)bidx * p.M + row_in;
      const uint32_t taddr = (uint32_t)(q * 32) << 16;   // (first row, column) of this warp in the parked tile
      const int first_contrib = (int)blockIdx.x + w.G;   // same member of the next group
      const int n_contrib = (SK && w.role == 2) ? w.n_contrib() : 0;
      if (SK && w.role == 1) {
        // stream-K contributor: this quadrant's rows of the fp32 partial -> workspace slot, then publish
        float* slot = p.sk_ws + (size_t)blockIdx.x * SK_SLOT_FLOATS;
#pragma unroll 1
        for (int c = 0; c < BN / 32; ++c) {
          uint32_t r[32];
          acc_ld(taddr + c * 32, r);
#pragma unroll
          for (int j = 0; j < 8; ++j)
            __stcg(reinterpret_cast<float4*>(slot + sk_slot_off(c, j, row_in_tile)),
                   make_float4(__uint_as_float(r[4 * j]), __uint_as_float(r[4 * j + 1]), __uint_as_float(r[4 * j + 2]),
                               __uint_as_float(r[4 * j + 3])));
        }
        __threadfence();
        __syncwarp();
        if (lane == 0) st_release_u32(p.sk_flags + blockIdx.x * 4 + q, 1u);
      } else {
        if (SK && w.role == 2) {
          // wait until every CTA that holds a later K range of this tile has published this quadrant's rows
          if (lane == 0) {
            for (int i = 0; i < n_contrib; ++i) {
              const int c = first_contrib + i * w.G;
              const uint32_t* f = p.sk_flags + c * 4 + q;
              const uint64_t t0 = globaltimer_ns();
              while (ld_acquire_u32(f) == 0u) {
                __nanosleep(64);
                if (globaltimer_ns() - t0 > 8000000000ull) __trap();   // no printf: a call anywhere in this kernel serialises its wgmma pipeline
              }
            }
          }
          __syncwarp();
        }
        // one 64-column x 32-row bf16 chunk (tail: 32 columns, pk[0..15]): registers -> this warp's swizzled staging
        // buffer -> TMA store at (col, rows)
        auto stage_store = [&](const CUtensorMap* map, const uint32_t (&pk)[32], int col, auto tail_c) {
          constexpr bool tail = decltype(tail_c)::value;
          const uint32_t sbuf = staging_base + (EW == 4 ? (uint32_t)warp * 8192u + (store_cnt & 1u) * 4096u : (uint32_t)warp * 4096u);
          if (lane == 0) {
            if constexpr (EW == 4) tma_store_wait_read<1>(); else tma_store_wait_read<0>();
          }
          __syncwarp();
#pragma unroll
          for (int j = 0; j < (tail ? 4 : 8); ++j) {
            asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(staging_addr(sbuf, lane, j, tail)), "r"(pk[4 * j]),
                         "r"(pk[4 * j + 1]), "r"(pk[4 * j + 2]), "r"(pk[4 * j + 3])
                         : "memory");
          }
          fence_proxy_async();
          __syncwarp();
          if (lane == 0) {
            tma_store_2d(tail ? &tmAux : map, sbuf, col, m0 + q * 32);
            tma_store_commit();
          }
          ++store_cnt;
        };
        // the epilogues below run the whole 64-column chunks of this warp with tail = false and, for BN = 224, the
        // 32-column tail chunk with tail = true (compile-time constants: one body, no run-time branches in it)
        auto for_chunks = [&](auto&& body) {
#pragma unroll 1
          for (int c2 = chalf * (NC64 / CS); c2 < (chalf + 1) * (NC64 / CS); ++c2) body(std::false_type{}, c2);
          if constexpr (TAIL) body(std::true_type{}, NC64);
        };
        if (!SK && p.tma_store && p.epi == SK_EPI_SWIGLU_FWD) {
          // ---- SwiGLU forward: tile columns [0,128) = gate, [128,256) = up of the same 128 hidden units ----
          if constexpr (BN == 256) {
#pragma unroll 1
#pragma unroll 1
            for (int i = chalf * (2 / CS); i < (chalf + 1) * (2 / CS); ++i) {   // 64 gate columns, the matching up and act columns
              uint32_t gpk[32], upk[32];
              {
                uint32_t r0[32], r1[32];
                acc_ld(taddr + i * 64, r0);
                acc_ld(taddr + i * 64 + 32, r1);
#pragma unroll
                for (int t = 0; t < 16; ++t) {
                  gpk[t] = pack_bf16(__uint_as_float(r0[2 * t]), __uint_as_float(r0[2 * t + 1]));
                  gpk[16 + t] = pack_bf16(__uint_as_float(r1[2 * t]), __uint_as_float(r1[2 * t + 1]));
                }
              }
              stage_store(&tmC, gpk, n0 + i * 64, std::false_type{});
              {
                uint32_t r0[32], r1[32];
                acc_ld(taddr + 128 + i * 64, r0);
                acc_ld(taddr + 128 + i * 64 + 32, r1);
#pragma unroll
                for (int t = 0; t < 16; ++t) {
                  upk[t] = pack_bf16(__uint_as_float(r0[2 * t]), __uint_as_float(r0[2 * t + 1]));
                  upk[16 + t] = pack_bf16(__uint_as_float(r1[2 * t]), __uint_as_float(r1[2 * t + 1]));
                }
              }
              stage_store(&tmC, upk, n0 + 128 + i * 64, std::false_type{});
#pragma unroll
              for (int t = 0; t < 32; ++t) {
                const float2 gf = unpack_bf16(gpk[t]), uf = unpack_bf16(upk[t]);
                const float2 sb = unpack_bf16(pack_bf16(silu_f(gf.x), silu_f(gf.y)));   // bf16(silu(g))
                gpk[t] = pack_bf16(sb.x * uf.x, sb.y * uf.y);
              }
              stage_store(&tmAux, gpk, (n0 >> 1) + i * 64, std::false_type{});
            }
          }
        } else if (!SK && p.tma_store && p.epi == SK_EPI_BIAS_ROPE && p.rope_rot < 64) {
          // ---- bias + partial RoPE (GPT-NeoX): in each head, element i < rope_rot/2 pairs with i + rope_rot/2; the
          // columns from rope_rot on get the bias only.  Same rounding points as the whole-head form below ----
          const int half = p.rope_rot >> 1;   // 8 or 16
          float cf[16], sf[16];
          {
            int pos = 0;
            if (row_ok) pos = p.rope_pos ? p.rope_pos[row] : (int)(row % (size_t)p.rope_T);
            pos = max(0, min(pos, p.rope_maxpos - 1));
#pragma unroll
            for (int j = 0; j < 2; ++j) {
              uint4 c = make_uint4(0u, 0u, 0u, 0u), sn = make_uint4(0u, 0u, 0u, 0u);
              if (8 * j < half) {
                c = ldg128(p.rope_cos + (size_t)pos * half + 8 * j);
                sn = ldg128(p.rope_sin + (size_t)pos * half + 8 * j);
              }
              const uint32_t cw[4] = {c.x, c.y, c.z, c.w}, sw[4] = {sn.x, sn.y, sn.z, sn.w};
#pragma unroll
              for (int e = 0; e < 4; ++e) {
                const float2 cc = unpack_bf16(cw[e]), ss = unpack_bf16(sw[e]);
                cf[8 * j + 2 * e] = cc.x; cf[8 * j + 2 * e + 1] = cc.y;
                sf[8 * j + 2 * e] = ss.x; sf[8 * j + 2 * e + 1] = ss.y;
              }
            }
          }
          auto rotate = [&](float (&a)[32], auto h_c) {
            constexpr int H = decltype(h_c)::value;
#pragma unroll
            for (int i = 0; i < H; ++i) {
              const float x1 = bf16_round(a[i]), x2 = bf16_round(a[i + H]);   // bf16 projection output
              a[i] = bf16_round(x1 * cf[i]) + bf16_round(-x2 * sf[i]);
              a[i + H] = bf16_round(x2 * cf[i]) + bf16_round(x1 * sf[i]);
            }
          };
#pragma unroll 1
          for (int c2 = chalf * (BN / 64 / CS); c2 < (chalf + 1) * (BN / 64 / CS); ++c2) {
            const int col64 = n0 + c2 * 64;
            if (col64 >= p.N) break;
            uint32_t r0[32], r1[32], pk[32];
            acc_ld(taddr + c2 * 64, r0);
            acc_ld(taddr + c2 * 64 + 32, r1);
            float a[32], b[32];
#pragma unroll
            for (int i = 0; i < 32; ++i) {
              a[i] = __uint_as_float(r0[i]);
              b[i] = __uint_as_float(r1[i]);
            }
            if (p.bias) {
#pragma unroll
              for (int g = 0; g < 4; ++g) {
                const uint4 b0 = ldg128(reinterpret_cast<const bf16*>(p.bias) + col64 + g * 8);
                const uint4 b1 = ldg128(reinterpret_cast<const bf16*>(p.bias) + col64 + 32 + g * 8);
                const uint32_t w0[4] = {b0.x, b0.y, b0.z, b0.w}, w1[4] = {b1.x, b1.y, b1.z, b1.w};
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                  const float2 f0 = unpack_bf16(w0[e]), f1 = unpack_bf16(w1[e]);
                  a[g * 8 + 2 * e] += f0.x; a[g * 8 + 2 * e + 1] += f0.y;
                  b[g * 8 + 2 * e] += f1.x; b[g * 8 + 2 * e + 1] += f1.y;
                }
              }
            }
            if (col64 < p.rope_cols) {
              if (half == 16) rotate(a, std::integral_constant<int, 16>{});
              else            rotate(a, std::integral_constant<int, 8>{});
            }
#pragma unroll
            for (int t = 0; t < 16; ++t) {
              pk[t] = pack_bf16(a[2 * t], a[2 * t + 1]);
              pk[16 + t] = pack_bf16(b[2 * t], b[2 * t + 1]);
            }
            stage_store(&tmC, pk, col64, std::false_type{});
          }
        } else if (!SK && p.tma_store && p.epi == SK_EPI_GELU_FWD) {
          // ---- GELU forward (GPT-NeoX dense_h_to_4h): pre = bf16(acc + bias) -> C, bf16(gelu(pre)) -> aux_out ----
#pragma unroll 1
          for (int c2 = chalf * (BN / 64 / CS); c2 < (chalf + 1) * (BN / 64 / CS); ++c2) {
            const int col64 = n0 + c2 * 64;
            if (col64 >= p.N) break;
            uint32_t r0[32], r1[32], pk[32];
            acc_ld(taddr + c2 * 64, r0);
            acc_ld(taddr + c2 * 64 + 32, r1);
#pragma unroll
            for (int g = 0; g < 8; ++g) {
              const uint32_t* r = g < 4 ? r0 + 8 * g : r1 + 8 * (g - 4);
              float v[8];
#pragma unroll
              for (int i = 0; i < 8; ++i) v[i] = __uint_as_float(r[i]);
              epi_bias_act(v, p, col64 + 8 * g);
#pragma unroll
              for (int e = 0; e < 4; ++e) pk[4 * g + e] = pack_bf16(v[2 * e], v[2 * e + 1]);
            }
            stage_store(&tmC, pk, col64, std::false_type{});
#pragma unroll
            for (int t = 0; t < 32; ++t) {
              const float2 f = unpack_bf16(pk[t]);
              pk[t] = pack_bf16(gelu_exact(f.x), gelu_exact(f.y));
            }
            stage_store(&tmAux, pk, col64, std::false_type{});
          }
        } else if (!SK && p.tma_store && p.epi == SK_EPI_GELU_BWD) {
          // ---- GELU backward (input gradient of dense_4h_to_h): d_pre = bf16(bf16(d_act) * gelu'(pre)) ----
#pragma unroll 1
          for (int c2 = chalf * (BN / 64 / CS); c2 < (chalf + 1) * (BN / 64 / CS); ++c2) {
            const int col64 = n0 + c2 * 64;
            if (col64 >= p.N) break;
            uint4 pv[8];
#pragma unroll
            for (int j = 0; j < 8; ++j)
              pv[j] = row_ok ? ldg128(p.aux + row * p.ld_aux + col64 + 8 * j) : make_uint4(0u, 0u, 0u, 0u);
            uint32_t r0[32], r1[32], pk[32];
            acc_ld(taddr + c2 * 64, r0);
            acc_ld(taddr + c2 * 64 + 32, r1);
#pragma unroll
            for (int j = 0; j < 8; ++j) {
              const uint32_t* r = j < 4 ? r0 + 8 * j : r1 + 8 * (j - 4);
              const uint32_t pw[4] = {pv[j].x, pv[j].y, pv[j].z, pv[j].w};
#pragma unroll
              for (int e = 0; e < 4; ++e) {
                const float2 x = unpack_bf16(pw[e]);
                const float2 d = unpack_bf16(pack_bf16(__uint_as_float(r[2 * e]), __uint_as_float(r[2 * e + 1])));
                pk[4 * j + e] = pack_bf16(d.x * gelu_exact_grad(x.x), d.y * gelu_exact_grad(x.y));
              }
            }
            stage_store(&tmC, pk, col64, std::false_type{});
          }
        } else if (!SK && p.tma_store && p.epi == SK_EPI_BIAS_ROPE) {
          // ---- bias + RoPE: a 64-column chunk is one attention head; element i pairs with element i + 32 ----
          uint32_t cw[16], sw[16];
          {
            int pos = 0;
            if (row_ok) pos = p.rope_pos ? p.rope_pos[row] : (int)(row % (size_t)p.rope_T);
            pos = max(0, min(pos, p.rope_maxpos - 1));
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              const uint4 c = ldg128(p.rope_cos + (size_t)pos * 32 + 8 * j), sn = ldg128(p.rope_sin + (size_t)pos * 32 + 8 * j);
              cw[4 * j] = c.x; cw[4 * j + 1] = c.y; cw[4 * j + 2] = c.z; cw[4 * j + 3] = c.w;
              sw[4 * j] = sn.x; sw[4 * j + 1] = sn.y; sw[4 * j + 2] = sn.z; sw[4 * j + 3] = sn.w;
            }
          }
#pragma unroll 1
          for (int c2 = chalf * (BN / 64 / CS); c2 < (chalf + 1) * (BN / 64 / CS); ++c2) {
            const int col64 = n0 + c2 * 64;
            if (col64 >= p.N) break;
            uint32_t r0[32], r1[32], pk[32];
            acc_ld(taddr + c2 * 64, r0);
            acc_ld(taddr + c2 * 64 + 32, r1);
#pragma unroll
            for (int g = 0; g < 4; ++g) {
              float v0[8], v1[8];
#pragma unroll
              for (int i = 0; i < 8; ++i) {
                v0[i] = __uint_as_float(r0[g * 8 + i]);
                v1[i] = __uint_as_float(r1[g * 8 + i]);
              }
              if (p.bias) {                                   // bf16 bias (the QKV projection's), no activation on this path
                const uint4 b0 = ldg128(reinterpret_cast<const bf16*>(p.bias) + col64 + g * 8);
                const uint4 b1 = ldg128(reinterpret_cast<const bf16*>(p.bias) + col64 + 32 + g * 8);
                const uint32_t w0[4] = {b0.x, b0.y, b0.z, b0.w}, w1[4] = {b1.x, b1.y, b1.z, b1.w};
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                  const float2 f0 = unpack_bf16(w0[e]), f1 = unpack_bf16(w1[e]);
                  v0[2 * e] += f0.x; v0[2 * e + 1] += f0.y;
                  v1[2 * e] += f1.x; v1[2 * e + 1] += f1.y;
                }
              }
              if (col64 < p.rope_cols) {
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                  const float2 c = unpack_bf16(cw[g * 4 + e]), sn = unpack_bf16(sw[g * 4 + e]);
                  const float2 x1 = unpack_bf16(pack_bf16(v0[2 * e], v0[2 * e + 1]));   // bf16 projection output
                  const float2 x2 = unpack_bf16(pack_bf16(v1[2 * e], v1[2 * e + 1]));
                  v0[2 * e] = bf16_round(x1.x * c.x) + bf16_round(-x2.x * sn.x);
                  v0[2 * e + 1] = bf16_round(x1.y * c.y) + bf16_round(-x2.y * sn.y);
                  v1[2 * e] = bf16_round(x2.x * c.x) + bf16_round(x1.x * sn.x);
                  v1[2 * e + 1] = bf16_round(x2.y * c.y) + bf16_round(x1.y * sn.y);
                }
              }
#pragma unroll
              for (int e = 0; e < 4; ++e) {
                pk[g * 4 + e] = pack_bf16(v0[2 * e], v0[2 * e + 1]);
                pk[16 + g * 4 + e] = pack_bf16(v1[2 * e], v1[2 * e + 1]);
              }
            }
            stage_store(&tmC, pk, col64, std::false_type{});
          }
        } else if (p.tma_store && !p.bias && !p.residual && !p.act) {
          // plain convert-and-store (dgrads, wgrads, gate/up ...): a straight-line instance without the per-column-group
          // bias / activation / residual tests of the general path below
          for_chunks([&](auto tail_c, int c2) {
            constexpr bool tail = decltype(tail_c)::value;
            uint32_t r0[32], r1[32], pk[32];
            acc_ld(taddr + c2 * 64, r0);
            if (SK && n_contrib > 0) sk_fixup_add(r0, p.sk_ws, c2 * 2, row_in_tile, first_contrib, w.G, n_contrib);
#pragma unroll
            for (int t = 0; t < 16; ++t) pk[t] = pack_bf16(__uint_as_float(r0[2 * t]), __uint_as_float(r0[2 * t + 1]));
            if constexpr (!tail) {
              acc_ld(taddr + c2 * 64 + 32, r1);
              if (SK && n_contrib > 0) sk_fixup_add(r1, p.sk_ws, c2 * 2 + 1, row_in_tile, first_contrib, w.G, n_contrib);
#pragma unroll
              for (int t = 0; t < 16; ++t) pk[16 + t] = pack_bf16(__uint_as_float(r1[2 * t]), __uint_as_float(r1[2 * t + 1]));
            }
            stage_store(&tmC, pk, n0 + c2 * 64, tail_c);
          });
        } else if (p.tma_store && !p.bias && !p.act && p.residual && !p.residual_lo && p.epi == 0) {
          // residual add only (o-proj and down-proj forward: x + linear(..), rounded like the unfused bf16 graph): the
          // row's 128 residual bytes are requested before the accumulator is read; straight-line
          for_chunks([&](auto tail_c, int c2) {
            constexpr bool tail = decltype(tail_c)::value;
            constexpr int nj = tail ? 4 : 8;     // 16-byte pieces of the chunk
            const int col64 = n0 + c2 * 64;
            if (col64 >= p.N) return;
            uint4 rv[8];
            if (row_ok) {
              const bf16* rp = p.residual + row * p.ldr + col64;
#pragma unroll
              for (int j = 0; j < 8; ++j) rv[j] = (j < nj && col64 + 8 * j < p.N) ? ldg128(rp + 8 * j) : make_uint4(0u, 0u, 0u, 0u);
            } else {
#pragma unroll
              for (int j = 0; j < 8; ++j) rv[j] = make_uint4(0u, 0u, 0u, 0u);
            }
            uint32_t r0[32], r1[32], pk[32];
            acc_ld(taddr + c2 * 64, r0);
            if (SK && n_contrib > 0) sk_fixup_add(r0, p.sk_ws, c2 * 2, row_in_tile, first_contrib, w.G, n_contrib);
            if constexpr (!tail) {
              acc_ld(taddr + c2 * 64 + 32, r1);
              if (SK && n_contrib > 0) sk_fixup_add(r1, p.sk_ws, c2 * 2 + 1, row_in_tile, first_contrib, w.G, n_contrib);
            }
#pragma unroll
            for (int j = 0; j < nj; ++j) {
              const uint32_t* r = j < 4 ? r0 + 8 * j : r1 + 8 * (j - 4);
              const uint32_t rw[4] = {rv[j].x, rv[j].y, rv[j].z, rv[j].w};
#pragma unroll
              for (int e = 0; e < 4; ++e) {
                const float2 f = unpack_bf16(rw[e]);
                float a0 = __uint_as_float(r[2 * e]), a1 = __uint_as_float(r[2 * e + 1]);
                if (p.round_before_res) {
                  const float2 t = unpack_bf16(pack_bf16(a0, a1));
                  a0 = t.x; a1 = t.y;
                }
                pk[4 * j + e] = pack_bf16(a0 + f.x, a1 + f.y);
              }
            }
            stage_store(&tmC, pk, col64, tail_c);
          });
        } else if (p.tma_store) {
          // coalesced path: parked accumulator -> registers -> 128B-swizzled smem (this warp's private 32-row buffer) -> TMA store
          for_chunks([&](auto tail_c, int c2) {
            constexpr bool tail = decltype(tail_c)::value;
            const uint32_t sbuf = staging_base + (EW == 4 ? (uint32_t)warp * 8192u + (store_cnt & 1u) * 4096u : (uint32_t)warp * 4096u);
            if (lane == 0) {
              if constexpr (EW == 4) tma_store_wait_read<1>(); else tma_store_wait_read<0>();
            }
            __syncwarp();
#pragma unroll
            for (int half = 0; half < (tail ? 1 : 2); ++half) {
              uint32_t r[32];
              acc_ld(taddr + c2 * 64 + half * 32, r);
              if (SK && n_contrib > 0) sk_fixup_add(r, p.sk_ws, c2 * 2 + half, row_in_tile, first_contrib, w.G, n_contrib);
#pragma unroll
              for (int g = 0; g < 4; ++g) {
                const int col = n0 + c2 * 64 + half * 32 + g * 8;
                float v[8];
#pragma unroll
                for (int i = 0; i < 8; ++i) v[i] = __uint_as_float(r[g * 8 + i]);
                if (col < p.N) {
                  epi_bias_act(v, p, col);
                  if (row_ok) epi_residual(v, p, row, col);
                }
                asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(staging_addr(sbuf, lane, half * 4 + g, tail)),
                             "r"(pack_bf16(v[0], v[1])), "r"(pack_bf16(v[2], v[3])), "r"(pack_bf16(v[4], v[5])),
                             "r"(pack_bf16(v[6], v[7]))
                             : "memory");
              }
            }
            fence_proxy_async();
            __syncwarp();
            if (lane == 0) {
              tma_store_2d(tail ? &tmAux : &tmC, sbuf, n0 + c2 * 64, m0 + q * 32);
              tma_store_commit();
            }
            ++store_cnt;
          });
        }
        else
#pragma unroll 1
        for (int c = chalf * (BN / 32 / CS); c < (chalf + 1) * (BN / 32 / CS); ++c) {
          uint32_t r[32];
          acc_ld(taddr + c * 32, r);
          if (SK && n_contrib > 0) sk_fixup_add(r, p.sk_ws, c, row_in_tile, first_contrib, w.G, n_contrib);
          const int col0 = n0 + c * 32;
          if (row_ok && col0 < p.N) {
#pragma unroll
            for (int g = 0; g < 4; ++g) {
              const int col = col0 + g * 8;
              if (col < p.N) {
                float v[8];
#pragma unroll
                for (int i = 0; i < 8; ++i) v[i] = __uint_as_float(r[g * 8 + i]);
                if (p.splits > 1) {
                  float* dst = p.splitk_ws + ((size_t)split_idx * p.M + row_in) * p.N + col;
                  *reinterpret_cast<float4*>(dst) = make_float4(v[0], v[1], v[2], v[3]);
                  *reinterpret_cast<float4*>(dst + 4) = make_float4(v[4], v[5], v[6], v[7]);
                  continue;
                }
                epi_bias_act(v, p, col);
                int ocol = col;
                if (p.col_gin > 0) {
                  const int gi = col / p.col_gin, ci = col - gi * p.col_gin;
                  if (ci >= p.col_gout) continue;
                  ocol = gi * p.col_gout + ci;
                }
                epi_residual(v, p, row, ocol);
                if (p.out_f32) {
                  float* dst = reinterpret_cast<float*>(p.C) + row * p.ldc + ocol;
                  *reinterpret_cast<float4*>(dst) = make_float4(v[0], v[1], v[2], v[3]);
                  *reinterpret_cast<float4*>(dst + 4) = make_float4(v[4], v[5], v[6], v[7]);
                } else {
                  uint4 o;
                  o.x = pack_bf16(v[0], v[1]);
                  o.y = pack_bf16(v[2], v[3]);
                  o.z = pack_bf16(v[4], v[5]);
                  o.w = pack_bf16(v[6], v[7]);
                  stg128(reinterpret_cast<bf16*>(p.C) + row * p.ldc + ocol, o);
                  if (p.C_lo) {
                    const float2 h0 = unpack_bf16(o.x), h1 = unpack_bf16(o.y), h2 = unpack_bf16(o.z), h3 = unpack_bf16(o.w);
                    uint4 l;
                    l.x = pack_bf16(v[0] - h0.x, v[1] - h0.y);
                    l.y = pack_bf16(v[2] - h1.x, v[3] - h1.y);
                    l.z = pack_bf16(v[4] - h2.x, v[5] - h2.y);
                    l.w = pack_bf16(v[6] - h3.x, v[7] - h3.y);
                    stg128(reinterpret_cast<bf16*>(p.C_lo) + row * p.ldc + ocol, l);
                  }
                }
              }
            }
          }
        }
        if (SK && w.role == 2) {
          // partials consumed: re-arm the flags for the next launch that shares this workspace
          __syncwarp();
          if (lane == 0)
            for (int i = 0; i < n_contrib; ++i) p.sk_flags[(first_contrib + i * w.G) * 4 + q] = 0u;
        }
      }
      release_acc();
    }
    if ((epi_warp || p.reg_epi) && p.tma_store && lane == 0) tma_store_wait<0>();   // all bulk stores retired before the CTA exits
  }
}

// C[m,n] = bf16( sum_s ws[s][m][n] (+ C when accumulate) ), fixed summation order -> deterministic split-K; the sum is
// rounded to bf16 before C is added when round_before_res is set (the same rounding points as the one-pass epilogue)
__global__ void splitk_reduce_kernel(const float* __restrict__ ws, bf16* __restrict__ C, int M, int N, int ldc, int splits,
                                     int accumulate, int round_before_res) {
  griddep_launch();
  griddep_wait();
  const long total = (long)M * N / 8;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const long e = i * 8;
    const int m = (int)(e / N), n = (int)(e % N);
    float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (int s = 0; s < splits; ++s) {
      const float* src = ws + ((size_t)s * M + m) * N + n;
      const float4 a = *reinterpret_cast<const float4*>(src), b = *reinterpret_cast<const float4*>(src + 4);
      acc[0] += a.x; acc[1] += a.y; acc[2] += a.z; acc[3] += a.w;
      acc[4] += b.x; acc[5] += b.y; acc[6] += b.z; acc[7] += b.w;
    }
    bf16* dst = C + (size_t)m * ldc + n;
    if (accumulate) {
      const uint4 o = *reinterpret_cast<const uint4*>(dst);
      const uint32_t ow[4] = {o.x, o.y, o.z, o.w};
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float2 f = unpack_bf16(ow[k]);
        acc[2 * k] = (round_before_res ? bf16_round(acc[2 * k]) : acc[2 * k]) + f.x;
        acc[2 * k + 1] = (round_before_res ? bf16_round(acc[2 * k + 1]) : acc[2 * k + 1]) + f.y;
      }
    }
    stg128(dst, make_uint4(pack_bf16(acc[0], acc[1]), pack_bf16(acc[2], acc[3]), pack_bf16(acc[4], acc[5]),
                           pack_bf16(acc[6], acc[7])));
  }
}

// ----------------------------------------------------------------------------------------------
// host side
// ----------------------------------------------------------------------------------------------
PFN_cuTensorMapEncodeTiled_v12000 g_encode = nullptr;
std::once_flag g_encode_once;

void load_encode() {
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult qres;
  cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres);
  if (e == cudaSuccess && qres == cudaDriverEntryPointSuccess) g_encode = (PFN_cuTensorMapEncodeTiled_v12000)fn;
}

}  // namespace

// Build a 2-D bf16 (elem_bytes=2) / fp32 (elem_bytes=4) tensor map: `inner` contiguous elements, `outer` rows of pitch
// ld elements, box (box_inner x box_outer), 128B swizzle (64B swizzle for a 64-byte box row).
int sk_make_tmap_2d(CUtensorMap* out, const void* ptr, int elem_bytes, uint64_t inner, uint64_t outer, uint64_t ld,
                    uint32_t box_inner, uint32_t box_outer) {
  std::call_once(g_encode_once, load_encode);
  SK_REQUIRE(g_encode != nullptr, "cuTensorMapEncodeTiled driver entry point not available");
  SK_REQUIRE((reinterpret_cast<uintptr_t>(ptr) & 15) == 0, "TMA base pointer must be 16-byte aligned");
  SK_REQUIRE((ld * elem_bytes) % 16 == 0, "TMA row pitch must be a multiple of 16 bytes (ld=%llu)",
             (unsigned long long)ld);
  SK_REQUIRE(box_inner * elem_bytes == 128 || box_inner * elem_bytes == 64, "box inner extent must be 128 (or 64) bytes");
  cuuint64_t dims[2] = {inner, outer};
  cuuint64_t strides[1] = {ld * (uint64_t)elem_bytes};
  cuuint32_t box[2] = {box_inner, box_outer};
  cuuint32_t estr[2] = {1, 1};
  CUtensorMapDataType dt = elem_bytes == 2 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32;
  CUresult r = g_encode(out, dt, 2, const_cast<void*>(ptr), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                        box_inner * elem_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B,
                        CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  SK_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed with CUresult %d (inner=%llu outer=%llu ld=%llu)", (int)r,
             (unsigned long long)inner, (unsigned long long)outer, (unsigned long long)ld);
  return 0;
}

// 3-D variant (inner, rows with pitch row_stride, batch with pitch batch_stride; all in elements), box (64 x box_rows x 1)
int sk_make_tmap_3d(CUtensorMap* out, const void* ptr, uint64_t inner, uint64_t rows, uint64_t batch, uint64_t row_stride,
                    uint64_t batch_stride, uint32_t box_rows) {
  std::call_once(g_encode_once, load_encode);
  SK_REQUIRE(g_encode != nullptr, "cuTensorMapEncodeTiled driver entry point not available");
  SK_REQUIRE((reinterpret_cast<uintptr_t>(ptr) & 15) == 0, "TMA base pointer must be 16-byte aligned");
  SK_REQUIRE((row_stride * 2) % 16 == 0 && (batch_stride * 2) % 16 == 0, "TMA strides must be multiples of 16 bytes");
  cuuint64_t dims[3] = {inner, rows, batch};
  cuuint64_t strides[2] = {row_stride * 2, batch_stride * 2};
  cuuint32_t box[3] = {64, box_rows, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = g_encode(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(ptr), dims, strides, box, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  SK_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled(3d) failed with CUresult %d", (int)r);
  return 0;
}

namespace {

template <int BN, bool A_MN, bool B_MN, bool SK, int EW = 4>
int launch_gemm(const CUtensorMap* tm, const GemmParams& p, int grid, cudaStream_t stream) {
  using Cfg = GemmCfg<BN, EW>;
  static bool attr_set = false;
  if (!attr_set) {
    SK_CUDA_CHECK(cudaFuncSetAttribute(gemm_wgmma_kernel<BN, A_MN, B_MN, SK, EW>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       Cfg::SMEM_BYTES));
    attr_set = true;
  }
  sk_prof_begin(0, stream);
  cudaError_t lerr = sk_launch_pdl_if(p.pdl != 0, gemm_wgmma_kernel<BN, A_MN, B_MN, SK, EW>, dim3(grid), dim3(GEMM_THREADS), (size_t)Cfg::SMEM_BYTES, stream,
                                   tm[0], tm[1], tm[2], tm[3], tm[4], tm[5], p);
  sk_prof_end(stream);
  SK_CUDA_CHECK(lerr);
  SK_LAUNCH_CHECK();
  return 0;
}

template <int BN, bool SK, int EW = 4>
int dispatch_major(bool a_mn, bool b_mn, const CUtensorMap* tm, const GemmParams& p, int grid, cudaStream_t s) {
  if (!a_mn && !b_mn) return launch_gemm<BN, false, false, SK, EW>(tm, p, grid, s);
  if (!a_mn && b_mn) return launch_gemm<BN, false, true, SK, EW>(tm, p, grid, s);
  if (a_mn && !b_mn) return launch_gemm<BN, true, false, SK, EW>(tm, p, grid, s);
  return launch_gemm<BN, true, true, SK, EW>(tm, p, grid, s);
}

// Relative cost of one 128 x BN tile (BN=256 == 100), a heuristic: narrow tiles pay the per-tile pipeline fill /
// epilogue overhead and re-read the A tile from shared memory more often per FLOP.  192 and 224 are put on the line
// through 128 and 256 (80 and 90).
inline int tile_cost(int bn) { return bn >= 256 ? 100 : (bn > 128 ? 61 + (bn - 128) * 39 / 128 : (bn == 128 ? 61 : 54)); }

constexpr size_t SK_FLAG_BYTES = 4096;   // tail of the scratch buffer: stream-K publish flags ([CTA][32-row quadrant])
// stream-K balancing pays when whole-tile waves would leave at least this share (%) of the SM-time idle and the K loop
// is at least this many k-blocks long; with less idle time or shorter K the fix-up traffic eats the gain
constexpr int STREAMK_MIN_IDLE_PCT = 20;
constexpr int STREAMK_MIN_KB = 32;
constexpr int STREAMK_RANGES = 4;   // row units: each leftover unit is cut into at most ~this many K ranges

}  // namespace

size_t sk_gemm_ws_min_bytes(void) { return (size_t)sk_num_sms() * SK_SLOT_FLOATS * sizeof(float) + SK_FLAG_BYTES; }

// Tile width.  The persistent kernel runs a GEMM in about ceil(tiles / SMs) tile times, and every tile pays for its
// whole BN columns (a half-empty last tile column costs a full one), so a width costs
// waves(tiles, sk_num_sms()) x tile_cost(bn).  256 is the default; 128 or 64 displaces it only when clearly cheaper
// (>= 25 %: near-ties favour the wide tile).  With `fit`, a 256 pick whose last tile column would be partly empty is
// then replaced by 224 or 192 when that costs >= 5 % less: the empty columns of 256 are often what pushes the GEMM into
// another wave (the LM's d = 896 = 4 x 224 and QKV = 1152 = 6 x 192).  Sizes that 256 divides keep it.  whole_heads
// keeps the widths to whole 64-column heads (the RoPE epilogue).  A forced width is taken as it is (192 / 224 when
// fit_forced).
int sk_pick_bn(int M, int N, int force_bn, bool fit_forced, bool fit, bool whole_heads) {
  if (force_bn == 64 || force_bn == 128 || force_bn == 256) return force_bn;
  if (fit_forced && (force_bn == 192 || (force_bn == 224 && !whole_heads))) return force_bn;
  const int nsm = sk_num_sms();
  auto cost = [&](int bn) {
    const long tiles = (long)((M + BM - 1) / BM) * ((N + bn - 1) / bn);
    return ((tiles + nsm - 1) / nsm) * tile_cost(bn);
  };
  int best = 256;
  long best_cost = cost(256);
  for (const int bn : {128, 64}) {
    if (cost(bn) * 100 < best_cost * 75) {
      best_cost = cost(bn);
      best = bn;
    }
  }
  if (best == 256 && fit && N % 256 != 0) {
    for (const int bn : {224, 192}) {
      if (!(whole_heads && bn % 64 != 0) && cost(bn) * 100 < best_cost * 95) {
        best_cost = cost(bn);
        best = bn;
      }
    }
  }
  return best;
}

namespace {

// Everything the launcher decides before it encodes tensor maps: argument checks, tile width (BN), split-K, TMA-store
// epilogue, the stream-K partition, epilogue warps (ew) and grid; p receives every kernel parameter.  sk_gemm_ex_launch
// runs exactly this plan (it only adds the tensor maps); sk_gemm_plan_ex reports it, so tests can tell which schedule ran.
int plan_gemm(const SkGemmEx& g, GemmParams& p, int& BN, int& ew, int& grid) {
  SK_REQUIRE(g.M > 0 && g.N > 0 && g.K > 0 && g.batch >= 1, "gemm: empty problem M=%d N=%d K=%d batch=%d", g.M, g.N, g.K,
             g.batch);
  SK_REQUIRE(g.N % 8 == 0, "gemm: N must be a multiple of 8 (N=%d)", g.N);
  SK_REQUIRE(g.ldc % 8 == 0 && (g.residual == nullptr || g.ldr % 8 == 0), "gemm: ldc/ldr must be multiples of 8");
  SK_REQUIRE((reinterpret_cast<uintptr_t>(g.C) & 15) == 0, "gemm: C must be 16-byte aligned");
  SK_REQUIRE(((reinterpret_cast<uintptr_t>(g.A) | reinterpret_cast<uintptr_t>(g.B) | reinterpret_cast<uintptr_t>(g.A_lo) |
               reinterpret_cast<uintptr_t>(g.B_lo)) & 15) == 0,
             "gemm: A and B must be 16-byte aligned");
  SK_REQUIRE((reinterpret_cast<uintptr_t>(g.bias) & 15) == 0 && (reinterpret_cast<uintptr_t>(g.residual) & 15) == 0,
             "gemm: bias and residual must be 16-byte aligned");
  SK_REQUIRE(g.passes == 1 || (g.passes == 3 && g.A_lo && g.B_lo), "gemm: passes must be 1, or 3 with lo operands");
  SK_REQUIRE(g.act >= 0 && g.act <= 2, "gemm: act must be 0 (none), 1 (GELU) or 2 (ReLU), got %d", g.act);
  const bool use3d = g.a_rows > 0;   // strided-window / batched A view
  SK_REQUIRE(!use3d || !g.a_mn, "gemm: a batched / windowed A operand must be K-major");
  SK_REQUIRE(g.a_mode == 0 || use3d, "gemm: a_mode 1 needs the 3-D A view");
  // pitches cover the rows they describe (a TMA map would otherwise read the next row's elements as this row's)
  SK_REQUIRE(use3d || g.lda >= (g.a_mn ? g.M : g.K), "gemm: lda=%d is smaller than the %s of A", g.lda, g.a_mn ? "M" : "K");
  SK_REQUIRE(g.ldb >= (g.b_mn ? g.N : g.K), "gemm: ldb=%d is smaller than the %s of B", g.ldb, g.b_mn ? "N" : "K");
  if (g.col_gin == 0) {   // (compacted columns are narrower than N)
    const int out_cols = g.epi == SK_EPI_SWIGLU_BWD ? 2 * g.N : g.N;
    SK_REQUIRE(g.ldc >= out_cols, "gemm: ldc=%d is smaller than the %d output columns", g.ldc, out_cols);
    SK_REQUIRE(g.residual == nullptr || g.ldr >= g.N, "gemm: ldr=%d is smaller than N=%d", g.ldr, g.N);
  }
  const int nsm = sk_num_sms();
  // stream-K needs the plain 2-D form and a scratch buffer of sk_gemm_ws_min_bytes() whose last 4 KB (flags) are zero
  static const int sk_env = [] { const char* e = getenv("SK_STREAMK"); return e ? atoi(e) : 1; }();
  const bool sk_ok = sk_env != 0 && g.batch == 1 && !use3d && g.passes == 1 && g.a_mode == 0 && g.splitk_ws != nullptr &&
                     g.splitk_ws_bytes >= sk_gemm_ws_min_bytes();
  const size_t ws_data_bytes = g.splitk_ws_bytes > SK_FLAG_BYTES ? g.splitk_ws_bytes - SK_FLAG_BYTES : 0;
  // the SwiGLU epilogues need both halves of a [128 gate | 128 up] block in one tile.  The 192 / 224 widths are for
  // plain one-pass 2-D problems; the auto planner leaves them to GEMMs without stream-K scratch (forward and dgrad):
  // with scratch, split-K / stream-K balance the last wave at the widths they were tuned for
  // (the GELU epilogues also stay on whole 64-column chunks: the forward's second output leaves through tmAux)
  const bool fit = g.passes == 1 && g.batch == 1 && !use3d && g.a_mode == 0 && g.epi != SK_EPI_SWIGLU_FWD &&
                   g.epi != SK_EPI_SWIGLU_BWD && g.epi != SK_EPI_GELU_FWD && g.epi != SK_EPI_GELU_BWD;
  SK_REQUIRE((g.force_bn != 192 && g.force_bn != 224) || (fit && !(g.force_bn == 224 && g.epi == SK_EPI_BIAS_ROPE)),
             "gemm: force_bn=%d needs a one-pass 2-D problem (and whole 64-column heads for RoPE)", g.force_bn);
  const bool swiglu = g.epi == SK_EPI_SWIGLU_FWD || g.epi == SK_EPI_SWIGLU_BWD;
  BN = (g.a_mode == 1) ? 64
                       : sk_pick_bn(g.M * g.batch, g.N, swiglu ? 256 : g.force_bn, fit, fit && !sk_ok, g.epi == SK_EPI_BIAS_ROPE);
  memset(&p, 0, sizeof(p));
  p.M = g.M; p.N = g.N; p.K = g.K;
  p.batch = g.batch;
  p.a_mode = (g.a_mode & 1) | (use3d ? 2 : 0);   // bit 1: A uses the 3-D TMA form
  p.passes = g.passes;
  p.C = g.C; p.C_lo = g.C_lo; p.ldc = g.ldc;
  p.bias = g.bias; p.bias_f32 = g.bias_f32;
  p.residual = reinterpret_cast<const bf16*>(g.residual);
  p.residual_lo = reinterpret_cast<const bf16*>(g.residual_lo);
  p.ldr = g.ldr;
  p.tiles_m = (g.M + BM - 1) / BM;
  p.tiles_n = (g.N + BN - 1) / BN;
  p.out_f32 = g.out_f32;
  p.round_before_res = g.round_before_res;
  p.act = g.act;
  p.col_gin = g.col_gin; p.col_gout = g.col_gout;
  p.pdl = g.pdl;
  const long tiles = (long)p.tiles_m * p.tiles_n * g.batch;
  // split-K: only for plain bf16-output GEMMs that leave most SMs idle and have a long K loop (the small wgrads)
  p.splits = 1;
  p.splitk_ws = nullptr;
  const int num_kb = (g.K + BK - 1) / BK;
  if (g.splitk_ws && g.batch == 1 && g.passes == 1 && !g.out_f32 && !g.bias && !g.act && !g.C_lo && g.col_gin == 0 &&
      g.epi == 0 &&
      (g.residual == nullptr || g.residual == g.C) && tiles * 2 <= nsm && num_kb >= 16) {
    int sp = (int)(nsm / tiles);
    if (sp > 8) sp = 8;
    if (sp > num_kb / 4) sp = num_kb / 4;
    if ((size_t)sp * g.M * g.N * sizeof(float) > ws_data_bytes) sp = (int)(ws_data_bytes / ((size_t)g.M * g.N * sizeof(float)));
    if (sp >= 2) {
      const int per = (num_kb + sp - 1) / sp;
      sp = (num_kb + per - 1) / per;   // no empty split: every work item issues at least one MMA
    }
    if (sp >= 2) {
      p.splits = sp;
      p.splitk_ws = reinterpret_cast<float*>(g.splitk_ws);
    }
  }
  // TMA-store epilogue for the plain bf16 outputs (everything on the LM path)
  p.tma_store = (!g.out_f32 && !g.C_lo && g.col_gin == 0 && p.splits == 1 && g.batch == 1 && !use3d && (g.ldc * 2) % 16 == 0)
                    ? 1 : 0;
  p.epi = g.epi;
  p.aux = reinterpret_cast<const bf16*>(g.aux);
  p.ld_aux = g.ld_aux;
  p.rope_cos = reinterpret_cast<const bf16*>(g.rope_cos);
  p.rope_sin = reinterpret_cast<const bf16*>(g.rope_sin);
  p.rope_pos = g.rope_pos;
  p.rope_T = g.rope_T; p.rope_cols = g.rope_cols; p.rope_maxpos = g.rope_maxpos;
  p.rope_rot = g.rope_rot == 0 ? 64 : g.rope_rot;
  if (g.epi == SK_EPI_RES2) {
    // two residuals: runs on every output path (epi_residual), stream-K included; split-K is not planned for it
    SK_REQUIRE(g.passes == 1 && g.batch == 1 && !use3d && g.residual && g.aux && !g.residual_lo && !g.act && !g.out_f32 &&
                   !g.C_lo && g.col_gin == 0 && g.round_before_res && g.ld_aux >= g.N && g.ld_aux % 8 == 0 &&
                   (reinterpret_cast<uintptr_t>(g.aux) & 15) == 0,
               "gemm: two-residual epilogue needs a plain one-pass bf16 GEMM, both residuals (16-byte aligned, pitch >= N) and "
               "round_before_res");
  } else if (g.epi != 0) {
    SK_REQUIRE(p.tma_store && g.passes == 1 && !g.residual && !g.act && g.splitk_ws == nullptr,
               "gemm: fused epilogue %d needs the plain bf16 TMA-store path (no residual / activation / scratch)", g.epi);
    if (g.epi == SK_EPI_SWIGLU_FWD) {
      SK_REQUIRE(BN == 256 && g.N % 256 == 0 && g.aux_out && g.ld_aux_out % 8 == 0 && !g.bias,
                 "gemm: SwiGLU-forward epilogue needs N = 2F with F %% 128 == 0 and an act output");
    } else if (g.epi == SK_EPI_SWIGLU_BWD) {
      SK_REQUIRE(BN == 256 && g.N % 128 == 0 && g.aux && g.ld_aux % 8 == 0 && !g.bias,
                 "gemm: SwiGLU-backward epilogue needs N = F with F %% 128 == 0 and the saved gu activation");
    } else if (g.epi == SK_EPI_BIAS_ROPE) {
      SK_REQUIRE(g.rope_cos && g.rope_sin && g.rope_T > 0 && g.rope_maxpos > 0 && g.rope_cols % 64 == 0 && g.N % 64 == 0 &&
                     !g.bias_f32,
                 "gemm: RoPE epilogue needs cos/sin tables, 64-column heads and a bf16 bias");
      SK_REQUIRE(p.rope_rot == 16 || p.rope_rot == 32 || p.rope_rot == 64,
                 "gemm: RoPE epilogue rotary width rope_rot=%d is not supported (16, 32 or 64)", g.rope_rot);
    } else if (g.epi == SK_EPI_GELU_FWD) {
      SK_REQUIRE(BN % 64 == 0 && g.N % 64 == 0 && g.aux_out && g.ld_aux_out >= g.N && g.ld_aux_out % 8 == 0 && !g.bias_f32 &&
                     (reinterpret_cast<uintptr_t>(g.aux_out) & 15) == 0,
                 "gemm: GELU-forward epilogue needs N %% 64 == 0, an act output (pitch >= N) and a bf16 bias");
    } else if (g.epi == SK_EPI_GELU_BWD) {
      SK_REQUIRE(BN % 64 == 0 && g.N % 64 == 0 && g.aux && g.ld_aux >= g.N && g.ld_aux % 8 == 0 && !g.bias &&
                     (reinterpret_cast<uintptr_t>(g.aux) & 15) == 0,
                 "gemm: GELU-backward epilogue needs N %% 64 == 0, the saved pre-activation (pitch >= N) and no bias");
    } else {
      SK_REQUIRE(false, "gemm: unknown fused epilogue %d", g.epi);
    }
  }
  // stream-K over the units (rows or columns of tiles) of the last, partial wave -- see WorkIter.  Row units (a tile
  // row of <= 8 tiles) cut the leftover units into at most ~4 ranges each.  Column units (<= 8 tile rows, more than 8
  // tile columns: the down-projection weight gradient, 7 x 19 tiles) balance the last of several waves by default: the
  // leftover units and the last full wave are laid end to end over every group, so each group runs 1 + rem / n_groups
  // units and a unit is cut into at most two ranges, the second continuing from the first's accumulator (carry-in: the
  // weight gradient comes out bit-identical to whole tiles).  SK_STREAMK=2 also takes single-wave shapes.
  p.sk_G = 1;
  if (sk_ok && BN == 256 && p.splits == 1 && num_kb >= STREAMK_MIN_KB && (p.tiles_n <= 8 || p.tiles_m <= 8)) {
    const int colunits = p.tiles_n <= 8 ? 0 : 1;
    const int G = colunits ? p.tiles_m : p.tiles_n;
    const int units = colunits ? p.tiles_n : p.tiles_m;
    const int n_groups = nsm / G;
    const int rem = units % n_groups;
    const long slots = ((long)(units + n_groups - 1) / n_groups) * n_groups;
    const bool multiwave = units > n_groups;
    if (n_groups >= 1 && rem != 0 && (slots - units) * 100 >= slots * STREAMK_MIN_IDLE_PCT &&   // enough SM-time would idle
        (!colunits || multiwave || sk_env >= 2)) {
      if (colunits && multiwave) {
        p.sk_units = rem + n_groups;
        p.sk_groups = n_groups;
        p.sk_carry = 1;
      } else {
        p.sk_units = rem;
        p.sk_groups = n_groups < rem * STREAMK_RANGES ? n_groups : rem * STREAMK_RANGES;
      }
      p.sk_G = G;
      p.sk_colunits = colunits;
      p.units = units;
      p.n_groups = n_groups;
      p.sk_ws = reinterpret_cast<float*>(g.splitk_ws);
      p.sk_flags = reinterpret_cast<uint32_t*>(reinterpret_cast<uint8_t*>(g.splitk_ws) + ws_data_bytes);
    }
  }
  const long work = tiles * p.splits;
  grid = p.sk_units > 0 ? p.n_groups * p.sk_G : (int)(work < nsm ? work : nsm);
  // 8 epilogue warps (two per 32-row quadrant) where the epilogue does real work per element; the plain
  // convert-and-store epilogue is faster with 4 (fewer warps contending with the TMA / MMA issue threads)
  static const int ew_env = [] { const char* e = getenv("SK_GEMM_EW"); return e ? atoi(e) : 0; }();
  const bool heavy_epi = g.epi == SK_EPI_SWIGLU_BWD || g.epi == SK_EPI_BIAS_ROPE || g.epi == SK_EPI_GELU_FWD ||
                         g.epi == SK_EPI_GELU_BWD;
  ew = (p.sk_units == 0 && BN == 256 && p.tma_store && (ew_env == 8 || (ew_env == 0 && heavy_epi))) ? 8 : 4;
  // the register epilogue takes the one-pass TMA-store tiles whose epilogue reads no operand (plain convert and SwiGLU
  // forward) on the 4-epilogue-warp kernels; the others keep the parked accumulator
  p.reg_epi = (p.tma_store && p.sk_units == 0 && ew == 4 && !g.bias && !g.act && !g.residual &&
               (g.epi == 0 || g.epi == SK_EPI_SWIGLU_FWD)) ? 1 : 0;
  return 0;
}

}  // namespace

int sk_gemm_plan_ex(const SkGemmEx& g, SkGemmPlan* out) {
  GemmParams p;
  int BN = 0, ew = 0, grid = 0;
  const int rc = plan_gemm(g, p, BN, ew, grid);
  if (rc) return rc;
  out->bn = BN;
  out->epi_warps = ew;
  out->splits = p.splits;
  out->sk_units = p.sk_units;
  out->sk_groups = p.sk_groups;
  out->sk_G = p.sk_G;
  out->sk_colunits = p.sk_colunits;
  out->tma_store = p.tma_store;
  out->grid = grid;
  return 0;
}

// General launcher (see SkGemmEx in kernels.h).
int sk_gemm_ex_launch(const SkGemmEx& g, cudaStream_t stream) {
  GemmParams p;
  int BN = 0, ew = 0, grid = 0;
  const int rc0 = plan_gemm(g, p, BN, ew, grid);
  if (rc0) return rc0;
  const bool use3d = g.a_rows > 0;
  CUtensorMap tm[6];
  const void* As[2] = {g.A, g.passes == 3 ? g.A_lo : g.A};
  const void* Bs[2] = {g.B, g.passes == 3 ? g.B_lo : g.B};
  for (int i = 0; i < 2; ++i) {
    int rc;
    CUtensorMap* ta = &tm[i == 0 ? 0 : 2];
    CUtensorMap* tb = &tm[i == 0 ? 1 : 3];
    if (use3d) {
      rc = sk_make_tmap_3d(ta, As[i], (uint64_t)g.a_inner, (uint64_t)g.a_rows, (uint64_t)g.batch, (uint64_t)g.a_row_stride,
                           (uint64_t)g.a_batch_stride, BM);
    } else if (!g.a_mn) {
      rc = sk_make_tmap_2d(ta, As[i], 2, (uint64_t)g.K, (uint64_t)g.M, (uint64_t)g.lda, BK, BM);
    } else {
      rc = sk_make_tmap_2d(ta, As[i], 2, (uint64_t)g.M, (uint64_t)g.K, (uint64_t)g.lda, 64, BK);
    }
    if (rc) return rc;
    if (!g.b_mn) rc = sk_make_tmap_2d(tb, Bs[i], 2, (uint64_t)g.K, (uint64_t)g.N, (uint64_t)g.ldb, BK, (uint32_t)BN);
    else         rc = sk_make_tmap_2d(tb, Bs[i], 2, (uint64_t)g.N, (uint64_t)g.K, (uint64_t)g.ldb, 64, BK);
    if (rc) return rc;
  }
  tm[4] = tm[0];
  // store boxes: 16 rows (one warp's rows of the wgmma fragment) for the register epilogue, 32 rows (one parked-epilogue
  // warp's quadrant) otherwise
  const uint32_t box_rows = p.reg_epi ? 16 : 32;
  if (p.tma_store) {
    // the SwiGLU backward writes d_gu [M, 2N] (the accumulator tile is d_act [M, N])
    const int rc2 = sk_make_tmap_2d(&tm[4], g.C, 2, (uint64_t)(g.epi == SK_EPI_SWIGLU_BWD ? 2 * g.N : g.N), (uint64_t)g.M,
                                    (uint64_t)g.ldc, 64, box_rows);
    if (rc2) return rc2;
  }
  tm[5] = tm[4];
  if (g.epi == SK_EPI_SWIGLU_FWD) {
    const int rc3 = sk_make_tmap_2d(&tm[5], g.aux_out, 2, (uint64_t)g.N / 2, (uint64_t)g.M, (uint64_t)g.ld_aux_out, 64, box_rows);
    if (rc3) return rc3;
  } else if (g.epi == SK_EPI_GELU_FWD) {   // the GELU output, same shape as C
    const int rc3 = sk_make_tmap_2d(&tm[5], g.aux_out, 2, (uint64_t)g.N, (uint64_t)g.M, (uint64_t)g.ld_aux_out, 64, 32);
    if (rc3) return rc3;
  } else if (p.tma_store && BN % 64 != 0) {   // the 32-column tail chunk of a 224-wide tile
    const int rc3 = sk_make_tmap_2d(&tm[5], g.C, 2, (uint64_t)g.N, (uint64_t)g.M, (uint64_t)g.ldc, 32, box_rows);
    if (rc3) return rc3;
  }
  int rc;
  if (p.sk_units > 0) {
    rc = dispatch_major<256, true>(g.a_mn, g.b_mn, tm, p, grid, stream);
  } else if (ew == 8) {
    rc = dispatch_major<256, false, 8>(g.a_mn, g.b_mn, tm, p, grid, stream);
  } else {
    switch (BN) {
      case 256: rc = dispatch_major<256, false>(g.a_mn, g.b_mn, tm, p, grid, stream); break;
      case 224: rc = dispatch_major<224, false>(g.a_mn, g.b_mn, tm, p, grid, stream); break;
      case 192: rc = dispatch_major<192, false>(g.a_mn, g.b_mn, tm, p, grid, stream); break;
      case 128: rc = dispatch_major<128, false>(g.a_mn, g.b_mn, tm, p, grid, stream); break;
      default:  rc = dispatch_major<64, false>(g.a_mn, g.b_mn, tm, p, grid, stream); break;
    }
  }
  if (rc) return rc;
  if (p.splits > 1) {
    // residual == C means "accumulate into C" (gradient accumulation); any other residual is not supported here
    SK_REQUIRE(g.residual == nullptr || g.residual == g.C, "gemm: split-K supports only in-place accumulation");
    const long n8 = (long)g.M * g.N / 8;
    int blocks = (int)((n8 + 255) / 256);
    if (blocks > sk_num_sms() * 8) blocks = sk_num_sms() * 8;
    sk_prof_begin(0, stream);
    SK_CUDA_CHECK(sk_launch_pdl(splitk_reduce_kernel, dim3(blocks), dim3(256), (size_t)(0), stream, p.splitk_ws, reinterpret_cast<bf16*>(g.C), g.M, g.N, g.ldc, p.splits,
                                                     g.residual != nullptr, g.round_before_res));
    sk_prof_end(stream);
    SK_LAUNCH_CHECK();
  }
  return 0;
}
