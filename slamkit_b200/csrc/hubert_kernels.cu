// HBM-bound kernels of the HuBERT unit-extraction path (path (i), SURVEY.md §8 a-1..a-6):
//   conv0 + GroupNorm(over time) + GELU front (two passes, the 12.6 GB fp32 intermediate of the reference is never
//   materialised), LayerNorm (+ residual add), channel regrouping for the positional conv, fp32 -> bf16 hi/lo
//   splitting, k-means argmin (first-min tie-break like sklearn) and run-length dedup.
//
// Activation format.  The reference computes this path in fp32 and the unit ids must match it, so bf16 tensor-core
// GEMMs are fed "split" operands: every activation x is stored as two bf16 tensors (hi = bf16(x), lo = bf16(x - hi));
// a GEMM then accumulates hi*hi + hi*lo + lo*hi in fp32 (error ~2^-16 per product instead of 2^-8).  Element-wise
// kernels here read hi+lo, compute in fp32, and write hi/lo again.
#include "kernels.h"
#include <algorithm>
#include <stdlib.h>

namespace {

SK_DEVINL float gelu_erf(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f)); }
// Branch-free GELU(erf) for the conv0 front, where it runs on 3.1e9 elements per batch and the kernel is bound by
// instruction issue, not by HBM.  erf from Abramowitz-Stegun 7.1.26
// (|error| <= 1.5e-7 absolute, below the 2^-17 relative quantisation of the hi/lo output it feeds), folded into the GELU:
//   gelu(y) = y/2 (1 + erf(y/sqrt2)),  erf|z| = 1 - P(t) exp(-z^2),  t = 1/(1 + p|z|)
//           = relu(y) - |y| * (P(t)/2) * exp(-y^2/2)
// -> 2 MUFU + 10 FMA-pipe + 1 ALU instruction, no sign fix-up, no separate 0.5x(1+erf) tail.
SK_DEVINL float gelu_fast(float y) {
  const float a = fabsf(y);
  float t;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(fmaf(0.3275911f * 0.70710678118654752440f, a, 1.0f)));
  float s = fmaf(0.5f * 1.061405429f, t, 0.5f * -1.453152027f);
  s = fmaf(s, t, 0.5f * 1.421413741f);
  s = fmaf(s, t, 0.5f * -0.284496736f);
  s = fmaf(s, t, 0.5f * 0.254829592f);
  const float e = ex2_approx((y * y) * -0.72134752044448170368f);   // exp(-y^2/2)
  const float q = (s * t) * e;
  return fmaf(-a, q, fmaxf(y, 0.0f));
}
SK_DEVINL void split_store(bf16* hi, bf16* lo, size_t idx, float v) {
  const bf16 h = __float2bfloat16_rn(v);
  hi[idx] = h;
  lo[idx] = __float2bfloat16_rn(v - __bfloat162float(h));
}
SK_DEVINL void split8(const float (&v)[8], uint4& hi, uint4& lo) {
  uint32_t h[4], l[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    // one packed convert for the hi pair, two integer ops to widen it back, one packed convert for the lo pair
    h[k] = pack_bf16(v[2 * k], v[2 * k + 1]);
    const float h0 = __uint_as_float(h[k] << 16), h1 = __uint_as_float(h[k] & 0xffff0000u);
    l[k] = pack_bf16(v[2 * k] - h0, v[2 * k + 1] - h1);
  }
  hi = make_uint4(h[0], h[1], h[2], h[3]);
  lo = make_uint4(l[0], l[1], l[2], l[3]);
}
SK_DEVINL void load8_hilo(const bf16* hi, const bf16* lo, size_t idx, float (&v)[8]) {
  const uint4 a = ldg128_stream(hi + idx);
  const uint32_t au[4] = {a.x, a.y, a.z, a.w};
  if (lo) {
    const uint4 b = ldg128_stream(lo + idx);
    const uint32_t bu[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float2 x = unpack_bf16(au[k]), y = unpack_bf16(bu[k]);
      v[2 * k] = x.x + y.x;
      v[2 * k + 1] = x.y + y.y;
    }
  } else {
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float2 x = unpack_bf16(au[k]);
      v[2 * k] = x.x;
      v[2 * k + 1] = x.y;
    }
  }
}

// ------------------------------------------------------------------------------------------------
// fp32 -> (hi, lo) bf16 split (weights at bind time)
// ------------------------------------------------------------------------------------------------
__global__ void split_f32_kernel(const float* __restrict__ x, bf16* __restrict__ hi, bf16* __restrict__ lo, long n) {
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x)
    split_store(hi, lo, i, x[i]);
}

// ------------------------------------------------------------------------------------------------
// conv0 (1 -> C channels, kernel KW, stride ST, no bias) + GroupNorm(C groups) over time + GELU.
// Pass 1: because the input has ONE channel, the per-(clip, channel) mean and second moment of the conv output are
// bilinear forms in the KW window sums  S[j] = sum_t x[ST t + j]  and  R[j][j'] = sum_t x[ST t + j] x[ST t + j']:
//   sum_t y_c = sum_j w_cj S_j ,  sum_t y_c^2 = sum_jj' w_cj w_cj' R_jj'.
// So the statistics pass reads the waveform once and never touches the C x T output.  Accumulated in fp64.
// Each stats block writes its partial sums to its own slot and the affine kernel adds the slots in block order, so the
// GroupNorm affine -- and every feature after it -- is bit-reproducible.  The block partition depends on T0 only (not on
// B or on the launch), so a clip gets the same statistics alone and inside any batch.
// The (pad,pad) zero padding of the reference (F.pad(wav,(40,40))) is applied by index arithmetic.
// ------------------------------------------------------------------------------------------------
constexpr int KW_MAX = 10;
constexpr int NSTAT = KW_MAX + KW_MAX * (KW_MAX + 1) / 2;  // 65
constexpr int STAT_BLOCKS_MAX = 64;                         // stats blocks (partial slots) per clip

inline int conv0_stat_blocks(int T0) { return std::max(1, std::min(STAT_BLOCKS_MAX, (T0 + 255) / 256)); }

SK_DEVINL float wav_at(const float* __restrict__ w, long i, int S, int pad) {
  const long j = i - pad;
  return (j >= 0 && j < S) ? w[j] : 0.f;
}

__global__ void __launch_bounds__(256)
conv0_stats_kernel(const float* __restrict__ wav, double* __restrict__ stats /*[B][STAT_BLOCKS_MAX][NSTAT]*/, int S,
                   int pad, int T0, int KW, int ST) {
  __shared__ double sred[8][NSTAT];
  const int b = blockIdx.y;
  const float* w = wav + (size_t)b * S;
  double acc[NSTAT];
#pragma unroll
  for (int i = 0; i < NSTAT; ++i) acc[i] = 0.0;
  for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < T0; t += gridDim.x * blockDim.x) {
    float x[KW_MAX];
#pragma unroll
    for (int j = 0; j < KW_MAX; ++j) x[j] = j < KW ? wav_at(w, (long)ST * t + j, S, pad) : 0.f;
    int q = KW_MAX;
#pragma unroll
    for (int j = 0; j < KW_MAX; ++j) {
      acc[j] += (double)x[j];
#pragma unroll
      for (int j2 = j; j2 < KW_MAX; ++j2) acc[q++] += (double)x[j] * (double)x[j2];
    }
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
  for (int i = 0; i < NSTAT; ++i) {
    double v = acc[i];
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (lane == 0) sred[warp][i] = v;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < NSTAT; i += blockDim.x) {
    double v = 0.0;
    for (int wi = 0; wi < 8; ++wi) v += sred[wi][i];
    stats[((size_t)b * STAT_BLOCKS_MAX + blockIdx.x) * NSTAT + i] = v;
  }
}

// per (clip, channel): scale = gamma * rstd, shift = beta - mean * gamma * rstd.  The block first adds the n_blk
// partial slots of its clip in slot order (fixed order: deterministic), then each thread forms its channel's affine.
__global__ void conv0_affine_kernel(const double* __restrict__ stats, const float* __restrict__ w /*[C][KW]*/,
                                    const float* __restrict__ gamma, const float* __restrict__ beta,
                                    float2* __restrict__ affine /*[B][C]*/, int C, int KW, int T0, int n_blk, float eps) {
  __shared__ double st[NSTAT];
  const int b = blockIdx.y;
  for (int i = threadIdx.x; i < NSTAT; i += blockDim.x) {
    const double* sp = stats + (size_t)b * STAT_BLOCKS_MAX * NSTAT + i;
    double v = 0.0;
    for (int k = 0; k < n_blk; ++k) v += sp[(size_t)k * NSTAT];
    st[i] = v;
  }
  __syncthreads();
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  double m = 0.0, e2 = 0.0;
  int q = KW_MAX;
  for (int j = 0; j < KW_MAX; ++j) {
    const double wj = j < KW ? (double)w[c * KW + j] : 0.0;
    m += wj * st[j];
    for (int j2 = j; j2 < KW_MAX; ++j2) {
      const double wj2 = j2 < KW ? (double)w[c * KW + j2] : 0.0;
      e2 += (j2 == j ? 1.0 : 2.0) * wj * wj2 * st[q++];
    }
  }
  m /= (double)T0;
  e2 /= (double)T0;
  const double var = e2 - m * m;
  const double rstd = 1.0 / sqrt((var > 0.0 ? var : 0.0) + (double)eps);
  const double sc = (double)gamma[c] * rstd;
  affine[(size_t)b * C + c] = make_float2((float)sc, (float)((double)beta[c] - m * sc));
}

// gelu_fast on NP packed pairs, written stage by stage so that the NP dependency chains (rcp -> 4 FMAs -> 2 muls ->
// FMA, with a parallel mul -> mul -> ex2) interleave in the instruction stream: 10 packed FMA-pipe instructions, 4 MUFU,
// 4 ALU per pair.  na = -|y| comes from OR-ing the sign bit, so t = 1 + p|y| = fma(-p, na, 1) and the tail is
// fma(na, q, relu(y)).
template <int NP>
SK_DEVINL void gelu_fast_pairs(f32x2 (&y)[NP]) {
  f32x2 na[NP], t[NP], e[NP], s[NP], r[NP];
#pragma unroll
  for (int i = 0; i < NP; ++i) {
    float y0, y1;
    upk2(y[i], y0, y1);
    na[i] = pk2(__uint_as_float(__float_as_uint(y0) | 0x80000000u), __uint_as_float(__float_as_uint(y1) | 0x80000000u));
    r[i] = pk2(fmaxf(y0, 0.0f), fmaxf(y1, 0.0f));
  }
#pragma unroll
  for (int i = 0; i < NP; ++i) t[i] = fma2(dup2(-0.3275911f * 0.70710678118654752440f), na[i], dup2(1.0f));
#pragma unroll
  for (int i = 0; i < NP; ++i) e[i] = mul2(mul2(y[i], y[i]), dup2(-0.72134752044448170368f));
#pragma unroll
  for (int i = 0; i < NP; ++i) {
    float a0, a1;
    upk2(t[i], a0, a1);
    asm volatile("rcp.approx.ftz.f32 %0, %1;" : "=f"(a0) : "f"(a0));
    asm volatile("rcp.approx.ftz.f32 %0, %1;" : "=f"(a1) : "f"(a1));
    t[i] = pk2(a0, a1);
  }
#pragma unroll
  for (int i = 0; i < NP; ++i) {
    float a0, a1;
    upk2(e[i], a0, a1);
    asm volatile("ex2.approx.ftz.f32 %0, %1;" : "=f"(a0) : "f"(a0));
    asm volatile("ex2.approx.ftz.f32 %0, %1;" : "=f"(a1) : "f"(a1));
    e[i] = pk2(a0, a1);
  }
#pragma unroll
  for (int i = 0; i < NP; ++i) s[i] = fma2(dup2(0.5f * 1.061405429f), t[i], dup2(0.5f * -1.453152027f));
#pragma unroll
  for (int i = 0; i < NP; ++i) s[i] = fma2(s[i], t[i], dup2(0.5f * 1.421413741f));
#pragma unroll
  for (int i = 0; i < NP; ++i) s[i] = fma2(s[i], t[i], dup2(0.5f * -0.284496736f));
#pragma unroll
  for (int i = 0; i < NP; ++i) s[i] = fma2(s[i], t[i], dup2(0.5f * 0.254829592f));
#pragma unroll
  for (int i = 0; i < NP; ++i) e[i] = mul2(e[i], t[i]);
#pragma unroll
  for (int i = 0; i < NP; ++i) s[i] = mul2(s[i], e[i]);
#pragma unroll
  for (int i = 0; i < NP; ++i) y[i] = fma2(na[i], s[i], r[i]);
}

// Pass 2 (generic geometry): out[b, t, c] = GELU(conv(x)[c,t] * scale + shift), channels-last, hi/lo bf16.  A thread
// owns CPT fixed channels (their CPT x KW taps, pre-multiplied by the GroupNorm scale, live in registers for the whole
// kernel; the shift seeds the accumulator) and walks over frames; a warp covers 32*CPT consecutive channels of one
// frame (coalesced 16-byte stores per thread).  No shared memory.  F2 = true pairs adjacent channels in packed fp32
// registers so the 10 taps issue as 5 FFMA2 per channel pair (same fp32 FMA chain per channel, half the issue slots).
// HuBERT's own front (kernel 10, stride 5) takes conv0_apply_k10s5_kernel below instead.
template <int CPT, bool F2>
__global__ void __launch_bounds__(256, 2)
conv0_apply_kernel(const float* __restrict__ wav, const float* __restrict__ w, const float2* __restrict__ affine,
                   bf16* __restrict__ out_hi, bf16* __restrict__ out_lo, int S, int pad, int T0, int C, int KW, int ST) {
  static_assert(CPT == 8, "conv0_apply: 8 channels per thread");
  const int b = blockIdx.y;
  const int groups = C / CPT;                     // channel groups per frame
  const int lanes_t = blockDim.x / groups > 0 ? blockDim.x / groups : 1;   // frames processed concurrently by a block
  const int cg = threadIdx.x % groups;
  const int tf = threadIdx.x / groups;
  if (tf >= lanes_t) return;
  // GroupNorm's per-(clip, channel) scale is folded into the taps, its shift seeds the accumulator
  float wr[F2 ? 1 : CPT][KW_MAX];
  f32x2 wr2[F2 ? CPT / 2 : 1][KW_MAX];
  float sh[CPT];
#pragma unroll
  for (int k = 0; k < CPT; ++k) sh[k] = affine[(size_t)b * C + cg * CPT + k].y;
  if (F2) {
#pragma unroll
    for (int k = 0; k < CPT / 2; ++k) {
      const float a0 = affine[(size_t)b * C + cg * CPT + 2 * k].x, a1 = affine[(size_t)b * C + cg * CPT + 2 * k + 1].x;
#pragma unroll
      for (int j = 0; j < KW_MAX; ++j)
        wr2[k][j] = pk2(j < KW ? __ldg(w + (cg * CPT + 2 * k) * KW + j) * a0 : 0.f,
                        j < KW ? __ldg(w + (cg * CPT + 2 * k + 1) * KW + j) * a1 : 0.f);
    }
  } else {
#pragma unroll
    for (int k = 0; k < CPT; ++k) {
      const float ax = affine[(size_t)b * C + cg * CPT + k].x;
#pragma unroll
      for (int j = 0; j < KW_MAX; ++j) wr[k][j] = j < KW ? __ldg(w + (cg * CPT + k) * KW + j) * ax : 0.f;
    }
  }
  const float* wv = wav + (size_t)b * S;
  auto load_x = [&](int t, float (&x)[KW_MAX]) {
    const long i0 = (long)ST * t - pad;          // first waveform sample of this frame (before the (pad,pad) padding)
    if (i0 >= 0 && i0 + KW_MAX <= S) {           // interior frame: no bounds checks
#pragma unroll
      for (int j = 0; j < KW_MAX; ++j) x[j] = __ldg(wv + i0 + j);
    } else {
#pragma unroll
      for (int j = 0; j < KW_MAX; ++j) x[j] = j < KW ? wav_at(wv, (long)ST * t + j, S, pad) : 0.f;
    }
  };
  const int t_step = gridDim.x * lanes_t;
  int t = blockIdx.x * lanes_t + tf;
  float xn[KW_MAX];
  if (t < T0) load_x(t, xn);
  for (; t < T0; t += t_step) {
    float x[KW_MAX];
#pragma unroll
    for (int j = 0; j < KW_MAX; ++j) x[j] = xn[j];
    if (t + t_step < T0) load_x(t + t_step, xn);   // prefetch the next frame's window: hides the global-load latency
    float v[CPT];
    if (F2) {
      f32x2 y2[CPT / 2];
#pragma unroll
      for (int k = 0; k < CPT / 2; ++k) y2[k] = pk2(sh[2 * k], sh[2 * k + 1]);
#pragma unroll
      for (int j = 0; j < KW_MAX; ++j) {
        const f32x2 xp = pk2(x[j], x[j]);
#pragma unroll
        for (int k = 0; k < CPT / 2; ++k) y2[k] = fma2(wr2[k][j], xp, y2[k]);
      }
#pragma unroll
      for (int k = 0; k < CPT / 2; ++k) {
        float y0, y1;
        upk2(y2[k], y0, y1);
        v[2 * k] = gelu_fast(y0);
        v[2 * k + 1] = gelu_fast(y1);
      }
    } else {
#pragma unroll
      for (int k = 0; k < CPT; ++k) {
        float y = sh[k];
#pragma unroll
        for (int j = 0; j < KW_MAX; ++j) y = fmaf(wr[k][j], x[j], y);
        v[k] = gelu_fast(y);
      }
    }
    const size_t idx = ((size_t)b * T0 + t) * C + cg * CPT;
    uint4 hi, lo;
    split8(v, hi, lo);
    stg128(out_hi + idx, hi);
    stg128(out_lo + idx, lo);
  }
}

// Fast path for the HuBERT geometry (kernel 10, stride 5).
//  * A thread owns 4 channels (2 packed pairs: 40 tap registers) and computes them for TWO consecutive frames per
//    iteration; the frames' windows overlap, so 15 samples feed both (8 outputs per thread-iteration).
//  * The waveform is staged through shared memory in chunks of CONV0_PCH frame pairs (coalesced loads, next chunk
//    fetched into registers while the current one is computed).  With per-iteration global loads the loop was bound by
//    the loaded HBM read latency (one load -> use dependency per iteration) no matter how the arithmetic was arranged.
//  * GELU runs on packed pairs, stage by stage (gelu_fast_pairs), so the four dependency chains interleave and the
//    FMA-pipe instruction count of the activation halves.
constexpr int CONV0_PCH = 256;                       // frame pairs per chunk
constexpr int CONV0_NS = 10 * CONV0_PCH + 8;         // samples per chunk (15 for the last pair, read as 8 float2; even)
constexpr int CONV0_NLD = (CONV0_NS + 255) / 256;    // staged loads per thread per chunk
__global__ void __launch_bounds__(256, 2)
conv0_apply_k10s5_kernel(const float* __restrict__ wav, const float* __restrict__ w, const float2* __restrict__ affine,
                         bf16* __restrict__ out_hi, bf16* __restrict__ out_lo, int S, int pad, int T0, int C) {
  constexpr int KW = 10, ST = 5, NX = 16, CPT = 4;
  __shared__ __align__(16) float sx[2][CONV0_NS];
  const int b = blockIdx.y;
  const int groups = C / CPT;                                             // channel groups per frame
  const int rows = blockDim.x / groups > 0 ? blockDim.x / groups : 1;     // frame pairs a block works on concurrently
  const int cg = threadIdx.x % groups;
  const int tr = threadIdx.x / groups;
  const bool active = tr < rows;
  f32x2 wr2[CPT / 2][KW];
  f32x2 sh2[CPT / 2];
#pragma unroll
  for (int k = 0; k < CPT / 2; ++k) {
    const float2 a0 = affine[(size_t)b * C + cg * CPT + 2 * k], a1 = affine[(size_t)b * C + cg * CPT + 2 * k + 1];
    sh2[k] = pk2(a0.y, a1.y);
#pragma unroll
    for (int j = 0; j < KW; ++j)
      wr2[k][j] = pk2(__ldg(w + (cg * CPT + 2 * k) * KW + j) * a0.x, __ldg(w + (cg * CPT + 2 * k + 1) * KW + j) * a1.x);
  }
  const float* wv = wav + (size_t)b * S;
  const int n_pairs = (T0 + 1) / 2;
  const int n_chunks = (n_pairs + CONV0_PCH - 1) / CONV0_PCH;
  float stage[CONV0_NLD];
  auto fetch = [&](int chunk) {      // samples [10 * PCH * chunk - pad, +NS) of the clip, zero outside [0, S)
    const long base = (long)2 * ST * CONV0_PCH * chunk - pad;
#pragma unroll
    for (int i = 0; i < CONV0_NLD; ++i) {
      const long g = base + threadIdx.x + 256 * i;
      stage[i] = (g >= 0 && g < S) ? __ldg(wv + g) : 0.f;
    }
  };
  auto commit = [&](int buf) {
#pragma unroll
    for (int i = 0; i < CONV0_NLD; ++i) {
      const int o = threadIdx.x + 256 * i;
      if (o < CONV0_NS) sx[buf][o] = stage[i];
    }
  };
  int chunk = blockIdx.x;
  int cur = 0;
  if (chunk < n_chunks) {
    fetch(chunk);
    commit(0);
  }
  __syncthreads();
  for (; chunk < n_chunks; chunk += gridDim.x) {
    const bool more = chunk + (int)gridDim.x < n_chunks;
    if (more) fetch(chunk + gridDim.x);            // in flight while this chunk is computed
    if (active) {
      const int p_end = min(CONV0_PCH, n_pairs - chunk * CONV0_PCH);
      // running output pointers (frame 2*pr of this row; the odd frame is C elements further)
      size_t idx = ((size_t)b * T0 + 2 * ((size_t)chunk * CONV0_PCH + tr)) * C + cg * CPT;
      const size_t idx_step = (size_t)2 * rows * C;
      for (int pp = tr; pp < p_end; pp += rows, idx += idx_step) {
        float x[NX];
        const float2* sp = reinterpret_cast<const float2*>(&sx[cur][2 * ST * pp]);   // 40 * pp bytes: 8-byte aligned
#pragma unroll
        for (int j = 0; j < NX / 2; ++j) {
          const float2 t2 = sp[j];
          x[2 * j] = t2.x;
          x[2 * j + 1] = t2.y;
        }
        f32x2 y2[2][CPT / 2];
#pragma unroll
        for (int f = 0; f < 2; ++f)
#pragma unroll
          for (int k = 0; k < CPT / 2; ++k) y2[f][k] = sh2[k];
#pragma unroll
        for (int j = 0; j < KW; ++j) {
#pragma unroll
          for (int f = 0; f < 2; ++f) {
            const f32x2 xp = pk2(x[ST * f + j], x[ST * f + j]);
#pragma unroll
            for (int k = 0; k < CPT / 2; ++k) y2[f][k] = fma2(wr2[k][j], xp, y2[f][k]);
          }
        }
        f32x2 gp[CPT];                    // 2 frames x 2 channel pairs
#pragma unroll
        for (int f = 0; f < 2; ++f)
#pragma unroll
          for (int k = 0; k < CPT / 2; ++k) gp[f * (CPT / 2) + k] = y2[f][k];
        gelu_fast_pairs<CPT>(gp);
        const int pr = chunk * CONV0_PCH + pp;
#pragma unroll
        for (int f = 0; f < 2; ++f) {
          const int t = 2 * pr + f;
          if (t < T0) {
            uint32_t h[2], l[2];
#pragma unroll
            for (int k = 0; k < 2; ++k) {
              float g0, g1, l0, l1;
              upk2(gp[f * 2 + k], g0, g1);
              h[k] = pack_bf16(g0, g1);
              upk2(sub2(gp[f * 2 + k], pk2(__uint_as_float(h[k] << 16), __uint_as_float(h[k] & 0xffff0000u))), l0, l1);
              l[k] = pack_bf16(l0, l1);
            }
            // streaming stores: 12.6 GB per batch must not push the waveform (and the next layer's weights) out of L2
            __stcs(reinterpret_cast<uint2*>(out_hi + idx + (size_t)f * C), make_uint2(h[0], h[1]));
            __stcs(reinterpret_cast<uint2*>(out_lo + idx + (size_t)f * C), make_uint2(l[0], l[1]));
          }
        }
      }
    }
    if (more) commit(cur ^ 1);
    __syncthreads();
    cur ^= 1;
  }
}

// ------------------------------------------------------------------------------------------------
// LayerNorm over the last dim (biased variance, eps inside sqrt; torch.nn.LayerNorm), input = (a_hi+a_lo) [+ (b_hi+b_lo)],
// fp32 gamma/beta, output hi/lo (+ optional fp32 copy for k-means).  One warp per row, D <= 1024.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
layernorm_hilo_kernel(const bf16* __restrict__ a_hi, const bf16* __restrict__ a_lo, const bf16* __restrict__ b_hi,
                      const bf16* __restrict__ b_lo, const float* __restrict__ gamma, const float* __restrict__ beta,
                      bf16* __restrict__ o_hi, bf16* __restrict__ o_lo, float* __restrict__ o_f32, int M, int D,
                      float eps) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int row = blockIdx.x * 8 + warp;
  if (row >= M) return;
  const int nvec = D / 8;
  float v[4][8];
  float sum = 0.f;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int c = lane + 32 * j;
    if (c < nvec) {
      const size_t idx = (size_t)row * D + c * 8;
      load8_hilo(a_hi, a_lo, idx, v[j]);
      if (b_hi) {
        float u[8];
        load8_hilo(b_hi, b_lo, idx, u);
#pragma unroll
        for (int k = 0; k < 8; ++k) v[j][k] += u[k];
      }
#pragma unroll
      for (int k = 0; k < 8; ++k) sum += v[j][k];
    }
  }
  const float mean = warp_sum(sum) / (float)D;
  float sq = 0.f;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int c = lane + 32 * j;
    if (c < nvec) {
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const float d = v[j][k] - mean;
        sq += d * d;
      }
    }
  }
  const float rstd = rsqrtf(warp_sum(sq) / (float)D + eps);
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int c = lane + 32 * j;
    if (c < nvec) {
      float o[8];
      const float4 g0 = *reinterpret_cast<const float4*>(gamma + c * 8), g1 = *reinterpret_cast<const float4*>(gamma + c * 8 + 4);
      const float4 b0 = *reinterpret_cast<const float4*>(beta + c * 8), b1 = *reinterpret_cast<const float4*>(beta + c * 8 + 4);
      const float gg[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
      const float bb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
      for (int k = 0; k < 8; ++k) o[k] = (v[j][k] - mean) * rstd * gg[k] + bb[k];
      const size_t idx = (size_t)row * D + c * 8;
      uint4 hi, lo;
      split8(o, hi, lo);
      stg128(o_hi + idx, hi);
      stg128(o_lo + idx, lo);
      if (o_f32) {
        *reinterpret_cast<float4*>(o_f32 + idx) = make_float4(o[0], o[1], o[2], o[3]);
        *reinterpret_cast<float4*>(o_f32 + idx + 4) = make_float4(o[4], o[5], o[6], o[7]);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Positional-conv input staging: [B*T, G*cg] -> [B, T + 2*halo, G*cgp] with zero halo rows and zero pad channels
// (cg = 48 channels per group padded to cgp = 64 so that every k-block of the grouped conv is one 128-byte TMA row).
// ------------------------------------------------------------------------------------------------
__global__ void regroup_pad_kernel(const bf16* __restrict__ in_hi, const bf16* __restrict__ in_lo,
                                   bf16* __restrict__ out_hi, bf16* __restrict__ out_lo, int B, int T, int halo, int G,
                                   int cg, int cgp) {
  const int Tp = T + 2 * halo;
  const int vec_per_row = G * cgp / 8;
  const long total = (long)B * Tp * vec_per_row;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int v = (int)(i % vec_per_row);
    const long r = i / vec_per_row;
    const int tp = (int)(r % Tp);
    const int b = (int)(r / Tp);
    const int g = (v * 8) / cgp, ci = (v * 8) % cgp;
    const int t = tp - halo;
    uint4 hi = make_uint4(0, 0, 0, 0), lo = hi;
    if (t >= 0 && t < T && ci < cg) {
      const size_t src = ((size_t)b * T + t) * (G * cg) + g * cg + ci;
      hi = ldg128_stream(in_hi + src);
      lo = ldg128_stream(in_lo + src);
    }
    const size_t dst = ((size_t)b * Tp + tp) * (G * cgp) + v * 8;
    stg128(out_hi + dst, hi);
    stg128(out_lo + dst, lo);
  }
}

// ------------------------------------------------------------------------------------------------
// k-means labels: label[m] = argmin_j (csq[j] - 2 * dot[m][j]), first minimum wins (SK:_k_means_lloyd.pyx:198-213).
// dot: fp32 [M, ld] from the split GEMM; one warp per row.  Every lane starts at label 0, as sklearn's loop does: a row
// with no distance below +inf (NaN features from non-finite audio) gets label 0, never an id outside [0, U).
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
kmeans_argmin_kernel(const float* __restrict__ dot, const float* __restrict__ csq, int32_t* __restrict__ labels, int M,
                     int U, int ld) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int row = blockIdx.x * 8 + warp;
  if (row >= M) return;
  float best = INFINITY;
  int bi = 0;
  for (int j = lane; j < U; j += 32) {
    const float d = csq[j] + (-2.0f) * dot[(size_t)row * ld + j];
    if (d < best) { best = d; bi = j; }   // ascending j per lane: strict '<' keeps the first minimum
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ob = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ob < best || (ob == best && oi < bi)) { best = ob; bi = oi; }
  }
  if (lane == 0) labels[row] = bi;
}

__global__ void row_sqnorm_kernel(const float* __restrict__ c, float* __restrict__ out, int U, int D) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= U) return;
  float s = 0.f;
  for (int i = lane; i < D; i += 32) s += c[(size_t)warp * D + i] * c[(size_t)warp * D + i];
  s = warp_sum(s);
  if (lane == 0) out[warp] = s;
}

// ------------------------------------------------------------------------------------------------
// Run-length dedup of each row's first n_frames[b] labels (itertools.groupby in UnitTokeniser.audio_represent,
// slamkit/tokeniser/unit_tokeniser.py:57): units / durations / count per row.  One warp per row, ballot scan.
// ------------------------------------------------------------------------------------------------
__global__ void rle_kernel(const int32_t* __restrict__ labels, const int32_t* __restrict__ n_frames,
                           int32_t* __restrict__ units, int32_t* __restrict__ durations, int32_t* __restrict__ counts,
                           int B, int T) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= B) return;
  const int32_t* row = labels + (size_t)warp * T;
  const int n = min(n_frames ? n_frames[warp] : T, T);
  int n_runs = 0;
  for (int base = 0; base < n; base += 32) {
    const int i = base + lane;
    const bool in = i < n;
    const int cur = in ? row[i] : -1;
    const bool head = in && (i == 0 || row[i - 1] != cur);
    const unsigned m = __ballot_sync(0xffffffffu, head);
    if (head) {
      const int slot = n_runs + __popc(m & ((1u << lane) - 1));
      units[(size_t)warp * T + slot] = cur;
      durations[(size_t)warp * T + slot] = i;   // start index for now
    }
    n_runs += __popc(m);
  }
  __syncwarp();
  // convert start indices to run lengths back-to-front within each 32-chunk to avoid read-after-write hazards
  for (int base = 0; base < n_runs; base += 32) {
    const int s = base + lane;
    int start = 0, next = n;
    if (s < n_runs) {
      start = durations[(size_t)warp * T + s];
      next = (s + 1 < n_runs) ? durations[(size_t)warp * T + s + 1] : n;
    }
    __syncwarp();
    if (s < n_runs) durations[(size_t)warp * T + s] = next - start;
    __syncwarp();
  }
  if (lane == 0) counts[warp] = n_runs;
}

// rel_l = ceil(float32(lens)/S * T) as int (hubert_feature_extractor.py:46), lens int64 or NULL (-> T)
__global__ void rel_len_kernel(const int64_t* __restrict__ lens, int32_t* __restrict__ n_frames, int B, int S, int T) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  if (!lens) { n_frames[b] = T; return; }
  const float r = ((float)lens[b] / (float)S) * (float)T;
  int v = (int)ceilf(r);
  n_frames[b] = v < 0 ? 0 : (v > T ? T : v);
}

__global__ void hilo_to_f32_kernel(const bf16* __restrict__ hi, const bf16* __restrict__ lo, float* __restrict__ out, long n) {
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x)
    out[i] = __bfloat162float(hi[i]) + (lo ? __bfloat162float(lo[i]) : 0.f);
}

inline int grid_for(long work_items, int threads, int max_blocks_per_sm = 16) {
  long b = (work_items + threads - 1) / threads;
  const long cap = (long)sk_num_sms() * max_blocks_per_sm;
  if (b > cap) b = cap;
  if (b < 1) b = 1;
  return (int)b;
}

}  // namespace

int sk_split_f32_launch(const float* x, bf16* hi, bf16* lo, long n, cudaStream_t s) {
  split_f32_kernel<<<grid_for(n, 256), 256, 0, s>>>(x, hi, lo, n);
  SK_LAUNCH_CHECK();
  return 0;
}
extern "C" int sk_conv0_nstat(void) { return STAT_BLOCKS_MAX * NSTAT; }
int sk_conv0_launch(const float* wav, const float* w, const float* gamma, const float* beta, double* stats,
                    float2* affine, bf16* out_hi, bf16* out_lo, int B, int S, int pad, int T0, int C, int KW, int ST,
                    float eps, cudaStream_t s) {
  SK_REQUIRE(KW <= KW_MAX, "conv0: kernel width %d > %d", KW, KW_MAX);
  SK_REQUIRE(C % 8 == 0 && C / 4 <= 256, "conv0: channel count must be a multiple of 8 and <= 1024");
  const int n_blk = conv0_stat_blocks(T0);
  conv0_stats_kernel<<<dim3(n_blk, B), 256, 0, s>>>(wav, stats, S, pad, T0, KW, ST);
  SK_LAUNCH_CHECK();
  dim3 g2((C + 127) / 128, B);
  conv0_affine_kernel<<<g2, 128, 0, s>>>(stats, w, gamma, beta, affine, C, KW, T0, n_blk, eps);
  SK_LAUNCH_CHECK();
  static const int mode = [] { const char* e = getenv("SK_CONV0_MODE"); return e ? atoi(e) : 2; }();
  // CUDA-core paths: HuBERT's kernel 10 / stride 5 front with 4 channels x 2 frames per thread; generic kernel otherwise
  const bool fast = mode == 2 && KW == 10 && ST == 5 && C % 4 == 0 && C / 4 <= 256;
  const int fpb = fast ? 2 * CONV0_PCH : std::max(1, 256 / (C / 8));   // frames per block-iteration (fast: per chunk)
  // grid (gx, B): a few CTAs per resident slot, gx chosen so that gx * B fills whole waves of resident CTAs
  static int occ[2] = {0, 0};
  if (occ[fast] == 0) {
    if (fast) SK_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ[1], conv0_apply_k10s5_kernel, 256, 0));
    else      SK_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ[0], conv0_apply_kernel<8, true>, 256, 0));
    if (occ[fast] < 1) occ[fast] = 1;
  }
  const long slots = (long)sk_num_sms() * occ[fast];
  const int gx_max = std::max(1, std::min((T0 + fpb - 1) / fpb, (int)std::max(1L, slots * 8 / B)));
  int gx = gx_max;
  double best = -1.0;
  for (int cand = gx_max; cand >= std::max(1, gx_max / 4); --cand) {
    const long ctas = (long)cand * B;
    const double eff = (double)ctas / (double)(((ctas + slots - 1) / slots) * slots);
    if (eff > best + 1e-9) { best = eff; gx = cand; }
  }
  sk_prof_begin(3, s);
  if (fast) conv0_apply_k10s5_kernel<<<dim3(gx, B), 256, 0, s>>>(wav, w, affine, out_hi, out_lo, S, pad, T0, C);
  else if (mode == 1) conv0_apply_kernel<8, true><<<dim3(gx, B), 256, 0, s>>>(wav, w, affine, out_hi, out_lo, S, pad, T0, C, KW, ST);
  else conv0_apply_kernel<8, false><<<dim3(gx, B), 256, 0, s>>>(wav, w, affine, out_hi, out_lo, S, pad, T0, C, KW, ST);
  sk_prof_end(s);
  SK_LAUNCH_CHECK();
  return 0;
}
int sk_layernorm_hilo_launch(const bf16* a_hi, const bf16* a_lo, const bf16* b_hi, const bf16* b_lo, const float* gamma,
                             const float* beta, bf16* o_hi, bf16* o_lo, float* o_f32, int M, int D, float eps,
                             cudaStream_t s) {
  SK_REQUIRE(D % 8 == 0 && D <= 1024, "layernorm: D must be a multiple of 8 and <= 1024");
  layernorm_hilo_kernel<<<(M + 7) / 8, 256, 0, s>>>(a_hi, a_lo, b_hi, b_lo, gamma, beta, o_hi, o_lo, o_f32, M, D, eps);
  SK_LAUNCH_CHECK();
  return 0;
}
int sk_regroup_pad_launch(const bf16* in_hi, const bf16* in_lo, bf16* out_hi, bf16* out_lo, int B, int T, int halo,
                          int G, int cg, int cgp, cudaStream_t s) {
  SK_REQUIRE(cg % 8 == 0 && cgp % 8 == 0 && cgp >= cg, "regroup: bad group sizes");
  regroup_pad_kernel<<<grid_for((long)B * (T + 2 * halo) * G * cgp / 8, 256), 256, 0, s>>>(in_hi, in_lo, out_hi, out_lo, B,
                                                                                         T, halo, G, cg, cgp);
  SK_LAUNCH_CHECK();
  return 0;
}
int sk_row_sqnorm_launch(const float* c, float* out, int U, int D, cudaStream_t s) {
  row_sqnorm_kernel<<<(U * 32 + 255) / 256, 256, 0, s>>>(c, out, U, D);
  SK_LAUNCH_CHECK();
  return 0;
}
int sk_kmeans_argmin_launch(const float* dot, const float* csq, int32_t* labels, int M, int U, int ld, cudaStream_t s) {
  kmeans_argmin_kernel<<<(M + 7) / 8, 256, 0, s>>>(dot, csq, labels, M, U, ld);
  SK_LAUNCH_CHECK();
  return 0;
}
int sk_rle_launch(const int32_t* labels, const int32_t* n_frames, int32_t* units, int32_t* durations, int32_t* counts,
                  int B, int T, cudaStream_t s) {
  rle_kernel<<<(B * 32 + 127) / 128, 128, 0, s>>>(labels, n_frames, units, durations, counts, B, T);
  SK_LAUNCH_CHECK();
  return 0;
}
int sk_rel_len_launch(const int64_t* lens, int32_t* n_frames, int B, int S, int T, cudaStream_t s) {
  rel_len_kernel<<<(B + 127) / 128, 128, 0, s>>>(lens, n_frames, B, S, T);
  SK_LAUNCH_CHECK();
  return 0;
}
int sk_hilo_to_f32_launch(const bf16* hi, const bf16* lo, float* out, long n, cudaStream_t s) {
  hilo_to_f32_kernel<<<grid_for(n, 256), 256, 0, s>>>(hi, lo, out, n);
  SK_LAUNCH_CHECK();
  return 0;
}
