// HBM-bound kernels of the causal-LM train step (path (ii), SURVEY.md §8 a-8..a-11): embedding gather/scatter,
// RMSNorm fwd/bwd, RoPE fwd/bwd, SwiGLU fwd/bwd, bias-grad column sums, cross-entropy fwd+bwd, gradient-norm
// clipping and fused AdamW.  All use 128-bit coalesced global accesses and warp-shuffle reductions; bf16 storage,
// fp32 math.  Rounding points follow the HF bf16 path so that parity with the reference is tight
// (HF:models/qwen2/modeling_qwen2.py:35-48 MLP, :102-146 RoPE, :249-262 RMSNorm).
#include "kernels.h"

namespace {

constexpr int WARPS_PER_BLOCK = 8;
constexpr int MAX_VEC_PER_LANE = 4;  // supports D <= 4*32*8 = 1024

// ------------------------------------------------------------------------------------------------
// embedding
// ------------------------------------------------------------------------------------------------
__global__ void embed_fwd_kernel(const int64_t* __restrict__ ids, const bf16* __restrict__ E, bf16* __restrict__ out,
                                 int M, int D, int V) {
  const int vec_per_row = D / 8;
  const long total = (long)M * vec_per_row;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int m = (int)(i / vec_per_row);
    const int c = (int)(i % vec_per_row);
    long id = ids[m];
    if (id < 0 || id >= V) id = 0;
    stg128(out + (size_t)m * D + c * 8, ldg128(E + (size_t)id * D + c * 8));
  }
}

// dE_fix[ids[m], :] += dx[m, :] in 64-bit FIXED POINT (2^-40 units): integer addition is associative, so the atomics may
// land in any order and the result is still bit-identical run to run (fp32 atomicAdd is not).  |sum| < 2^23 and terms
// below 2^-41 vanish -- both far outside what a bf16 gradient row can hold.  Vocab is tiny for unit LMs (heavy
// collisions, negligible traffic next to the GEMMs); for text+unit vocabularies the scratch is Vpad x D x 8 bytes.
constexpr float EMBED_FIX_SCALE = 1099511627776.0f;          // 2^40
__global__ void embed_bwd_scatter_kernel(const int64_t* __restrict__ ids, const bf16* __restrict__ dx,
                                         unsigned long long* __restrict__ scratch, int M, int D, int V) {
  const int vec_per_row = D / 8;
  const long total = (long)M * vec_per_row;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int m = (int)(i / vec_per_row);
    const int c = (int)(i % vec_per_row);
    long id = ids[m];
    if (id < 0 || id >= V) continue;
    const uint4 v = ldg128_stream(dx + (size_t)m * D + c * 8);
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
    unsigned long long* dst = scratch + (size_t)id * D + c * 8;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float2 f = unpack_bf16(w[k]);
      if (f.x != 0.f) atomicAdd(dst + 2 * k, (unsigned long long)__float2ll_rn(f.x * EMBED_FIX_SCALE));
      if (f.y != 0.f) atomicAdd(dst + 2 * k + 1, (unsigned long long)__float2ll_rn(f.y * EMBED_FIX_SCALE));
    }
  }
}

// grad[i] = bf16(float(grad[i]) * keep + fix[i] * 2^-40)
__global__ void add_fix_into_bf16_kernel(bf16* __restrict__ grad, const unsigned long long* __restrict__ scratch, long n, int keep) {
  for (long i = (blockIdx.x * (long)blockDim.x + threadIdx.x) * 8; i < n; i += (long)gridDim.x * blockDim.x * 8) {
    float s[8];
#pragma unroll
    for (int k = 0; k < 8; k += 2) {
      const ulonglong2 a = *reinterpret_cast<const ulonglong2*>(scratch + i + k);
      s[k] = (float)((double)(long long)a.x * (1.0 / 1099511627776.0));
      s[k + 1] = (float)((double)(long long)a.y * (1.0 / 1099511627776.0));
    }
    if (keep) {
      const uint4 g = *reinterpret_cast<const uint4*>(grad + i);
      const uint32_t w[4] = {g.x, g.y, g.z, g.w};
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float2 f = unpack_bf16(w[k]);
        s[2 * k] += f.x;
        s[2 * k + 1] += f.y;
      }
    }
    uint4 o;
    o.x = pack_bf16(s[0], s[1]);
    o.y = pack_bf16(s[2], s[3]);
    o.z = pack_bf16(s[4], s[5]);
    o.w = pack_bf16(s[6], s[7]);
    stg128(grad + i, o);
  }
}

// ------------------------------------------------------------------------------------------------
// RMSNorm:  y = w * bf16(x * rsqrt(mean(x^2) + eps))      one warp per row
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(WARPS_PER_BLOCK * 32)
rmsnorm_fwd_kernel(const bf16* __restrict__ x, const bf16* __restrict__ w, bf16* __restrict__ y,
                   float* __restrict__ rstd_out, int M, int D, float eps) {
  griddep_launch();
  griddep_wait();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int row = blockIdx.x * WARPS_PER_BLOCK + warp;
  if (row >= M) return;
  const int nvec = D / 8;
  uint4 xv[MAX_VEC_PER_LANE];
  float ss = 0.f;
#pragma unroll
  for (int j = 0; j < MAX_VEC_PER_LANE; ++j) {
    const int c = lane + 32 * j;
    if (c < nvec) {
      xv[j] = ldg128_stream(x + (size_t)row * D + c * 8);
      const uint32_t u[4] = {xv[j].x, xv[j].y, xv[j].z, xv[j].w};
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float2 f = unpack_bf16(u[k]);
        ss += f.x * f.x + f.y * f.y;
      }
    }
  }
  ss = warp_sum(ss);
  const float rstd = rsqrtf(ss / (float)D + eps);
  if (lane == 0 && rstd_out) rstd_out[row] = rstd;
#pragma unroll
  for (int j = 0; j < MAX_VEC_PER_LANE; ++j) {
    const int c = lane + 32 * j;
    if (c < nvec) {
      const uint4 wv = ldg128(w + c * 8);
      const uint32_t u[4] = {xv[j].x, xv[j].y, xv[j].z, xv[j].w};
      const uint32_t ww[4] = {wv.x, wv.y, wv.z, wv.w};
      uint32_t o[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float2 f = unpack_bf16(u[k]);
        const float2 g = unpack_bf16(ww[k]);
        o[k] = pack_bf16(g.x * bf16_round(f.x * rstd), g.y * bf16_round(f.y * rstd));
      }
      stg128(y + (size_t)row * D + c * 8, make_uint4(o[0], o[1], o[2], o[3]));
    }
  }
}

// backward: g = bf16(dy*w) ; xhat = x*rstd ; dx = rstd*g - rstd^2*mean(g*xhat)*x (+ dres) ; dw partial = sum_rows dy*bf16(xhat)
// grid-stride over rows so every block owns a fixed slice; per-block partial dw rows are written to `dw_partial`
// [gridDim.x, D] and reduced by colsum_reduce_kernel in a fixed order (deterministic).
// All three row operands (x, dy, dres) are requested before anything is consumed, g is formed by one packed bf16
// multiply per pair (HMUL2.BF16: the exact product rounded once, the same value as rounding the fp32 product) and
// kept packed for the second phase.
__global__ void __launch_bounds__(WARPS_PER_BLOCK * 32, 2)
rmsnorm_bwd_kernel(const bf16* __restrict__ dy, const bf16* __restrict__ x, const bf16* __restrict__ w,
                   const float* __restrict__ rstd_in, const bf16* __restrict__ dres, bf16* __restrict__ dx,
                   float* __restrict__ dw_partial, int M, int D) {
  griddep_launch();
  griddep_wait();
  extern __shared__ float sdw[];  // [WARPS_PER_BLOCK][D]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nvec = D / 8;
  float dwacc[MAX_VEC_PER_LANE][8];
#pragma unroll
  for (int j = 0; j < MAX_VEC_PER_LANE; ++j)
#pragma unroll
    for (int k = 0; k < 8; ++k) dwacc[j][k] = 0.f;
  uint4 wv[MAX_VEC_PER_LANE];
#pragma unroll
  for (int j = 0; j < MAX_VEC_PER_LANE; ++j) {
    const int c = lane + 32 * j;
    wv[j] = c < nvec ? ldg128(w + c * 8) : make_uint4(0, 0, 0, 0);
  }
  for (int row = blockIdx.x * WARPS_PER_BLOCK + warp; row < M; row += gridDim.x * WARPS_PER_BLOCK) {
    uint4 xq[MAX_VEC_PER_LANE], gq[MAX_VEC_PER_LANE], rq[MAX_VEC_PER_LANE];   // packed bf16 (gq: dy, then g = dy*w)
#pragma unroll
    for (int j = 0; j < MAX_VEC_PER_LANE; ++j) {
      const int c = lane + 32 * j;
      if (c < nvec) {
        xq[j] = ldg128_stream(x + (size_t)row * D + c * 8);
        gq[j] = ldg128_stream(dy + (size_t)row * D + c * 8);
        rq[j] = dres ? ldg128_stream(dres + (size_t)row * D + c * 8) : make_uint4(0, 0, 0, 0);
      }
    }
    const float rstd = rstd_in[row];
    float dot = 0.f;
#pragma unroll
    for (int j = 0; j < MAX_VEC_PER_LANE; ++j) {
      const int c = lane + 32 * j;
      if (c < nvec) {
        const uint32_t xu[4] = {xq[j].x, xq[j].y, xq[j].z, xq[j].w};
        uint32_t du[4] = {gq[j].x, gq[j].y, gq[j].z, gq[j].w};
        const uint32_t wu[4] = {wv[j].x, wv[j].y, wv[j].z, wv[j].w};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const float2 xf = unpack_bf16(xu[k]);
          const float2 df = unpack_bf16(du[k]);
          const float xh0 = xf.x * rstd, xh1 = xf.y * rstd;
          const float2 xb = unpack_bf16(pack_bf16(xh0, xh1));          // bf16(xhat): what the forward multiplied by w
          dwacc[j][2 * k] = fmaf(df.x, xb.x, dwacc[j][2 * k]);
          dwacc[j][2 * k + 1] = fmaf(df.y, xb.y, dwacc[j][2 * k + 1]);
          bf162 gp = __hmul2(*reinterpret_cast<const bf162*>(&du[k]), *reinterpret_cast<const bf162*>(&wu[k]));
          du[k] = *reinterpret_cast<uint32_t*>(&gp);
          const float2 gf = unpack_bf16(du[k]);
          dot = fmaf(gf.x, xh0, dot);
          dot = fmaf(gf.y, xh1, dot);
        }
        gq[j] = make_uint4(du[0], du[1], du[2], du[3]);
      }
    }
    dot = warp_sum(dot) / (float)D;
    const float c2 = -(rstd * rstd) * dot;
#pragma unroll
    for (int j = 0; j < MAX_VEC_PER_LANE; ++j) {
      const int c = lane + 32 * j;
      if (c < nvec) {
        const uint32_t xu[4] = {xq[j].x, xq[j].y, xq[j].z, xq[j].w};
        const uint32_t gu[4] = {gq[j].x, gq[j].y, gq[j].z, gq[j].w};
        const uint32_t ru[4] = {rq[j].x, rq[j].y, rq[j].z, rq[j].w};
        uint32_t o[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const float2 xf = unpack_bf16(xu[k]);
          const float2 gf = unpack_bf16(gu[k]);
          const float2 rf = unpack_bf16(ru[k]);
          o[k] = pack_bf16(fmaf(c2, xf.x, rstd * gf.x) + rf.x, fmaf(c2, xf.y, rstd * gf.y) + rf.y);
        }
        stg128(dx + (size_t)row * D + c * 8, make_uint4(o[0], o[1], o[2], o[3]));
      }
    }
  }
  // block reduce dw
#pragma unroll
  for (int j = 0; j < MAX_VEC_PER_LANE; ++j) {
    const int c = lane + 32 * j;
    if (c < nvec) {
#pragma unroll
      for (int k = 0; k < 8; ++k) sdw[warp * D + c * 8 + k] = dwacc[j][k];
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < D; i += blockDim.x) {
    float s = 0.f;
#pragma unroll
    for (int wi = 0; wi < WARPS_PER_BLOCK; ++wi) s += sdw[wi * D + i];
    dw_partial[(size_t)blockIdx.x * D + i] = s;
  }
}

SK_DEVINL float to_f32(bf16 v) { return __bfloat162float(v); }
SK_DEVINL float to_f32(float v) { return v; }
SK_DEVINL void store_f32(bf16* p, float v) { *p = __float2bfloat16_rn(v); }
SK_DEVINL void store_f32(float* p, float v) { *p = v; }

// out[j] = OutT( (accumulate ? out[j] : 0) + sum_b partial[b][j] ).  Block = 32 columns x 32 row groups (1024 threads);
// every thread sums a fixed strided subset of rows, then a fixed-order tree over the 32 groups (deterministic).
template <typename OutT>
__global__ void __launch_bounds__(1024)
colsum_reduce_kernel(const float* __restrict__ partial, OutT* __restrict__ out, int nblocks, int D, int accumulate) {
  griddep_launch();
  griddep_wait();
  __shared__ float sred[32][33];
  const int c = threadIdx.x & 31, rg = threadIdx.x >> 5;
  const int j = blockIdx.x * 32 + c;
  float s = 0.f;
  if (j < D)
    for (int b = rg; b < nblocks; b += 32) s += partial[(size_t)b * D + j];
  sred[rg][c] = s;
  __syncthreads();
#pragma unroll
  for (int st = 16; st > 0; st >>= 1) {
    if (rg < st) sred[rg][c] += sred[rg + st][c];
    __syncthreads();
  }
  if (rg == 0 && j < D) {
    float t = sred[0][c];
    if (accumulate) t += to_f32(out[j]);
    store_f32(out + j, t);
  }
}

// column sums of a bf16 [M, N] matrix (leading dim ld) -> partial[gridDim.y][N]; used for the q/k/v bias gradient
__global__ void colsum_partial_kernel(const bf16* __restrict__ x, float* __restrict__ partial, int M, int N, int ld) {
  griddep_launch();
  griddep_wait();
  const int col = (blockIdx.x * blockDim.x + threadIdx.x) * 8;
  if (col >= N) return;
  float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  const int rows_per = (M + gridDim.y - 1) / gridDim.y;
  const int r0 = blockIdx.y * rows_per;
  const int r1 = min(M, r0 + rows_per);
  for (int r = r0; r < r1; ++r) {
    const uint4 v = ldg128_stream(x + (size_t)r * ld + col);
    const uint32_t u[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float2 f = unpack_bf16(u[k]);
      acc[2 * k] += f.x;
      acc[2 * k + 1] += f.y;
    }
  }
#pragma unroll
  for (int k = 0; k < 8; ++k) partial[(size_t)blockIdx.y * N + col + k] = acc[k];
}

// ------------------------------------------------------------------------------------------------
// RoPE (rotate_half form), in place on the q and k head slices of the fused qkv activation [M, ld].
//   out[i]      = bf16(bf16(x[i]*c) + bf16(-x[i+hd/2]*s))
//   out[i+hd/2] = bf16(bf16(x[i+hd/2]*c) + bf16(x[i]*s))          c,s: bf16 tables [maxpos, hd/2]
// inverse=1 applies the transposed rotation (backward).  rot < head_dim (GPT-NeoX partial rotary): only the first rot
// columns of each head rotate, pairing i with i + rot/2, with [maxpos, rot/2] tables; the other columns are untouched.
// ------------------------------------------------------------------------------------------------
__global__ void rope_kernel(bf16* __restrict__ qkv, const bf16* __restrict__ cos_t, const bf16* __restrict__ sin_t,
                            const int* __restrict__ pos_ids, int M, int T, int ld, int n_rot_heads, int head_dim,
                            int inverse, int max_pos, int rot) {
  griddep_launch();
  griddep_wait();
  const int half = rot / 2;               // 32 (full rotary) / 16 / 8
  const int vec_per_head = half / 8;      // 4 / 2 / 1 threads per (token, head)
  const long total = (long)M * n_rot_heads * vec_per_head;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int v = (int)(i % vec_per_head);
    const int h = (int)((i / vec_per_head) % n_rot_heads);
    const int m = (int)(i / ((long)vec_per_head * n_rot_heads));
    int pos = pos_ids ? pos_ids[m] : (m % T);
    pos = max(0, min(pos, max_pos - 1));     // caller-supplied positions never index outside the tables
    bf16* p1 = qkv + (size_t)m * ld + h * head_dim + v * 8;
    bf16* p2 = p1 + half;
    const uint4 a = *reinterpret_cast<const uint4*>(p1);
    const uint4 b = *reinterpret_cast<const uint4*>(p2);
    const uint4 cv = ldg128(cos_t + (size_t)pos * half + v * 8);
    const uint4 sv = ldg128(sin_t + (size_t)pos * half + v * 8);
    const uint32_t au[4] = {a.x, a.y, a.z, a.w}, bu[4] = {b.x, b.y, b.z, b.w};
    const uint32_t cu[4] = {cv.x, cv.y, cv.z, cv.w}, su[4] = {sv.x, sv.y, sv.z, sv.w};
    uint32_t o1[4], o2[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float2 x1 = unpack_bf16(au[k]), x2 = unpack_bf16(bu[k]);
      const float2 c = unpack_bf16(cu[k]);
      float2 s = unpack_bf16(su[k]);
      if (inverse) { s.x = -s.x; s.y = -s.y; }
      o1[k] = pack_bf16(bf16_round(x1.x * c.x) + bf16_round(-x2.x * s.x), bf16_round(x1.y * c.y) + bf16_round(-x2.y * s.y));
      o2[k] = pack_bf16(bf16_round(x2.x * c.x) + bf16_round(x1.x * s.x), bf16_round(x2.y * c.y) + bf16_round(x1.y * s.y));
    }
    *reinterpret_cast<uint4*>(p1) = make_uint4(o1[0], o1[1], o1[2], o1[3]);
    *reinterpret_cast<uint4*>(p2) = make_uint4(o2[0], o2[1], o2[2], o2[3]);
  }
}

// ------------------------------------------------------------------------------------------------
// SwiGLU: gu = [gate | up] (each F wide).  act = bf16(bf16(silu(g)) * u)
// ------------------------------------------------------------------------------------------------
// (sigmoid_f / silu_f: common.cuh)

// two independent 16-byte vectors per thread and iteration (more loads in flight per thread)
__global__ void __launch_bounds__(256)
swiglu_fwd_kernel(const bf16* __restrict__ gu, bf16* __restrict__ act, int M, int F) {
  griddep_launch();
  griddep_wait();
  const int vec_per_row = F / 8;
  const long total = (long)M * vec_per_row;
  const long half = (total + 1) / 2;
  for (long i0 = blockIdx.x * (long)blockDim.x + threadIdx.x; i0 < half; i0 += (long)gridDim.x * blockDim.x) {
    uint4 gv[2], uv[2];
    long idx[2] = {i0, i0 + half};
#pragma unroll
    for (int v = 0; v < 2; ++v) {
      if (idx[v] < total) {
        const int m = (int)(idx[v] / vec_per_row), c = (int)(idx[v] % vec_per_row);
        gv[v] = ldg128_stream(gu + (size_t)m * 2 * F + c * 8);
        uv[v] = ldg128_stream(gu + (size_t)m * 2 * F + F + c * 8);
      }
    }
#pragma unroll
    for (int v = 0; v < 2; ++v) {
      if (idx[v] < total) {
        const int m = (int)(idx[v] / vec_per_row), c = (int)(idx[v] % vec_per_row);
        const uint32_t g[4] = {gv[v].x, gv[v].y, gv[v].z, gv[v].w}, u[4] = {uv[v].x, uv[v].y, uv[v].z, uv[v].w};
        uint32_t o[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const float2 gf = unpack_bf16(g[k]), uf = unpack_bf16(u[k]);
          const float2 sb = unpack_bf16(pack_bf16(silu_f(gf.x), silu_f(gf.y)));   // bf16(silu(g))
          o[k] = pack_bf16(sb.x * uf.x, sb.y * uf.y);
        }
        stg128(act + (size_t)m * F + c * 8, make_uint4(o[0], o[1], o[2], o[3]));
      }
    }
  }
}

// d_gu = [ d_act*u*silu'(g) | d_act*silu(g) ]
__global__ void swiglu_bwd_kernel(const bf16* __restrict__ gu, const bf16* __restrict__ dact, bf16* __restrict__ dgu,
                                  int M, int F) {
  griddep_launch();
  griddep_wait();
  const int vec_per_row = F / 8;
  const long total = (long)M * vec_per_row;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int m = (int)(i / vec_per_row);
    const int c = (int)(i % vec_per_row);
    const uint4 gv = ldg128_stream(gu + (size_t)m * 2 * F + c * 8);
    const uint4 uv = ldg128_stream(gu + (size_t)m * 2 * F + F + c * 8);
    const uint4 dv = ldg128_stream(dact + (size_t)m * F + c * 8);
    const uint32_t g[4] = {gv.x, gv.y, gv.z, gv.w}, u[4] = {uv.x, uv.y, uv.z, uv.w}, d[4] = {dv.x, dv.y, dv.z, dv.w};
    uint32_t og[4], ou[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float2 gf = unpack_bf16(g[k]), uf = unpack_bf16(u[k]), df = unpack_bf16(d[k]);
      const float s0 = sigmoid_f(gf.x), s1 = sigmoid_f(gf.y);
      const float sil0 = bf16_round(gf.x * s0), sil1 = bf16_round(gf.y * s1);
      const float ds0 = s0 * (1.0f + gf.x * (1.0f - s0)), ds1 = s1 * (1.0f + gf.y * (1.0f - s1));
      // d(silu)*u rounded like the bf16 autograd chain: d_silu = bf16(dact*u); dg = bf16(d_silu * silu'(g))
      og[k] = pack_bf16(bf16_round(df.x * uf.x) * ds0, bf16_round(df.y * uf.y) * ds1);
      ou[k] = pack_bf16(df.x * sil0, df.y * sil1);
    }
    stg128(dgu + (size_t)m * 2 * F + c * 8, make_uint4(og[0], og[1], og[2], og[3]));
    stg128(dgu + (size_t)m * 2 * F + F + c * 8, make_uint4(ou[0], ou[1], ou[2], ou[3]));
  }
}

// ------------------------------------------------------------------------------------------------
// Cross entropy over bf16 logits [M, ldl] with V valid columns; shifted labels (row (b,t) predicts labels[b,t+1]).
// Matches slamkit/model/unit_lm.py:13-29: fp32 upcast, ignore_index=-100, reduction sum (then / num_items) or mean.
// One warp per row.  Writes per-block partial {loss_sum, n_valid} and dlogits (bf16, unscaled = softmax - onehot);
// the scale 1/num_items (or 1/n_valid) * dloss is applied by ce_scale_kernel once the count is known when reduction
// is 'mean'; for the 'sum / num_items' path the scale is known up front and applied here.
// ------------------------------------------------------------------------------------------------
constexpr int CE_MAX_VEC = 2;  // up to 512 padded columns per row

__global__ void __launch_bounds__(WARPS_PER_BLOCK * 32)
ce_fwd_bwd_kernel(const bf16* __restrict__ logits, const int64_t* __restrict__ labels, bf16* __restrict__ dlogits,
                  float* __restrict__ partial /*[grid][2]*/, float* __restrict__ row_nll /*[M] or null*/,
                  const float* __restrict__ row_weight /*[M] or null*/, int M, int T, int V, int ldl, float grad_scale) {
  __shared__ float s_loss[WARPS_PER_BLOCK], s_cnt[WARPS_PER_BLOCK];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int row = blockIdx.x * WARPS_PER_BLOCK + warp;
  float my_loss = 0.f, my_cnt = 0.f;
  if (row < M) {
    const int t = row % T;
    long target = -100;
    if (t < T - 1) target = labels[row + 1];
    const bool valid = (target >= 0 && target < V);
    float v[CE_MAX_VEC][8];
    float mx = -INFINITY;
#pragma unroll
    for (int j = 0; j < CE_MAX_VEC; ++j) {
      const int c = (lane + 32 * j) * 8;
      if (c < ldl) {
        const uint4 lv = ldg128_stream(logits + (size_t)row * ldl + c);
        const uint32_t u[4] = {lv.x, lv.y, lv.z, lv.w};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const float2 f = unpack_bf16(u[k]);
          v[j][2 * k] = (c + 2 * k < V) ? f.x : -INFINITY;
          v[j][2 * k + 1] = (c + 2 * k + 1 < V) ? f.y : -INFINITY;
        }
#pragma unroll
        for (int k = 0; k < 8; ++k) mx = fmaxf(mx, v[j][k]);
      } else {
#pragma unroll
        for (int k = 0; k < 8; ++k) v[j][k] = -INFINITY;
      }
    }
    mx = warp_max(mx);
    float se = 0.f, tgt_logit = 0.f;
#pragma unroll
    for (int j = 0; j < CE_MAX_VEC; ++j) {
      const int c = (lane + 32 * j) * 8;
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        se += expf(v[j][k] - mx);
        if (valid && c + k == (int)target) tgt_logit = v[j][k];
      }
    }
    se = warp_sum(se);
    tgt_logit = warp_sum(tgt_logit);
    const float lse = mx + logf(se);
    if (valid) {
      my_loss = lse - tgt_logit;
      my_cnt = 1.f;
    }
    if (row_nll && lane == 0) row_nll[row] = valid ? (lse - tgt_logit) : 0.f;
    if (dlogits) {
      const float inv = 1.0f / se;
      const float gs = row_weight ? grad_scale * row_weight[row] : grad_scale;
#pragma unroll
      for (int j = 0; j < CE_MAX_VEC; ++j) {
        const int c = (lane + 32 * j) * 8;
        if (c < ldl) {
          float o[8];
#pragma unroll
          for (int k = 0; k < 8; ++k) {
            float pr = valid ? expf(v[j][k] - mx) * inv : 0.f;
            if (valid && c + k == (int)target) pr -= 1.f;
            o[k] = pr * gs;
          }
          stg128(dlogits + (size_t)row * ldl + c,
                 make_uint4(pack_bf16(o[0], o[1]), pack_bf16(o[2], o[3]), pack_bf16(o[4], o[5]), pack_bf16(o[6], o[7])));
        }
      }
    }
  }
  if (lane == 0) { s_loss[warp] = my_loss; s_cnt[warp] = my_cnt; }
  __syncthreads();
  if (threadIdx.x == 0) {
    float a = 0.f, b = 0.f;
    for (int i = 0; i < WARPS_PER_BLOCK; ++i) { a += s_loss[i]; b += s_cnt[i]; }
    partial[2 * blockIdx.x] = a;
    partial[2 * blockIdx.x + 1] = b;
  }
}

// Large-vocabulary variant (interleaved text+unit vocabularies, ~152 k columns: SURVEY.md f-1): one block per row, an
// online (max, sum) pass over the row, then a second pass that writes the gradient -- logits are read twice and the
// gradient written once (3 x M x V x 2 B; 7.5 GB at [8192, 152 k]).  Same outputs and rounding as the warp-per-row kernel.
__global__ void __launch_bounds__(256)
ce_large_kernel(const bf16* __restrict__ logits, const int64_t* __restrict__ labels, bf16* __restrict__ dlogits,
                float* __restrict__ partial /*[M][2]*/, float* __restrict__ row_nll, const float* __restrict__ row_weight,
                int M, int T, int V, int ldl, float grad_scale, int row0) {
  // row0 > 0: `logits` / `dlogits` hold a CHUNK of rows starting at global row row0 (chunked lm_head, lm_step.cu);
  // labels, partial, row_nll and row_weight are always indexed by the global row
  __shared__ float s_m[8], s_s[8];
  const int row = row0 + blockIdx.x;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int t = row % T;
  long target = -100;
  if (t < T - 1) target = labels[row + 1];
  const bool valid = (target >= 0 && target < V);
  const bf16* lrow = logits + (size_t)blockIdx.x * ldl;
  const int nvec = ldl / 8;
  float m = -INFINITY, sum = 0.f;
  for (int c = threadIdx.x; c < nvec; c += 256) {
    const uint4 lv = ldg128_stream(lrow + c * 8);
    const uint32_t u[4] = {lv.x, lv.y, lv.z, lv.w};
    float v[8];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float2 f = unpack_bf16(u[k]);
      v[2 * k] = (c * 8 + 2 * k < V) ? f.x : -INFINITY;
      v[2 * k + 1] = (c * 8 + 2 * k + 1 < V) ? f.y : -INFINITY;
    }
    float cm = v[0];
#pragma unroll
    for (int k = 1; k < 8; ++k) cm = fmaxf(cm, v[k]);
    if (cm > -INFINITY) {
      const float mn = fmaxf(m, cm);
      float acc = 0.f;
#pragma unroll
      for (int k = 0; k < 8; ++k) acc += ex2_approx((v[k] - mn) * 1.4426950408889634f);
      sum = sum * ex2_approx((m - mn) * 1.4426950408889634f) + acc;   // m == -inf: sum is 0 and 0 * 0 = 0
      m = mn;
    }
  }
  // combine (m, sum) pairs: warp, then block
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float m2 = __shfl_xor_sync(0xffffffffu, m, o), s2 = __shfl_xor_sync(0xffffffffu, sum, o);
    const float mn = fmaxf(m, m2);
    if (mn > -INFINITY) sum = sum * ex2_approx((m - mn) * 1.4426950408889634f) + s2 * ex2_approx((m2 - mn) * 1.4426950408889634f);
    m = mn;
  }
  if (lane == 0) { s_m[warp] = m; s_s[warp] = sum; }
  __syncthreads();
  m = s_m[0]; sum = s_s[0];
#pragma unroll
  for (int i = 1; i < 8; ++i) {
    const float mn = fmaxf(m, s_m[i]);
    if (mn > -INFINITY) sum = sum * ex2_approx((m - mn) * 1.4426950408889634f) + s_s[i] * ex2_approx((s_m[i] - mn) * 1.4426950408889634f);
    m = mn;
  }
  const float lse = m + logf(sum);
  const float tgt_logit = valid ? __bfloat162float(lrow[target]) : 0.f;
  if (threadIdx.x == 0) {
    partial[2 * row] = valid ? (lse - tgt_logit) : 0.f;
    partial[2 * row + 1] = valid ? 1.f : 0.f;
    if (row_nll) row_nll[row] = valid ? (lse - tgt_logit) : 0.f;
  }
  if (dlogits) {
    const float gs = row_weight ? grad_scale * row_weight[row] : grad_scale;
    const float nlse2 = -lse * 1.4426950408889634f;
    bf16* drow = dlogits + (size_t)blockIdx.x * ldl;
    for (int c = threadIdx.x; c < nvec; c += 256) {
      float o[8];
      if (valid) {
        const uint4 lv = ldg128_stream(lrow + c * 8);
        const uint32_t u[4] = {lv.x, lv.y, lv.z, lv.w};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const float2 f = unpack_bf16(u[k]);
          o[2 * k] = (c * 8 + 2 * k < V) ? ex2_approx(fmaf(f.x, 1.4426950408889634f, nlse2)) : 0.f;
          o[2 * k + 1] = (c * 8 + 2 * k + 1 < V) ? ex2_approx(fmaf(f.y, 1.4426950408889634f, nlse2)) : 0.f;
        }
        const int d = (int)target - c * 8;
#pragma unroll
        for (int k = 0; k < 8; ++k) o[k] = (o[k] - (k == d ? 1.f : 0.f)) * gs;
      } else {
#pragma unroll
        for (int k = 0; k < 8; ++k) o[k] = 0.f;
      }
      stg128(drow + c * 8, make_uint4(pack_bf16(o[0], o[1]), pack_bf16(o[2], o[3]), pack_bf16(o[4], o[5]), pack_bf16(o[6], o[7])));
    }
  }
}

// out[0] = loss (sum/denom), out[1] = n_valid, out[2] = raw nll sum.   denom<=0 -> mean over valid tokens.
__global__ void ce_finalize_kernel(const float* __restrict__ partial, int nblocks, float denom, float* __restrict__ out) {
  __shared__ double sa[256], sb[256];
  double a = 0, b = 0;
  for (int i = threadIdx.x; i < nblocks; i += blockDim.x) { a += partial[2 * i]; b += partial[2 * i + 1]; }
  sa[threadIdx.x] = a; sb[threadIdx.x] = b;
  __syncthreads();
  for (int s = blockDim.x / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s) { sa[threadIdx.x] += sa[threadIdx.x + s]; sb[threadIdx.x] += sb[threadIdx.x + s]; }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    const double d = denom > 0.f ? (double)denom : (sb[0] > 0 ? sb[0] : 1.0);
    out[0] = (float)(sa[0] / d);
    out[1] = (float)sb[0];
    out[2] = (float)sa[0];
  }
}

// dlogits *= 1/n_valid (mean reduction, count only known after the forward pass)
__global__ void scale_by_inv_count_kernel(bf16* __restrict__ x, long n, const float* __restrict__ stats) {
  const float sc = 1.0f / fmaxf(stats[1], 1.0f);
  for (long i = (blockIdx.x * (long)blockDim.x + threadIdx.x) * 8; i < n; i += (long)gridDim.x * blockDim.x * 8) {
    const uint4 v = *reinterpret_cast<const uint4*>(x + i);
    const uint32_t u[4] = {v.x, v.y, v.z, v.w};
    uint32_t o[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float2 f = unpack_bf16(u[k]);
      o[k] = pack_bf16(f.x * sc, f.y * sc);
    }
    stg128(x + i, make_uint4(o[0], o[1], o[2], o[3]));
  }
}

// ------------------------------------------------------------------------------------------------
// gradient norm (torch.nn.utils.clip_grad_norm_ semantics on bf16 grads) + fused AdamW
// ------------------------------------------------------------------------------------------------
// acc += the squares of one 16-byte vector of gradients (pairwise for bf16, as the bf16 path has always summed them)
SK_DEVINL void add_sq16(float& acc, const uint4 v, const bf16*) {
  const uint32_t u[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const float2 f = unpack_bf16(u[k]);
    acc += f.x * f.x + f.y * f.y;
  }
}
SK_DEVINL void add_sq16(float& acc, const uint4 v, const float*) {
  const float f[4] = {__uint_as_float(v.x), __uint_as_float(v.y), __uint_as_float(v.z), __uint_as_float(v.w)};
#pragma unroll
  for (int k = 0; k < 4; ++k) acc += f[k] * f[k];
}

// chunk c covers grads[chunk_start[c] .. +chunk_len[c]) and never straddles a tensor; partial[c] = sum of squares
template <typename T>
__global__ void sumsq_chunks_kernel(const T* __restrict__ g, const long* __restrict__ chunk_start,
                                    const int* __restrict__ chunk_len, float* __restrict__ partial) {
  __shared__ float sred[32];
  constexpr int VEC = 16 / sizeof(T);
  const long s = chunk_start[blockIdx.x];
  const int n = chunk_len[blockIdx.x];
  float acc = 0.f;
  const int nvec = n / VEC;
  for (int i = threadIdx.x; i < nvec; i += blockDim.x) add_sq16(acc, ldg128_stream(g + s + (long)i * VEC), g);
  for (int i = nvec * VEC + threadIdx.x; i < n; i += blockDim.x) {
    const float f = to_f32(g[s + i]);
    acc += f * f;
  }
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) sred[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x < 32) {
    float v = threadIdx.x < (blockDim.x >> 5) ? sred[threadIdx.x] : 0.f;
    v = warp_sum(v);
    if (threadIdx.x == 0) partial[blockIdx.x] = v;
  }
}

// one block: per-tensor norms (rounded to bf16 like torch._foreach_norm on bf16 grads), total norm (bf16), and
// clip coefficient  min(1, max_norm/(total+1e-6))  (bf16, as torch computes it on bf16 tensors).
// out[0] = total_norm, out[1] = clip_coef (1.0 if max_norm <= 0), out[2] = exact fp32 total norm
__global__ void gradnorm_finalize_kernel(const float* __restrict__ partial, const int* __restrict__ tensor_chunk_begin,
                                         int n_tensors, float max_norm, int emulate_bf16, float* __restrict__ out) {
  __shared__ double s1[256], s2[256];
  double a = 0, b = 0;
  for (int t = threadIdx.x; t < n_tensors; t += blockDim.x) {
    float ss = 0.f;
    for (int c = tensor_chunk_begin[t]; c < tensor_chunk_begin[t + 1]; ++c) ss += partial[c];
    float nt = sqrtf(ss);
    b += (double)ss;
    if (emulate_bf16) nt = bf16_round(nt);
    a += (double)nt * (double)nt;
  }
  s1[threadIdx.x] = a; s2[threadIdx.x] = b;
  __syncthreads();
  for (int s = blockDim.x / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s) { s1[threadIdx.x] += s1[threadIdx.x + s]; s2[threadIdx.x] += s2[threadIdx.x + s]; }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    float total = sqrtf((float)s1[0]);
    if (emulate_bf16) total = bf16_round(total);
    float coef = 1.0f;
    if (max_norm > 0.f) {
      coef = max_norm / (total + 1e-6f);
      if (emulate_bf16) coef = bf16_round(coef);
      // torch.clamp(coef, max=1) keeps a NaN (a NaN gradient makes every gradient NaN); fminf would return 1
      coef = coef > 1.0f ? 1.0f : coef;
    }
    out[0] = total;
    out[1] = coef;
    out[2] = sqrtf((float)s2[0]);
  }
}

// torch fused AdamW semantics (fp32 math per element, bf16 storage of p, m, v; decoupled weight decay):
//   g = bf16(g * clip_coef) ; p -= lr*wd*p ; m = m + (1-b1)*(g-m) ; v = b2*v + (1-b2)*g*g
//   p -= (lr/bc1) * m / (sqrt(v)/sqrt(bc2) + eps)
__global__ void adamw_kernel(bf16* __restrict__ p, const bf16* __restrict__ g, bf16* __restrict__ m,
                             bf16* __restrict__ v, long n, float lr, float beta1, float beta2, float eps, float wd,
                             float bc1, float bc2_sqrt, const float* __restrict__ clip_stats) {
  const float coef = clip_stats ? clip_stats[1] : 1.0f;
  const float step_size = lr / bc1;
  for (long i = (blockIdx.x * (long)blockDim.x + threadIdx.x) * 8; i < n; i += (long)gridDim.x * blockDim.x * 8) {
    const uint4 pv = *reinterpret_cast<const uint4*>(p + i);
    const uint4 gv = ldg128_stream(g + i);
    const uint4 mv = *reinterpret_cast<const uint4*>(m + i);
    const uint4 vv = *reinterpret_cast<const uint4*>(v + i);
    const uint32_t pu[4] = {pv.x, pv.y, pv.z, pv.w}, gu[4] = {gv.x, gv.y, gv.z, gv.w};
    const uint32_t mu[4] = {mv.x, mv.y, mv.z, mv.w}, vu[4] = {vv.x, vv.y, vv.z, vv.w};
    uint32_t po[4], mo[4], vo[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      float2 pf = unpack_bf16(pu[k]), gf = unpack_bf16(gu[k]), mf = unpack_bf16(mu[k]), vf = unpack_bf16(vu[k]);
      float pp[2] = {pf.x, pf.y}, gg[2] = {gf.x, gf.y}, mm[2] = {mf.x, mf.y}, vv2[2] = {vf.x, vf.y};
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        float grad = (coef != 1.0f) ? bf16_round(gg[e] * coef) : gg[e];
        float param = pp[e];
        param -= lr * wd * param;
        float ea = mm[e] + (1.0f - beta1) * (grad - mm[e]);
        float es = beta2 * vv2[e] + (1.0f - beta2) * grad * grad;
        const float denom = sqrtf(es) / bc2_sqrt + eps;
        param -= step_size * ea / denom;
        pp[e] = param; mm[e] = ea; vv2[e] = es;
      }
      po[k] = pack_bf16(pp[0], pp[1]);
      mo[k] = pack_bf16(mm[0], mm[1]);
      vo[k] = pack_bf16(vv2[0], vv2[1]);
    }
    stg128(p + i, make_uint4(po[0], po[1], po[2], po[3]));
    stg128(m + i, make_uint4(mo[0], mo[1], mo[2], mo[3]));
    stg128(v + i, make_uint4(vo[0], vo[1], vo[2], vo[3]));
  }
}

// out[N, M] = in[M, N]^T (bf16), 32x32 tiles through shared memory; used only by tests / the transposed-copy fallback
__global__ void transpose_kernel(const bf16* __restrict__ in, bf16* __restrict__ out, int M, int N) {
  __shared__ bf16 tile[32][33];
  int x = blockIdx.x * 32 + threadIdx.x, y = blockIdx.y * 32 + threadIdx.y;
  for (int j = 0; j < 32; j += 8)
    if (x < N && y + j < M) tile[threadIdx.y + j][threadIdx.x] = in[(size_t)(y + j) * N + x];
  __syncthreads();
  x = blockIdx.y * 32 + threadIdx.x;
  y = blockIdx.x * 32 + threadIdx.y;
  for (int j = 0; j < 32; j += 8)
    if (x < M && y + j < N) out[(size_t)(y + j) * M + x] = tile[threadIdx.x][threadIdx.y + j];
}

// ------------------------------------------------------------------------------------------------
// Packed batches: a document starts wherever position_ids == 0 (and at column 0).  seg_start[t] = index of the last
// start <= t, seg_end[t] = index of the first start > t (or T).  One block per batch row; threads own contiguous
// chunks, chunk summaries are combined serially (T <= a few thousand: this is a ~3 us kernel).
// Reference: HF derives cu_seqlens for its varlen flash-attention path the same way (HF:modeling_flash_attention_utils.py
// prepare_fa_kwargs_from_position_ids: boundaries at position_ids == 0), used by DataCollatorWithFlattening batches
// (slamkit/data/hf_dataset.py:61-62).
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
seg_bounds_kernel(const int32_t* __restrict__ pos, int32_t* __restrict__ seg_start, int32_t* __restrict__ seg_end, int T) {
  __shared__ int s_last[256], s_first[256];
  const int b = blockIdx.x, tid = threadIdx.x;
  const int per = (T + 255) / 256;
  const int t0 = min(T, tid * per), t1 = min(T, t0 + per);
  const int32_t* p = pos + (size_t)b * T;
  int last = -1, first = T;                      // last / first document start inside this thread's chunk
  for (int t = t0; t < t1; ++t) {
    if (t == 0 || p[t] == 0) {
      last = t;
      if (first == T) first = t;
    }
  }
  s_last[tid] = last;
  s_first[tid] = first;
  __syncthreads();
  int carry_last = 0;                            // last start before this chunk
  for (int i = 0; i < tid; ++i) carry_last = s_last[i] >= 0 ? s_last[i] : carry_last;
  int carry_first = T;                           // first start after this chunk
  for (int i = 255; i > tid; --i) carry_first = s_first[i] < T ? s_first[i] : carry_first;
  int cur = carry_last;
  for (int t = t0; t < t1; ++t) {
    if (t == 0 || p[t] == 0) cur = t;
    seg_start[(size_t)b * T + t] = cur;
  }
  int nxt = carry_first;
  for (int t = t1 - 1; t >= t0; --t) {
    seg_end[(size_t)b * T + t] = nxt;
    if (t == 0 || p[t] == 0) nxt = t;
  }
}

inline int grid_for(long work_items, int threads, int max_blocks_per_sm = 16) {
  long b = (work_items + threads - 1) / threads;
  long cap = (long)sk_num_sms() * max_blocks_per_sm;
  if (b > cap) b = cap;
  if (b < 1) b = 1;
  return (int)b;
}

}  // namespace

// ------------------------------------------------------------------------------------------------
// launchers (C++ linkage; the extern "C" ABI in api.cu forwards to these)
// ------------------------------------------------------------------------------------------------
int sk_embed_fwd_launch(const int64_t* ids, const bf16* E, bf16* out, int M, int D, int V, cudaStream_t s) {
  SK_REQUIRE(D % 8 == 0, "embed: D must be a multiple of 8");
  embed_fwd_kernel<<<grid_for((long)M * D / 8, 256), 256, 0, s>>>(ids, E, out, M, D, V);
  SK_LAUNCH_CHECK();
  return 0;
}
int sk_embed_bwd_launch(const int64_t* ids, const bf16* dx, float* scratch, bf16* dE, int M, int D, int V, int Vpad,
                        int accumulate, cudaStream_t s) {
  SK_REQUIRE(D % 8 == 0, "embed: D must be a multiple of 8");
  unsigned long long* fix = reinterpret_cast<unsigned long long*>(scratch);   // Vpad * D 64-bit words
  SK_CUDA_CHECK(cudaMemsetAsync(fix, 0, (size_t)Vpad * D * sizeof(unsigned long long), s));
  embed_bwd_scatter_kernel<<<grid_for((long)M * D / 8, 256), 256, 0, s>>>(ids, dx, fix, M, D, V);
  SK_LAUNCH_CHECK();
  add_fix_into_bf16_kernel<<<grid_for((long)Vpad * D / 8, 256), 256, 0, s>>>(dE, fix, (long)Vpad * D, accumulate);
  SK_LAUNCH_CHECK();
  return 0;
}
int sk_rmsnorm_fwd_launch(const bf16* x, const bf16* w, bf16* y, float* rstd, int M, int D, float eps, cudaStream_t s) {
  SK_REQUIRE(D % 8 == 0 && D <= 1024, "rmsnorm: D must be a multiple of 8 and <= 1024 (D=%d)", D);
  SK_CUDA_CHECK(sk_launch_pdl(rmsnorm_fwd_kernel, dim3((M + WARPS_PER_BLOCK - 1) / WARPS_PER_BLOCK), dim3(WARPS_PER_BLOCK * 32), (size_t)(0), s, x, w, y, rstd, M, D, eps));
  SK_LAUNCH_CHECK();
  return 0;
}
// dw_partial must hold sk_rmsnorm_bwd_blocks() * D floats
extern "C" int sk_rmsnorm_bwd_blocks(void) { return sk_num_sms() * 4; }
int sk_rmsnorm_bwd_launch(const bf16* dy, const bf16* x, const bf16* w, const float* rstd, const bf16* dres, bf16* dx,
                          bf16* dw, float* dw_partial, int M, int D, int accumulate_dw, cudaStream_t s) {
  SK_REQUIRE(D % 8 == 0 && D <= 1024, "rmsnorm: D must be a multiple of 8 and <= 1024 (D=%d)", D);
  int blocks = sk_rmsnorm_bwd_blocks();
  const int need = (M + WARPS_PER_BLOCK - 1) / WARPS_PER_BLOCK;
  if (blocks > need) blocks = need;
  const size_t smem = (size_t)WARPS_PER_BLOCK * D * sizeof(float);
  SK_CUDA_CHECK(sk_launch_pdl(rmsnorm_bwd_kernel, dim3(blocks), dim3(WARPS_PER_BLOCK * 32), (size_t)(smem), s, dy, x, w, rstd, dres, dx, dw_partial, M, D));
  SK_LAUNCH_CHECK();
  SK_CUDA_CHECK(sk_launch_pdl(colsum_reduce_kernel<bf16>, dim3((D + 31) / 32), dim3(1024), (size_t)(0), s, dw_partial, dw, blocks, D, accumulate_dw));
  SK_LAUNCH_CHECK();
  return 0;
}
constexpr int COLSUM_SPLITS = 512;
extern "C" int sk_colsum_splits(void) { return COLSUM_SPLITS; }
int sk_colsum_launch(const bf16* x, bf16* out, float* partial, int M, int N, int ld, int accumulate, cudaStream_t s) {
  SK_REQUIRE(N % 8 == 0 && ld % 8 == 0, "colsum: N and ld must be multiples of 8");
  dim3 grid((N / 8 + 127) / 128, COLSUM_SPLITS);
  SK_CUDA_CHECK(sk_launch_pdl(colsum_partial_kernel, dim3(grid), dim3(128), (size_t)(0), s, x, partial, M, N, ld));
  SK_LAUNCH_CHECK();
  SK_CUDA_CHECK(sk_launch_pdl(colsum_reduce_kernel<bf16>, dim3((N + 31) / 32), dim3(1024), (size_t)(0), s, partial, out, COLSUM_SPLITS, N, accumulate));
  SK_LAUNCH_CHECK();
  return 0;
}
int sk_rope_launch(bf16* qkv, const bf16* cos_t, const bf16* sin_t, const int* pos_ids, int M, int T, int ld,
                   int n_rot_heads, int head_dim, int inverse, int max_positions, cudaStream_t s, int rot_dims) {
  SK_REQUIRE(head_dim % 16 == 0 && ld % 8 == 0, "rope: head_dim must be a multiple of 16");
  SK_REQUIRE(max_positions > 0 && (pos_ids != nullptr || T <= max_positions), "rope: table rows (%d) do not cover T=%d", max_positions, T);
  const int rot = rot_dims > 0 ? rot_dims : head_dim;
  SK_REQUIRE(rot == head_dim || (head_dim == 64 && (rot == 16 || rot == 32)),
             "rope: rotary width %d not supported (16, 32 or the head_dim %d)", rot, head_dim);
  SK_CUDA_CHECK(sk_launch_pdl(rope_kernel, dim3(grid_for((long)M * n_rot_heads * (rot / 16), 256)), dim3(256), (size_t)(0), s, qkv, cos_t, sin_t, pos_ids, M, T, ld,
                                                                                   n_rot_heads, head_dim, inverse, max_positions, rot));
  SK_LAUNCH_CHECK();
  return 0;
}
int sk_swiglu_fwd_launch(const bf16* gu, bf16* act, int M, int F, cudaStream_t s) {
  SK_REQUIRE(F % 8 == 0, "swiglu: F must be a multiple of 8");
  SK_CUDA_CHECK(sk_launch_pdl(swiglu_fwd_kernel, dim3(grid_for(((long)M * F / 8 + 1) / 2, 256)), dim3(256), (size_t)(0), s, gu, act, M, F));
  SK_LAUNCH_CHECK();
  return 0;
}
int sk_swiglu_bwd_launch(const bf16* gu, const bf16* dact, bf16* dgu, int M, int F, cudaStream_t s) {
  SK_REQUIRE(F % 8 == 0, "swiglu: F must be a multiple of 8");
  SK_CUDA_CHECK(sk_launch_pdl(swiglu_bwd_kernel, dim3(grid_for((long)M * F / 8, 256)), dim3(256), (size_t)(0), s, gu, dact, dgu, M, F));
  SK_LAUNCH_CHECK();
  return 0;
}
// partial[] entries sk_ce_launch may write: one pair per row in the large-vocabulary kernel (a superset of the per-block
// pairs of the small one)
extern "C" int sk_ce_blocks(int M) { return M; }
// stats_out: float[3] = {loss, n_valid, nll_sum}.  num_items > 0: loss = sum/num_items (reference 'sum' path);
// num_items <= 0: mean over valid tokens.  dloss scales the gradient.
int sk_ce_launch(const bf16* logits, const int64_t* labels, bf16* dlogits, float* partial, float* row_nll,
                 float* stats_out, int M, int T, int V, int ldl, float num_items, float dloss, cudaStream_t s,
                 const float* row_weight) {
  SK_REQUIRE(ldl % 8 == 0 && V <= ldl, "ce: padded vocab must be a multiple of 8 and >= the vocabulary");
  const float gs = num_items > 0.f ? dloss / num_items : dloss;
  int blocks;
  if (ldl <= CE_MAX_VEC * 256) {             // unit vocabularies (502): one warp per row, the row lives in registers
    blocks = (M + WARPS_PER_BLOCK - 1) / WARPS_PER_BLOCK;
    ce_fwd_bwd_kernel<<<blocks, WARPS_PER_BLOCK * 32, 0, s>>>(logits, labels, dlogits, partial, row_nll, row_weight, M, T, V, ldl, gs);
  } else {                                   // text + unit vocabularies: one block per row, two passes
    blocks = M;
    ce_large_kernel<<<blocks, 256, 0, s>>>(logits, labels, dlogits, partial, row_nll, row_weight, M, T, V, ldl, gs, 0);
  }
  SK_LAUNCH_CHECK();
  ce_finalize_kernel<<<1, 256, 0, s>>>(partial, blocks, num_items, stats_out);
  SK_LAUNCH_CHECK();
  if (dlogits && num_items <= 0.f) {
    scale_by_inv_count_kernel<<<grid_for((long)M * ldl / 8, 256), 256, 0, s>>>(dlogits, (long)M * ldl, stats_out);
    SK_LAUNCH_CHECK();
  }
  return 0;
}
// Chunked form for large vocabularies: rows [row0, row0 + rows) of the batch, whose logits sit at `logits_chunk` (the
// gradient is written in place when dlogits_chunk == logits_chunk: every element is read, then overwritten, by the same
// thread).  partial holds one (nll, valid) pair per GLOBAL row; sk_ce_finalize_launch sums them once all chunks are done.
int sk_ce_chunk_launch(const bf16* logits_chunk, const int64_t* labels, bf16* dlogits_chunk, float* partial, int row0, int rows,
                       int M, int T, int V, int ldl, float grad_scale, cudaStream_t s) {
  SK_REQUIRE(ldl % 8 == 0 && V <= ldl && rows > 0 && row0 >= 0 && row0 + rows <= M, "ce chunk: bad arguments");
  ce_large_kernel<<<rows, 256, 0, s>>>(logits_chunk, labels, dlogits_chunk, partial, nullptr, nullptr, M, T, V, ldl, grad_scale, row0);
  SK_LAUNCH_CHECK();
  return 0;
}
int sk_ce_finalize_launch(const float* partial, int M, float num_items, float* stats_out, cudaStream_t s) {
  ce_finalize_kernel<<<1, 256, 0, s>>>(partial, M, num_items, stats_out);
  SK_LAUNCH_CHECK();
  return 0;
}
int sk_gradnorm_launch(const bf16* g, const long* chunk_start, const int* chunk_len, int n_chunks,
                       const int* tensor_chunk_begin, int n_tensors, float* partial, float max_norm, int emulate_bf16,
                       float* stats_out, cudaStream_t s) {
  sumsq_chunks_kernel<<<n_chunks, 256, 0, s>>>(g, chunk_start, chunk_len, partial);
  SK_LAUNCH_CHECK();
  gradnorm_finalize_kernel<<<1, 256, 0, s>>>(partial, tensor_chunk_begin, n_tensors, max_norm, emulate_bf16, stats_out);
  SK_LAUNCH_CHECK();
  return 0;
}
// fp32 gradients: per-tensor fp32 norms and their fp32 norm, no bf16 rounding anywhere (clip_grad_norm_ on fp32 .grad)
int sk_gradnorm_f32_launch(const float* g, const long* chunk_start, const int* chunk_len, int n_chunks,
                           const int* tensor_chunk_begin, int n_tensors, float* partial, float max_norm, float* stats_out,
                           cudaStream_t s) {
  sumsq_chunks_kernel<<<n_chunks, 256, 0, s>>>(g, chunk_start, chunk_len, partial);
  SK_LAUNCH_CHECK();
  gradnorm_finalize_kernel<<<1, 256, 0, s>>>(partial, tensor_chunk_begin, n_tensors, max_norm, 0, stats_out);
  SK_LAUNCH_CHECK();
  return 0;
}
int sk_adamw_launch(bf16* p, const bf16* g, bf16* m, bf16* v, long n, float lr, float beta1, float beta2, float eps,
                    float wd, int step, const float* clip_stats, cudaStream_t s) {
  SK_REQUIRE(n % 8 == 0, "adamw: flat parameter count must be a multiple of 8 (n=%ld)", n);
  SK_REQUIRE(step >= 1, "adamw: step counts from 1");
  const float bc1 = (float)(1.0 - pow((double)beta1, (double)step));
  const float bc2_sqrt = (float)sqrt(1.0 - pow((double)beta2, (double)step));
  adamw_kernel<<<grid_for(n / 8, 256, 8), 256, 0, s>>>(p, g, m, v, n, lr, beta1, beta2, eps, wd, bc1, bc2_sqrt, clip_stats);
  SK_LAUNCH_CHECK();
  return 0;
}
int sk_seg_bounds_launch(const int32_t* pos_ids, int32_t* seg_start, int32_t* seg_end, int B, int T, cudaStream_t s) {
  SK_REQUIRE(pos_ids && seg_start && seg_end && B > 0 && T > 0, "seg_bounds: bad arguments");
  seg_bounds_kernel<<<B, 256, 0, s>>>(pos_ids, seg_start, seg_end, T);
  SK_LAUNCH_CHECK();
  return 0;
}
int sk_transpose_launch(const bf16* in, bf16* out, int M, int N, cudaStream_t s) {
  dim3 grid((N + 31) / 32, (M + 31) / 32), block(32, 8);
  transpose_kernel<<<grid, block, 0, s>>>(in, out, M, N);
  SK_LAUNCH_CHECK();
  return 0;
}

// ------------------------------------------------------------------------------------------------
// OPT decoder (pre-LayerNorm, learned positions, ReLU MLP; HF:models/opt/modeling_opt.py:45-70,170-260,480-560)
// ------------------------------------------------------------------------------------------------
namespace {

constexpr int LN_BWD_WARPS = 4;

// LayerNorm forward, one warp per row: y = bf16((x - mean) * rstd * g + b) in fp32 (nn.LayerNorm on a bf16 input, and
// its autocast form that runs in fp32 and feeds the next linear a bf16 copy, both round once).  The row stays in
// registers between the mean pass, the variance pass and the output pass.  NOUT = 2 (GPT-NeoX's parallel residual,
// HF:models/gpt_neox/modeling_gpt_neox.py use_parallel_residual) also writes y2 = LN(x; w2, b2) from the same registers
// and statistics: each output is the NOUT = 1 value by construction.
template <int MAXV, int NOUT = 1>
__global__ void __launch_bounds__(WARPS_PER_BLOCK * 32)
layernorm_fwd_kernel(const bf16* __restrict__ x, const bf16* __restrict__ w, const bf16* __restrict__ b, bf16* __restrict__ y,
                     const bf16* __restrict__ w2, const bf16* __restrict__ b2, bf16* __restrict__ y2,
                     float* __restrict__ mean_out, float* __restrict__ rstd_out, int M, int D, float eps) {
  griddep_launch();
  griddep_wait();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int row = blockIdx.x * WARPS_PER_BLOCK + warp;
  if (row >= M) return;
  const int nvec = D / 8;
  uint4 xv[MAXV];
  float s = 0.f;
#pragma unroll
  for (int j = 0; j < MAXV; ++j) {
    const int c = lane + 32 * j;
    if (c < nvec) {
      xv[j] = ldg128_stream(x + (size_t)row * D + c * 8);
      const uint32_t u[4] = {xv[j].x, xv[j].y, xv[j].z, xv[j].w};
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float2 f = unpack_bf16(u[k]);
        s += f.x + f.y;
      }
    }
  }
  const float mean = warp_sum(s) / (float)D;
  float ss = 0.f;
#pragma unroll
  for (int j = 0; j < MAXV; ++j) {
    const int c = lane + 32 * j;
    if (c < nvec) {
      const uint32_t u[4] = {xv[j].x, xv[j].y, xv[j].z, xv[j].w};
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float2 f = unpack_bf16(u[k]);
        ss += (f.x - mean) * (f.x - mean) + (f.y - mean) * (f.y - mean);
      }
    }
  }
  const float rstd = rsqrtf(warp_sum(ss) / (float)D + eps);
  if (lane == 0) {
    if (mean_out) mean_out[row] = mean;
    if (rstd_out) rstd_out[row] = rstd;
  }
#pragma unroll
  for (int j = 0; j < MAXV; ++j) {
    const int c = lane + 32 * j;
    if (c < nvec) {
      const uint32_t u[4] = {xv[j].x, xv[j].y, xv[j].z, xv[j].w};
#pragma unroll
      for (int t = 0; t < NOUT; ++t) {
        const uint4 wv = ldg128((t ? w2 : w) + c * 8), bv = ldg128((t ? b2 : b) + c * 8);
        const uint32_t wu[4] = {wv.x, wv.y, wv.z, wv.w}, bu[4] = {bv.x, bv.y, bv.z, bv.w};
        uint32_t o[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const float2 f = unpack_bf16(u[k]), g = unpack_bf16(wu[k]), bb = unpack_bf16(bu[k]);
          o[k] = pack_bf16(fmaf((f.x - mean) * rstd, g.x, bb.x), fmaf((f.y - mean) * rstd, g.y, bb.y));
        }
        stg128((t ? y2 : y) + (size_t)row * D + c * 8, make_uint4(o[0], o[1], o[2], o[3]));
      }
    }
  }
}

// LayerNorm backward, one warp per row, grid-stride over rows with a fixed grid:
//   xhat = (x - mean) * rstd ; g = dy * w ; dx = rstd * (g - mean(g) - xhat * mean(g * xhat)) (+ dres)
//   dw (+)= sum_rows dy * xhat ; db (+)= sum_rows dy
// Each warp adds its rows' dw / db terms into its own shared-memory slab (a lane owns its columns: no conflicts); the
// block writes one partial row per block, and colsum_reduce_kernel sums the partials in a fixed order (deterministic).
// NIN = 2 is the backward of the two LayerNorms of one x (GPT-NeoX's parallel residual): the input gradient is linear in
// g, so one pass takes g = dy * w + dy2 * w2 in fp32, and dw2 / db2 get their own slabs and partial rows.
template <int MAXV, int NIN = 1>
__global__ void __launch_bounds__(LN_BWD_WARPS * 32)
layernorm_bwd_kernel(const bf16* __restrict__ dy, const bf16* __restrict__ dy2, const bf16* __restrict__ x,
                     const bf16* __restrict__ w, const bf16* __restrict__ w2, const float* __restrict__ mean_in,
                     const float* __restrict__ rstd_in, const bf16* __restrict__ dres, bf16* __restrict__ dx,
                     float* __restrict__ dw_partial, float* __restrict__ db_partial, float* __restrict__ dw2_partial,
                     float* __restrict__ db2_partial, int M, int D) {
  griddep_launch();
  griddep_wait();
  extern __shared__ float sacc[];   // [2 * NIN][LN_BWD_WARPS][D]: dw, db (then dw2, db2)
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nvec = D / 8;
  float* sl[2 * NIN];
#pragma unroll
  for (int t = 0; t < 2 * NIN; ++t) sl[t] = sacc + ((size_t)t * LN_BWD_WARPS + warp) * D;
  for (int c = lane; c < nvec; c += 32)
#pragma unroll
    for (int k = 0; k < 8; ++k)
#pragma unroll
      for (int t = 0; t < 2 * NIN; ++t) sl[t][c * 8 + k] = 0.f;
  for (int row = blockIdx.x * LN_BWD_WARPS + warp; row < M; row += gridDim.x * LN_BWD_WARPS) {
    uint4 xq[MAXV], dq[MAXV], dq2[MAXV];
#pragma unroll
    for (int j = 0; j < MAXV; ++j) {
      const int c = lane + 32 * j;
      if (c < nvec) {
        xq[j] = ldg128_stream(x + (size_t)row * D + c * 8);
        dq[j] = ldg128_stream(dy + (size_t)row * D + c * 8);
        if constexpr (NIN == 2) dq2[j] = ldg128_stream(dy2 + (size_t)row * D + c * 8);
      }
    }
    const float mean = mean_in[row], rstd = rstd_in[row];
    // g of element pair k of vector j (the only place the two forms differ)
    auto gpair = [&](int j, int k, const uint4& wv, const uint4& wv2) {
      const uint32_t du[4] = {dq[j].x, dq[j].y, dq[j].z, dq[j].w}, wu[4] = {wv.x, wv.y, wv.z, wv.w};
      const float2 df = unpack_bf16(du[k]), wf = unpack_bf16(wu[k]);
      if constexpr (NIN == 2) {
        const uint32_t eu[4] = {dq2[j].x, dq2[j].y, dq2[j].z, dq2[j].w}, vu[4] = {wv2.x, wv2.y, wv2.z, wv2.w};
        const float2 ef = unpack_bf16(eu[k]), vf = unpack_bf16(vu[k]);
        return make_float2(fmaf(df.x, wf.x, ef.x * vf.x), fmaf(df.y, wf.y, ef.y * vf.y));
      } else {
        return make_float2(df.x * wf.x, df.y * wf.y);
      }
    };
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int j = 0; j < MAXV; ++j) {
      const int c = lane + 32 * j;
      if (c < nvec) {
        const uint4 wv = ldg128(w + c * 8);
        const uint4 wv2 = NIN == 2 ? ldg128(w2 + c * 8) : wv;
        const uint32_t xu[4] = {xq[j].x, xq[j].y, xq[j].z, xq[j].w}, du[4] = {dq[j].x, dq[j].y, dq[j].z, dq[j].w};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const float2 xf = unpack_bf16(xu[k]), df = unpack_bf16(du[k]);
          const float xh0 = (xf.x - mean) * rstd, xh1 = (xf.y - mean) * rstd;
          const float2 g = gpair(j, k, wv, wv2);
          s1 += g.x + g.y;
          s2 = fmaf(g.x, xh0, fmaf(g.y, xh1, s2));
          const int e = c * 8 + 2 * k;
          sl[0][e] = fmaf(df.x, xh0, sl[0][e]);
          sl[0][e + 1] = fmaf(df.y, xh1, sl[0][e + 1]);
          sl[1][e] += df.x;
          sl[1][e + 1] += df.y;
          if constexpr (NIN == 2) {
            const uint32_t eu[4] = {dq2[j].x, dq2[j].y, dq2[j].z, dq2[j].w};
            const float2 ef = unpack_bf16(eu[k]);
            sl[2][e] = fmaf(ef.x, xh0, sl[2][e]);
            sl[2][e + 1] = fmaf(ef.y, xh1, sl[2][e + 1]);
            sl[3][e] += ef.x;
            sl[3][e + 1] += ef.y;
          }
        }
      }
    }
    const float m1 = warp_sum(s1) / (float)D, m2 = warp_sum(s2) / (float)D;
#pragma unroll
    for (int j = 0; j < MAXV; ++j) {
      const int c = lane + 32 * j;
      if (c < nvec) {
        const uint4 wv = ldg128(w + c * 8);
        const uint4 wv2 = NIN == 2 ? ldg128(w2 + c * 8) : wv;
        const uint4 rv = dres ? ldg128_stream(dres + (size_t)row * D + c * 8) : make_uint4(0, 0, 0, 0);
        const uint32_t xu[4] = {xq[j].x, xq[j].y, xq[j].z, xq[j].w}, ru[4] = {rv.x, rv.y, rv.z, rv.w};
        uint32_t o[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const float2 xf = unpack_bf16(xu[k]), rf = unpack_bf16(ru[k]);
          const float xh0 = (xf.x - mean) * rstd, xh1 = (xf.y - mean) * rstd;
          const float2 g = gpair(j, k, wv, wv2);
          const float d0 = rstd * (g.x - m1 - xh0 * m2), d1 = rstd * (g.y - m1 - xh1 * m2);
          o[k] = pack_bf16(d0 + rf.x, d1 + rf.y);
        }
        stg128(dx + (size_t)row * D + c * 8, make_uint4(o[0], o[1], o[2], o[3]));
      }
    }
  }
  __syncthreads();
  float* outs[4] = {dw_partial, db_partial, dw2_partial, db2_partial};
  for (int i = threadIdx.x; i < D; i += blockDim.x) {
#pragma unroll
    for (int t = 0; t < 2 * NIN; ++t) {
      float a = 0.f;
#pragma unroll
      for (int wi = 0; wi < LN_BWD_WARPS; ++wi) a += sacc[((size_t)t * LN_BWD_WARPS + wi) * D + i];
      outs[t][(size_t)blockIdx.x * D + i] = a;
    }
  }
}

// OPTLearnedPositionalEmbedding: table row of a position (offset 2, clamped to the table like the RoPE tables)
SK_DEVINL int opt_pos_row(const int32_t* pos_ids, int m, int T, int n_rows) {
  const int p = (pos_ids ? pos_ids[m] : m % T) + 2;
  return max(0, min(p, n_rows - 1));
}

// x0 = bf16(E[id] + P[pos + 2]) (embed_tokens + embed_positions in bf16: one rounding)
__global__ void opt_embed_fwd_kernel(const int64_t* __restrict__ ids, const int32_t* __restrict__ pos_ids, const bf16* __restrict__ E,
                                     const bf16* __restrict__ P, bf16* __restrict__ out, int M, int T, int D, int V, int n_pos) {
  const int vec_per_row = D / 8;
  const long total = (long)M * vec_per_row;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int m = (int)(i / vec_per_row);
    const int c = (int)(i % vec_per_row);
    const int pr = opt_pos_row(pos_ids, m, T, n_pos);
    uint4 a = make_uint4(0u, 0u, 0u, 0u);   // E == nullptr: the position rows alone (post-LN OPT with project_in)
    if (E) {
      long id = ids[m];
      if (id < 0 || id >= V) id = 0;
      a = ldg128(E + (size_t)id * D + c * 8);
    }
    const uint4 b = ldg128(P + (size_t)pr * D + c * 8);
    const uint32_t au[4] = {a.x, a.y, a.z, a.w}, bu[4] = {b.x, b.y, b.z, b.w};
    uint32_t o[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float2 fa = unpack_bf16(au[k]), fb = unpack_bf16(bu[k]);
      o[k] = pack_bf16(fa.x + fb.x, fa.y + fb.y);
    }
    stg128(out + (size_t)m * D + c * 8, make_uint4(o[0], o[1], o[2], o[3]));
  }
}

// dP_fix[pos_row(m)] += dx[m] in the 64-bit fixed point of embed_bwd_scatter_kernel (order-independent)
__global__ void opt_pos_bwd_scatter_kernel(const int32_t* __restrict__ pos_ids, const bf16* __restrict__ dx,
                                           unsigned long long* __restrict__ scratch, int M, int T, int D, int n_pos) {
  const int vec_per_row = D / 8;
  const long total = (long)M * vec_per_row;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int m = (int)(i / vec_per_row);
    const int c = (int)(i % vec_per_row);
    const int pr = opt_pos_row(pos_ids, m, T, n_pos);
    const uint4 v = ldg128_stream(dx + (size_t)m * D + c * 8);
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
    unsigned long long* dst = scratch + (size_t)pr * D + c * 8;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float2 f = unpack_bf16(w[k]);
      if (f.x != 0.f) atomicAdd(dst + 2 * k, (unsigned long long)__float2ll_rn(f.x * EMBED_FIX_SCALE));
      if (f.y != 0.f) atomicAdd(dst + 2 * k + 1, (unsigned long long)__float2ll_rn(f.y * EMBED_FIX_SCALE));
    }
  }
}

// torch threshold_backward(grad, relu_out, 0) = where(relu_out <= 0, 0, grad), in place on grad: a NaN activation passes
// the gradient through, as autograd's ReLU backward does
__global__ void relu_bwd_kernel(bf16* __restrict__ g, const bf16* __restrict__ a, long n) {
  griddep_launch();
  griddep_wait();
  for (long i = (blockIdx.x * (long)blockDim.x + threadIdx.x) * 8; i < n; i += (long)gridDim.x * blockDim.x * 8) {
    const uint4 gv = *reinterpret_cast<const uint4*>(g + i);
    const uint4 av = ldg128_stream(a + i);
    const uint32_t gu[4] = {gv.x, gv.y, gv.z, gv.w}, au[4] = {av.x, av.y, av.z, av.w};
    uint32_t o[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float2 fa = unpack_bf16(au[k]);
      o[k] = (fa.x <= 0.f ? 0u : (gu[k] & 0xffffu)) | (fa.y <= 0.f ? 0u : (gu[k] & 0xffff0000u));
    }
    stg128(g + i, make_uint4(o[0], o[1], o[2], o[3]));
  }
}

}  // namespace

int sk_layernorm_fwd_launch(const bf16* x, const bf16* w, const bf16* b, bf16* y, float* mean, float* rstd, int M, int D,
                            float eps, cudaStream_t s) {
  SK_REQUIRE(D % 8 == 0 && D <= 2048, "layernorm: D must be a multiple of 8 and <= 2048 (D=%d)", D);
  const dim3 grid((M + WARPS_PER_BLOCK - 1) / WARPS_PER_BLOCK), block(WARPS_PER_BLOCK * 32);
  const bf16* none = nullptr;
  bf16* no_out = nullptr;
  if (D <= 1024) SK_CUDA_CHECK(sk_launch_pdl(layernorm_fwd_kernel<4>, grid, block, (size_t)0, s, x, w, b, y, none, none, no_out, mean, rstd, M, D, eps));
  else           SK_CUDA_CHECK(sk_launch_pdl(layernorm_fwd_kernel<8>, grid, block, (size_t)0, s, x, w, b, y, none, none, no_out, mean, rstd, M, D, eps));
  SK_LAUNCH_CHECK();
  return 0;
}
// dw_partial / db_partial must each hold sk_layernorm_bwd_blocks() * D floats
extern "C" int sk_layernorm_bwd_blocks(void) { return sk_num_sms() * 2; }
int sk_layernorm_bwd_launch(const bf16* dy, const bf16* x, const bf16* w, const float* mean, const float* rstd, const bf16* dres,
                            bf16* dx, bf16* dw, bf16* db, float* dw_partial, float* db_partial, int M, int D, int accumulate,
                            cudaStream_t s) {
  SK_REQUIRE(D % 8 == 0 && D <= 2048, "layernorm: D must be a multiple of 8 and <= 2048 (D=%d)", D);
  int blocks = sk_layernorm_bwd_blocks();
  const int need = (M + LN_BWD_WARPS - 1) / LN_BWD_WARPS;
  if (blocks > need) blocks = need;
  const size_t smem = (size_t)2 * LN_BWD_WARPS * D * sizeof(float);
  if (smem > 48 * 1024)   // D > 1536
    SK_CUDA_CHECK(cudaFuncSetAttribute(layernorm_bwd_kernel<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const bf16* none = nullptr;
  float* no_partial = nullptr;
  if (D <= 1024)
    SK_CUDA_CHECK(sk_launch_pdl(layernorm_bwd_kernel<4>, dim3(blocks), dim3(LN_BWD_WARPS * 32), smem, s, dy, none, x, w, none, mean, rstd,
                                dres, dx, dw_partial, db_partial, no_partial, no_partial, M, D));
  else
    SK_CUDA_CHECK(sk_launch_pdl(layernorm_bwd_kernel<8>, dim3(blocks), dim3(LN_BWD_WARPS * 32), smem, s, dy, none, x, w, none, mean, rstd,
                                dres, dx, dw_partial, db_partial, no_partial, no_partial, M, D));
  SK_LAUNCH_CHECK();
  SK_CUDA_CHECK(sk_launch_pdl(colsum_reduce_kernel<bf16>, dim3((D + 31) / 32), dim3(1024), (size_t)0, s, (const float*)dw_partial, dw, blocks, D, accumulate));
  SK_LAUNCH_CHECK();
  SK_CUDA_CHECK(sk_launch_pdl(colsum_reduce_kernel<bf16>, dim3((D + 31) / 32), dim3(1024), (size_t)0, s, (const float*)db_partial, db, blocks, D, accumulate));
  SK_LAUNCH_CHECK();
  return 0;
}
int sk_opt_embed_fwd_launch(const int64_t* ids, const int32_t* pos_ids, const bf16* E, const bf16* P, bf16* out, int M, int T, int D,
                            int V, int n_pos, cudaStream_t s) {
  SK_REQUIRE(D % 8 == 0 && n_pos > 0 && T > 0, "opt embed: D must be a multiple of 8");
  opt_embed_fwd_kernel<<<grid_for((long)M * D / 8, 256), 256, 0, s>>>(ids, pos_ids, E, P, out, M, T, D, V, n_pos);
  SK_LAUNCH_CHECK();
  return 0;
}
int sk_opt_pos_bwd_launch(const int32_t* pos_ids, const bf16* dx, float* scratch, bf16* dP, int M, int T, int D, int n_pos,
                          int accumulate, cudaStream_t s) {
  SK_REQUIRE(D % 8 == 0 && n_pos > 0 && T > 0, "opt positions: D must be a multiple of 8");
  unsigned long long* fix = reinterpret_cast<unsigned long long*>(scratch);   // n_pos * D 64-bit words
  const long n = (long)n_pos * D;
  SK_CUDA_CHECK(cudaMemsetAsync(fix, 0, (size_t)n * sizeof(unsigned long long), s));
  opt_pos_bwd_scatter_kernel<<<grid_for((long)M * D / 8, 256), 256, 0, s>>>(pos_ids, dx, fix, M, T, D, n_pos);
  SK_LAUNCH_CHECK();
  SK_REQUIRE(n % 8 == 0, "opt positions: table size must be a multiple of 8");
  add_fix_into_bf16_kernel<<<grid_for(n / 8, 256), 256, 0, s>>>(dP, fix, n, accumulate);
  SK_LAUNCH_CHECK();
  return 0;
}
int sk_layernorm2_fwd_launch(const bf16* x, const bf16* w1, const bf16* b1, const bf16* w2, const bf16* b2, bf16* y1, bf16* y2,
                             float* mean, float* rstd, int M, int D, float eps, cudaStream_t s) {
  SK_REQUIRE(D % 8 == 0 && D <= 2048, "layernorm2: D must be a multiple of 8 and <= 2048 (D=%d)", D);
  const dim3 grid((M + WARPS_PER_BLOCK - 1) / WARPS_PER_BLOCK), block(WARPS_PER_BLOCK * 32);
  if (D <= 1024) SK_CUDA_CHECK(sk_launch_pdl(layernorm_fwd_kernel<4, 2>, grid, block, (size_t)0, s, x, w1, b1, y1, w2, b2, y2, mean, rstd, M, D, eps));
  else           SK_CUDA_CHECK(sk_launch_pdl(layernorm_fwd_kernel<8, 2>, grid, block, (size_t)0, s, x, w1, b1, y1, w2, b2, y2, mean, rstd, M, D, eps));
  SK_LAUNCH_CHECK();
  return 0;
}
// partial must hold 4 * sk_layernorm_bwd_blocks() * D floats
int sk_layernorm2_bwd_launch(const bf16* dy1, const bf16* dy2, const bf16* x, const bf16* w1, const bf16* w2, const float* mean,
                             const float* rstd, const bf16* dres, bf16* dx, bf16* dw1, bf16* db1, bf16* dw2, bf16* db2,
                             float* partial, int M, int D, int accumulate, cudaStream_t s) {
  SK_REQUIRE(D % 8 == 0 && D <= 2048, "layernorm2: D must be a multiple of 8 and <= 2048 (D=%d)", D);
  SK_REQUIRE(M > 0, "layernorm2: M must be positive");
  int blocks = sk_layernorm_bwd_blocks();
  const int need = (M + LN_BWD_WARPS - 1) / LN_BWD_WARPS;
  if (blocks > need) blocks = need;
  const size_t smem = (size_t)4 * LN_BWD_WARPS * D * sizeof(float);
  float* pt[4];
  for (int t = 0; t < 4; ++t) pt[t] = partial + (size_t)t * blocks * D;
  if (D <= 1024) {
    if (smem > 48 * 1024)
      SK_CUDA_CHECK(cudaFuncSetAttribute(layernorm_bwd_kernel<4, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    SK_CUDA_CHECK(sk_launch_pdl(layernorm_bwd_kernel<4, 2>, dim3(blocks), dim3(LN_BWD_WARPS * 32), smem, s, dy1, dy2, x, w1, w2, mean,
                                rstd, dres, dx, pt[0], pt[1], pt[2], pt[3], M, D));
  } else {
    SK_CUDA_CHECK(cudaFuncSetAttribute(layernorm_bwd_kernel<8, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    SK_CUDA_CHECK(sk_launch_pdl(layernorm_bwd_kernel<8, 2>, dim3(blocks), dim3(LN_BWD_WARPS * 32), smem, s, dy1, dy2, x, w1, w2, mean,
                                rstd, dres, dx, pt[0], pt[1], pt[2], pt[3], M, D));
  }
  SK_LAUNCH_CHECK();
  bf16* outs[4] = {dw1, db1, dw2, db2};
  for (int t = 0; t < 4; ++t) {
    SK_CUDA_CHECK(sk_launch_pdl(colsum_reduce_kernel<bf16>, dim3((D + 31) / 32), dim3(1024), (size_t)0, s, (const float*)pt[t], outs[t],
                                blocks, D, accumulate));
    SK_LAUNCH_CHECK();
  }
  return 0;
}
int sk_relu_bwd_launch(bf16* g, const bf16* a, long n, cudaStream_t s) {
  SK_REQUIRE(n % 8 == 0, "relu backward: size must be a multiple of 8");
  SK_CUDA_CHECK(sk_launch_pdl(relu_bwd_kernel, dim3(grid_for(n / 8, 256)), dim3(256), (size_t)0, s, g, a, n));
  SK_LAUNCH_CHECK();
  return 0;
}

// ------------------------------------------------------------------------------------------------
// OPT with fp32 master weights: HF OPTForCausalLM with fp32 parameters under torch.autocast(bfloat16), the precision of
// the reference's default recipe (torch_dtype null, bf16: true).  The residual stream, the embedding tables, the
// LayerNorm parameters and every gradient are fp32; each linear reads bf16 operands (the bf16 shadow of the masters)
// and writes a bf16 output, so the GEMMs are the bf16 path's own.
// ------------------------------------------------------------------------------------------------
namespace {

constexpr int VEC4_PER_WARP = 32 * 4;   // fp32 row elements per warp pass (one float4 per lane)

SK_DEVINL float4 ldg4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }
SK_DEVINL float4 ldg4_stream(const float* p) {
  const uint4 u = ldg128_stream(p);
  return make_float4(__uint_as_float(u.x), __uint_as_float(u.y), __uint_as_float(u.z), __uint_as_float(u.w));
}
SK_DEVINL float4 ld_bf16x4(const bf16* p) {
  const uint2 u = *reinterpret_cast<const uint2*>(p);
  const float2 a = unpack_bf16(u.x), b = unpack_bf16(u.y);
  return make_float4(a.x, a.y, b.x, b.y);
}
SK_DEVINL void st_bf16x4(bf16* p, float4 v) {
  *reinterpret_cast<uint2*>(p) = make_uint2(pack_bf16(v.x, v.y), pack_bf16(v.z, v.w));
}

// x0 = E[id] + P[pos + 2] in fp32 (embed_tokens + embed_positions of the fp32 tables: the residual stream starts fp32)
__global__ void opt_embed_fwd_f32_kernel(const int64_t* __restrict__ ids, const int32_t* __restrict__ pos_ids,
                                         const float* __restrict__ E, const float* __restrict__ P, float* __restrict__ out,
                                         int M, int T, int D, int V, int n_pos) {
  const int vec_per_row = D / 4;
  const long total = (long)M * vec_per_row;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int m = (int)(i / vec_per_row);
    const int c = (int)(i % vec_per_row);
    // E == nullptr: the position rows alone; P == nullptr: the token rows alone (post-LN OPT with project_in, whose
    // token rows are proj_dim wide)
    float4 a = make_float4(0.f, 0.f, 0.f, 0.f), b = a;
    if (E) {
      long id = ids[m];
      if (id < 0 || id >= V) id = 0;
      a = ldg4(E + (size_t)id * D + c * 4);
    }
    if (P) b = ldg4(P + (size_t)opt_pos_row(pos_ids, m, T, n_pos) * D + c * 4);
    *reinterpret_cast<float4*>(out + (size_t)m * D + c * 4) = make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w);
  }
}

// Residual add + LayerNorm, one warp per row, the row in registers:
//   x' = x + float(y)  (fp32 + bf16 promotes to fp32: the residual is never rounded to bf16; y == nullptr: x' = x)
//   h  = bf16((x' - mean) * rstd * g + b)   (fp32 LayerNorm of fp32 parameters; the next linear's autocast rounds once)
// x' is written to xo when y is given (the backward pass reads it), mean / rstd when their pointers are.
template <int MAXV>
__global__ void __launch_bounds__(WARPS_PER_BLOCK * 32)
add_layernorm_f32_kernel(const float* __restrict__ x, const bf16* __restrict__ y, const float* __restrict__ w,
                         const float* __restrict__ b, float* __restrict__ xo, bf16* __restrict__ h,
                         float* __restrict__ mean_out, float* __restrict__ rstd_out, int M, int D, float eps) {
  griddep_launch();
  griddep_wait();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int row = blockIdx.x * WARPS_PER_BLOCK + warp;
  if (row >= M) return;
  const int nvec = D / 4;
  float4 xv[MAXV];
  float s = 0.f;
#pragma unroll
  for (int j = 0; j < MAXV; ++j) {
    const int c = lane + 32 * j;
    if (c < nvec) {
      xv[j] = ldg4_stream(x + (size_t)row * D + c * 4);
      if (y) {
        const float4 yv = ld_bf16x4(y + (size_t)row * D + c * 4);
        xv[j] = make_float4(xv[j].x + yv.x, xv[j].y + yv.y, xv[j].z + yv.z, xv[j].w + yv.w);
        *reinterpret_cast<float4*>(xo + (size_t)row * D + c * 4) = xv[j];
      }
      s += (xv[j].x + xv[j].y) + (xv[j].z + xv[j].w);
    }
  }
  const float mean = warp_sum(s) / (float)D;
  float ss = 0.f;
#pragma unroll
  for (int j = 0; j < MAXV; ++j) {
    const int c = lane + 32 * j;
    if (c < nvec) {
      const float a0 = xv[j].x - mean, a1 = xv[j].y - mean, a2 = xv[j].z - mean, a3 = xv[j].w - mean;
      ss += (a0 * a0 + a1 * a1) + (a2 * a2 + a3 * a3);
    }
  }
  const float rstd = rsqrtf(warp_sum(ss) / (float)D + eps);
  if (lane == 0) {
    if (mean_out) mean_out[row] = mean;
    if (rstd_out) rstd_out[row] = rstd;
  }
#pragma unroll
  for (int j = 0; j < MAXV; ++j) {
    const int c = lane + 32 * j;
    if (c < nvec) {
      const float4 g = ldg4(w + c * 4), bb = ldg4(b + c * 4);
      st_bf16x4(h + (size_t)row * D + c * 4,
                make_float4(fmaf((xv[j].x - mean) * rstd, g.x, bb.x), fmaf((xv[j].y - mean) * rstd, g.y, bb.y),
                            fmaf((xv[j].z - mean) * rstd, g.z, bb.z), fmaf((xv[j].w - mean) * rstd, g.w, bb.w)));
    }
  }
}

// LayerNorm backward on the fp32 residual, one warp per row, grid-stride over rows with a fixed grid:
//   xhat = (x - mean) * rstd ; g = float(dy) * w ; dres' = dres + rstd * (g - mean(g) - xhat * mean(g * xhat))
// dres' is written in fp32 (dres_out may alias dres_in: each element is read, then written, by the same lane) and as a
// bf16 copy for the next branch's GEMMs; dres_in == nullptr reads zeros.  dw / db partial rows as in
// layernorm_bwd_kernel (per-warp shared slabs, one partial row per block, fixed-order reduction afterwards).
template <int MAXV>
__global__ void __launch_bounds__(LN_BWD_WARPS * 32)
layernorm_bwd_f32_kernel(const bf16* __restrict__ dy, const float* __restrict__ x, const float* __restrict__ w,
                         const float* __restrict__ mean_in, const float* __restrict__ rstd_in, const float* dres_in,
                         float* dres_out, bf16* __restrict__ dres16, float* __restrict__ dw_partial,
                         float* __restrict__ db_partial, int M, int D) {
  griddep_launch();
  griddep_wait();
  extern __shared__ float sacc[];   // [2][LN_BWD_WARPS][D]: dw, db
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nvec = D / 4;
  float* sw = sacc + (size_t)warp * D;
  float* sb = sacc + ((size_t)LN_BWD_WARPS + warp) * D;
  for (int e = lane; e < D; e += 32) sw[e] = sb[e] = 0.f;
  for (int row = blockIdx.x * LN_BWD_WARPS + warp; row < M; row += gridDim.x * LN_BWD_WARPS) {
    float4 xh[MAXV], gv[MAXV];
    const float mean = mean_in[row], rstd = rstd_in[row];
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int j = 0; j < MAXV; ++j) {
      const int c = lane + 32 * j;
      if (c < nvec) {
        const float4 xv = ldg4_stream(x + (size_t)row * D + c * 4);
        const float4 dv = ld_bf16x4(dy + (size_t)row * D + c * 4);
        const float4 wv = ldg4(w + c * 4);
        xh[j] = make_float4((xv.x - mean) * rstd, (xv.y - mean) * rstd, (xv.z - mean) * rstd, (xv.w - mean) * rstd);
        gv[j] = make_float4(dv.x * wv.x, dv.y * wv.y, dv.z * wv.z, dv.w * wv.w);
        s1 += (gv[j].x + gv[j].y) + (gv[j].z + gv[j].w);
        s2 += (gv[j].x * xh[j].x + gv[j].y * xh[j].y) + (gv[j].z * xh[j].z + gv[j].w * xh[j].w);
        const int e = c * 4;
        sw[e] = fmaf(dv.x, xh[j].x, sw[e]);
        sw[e + 1] = fmaf(dv.y, xh[j].y, sw[e + 1]);
        sw[e + 2] = fmaf(dv.z, xh[j].z, sw[e + 2]);
        sw[e + 3] = fmaf(dv.w, xh[j].w, sw[e + 3]);
        sb[e] += dv.x;
        sb[e + 1] += dv.y;
        sb[e + 2] += dv.z;
        sb[e + 3] += dv.w;
      }
    }
    const float m1 = warp_sum(s1) / (float)D, m2 = warp_sum(s2) / (float)D;
#pragma unroll
    for (int j = 0; j < MAXV; ++j) {
      const int c = lane + 32 * j;
      if (c < nvec) {
        const size_t o = (size_t)row * D + c * 4;
        const float4 r = dres_in ? *reinterpret_cast<const float4*>(dres_in + o) : make_float4(0.f, 0.f, 0.f, 0.f);
        const float4 d = make_float4(r.x + rstd * (gv[j].x - m1 - xh[j].x * m2), r.y + rstd * (gv[j].y - m1 - xh[j].y * m2),
                                     r.z + rstd * (gv[j].z - m1 - xh[j].z * m2), r.w + rstd * (gv[j].w - m1 - xh[j].w * m2));
        *reinterpret_cast<float4*>(dres_out + o) = d;
        st_bf16x4(dres16 + o, d);
      }
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < D; i += blockDim.x) {
    float a = 0.f, bsum = 0.f;
#pragma unroll
    for (int wi = 0; wi < LN_BWD_WARPS; ++wi) {
      a += sacc[(size_t)wi * D + i];
      bsum += sacc[((size_t)LN_BWD_WARPS + wi) * D + i];
    }
    dw_partial[(size_t)blockIdx.x * D + i] = a;
    db_partial[(size_t)blockIdx.x * D + i] = bsum;
  }
}

// table_fix[row(m)] += dx[m] for fp32 rows, in the 64-bit fixed point of embed_bwd_scatter_kernel (2^-40 units,
// order-independent).  row(m) = ids[m] (ids given; out-of-range ids are skipped) or the position-table row of m.
__global__ void scatter_rows_fix_f32_kernel(const int64_t* __restrict__ ids, const int32_t* __restrict__ pos_ids,
                                            const float* __restrict__ dx, unsigned long long* __restrict__ scratch, int M,
                                            int T, int D, int n_rows) {
  const int vec_per_row = D / 4;
  const long total = (long)M * vec_per_row;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int m = (int)(i / vec_per_row);
    const int c = (int)(i % vec_per_row);
    long r;
    if (ids) {
      r = ids[m];
      if (r < 0 || r >= n_rows) continue;
    } else {
      r = opt_pos_row(pos_ids, m, T, n_rows);
    }
    const float4 v = ldg4_stream(dx + (size_t)m * D + c * 4);
    const float f[4] = {v.x, v.y, v.z, v.w};
    unsigned long long* dst = scratch + (size_t)r * D + c * 4;
#pragma unroll
    for (int k = 0; k < 4; ++k)
      if (f[k] != 0.f) atomicAdd(dst + k, (unsigned long long)__float2ll_rn(f[k] * EMBED_FIX_SCALE));
  }
}

// grad = (keep ? grad : 0) + (float(head) + fix * 2^-40): the tied lm_head's bf16 gradient widened (head may be null)
// plus the embedding's own fp32 gradient, added to the fp32 .grad as autograd accumulates a leaf used twice
__global__ void add_fix_into_f32_kernel(float* __restrict__ grad, const unsigned long long* __restrict__ scratch,
                                        const bf16* __restrict__ head, long n, int keep) {
  for (long i = (blockIdx.x * (long)blockDim.x + threadIdx.x) * 4; i < n; i += (long)gridDim.x * blockDim.x * 4) {
    const ulonglong2 a = *reinterpret_cast<const ulonglong2*>(scratch + i);
    const ulonglong2 b = *reinterpret_cast<const ulonglong2*>(scratch + i + 2);
    float t[4] = {(float)((double)(long long)a.x * (1.0 / 1099511627776.0)), (float)((double)(long long)a.y * (1.0 / 1099511627776.0)),
                  (float)((double)(long long)b.x * (1.0 / 1099511627776.0)), (float)((double)(long long)b.y * (1.0 / 1099511627776.0))};
    if (head) {
      const float4 hv = ld_bf16x4(head + i);
      t[0] = hv.x + t[0]; t[1] = hv.y + t[1]; t[2] = hv.z + t[2]; t[3] = hv.w + t[3];
    }
    float4* g = reinterpret_cast<float4*>(grad + i);
    if (keep) {
      const float4 o = *g;
      t[0] = o.x + t[0]; t[1] = o.y + t[1]; t[2] = o.z + t[2]; t[3] = o.w + t[3];
    }
    *g = make_float4(t[0], t[1], t[2], t[3]);
  }
}

// g32 = (keep ? g32 : 0) + float(g16) over the listed chunks (the linear weights and biases, whose bf16 gradients the
// wgrad GEMMs and column sums write): the widening of autocast's bf16 dW into the fp32 .grad, one pass per micro-batch
__global__ void widen_grads_kernel(const bf16* __restrict__ g16, float* __restrict__ g32, const long* __restrict__ chunk_start,
                                   const int* __restrict__ chunk_len, int keep) {
  const long s = chunk_start[blockIdx.x];
  const int n = chunk_len[blockIdx.x];
  for (int i = threadIdx.x * 8; i < n; i += blockDim.x * 8) {
    const uint4 v = ldg128_stream(g16 + s + i);
    const float2 a = unpack_bf16(v.x), b = unpack_bf16(v.y), c = unpack_bf16(v.z), d = unpack_bf16(v.w);
    float4* o = reinterpret_cast<float4*>(g32 + s + i);
    float4 lo = make_float4(a.x, a.y, b.x, b.y), hi = make_float4(c.x, c.y, d.x, d.y);
    if (keep) {
      const float4 p = o[0], q = o[1];
      lo = make_float4(p.x + lo.x, p.y + lo.y, p.z + lo.z, p.w + lo.w);
      hi = make_float4(q.x + hi.x, q.y + hi.y, q.z + hi.z, q.w + hi.w);
    }
    o[0] = lo;
    o[1] = hi;
  }
}

// AdamW on fp32 master weights, element for element the arithmetic of torch's AdamW (fused=True) on fp32 tensors as
// written out in ATen's adam_math: every product, sum and quotient rounded on its own (no contraction), the clip
// coefficient applied to the gradient first.  Writes the master, both moments and the bf16 shadow the kernels read.
__global__ void adamw_master_kernel(float* __restrict__ p, bf16* __restrict__ shadow, const float* __restrict__ g,
                                    float* __restrict__ m, float* __restrict__ v, long n, float lr_wd, float one_m_b1,
                                    float beta2, float one_m_b2, float eps, float step_size, float bc2_sqrt,
                                    const float* __restrict__ clip_stats) {
  const float coef = clip_stats ? clip_stats[1] : 1.0f;
  for (long i = (blockIdx.x * (long)blockDim.x + threadIdx.x) * 4; i < n; i += (long)gridDim.x * blockDim.x * 4) {
    float4 pv = *reinterpret_cast<const float4*>(p + i), mv = *reinterpret_cast<const float4*>(m + i);
    float4 vv = *reinterpret_cast<const float4*>(v + i);
    const float4 gv = ldg4_stream(g + i);
    float* pp = &pv.x;
    float* mm = &mv.x;
    float* ss = &vv.x;
    const float gg[4] = {gv.x, gv.y, gv.z, gv.w};
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float grad = __fmul_rn(gg[e], coef);
      float param = __fsub_rn(pp[e], __fmul_rn(lr_wd, pp[e]));
      const float ea = __fadd_rn(mm[e], __fmul_rn(one_m_b1, __fsub_rn(grad, mm[e])));
      const float es = __fadd_rn(__fmul_rn(beta2, ss[e]), __fmul_rn(__fmul_rn(one_m_b2, grad), grad));
      const float denom = __fadd_rn(__fdiv_rn(__fsqrt_rn(es), bc2_sqrt), eps);
      param = __fsub_rn(param, __fdiv_rn(__fmul_rn(step_size, ea), denom));
      pp[e] = param;
      mm[e] = ea;
      ss[e] = es;
    }
    *reinterpret_cast<float4*>(p + i) = pv;
    *reinterpret_cast<float4*>(m + i) = mv;
    *reinterpret_cast<float4*>(v + i) = vv;
    st_bf16x4(shadow + i, pv);
  }
}

}  // namespace

int sk_opt_embed_fwd_f32_launch(const int64_t* ids, const int32_t* pos_ids, const float* E, const float* P, float* out, int M,
                                int T, int D, int V, int n_pos, cudaStream_t s) {
  SK_REQUIRE(D % 8 == 0 && n_pos > 0 && T > 0, "opt embed (fp32): D must be a multiple of 8");
  opt_embed_fwd_f32_kernel<<<grid_for((long)M * D / 4, 256), 256, 0, s>>>(ids, pos_ids, E, P, out, M, T, D, V, n_pos);
  SK_LAUNCH_CHECK();
  return 0;
}
int sk_add_layernorm_f32_launch(const float* x, const bf16* y, const float* w, const float* b, float* xo, bf16* h, float* mean,
                                float* rstd, int M, int D, float eps, cudaStream_t s) {
  SK_REQUIRE(D % 8 == 0 && D <= 2048, "add+layernorm (fp32): D must be a multiple of 8 and <= 2048 (D=%d)", D);
  SK_REQUIRE(y == nullptr || xo != nullptr, "add+layernorm (fp32): the sum x + y needs an output");
  const dim3 grid((M + WARPS_PER_BLOCK - 1) / WARPS_PER_BLOCK), block(WARPS_PER_BLOCK * 32);
  if (D <= 4 * VEC4_PER_WARP)
    SK_CUDA_CHECK(sk_launch_pdl(add_layernorm_f32_kernel<4>, grid, block, (size_t)0, s, x, y, w, b, xo, h, mean, rstd, M, D, eps));
  else if (D <= 8 * VEC4_PER_WARP)
    SK_CUDA_CHECK(sk_launch_pdl(add_layernorm_f32_kernel<8>, grid, block, (size_t)0, s, x, y, w, b, xo, h, mean, rstd, M, D, eps));
  else
    SK_CUDA_CHECK(sk_launch_pdl(add_layernorm_f32_kernel<16>, grid, block, (size_t)0, s, x, y, w, b, xo, h, mean, rstd, M, D, eps));
  SK_LAUNCH_CHECK();
  return 0;
}
// partial must hold 2 * sk_layernorm_bwd_blocks() * D floats
int sk_layernorm_bwd_f32_launch(const bf16* dy, const float* x, const float* w, const float* mean, const float* rstd,
                                const float* dres_in, float* dres_out, bf16* dres16, float* dw, float* db, float* partial, int M,
                                int D, int accumulate, cudaStream_t s) {
  SK_REQUIRE(D % 8 == 0 && D <= 2048, "layernorm backward (fp32): D must be a multiple of 8 and <= 2048 (D=%d)", D);
  SK_REQUIRE(M > 0, "layernorm backward (fp32): M must be positive");
  int blocks = sk_layernorm_bwd_blocks();
  const int need = (M + LN_BWD_WARPS - 1) / LN_BWD_WARPS;
  if (blocks > need) blocks = need;
  const size_t smem = (size_t)2 * LN_BWD_WARPS * D * sizeof(float);
  float* dwp = partial;
  float* dbp = partial + (size_t)blocks * D;
  const dim3 grid(blocks), block(LN_BWD_WARPS * 32);
  if (D <= 4 * VEC4_PER_WARP) {
    SK_CUDA_CHECK(sk_launch_pdl(layernorm_bwd_f32_kernel<4>, grid, block, smem, s, dy, x, w, mean, rstd, dres_in, dres_out, dres16,
                                dwp, dbp, M, D));
  } else if (D <= 8 * VEC4_PER_WARP) {
    SK_CUDA_CHECK(sk_launch_pdl(layernorm_bwd_f32_kernel<8>, grid, block, smem, s, dy, x, w, mean, rstd, dres_in, dres_out, dres16,
                                dwp, dbp, M, D));
  } else {
    SK_CUDA_CHECK(cudaFuncSetAttribute(layernorm_bwd_f32_kernel<16>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    SK_CUDA_CHECK(sk_launch_pdl(layernorm_bwd_f32_kernel<16>, grid, block, smem, s, dy, x, w, mean, rstd, dres_in, dres_out, dres16,
                                dwp, dbp, M, D));
  }
  SK_LAUNCH_CHECK();
  SK_CUDA_CHECK(sk_launch_pdl(colsum_reduce_kernel<float>, dim3((D + 31) / 32), dim3(1024), (size_t)0, s, (const float*)dwp, dw, blocks,
                              D, accumulate));
  SK_LAUNCH_CHECK();
  SK_CUDA_CHECK(sk_launch_pdl(colsum_reduce_kernel<float>, dim3((D + 31) / 32), dim3(1024), (size_t)0, s, (const float*)dbp, db, blocks,
                              D, accumulate));
  SK_LAUNCH_CHECK();
  return 0;
}
// Gradient of a table from fp32 rows: the 64-bit fixed point (2^-40 units; exact integer sums, so bit-identical run to
// run) resolves 9.1e-13 absolute per term -- fp32's own resolution for terms near 1e-5, finer above -- and holds sums
// below 2^23.  ids given: token table (n_rows = vocabulary), head = the tied lm_head's bf16 gradient or null; ids null:
// position table (n_rows = max_positions + 2).  keep: add to the fp32 gradient instead of overwriting it.
int sk_table_bwd_f32_launch(const int64_t* ids, const int32_t* pos_ids, const float* dx, float* scratch, float* dtable,
                            const bf16* head, int M, int T, int D, int n_rows, int n_rows_padded, int keep, cudaStream_t s) {
  SK_REQUIRE(D % 8 == 0 && n_rows > 0 && T > 0, "table backward (fp32): D must be a multiple of 8");
  unsigned long long* fix = reinterpret_cast<unsigned long long*>(scratch);
  const long n = (long)n_rows_padded * D;
  SK_CUDA_CHECK(cudaMemsetAsync(fix, 0, (size_t)n * sizeof(unsigned long long), s));
  scatter_rows_fix_f32_kernel<<<grid_for((long)M * D / 4, 256), 256, 0, s>>>(ids, pos_ids, dx, fix, M, T, D, n_rows);
  SK_LAUNCH_CHECK();
  add_fix_into_f32_kernel<<<grid_for(n / 4, 256), 256, 0, s>>>(dtable, fix, head, n, keep);
  SK_LAUNCH_CHECK();
  return 0;
}
int sk_widen_grads_launch(const bf16* g16, float* g32, const long* chunk_start, const int* chunk_len, int n_chunks, int keep,
                          cudaStream_t s) {
  if (n_chunks == 0) return 0;
  widen_grads_kernel<<<n_chunks, 256, 0, s>>>(g16, g32, chunk_start, chunk_len, keep);
  SK_LAUNCH_CHECK();
  return 0;
}
// The fp32 hyperparameters are combined on the host in double, as Python does before torch sees them: 1 - beta,
// lr * weight_decay, lr / (1 - beta1^step) and sqrt(1 - beta2^step), each rounded to fp32 once.
int sk_adamw_master_launch(float* p, bf16* shadow, const float* g, float* m, float* v, long n, float lr, float beta1, float beta2,
                           float eps, float wd, int step, const float* clip_stats, cudaStream_t s) {
  SK_REQUIRE(n % 8 == 0, "adamw (fp32): flat parameter count must be a multiple of 8 (n=%ld)", n);
  SK_REQUIRE(step >= 1, "adamw (fp32): step counts from 1");
  const double bc1 = 1.0 - pow((double)beta1, (double)step);
  const float bc2_sqrt = (float)sqrt(1.0 - pow((double)beta2, (double)step));
  adamw_master_kernel<<<grid_for(n / 4, 256, 8), 256, 0, s>>>(p, shadow, g, m, v, n, (float)((double)lr * (double)wd),
                                                              (float)(1.0 - (double)beta1), beta2, (float)(1.0 - (double)beta2),
                                                              eps, (float)((double)lr / bc1), bc2_sqrt, clip_stats);
  SK_LAUNCH_CHECK();
  return 0;
}
