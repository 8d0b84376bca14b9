// HiFi-GAN unit vocoder (CodeGenerator in eval mode, weight norm folded), sm_90a.
//
// Layout.  A batch is one time-major packed timeline: at unit-frame resolution row b occupies frames
// [start_b, start_b + F_b), rows are separated (and the timeline starts and ends) with G0 zero frames.  After upsampling
// stage i every frame is U_i positions, so the whole timeline scales uniformly (T_i = T0 * U_i) and a transposed
// convolution maps the packed input onto the packed output with one global index formula.  G0 is chosen at create
// time so that G0 * U_i covers the widest one-sided reach of every convolution at that resolution: no output of a
// row ever reads a neighbouring row.  Every layer writes zeros over the gap positions, so the gaps stay zero from layer
// to layer and from call to call.  Each output element then depends only on its own row's values and on a reduction
// order that does not depend on where the row sits: a row's waveform is bit-identical alone, in any batch and at any
// position.
//
// Convolutions are implicit GEMMs on the tensor cores (M = time, N = output channels, K = taps x input channels) with
// mma.sync m16n8k16 bf16 and fp32 accumulation, in the split-bf16 three-product form (hi*hi + hi*lo + lo*hi).  A time
// tile plus its halo is staged into shared memory once per 32-channel chunk, with the leaky ReLU and the hi/lo split
// fused into the staging, and every tap reads it at a row shift of tap * dilation.  That shift breaks the 8-row swizzle
// atom a wgmma shared-memory descriptor needs, so the A fragments come from ldmatrix of the shifted rows and the
// products run on mma.sync.  Transposed convolutions run polyphase: phase r of stride u uses taps r, r+u, ... and
// writes every u-th output.  Bias, gap masking, the ResBlock residual and the running ResBlock mean are fused into the
// epilogue.  conv_post (one output channel), the embeddings and the duration predictor run on CUDA cores in fp32.
#include "kernels.h"
#include "../../include/slamkit_b200.h"

#include <algorithm>
#include <new>
#include <string.h>
#include <vector>

namespace {

constexpr int BM = 128;      // time positions per CTA tile
constexpr int KC = 32;       // input channels per staged chunk
constexpr int LDS = KC + 8;  // smem row pitch in bf16 (80 bytes: 16-byte aligned rows, conflict-free ldmatrix)
constexpr int CPAD = 64;     // prepared weights: output channels padded to a multiple of this
constexpr int MAX_TAPS = 32;
constexpr size_t CONV_SMEM_MAX = 96 * 1024;   // dynamic shared memory a convolution may request
constexpr size_t DUR_SMEM_MAX = 48 * 1024;    // dur_kernel runs without raising the default limit

inline int64_t align_up(int64_t x, int64_t a) { return (x + a - 1) / a * a; }
inline int round_up(int x, int a) { return (x + a - 1) / a * a; }

// ---- one convolution layer as the kernel sees it ----------------------------------------------------------------
struct ConvParams {
  const float* x;             // [T_in, Cin] fp32
  int T_in, Cin, Cin_pad;
  const bf16* w_hi;           // [taps][Cout_pad][Cin_pad]
  const bf16* w_lo;
  int Cout, Cout_pad;
  int n_phase;                // 1 (conv) or u (transposed)
  int ntaps[MAX_TAPS];        // taps of each phase
  int tap_base[MAX_TAPS];     // first prepared tap of each phase
  int in_off0, in_step;       // input row of tap m = q + in_off0 + m * in_step
  int out_mul, out_off;       // output row = q * out_mul + phase + out_off
  int Q;                      // q in [0, Q)
  int T_out;
  float slope;                // leaky ReLU slope applied to the input as it is staged (1 = identity)
  const float* bias;          // [Cout]
  float* y;                   // [T_out, Cout] (mode 0)
  const float* res;           // residual [T_out, Cout] or null
  float* sum;                 // ResBlock mean accumulator [T_out, Cout] (modes 1, 2)
  int mode;                   // 0: y = v;  1: sum = v;  2: sum = sum + v
  int divide;                 // > 0: the stored sum is divided by this (the last ResBlock of a stage)
  const uint8_t* valid;       // [T0] frame-level row mask
  int up;                     // positions per frame at the output resolution
};


SK_DEVINL void ldsm_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];\n"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
SK_DEVINL void ldsm_x2(uint32_t addr, uint32_t& r0, uint32_t& r1) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x2.shared.b16 {%0,%1}, [%2];\n" : "=r"(r0), "=r"(r1) : "r"(addr));
}
SK_DEVINL void mma_bf16(float* c, const uint32_t* a, uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
               "{%0,%1,%2,%3};\n"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// CTA: BM time positions x BN = 16 * NT output channels, 8 warps as 4 (time) x 2 (channels); each warp owns two m16
// tiles x NT n8 tiles.  grid = (time tiles, channel tiles, phases).
template <int NT>
__global__ void __launch_bounds__(256, 2) vocoder_conv_kernel(const ConvParams p) {
  constexpr int BN = 16 * NT;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int phase = blockIdx.z;
  const int ntaps = p.ntaps[phase];
  const int tbase = p.tap_base[phase];
  const int off_min = p.in_off0 + min(0, (ntaps - 1) * p.in_step);
  const int span = (ntaps - 1) * abs(p.in_step);
  const int arows = BM + span;
  bf16* a_hi = reinterpret_cast<bf16*>(smem_raw);
  bf16* a_lo = a_hi + arows * LDS;
  bf16* b_hi = a_lo + arows * LDS;
  bf16* b_lo = b_hi + BN * LDS;

  const int q0 = blockIdx.x * BM;
  const int n0 = blockIdx.y * BN;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int wm = warp & 3, wn = warp >> 2;

  float acc[2][NT][4];
#pragma unroll
  for (int a = 0; a < 2; ++a)
#pragma unroll
    for (int b = 0; b < NT; ++b)
#pragma unroll
      for (int c = 0; c < 4; ++c) acc[a][b][c] = 0.f;

  for (int c0 = 0; c0 < p.Cin_pad; c0 += KC) {
    __syncthreads();
    // stage the activation tile + halo: leaky ReLU, then the hi / lo split
    for (int e = tid; e < arows * (KC / 4); e += 256) {
      const int r = e / (KC / 4), c = (e % (KC / 4)) * 4;
      const int g = q0 + off_min + r;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (g >= 0 && g < p.T_in && c0 + c < p.Cin) v = *reinterpret_cast<const float4*>(p.x + (int64_t)g * p.Cin + c0 + c);
      float f[4] = {v.x, v.y, v.z, v.w};
      bf16 h[4], l[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        float t = f[i] > 0.f ? f[i] : f[i] * p.slope;
        h[i] = __float2bfloat16_rn(t);
        l[i] = __float2bfloat16_rn(t - __bfloat162float(h[i]));
      }
      bf162* dh = reinterpret_cast<bf162*>(a_hi + r * LDS + c);
      bf162* dl = reinterpret_cast<bf162*>(a_lo + r * LDS + c);
      dh[0] = bf162(h[0], h[1]); dh[1] = bf162(h[2], h[3]);
      dl[0] = bf162(l[0], l[1]); dl[1] = bf162(l[2], l[3]);
    }
    const int ksteps = min(2, (p.Cin - c0 + 15) / 16);
    for (int m = 0; m < ntaps; ++m) {
      if (m > 0) __syncthreads();
      // stage the weights of this tap (already split at bind time)
      const int64_t wbase = ((int64_t)(tbase + m) * p.Cout_pad + n0) * p.Cin_pad + c0;
      for (int e = tid; e < 2 * BN * (KC / 8); e += 256) {
        const int which = e / (BN * (KC / 8)), rem = e % (BN * (KC / 8));
        const int r = rem / (KC / 8), c = (rem % (KC / 8)) * 8;
        const bf16* src = (which ? p.w_lo : p.w_hi) + wbase + (int64_t)r * p.Cin_pad + c;
        *reinterpret_cast<uint4*>((which ? b_lo : b_hi) + r * LDS + c) = *reinterpret_cast<const uint4*>(src);
      }
      __syncthreads();
      const int ashift = p.in_off0 + m * p.in_step - off_min;
      for (int ks = 0; ks < ksteps; ++ks) {
        uint32_t ah[2][4], al[2][4];
#pragma unroll
        for (int mt = 0; mt < 2; ++mt) {
          const int row = ashift + wm * 32 + mt * 16 + (lane & 15);
          const int col = ks * 16 + (lane >> 4) * 8;
          ldsm_x4(smem_u32(a_hi + row * LDS + col), ah[mt][0], ah[mt][1], ah[mt][2], ah[mt][3]);
          ldsm_x4(smem_u32(a_lo + row * LDS + col), al[mt][0], al[mt][1], al[mt][2], al[mt][3]);
        }
#pragma unroll
        for (int nt = 0; nt < NT; ++nt) {
          const int nrow = wn * (BN / 2) + nt * 8 + (lane & 7);
          const int col = ks * 16 + ((lane >> 3) & 1) * 8;
          uint32_t bh0, bh1, bl0, bl1;
          ldsm_x2(smem_u32(b_hi + nrow * LDS + col), bh0, bh1);
          ldsm_x2(smem_u32(b_lo + nrow * LDS + col), bl0, bl1);
#pragma unroll
          for (int mt = 0; mt < 2; ++mt) {
            mma_bf16(acc[mt][nt], ah[mt], bh0, bh1);
            mma_bf16(acc[mt][nt], ah[mt], bl0, bl1);
            mma_bf16(acc[mt][nt], al[mt], bh0, bh1);
          }
        }
      }
    }
  }

  // epilogue: bias, gap mask, residual, ResBlock mean
  const int g = lane >> 2, t4 = lane & 3;
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int half = 0; half < 2; ++half) {
      const int q = q0 + wm * 32 + mt * 16 + g + half * 8;
      if (q >= p.Q) continue;
      const int o = q * p.out_mul + phase + p.out_off;
      if (o < 0 || o >= p.T_out) continue;
      const bool live = p.valid[o / p.up] != 0;
#pragma unroll
      for (int nt = 0; nt < NT; ++nt) {
        const int co = n0 + wn * (BN / 2) + nt * 8 + 2 * t4;
        if (co >= p.Cout) continue;
        const int64_t idx = (int64_t)o * p.Cout + co;
        float v0 = 0.f, v1 = 0.f;
        if (live) {
          v0 = acc[mt][nt][half * 2 + 0] + p.bias[co];
          v1 = acc[mt][nt][half * 2 + 1] + p.bias[co + 1];
          if (p.res) {
            const float2 r = *reinterpret_cast<const float2*>(p.res + idx);
            v0 += r.x; v1 += r.y;
          }
          if (p.mode == 2) {
            const float2 s = *reinterpret_cast<const float2*>(p.sum + idx);
            v0 = s.x + v0; v1 = s.y + v1;
          }
          if (p.divide > 0) { v0 = v0 / (float)p.divide; v1 = v1 / (float)p.divide; }
        }
        *reinterpret_cast<float2*>((p.mode ? p.sum : p.y) + idx) = make_float2(v0, v1);
      }
    }
}

// ---- codes -> units -> durations -> frames --------------------------------------------------------------------------
// One warp per row: drop negative codes (CodeHiFiGANVocoder.forward's `code >= 0` mask), flag and zero codes past the
// embedding table so nothing is ever read out of bounds.
__global__ void compact_kernel(const int64_t* codes, int ld, const int32_t* counts, int B, int num_emb, int max_units,
                               int32_t* units, int32_t* n_units, int32_t* bad) {
  const int b = blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32, lane = threadIdx.x & 31;
  if (b >= B) return;
  const int n = min(max(counts[b], 0), ld);
  int k = 0, nbad = 0;
  for (int i0 = 0; i0 < n; i0 += 32) {
    const int i = i0 + lane;
    const int64_t c = i < n ? codes[(int64_t)b * ld + i] : -1;
    const bool keep = c >= 0;
    const unsigned m = __ballot_sync(0xffffffffu, keep);
    const int pos = k + __popc(m & ((1u << lane) - 1));
    if (keep) {
      const bool oob = c >= num_emb;
      nbad += oob;
      if (pos < max_units) units[(int64_t)b * max_units + pos] = oob ? 0 : (int32_t)c;
    }
    k += __popc(m);
  }
  for (int o = 16; o; o >>= 1) nbad += __shfl_xor_sync(0xffffffffu, nbad, o);
  if (lane == 0) {
    n_units[b] = k;
    if (nbad) atomicAdd(bad, nbad);
    if (k > max_units) atomicAdd(bad + 1, 1);
  }
}

SK_DEVINL float block_sum(float v, float* red) {
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  const int w = threadIdx.x >> 5, nw = blockDim.x >> 5;
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[w] = v;
  __syncthreads();
  float s = 0.f;
  for (int i = 0; i < nw; ++i) s += red[i];
  return s;
}

// VariancePredictor (conv k=3 + ReLU + LayerNorm, twice, then Linear) for one unit per CTA, fp32, blockDim = round_up(H, 32).
// The three LayerNorm-1 outputs conv2 needs are recomputed here rather than stored.
__global__ void dur_kernel(const int32_t* units, const int32_t* n_units, int max_units, const float* emb, int E, int H,
                           const float* c1w, const float* c1b, const float* l1w, const float* l1b, const float* c2w,
                           const float* c2b, const float* l2w, const float* l2b, const float* pw, const float* pb,
                           int32_t* dur, float* logd) {
  extern __shared__ float sm[];
  float* xe = sm;              // [5][E] embeddings at i-2 .. i+2
  float* h1 = xe + 5 * E;      // [3][H] LayerNorm-1 outputs at i-1 .. i+1
  float* red = h1 + 3 * H;     // [32]
  const int b = blockIdx.y, i = blockIdx.x, n = n_units[b];
  if (i >= min(n, max_units)) return;
  const int32_t* u = units + (int64_t)b * max_units;
  for (int e = threadIdx.x; e < 5 * E; e += blockDim.x) {
    const int j = i - 2 + e / E;
    xe[e] = (j >= 0 && j < n) ? emb[(int64_t)u[j] * E + e % E] : 0.f;
  }
  __syncthreads();
  const int h = threadIdx.x;
  for (int s = 0; s < 3; ++s) {
    const int j = i - 1 + s;
    float a = 0.f;
    if (h < H) {
      a = c1b[h];
      for (int c = 0; c < E; ++c)
        for (int k = 0; k < 3; ++k) a += c1w[((int64_t)h * E + c) * 3 + k] * xe[(s + k) * E + c];
      a = fmaxf(a, 0.f);
    }
    const float mean = block_sum(h < H ? a : 0.f, red) / H;
    const float d = h < H ? a - mean : 0.f;
    const float var = block_sum(d * d, red) / H;
    if (h < H) h1[s * H + h] = (j >= 0 && j < n) ? d * rsqrtf(var + 1e-5f) * l1w[h] + l1b[h] : 0.f;
  }
  __syncthreads();
  float a = 0.f;
  if (h < H) {
    a = c2b[h];
    for (int c = 0; c < H; ++c)
      for (int k = 0; k < 3; ++k) a += c2w[((int64_t)h * H + c) * 3 + k] * h1[k * H + c];
    a = fmaxf(a, 0.f);
  }
  const float mean = block_sum(h < H ? a : 0.f, red) / H;
  const float d = h < H ? a - mean : 0.f;
  const float var = block_sum(d * d, red) / H;
  const float z = h < H ? (d * rsqrtf(var + 1e-5f) * l2w[h] + l2b[h]) * pw[h] : 0.f;
  const float v = block_sum(z, red) + pb[0];
  if (threadIdx.x == 0) {
    // torch.clamp(torch.round(torch.exp(v) - 1), min=1): round half to even
    dur[(int64_t)b * max_units + i] = max(1, (int)rintf(expf(v) - 1.f));
    if (logd) logd[(int64_t)b * max_units + i] = v;
  }
}

// Inclusive prefix of each row's durations (1 per unit without a predictor) and the row's frame count.
__global__ void cum_kernel(const int32_t* n_units, int B, int max_units, int has_dur, int32_t* dur, int32_t* cum,
                           int32_t* frames) {
  const int b = blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32, lane = threadIdx.x & 31;
  if (b >= B) return;
  const int n = min(n_units[b], max_units);
  int run = 0;
  for (int i0 = 0; i0 < n; i0 += 32) {
    const int i = i0 + lane;
    int d = 0;
    if (i < n) {
      if (!has_dur) dur[(int64_t)b * max_units + i] = 1;
      d = has_dur ? dur[(int64_t)b * max_units + i] : 1;
    }
    int x = d;
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, x, o);
      if (lane >= o) x += y;
    }
    if (i < n) cum[(int64_t)b * max_units + i] = run + x;
    run += __shfl_sync(0xffffffffu, x, 31);
  }
  if (lane == 0) frames[b] = run;
}

__global__ void starts_kernel(const int32_t* frames, int B, int G0, int32_t* starts) {
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    int s = G0;
    for (int b = 0; b < B; ++b) { starts[b] = s; s += frames[b] + G0; }
    starts[B] = s;
  }
}

// Frame-level input of conv_pre: [code embedding | speaker 0 | style 0] of the unit covering each frame, zero in gaps.
__global__ void expand_kernel(const int32_t* units, const int32_t* n_units, const int32_t* cum, const int32_t* starts,
                              const int32_t* frames, int B, int max_units, int T0, const float* emb, const float* spk, const float* sty, int E,
                              int Cin, float* x0, uint8_t* valid) {
  const int f = blockIdx.x;
  if (f >= T0) return;
  int lo = 0, hi = B - 1;    // last row with starts[row] <= f
  if (f < starts[0]) hi = -1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (starts[mid] <= f) lo = mid; else hi = mid - 1;
  }
  const int b = hi;
  const int local = b >= 0 ? f - starts[b] : -1;
  const bool live = b >= 0 && local < frames[b];
  int unit = 0;
  if (live) {
    const int32_t* c = cum + (int64_t)b * max_units;
    int a = 0, z = min(n_units[b], max_units) - 1;   // first unit with cum > local
    while (a < z) {
      const int mid = (a + z) >> 1;
      if (c[mid] > local) z = mid; else a = mid + 1;
    }
    unit = units[(int64_t)b * max_units + a];
  }
  if (threadIdx.x == 0) valid[f] = live;
  for (int ch = threadIdx.x; ch < Cin; ch += blockDim.x) {
    float v = 0.f;
    if (live) v = ch < E ? emb[(int64_t)unit * E + ch] : (spk && ch < 2 * E) ? spk[ch - E] : sty[ch - (spk ? 2 * E : E)];
    x0[(int64_t)f * Cin + ch] = v;
  }
}

// conv_post (Cout = 1, k = 7, padding 3) after leaky_relu(0.01), then tanh, written per row into the padded waveform.
__global__ void post_kernel(const float* x, int C, const float* w, const float* bias, const int32_t* starts,
                            const int32_t* frames, int U, int B, float* wave, int ldw) {
  const int b = blockIdx.y;
  const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B || p >= ldw) return;
  const int64_t len = (int64_t)frames[b] * U;
  float out = 0.f;
  if (p < len) {
    const int64_t o = (int64_t)starts[b] * U + p;
    float a = 0.f;
    for (int c = 0; c < C; ++c)
      for (int k = 0; k < 7; ++k) {
        const float v = x[(o + k - 3) * C + c];
        a += w[c * 7 + k] * (v > 0.f ? v : 0.01f * v);
      }
    out = tanhf(a + bias[0]);
  }
  wave[(int64_t)b * ldw + p] = out;
}

// folded fp32 conv weight [Cout][Cin][k] (or [Cin][Cout][k] transposed) -> split bf16 [tap][Cout_pad][Cin_pad]
__global__ void prepare_kernel(const float* w, int Cout, int Cin, int k, int transposed, int u, int Cout_pad, int Cin_pad,
                               bf16* hi, bf16* lo) {
  const int64_t n = (int64_t)k * Cout_pad * Cin_pad;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (int64_t)gridDim.x * blockDim.x) {
    const int ci = e % Cin_pad, co = (e / Cin_pad) % Cout_pad, tap = e / ((int64_t)Cin_pad * Cout_pad);
    float v = 0.f;
    if (ci < Cin && co < Cout) {
      if (!transposed) {
        v = w[((int64_t)co * Cin + ci) * k + tap];
      } else {   // tap index runs over phases r = 0..u-1, then taps j = r, r+u, ...
        int r = 0, base = 0;
        while (base + (k - r + u - 1) / u <= tap) { base += (k - r + u - 1) / u; ++r; }
        const int j = r + (tap - base) * u;
        v = w[((int64_t)ci * Cout + co) * k + j];
      }
    }
    const bf16 h = __float2bfloat16_rn(v);
    hi[e] = h;
    lo[e] = __float2bfloat16_rn(v - __bfloat162float(h));
  }
}

struct Tensor {
  char name[64];
  int64_t off, numel;
};

// One convolution layer: offsets of its fp32 weight and bias in the flat buffer and of its prepared split weights.
struct ConvLayer { int64_t w, b, prep; int Cout, Cin, k, transposed, u, dil, Cout_pad, Cin_pad; };

ConvLayer conv_layer(int Cout, int Cin, int k, int transposed, int u, int dil) {
  ConvLayer L;
  L.w = L.b = L.prep = 0;
  L.Cout = Cout; L.Cin = Cin; L.k = k; L.transposed = transposed; L.u = u; L.dil = dil;
  L.Cout_pad = round_up(Cout, CPAD);
  L.Cin_pad = round_up(Cin, KC);
  return L;
}

int64_t prep_elems(const ConvLayer& L) { return (int64_t)L.k * L.Cout_pad * L.Cin_pad; }

// tile width (n8 tiles per warp) the launcher picks from the output channels
int conv_nt(int Cout) { return Cout >= 64 ? 4 : Cout >= 32 ? 2 : 1; }

// dynamic shared memory of a conv CTA: the activation tile plus a halo of `span` rows (hi and lo), and one tap's weights
size_t conv_smem_bytes(int span, int NT) { return ((size_t)2 * (BM + span) * LDS + 2 * 16 * NT * LDS) * sizeof(bf16); }

// widest halo of the layer's phases, in rows
int halo_span(const ConvLayer& L) { return L.transposed ? (L.k + L.u - 1) / L.u - 1 : (L.k - 1) * L.dil; }

size_t dur_smem_bytes(int E, int H) { return (5 * (size_t)E + 3 * (size_t)H + 32) * sizeof(float); }

int prepare_layer(const ConvLayer& L, const float* w, bf16* hi, bf16* lo, cudaStream_t s) {
  const int blocks = (int)std::min<int64_t>((prep_elems(L) + 255) / 256, 4096);
  prepare_kernel<<<blocks, 256, 0, s>>>(w, L.Cout, L.Cin, L.k, L.transposed, L.u, L.Cout_pad, L.Cin_pad, hi, lo);
  SK_LAUNCH_CHECK();
  return 0;
}

}  // namespace

struct SkVocoder {
  SkVocoderConfig cfg;
  int in_dim, G0, U_total;
  std::vector<Tensor> tensors;
  int64_t n_params = 0;
  // prepared conv layers (order: conv_pre, per stage: ups, resblocks' convs1/convs2 interleaved)
  std::vector<ConvLayer> layers;
  int64_t prep_elems = 0;
  int64_t t_dict = -1, t_spk = -1, t_sty = -1, t_dur = -1, t_post_w = -1, t_post_b = -1;
  int64_t T0_cap = 0, act_elems = 0;
  const float* w = nullptr;
  bf16 *hi = nullptr, *lo = nullptr;
  unsigned char* ws = nullptr;
  // workspace carve-up
  int32_t *units, *n_units, *dur, *cum, *frames, *starts, *bad;
  float *logd, *x0, *buf[4];
  uint8_t* valid;
};

namespace {

int64_t add_tensor(SkVocoder* v, const char* name, int64_t numel) {
  Tensor t;
  snprintf(t.name, sizeof t.name, "%s", name);
  t.off = v->n_params;
  t.numel = numel;
  v->tensors.push_back(t);
  v->n_params += align_up(numel, 4);
  return t.off;
}

void add_conv(SkVocoder* v, const char* base, int Cout, int Cin, int k, int transposed, int u, int dil) {
  char nm[64];
  ConvLayer L = conv_layer(Cout, Cin, k, transposed, u, dil);
  snprintf(nm, sizeof nm, "%s.weight", base);
  L.w = add_tensor(v, nm, (int64_t)Cout * Cin * k);
  snprintf(nm, sizeof nm, "%s.bias", base);
  L.b = add_tensor(v, nm, Cout);
  L.prep = v->prep_elems;
  v->prep_elems += align_up(prep_elems(L), 128);
  v->layers.push_back(L);
}

template <int NT>
int launch_conv_nt(const ConvParams& p, int n_tiles_m, cudaStream_t s) {
  constexpr int BN = 16 * NT;
  int maxspan = 0;
  for (int r = 0; r < p.n_phase; ++r) maxspan = std::max(maxspan, (p.ntaps[r] - 1) * abs(p.in_step));
  const size_t smem = conv_smem_bytes(maxspan, NT);
  SK_REQUIRE(smem <= CONV_SMEM_MAX, "sk_vocoder: convolution halo too wide (%zu bytes of shared memory)", smem);
  SK_CUDA_CHECK(cudaFuncSetAttribute(vocoder_conv_kernel<NT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  dim3 grid(n_tiles_m, (p.Cout + BN - 1) / BN, p.n_phase);
  vocoder_conv_kernel<NT><<<grid, 256, smem, s>>>(p);
  SK_LAUNCH_CHECK();
  return 0;
}

int launch_conv(const ConvParams& p, cudaStream_t s) {
  const int tiles = (p.Q + BM - 1) / BM;
  switch (conv_nt(p.Cout)) {
    case 4: return launch_conv_nt<4>(p, tiles, s);
    case 2: return launch_conv_nt<2>(p, tiles, s);
    default: return launch_conv_nt<1>(p, tiles, s);
  }
}

// One convolution layer over the packed timeline at `up` positions per frame, from its prepared (split) weights.
// The network and the sk_vocoder_conv test hook both run every layer through here.
int run_layer(const ConvLayer& L, const bf16* w_hi, const bf16* w_lo, const float* bias, const uint8_t* valid,
              const float* x, int T_in, int T_out, float slope, float* y, const float* res, float* sum, int mode, int divide,
              int up, cudaStream_t s) {
  ConvParams p;
  memset(&p, 0, sizeof p);
  p.x = x; p.T_in = T_in; p.Cin = L.Cin; p.Cin_pad = L.Cin_pad;
  p.w_hi = w_hi; p.w_lo = w_lo;
  p.Cout = L.Cout; p.Cout_pad = L.Cout_pad;
  if (!L.transposed) {
    const int pad = (L.k * L.dil - L.dil) / 2;
    p.n_phase = 1; p.ntaps[0] = L.k; p.tap_base[0] = 0;
    p.in_off0 = -pad; p.in_step = L.dil;
    p.out_mul = 1; p.out_off = 0; p.Q = T_out;
  } else {
    const int u = L.u, pad = (L.k - u) / 2;
    p.n_phase = u;
    int base = 0;
    for (int r = 0; r < u; ++r) { p.ntaps[r] = (L.k - r + u - 1) / u; p.tap_base[r] = base; base += p.ntaps[r]; }
    p.in_off0 = 0; p.in_step = -1;
    p.out_mul = u; p.out_off = -pad; p.Q = T_in + (pad + u - 1) / u;
  }
  p.T_out = T_out; p.slope = slope;
  p.bias = bias; p.y = y; p.res = res; p.sum = sum; p.mode = mode; p.divide = divide;
  p.valid = valid; p.up = up;
  return launch_conv(p, s);
}

#define VOC_TRY(x) do { int _r = (x); if (_r) return _r; } while (0)

// Durations and frame counts of rows [0, B) of the given codes into the workspace (no host synchronisation).
int enqueue_durations(SkVocoder* v, const int64_t* codes, int ld, const int32_t* counts, int B, cudaStream_t s) {
  const SkVocoderConfig& c = v->cfg;
  const int MU = c.max_frames;
  compact_kernel<<<(B + 3) / 4, 128, 0, s>>>(codes, ld, counts, B, c.num_embeddings, MU, v->units, v->n_units, v->bad);
  SK_LAUNCH_CHECK();
  if (c.dur_predictor) {
    const int H = c.dur_hidden, E = c.embedding_dim;
    const int64_t d = v->t_dur;
    const float* W = v->w;
    const int threads = round_up(H, 32);
    const size_t smem = dur_smem_bytes(E, H);
    dim3 grid(std::min(ld, MU), B);
    // tensor order: conv1.w, conv1.b, ln1.w, ln1.b, conv2.w, conv2.b, ln2.w, ln2.b, proj.w, proj.b
    const int64_t o_c1w = d, o_c1b = o_c1w + align_up((int64_t)H * E * 3, 4), o_l1w = o_c1b + align_up(H, 4),
                  o_l1b = o_l1w + align_up(H, 4), o_c2w = o_l1b + align_up(H, 4), o_c2b = o_c2w + align_up((int64_t)H * H * 3, 4),
                  o_l2w = o_c2b + align_up(H, 4), o_l2b = o_l2w + align_up(H, 4), o_pw = o_l2b + align_up(H, 4),
                  o_pb = o_pw + align_up(H, 4);
    dur_kernel<<<grid, threads, smem, s>>>(v->units, v->n_units, MU, W + v->t_dict, E, H, W + o_c1w, W + o_c1b, W + o_l1w,
                                           W + o_l1b, W + o_c2w, W + o_c2b, W + o_l2w, W + o_l2b, W + o_pw, W + o_pb,
                                           v->dur, v->logd);
    SK_LAUNCH_CHECK();
  }
  cum_kernel<<<(B + 3) / 4, 128, 0, s>>>(v->n_units, B, MU, c.dur_predictor, v->dur, v->cum, v->frames);
  SK_LAUNCH_CHECK();
  return 0;
}

int enqueue_network(SkVocoder* v, int B, int T0, float* wave, int ldw, cudaStream_t s) {
  const SkVocoderConfig& c = v->cfg;
  const float* W = v->w;
  starts_kernel<<<1, 32, 0, s>>>(v->frames, B, v->G0, v->starts);
  SK_LAUNCH_CHECK();
  expand_kernel<<<T0, 128, 0, s>>>(v->units, v->n_units, v->cum, v->starts, v->frames, B, c.max_frames, T0, W + v->t_dict,
                                   v->t_spk >= 0 ? W + v->t_spk : nullptr, v->t_sty >= 0 ? W + v->t_sty : nullptr,
                                   c.embedding_dim, v->in_dim, v->x0, v->valid);
  SK_LAUNCH_CHECK();
  const int nk = c.n_resblocks;
  size_t li = 0;
  float *X = v->buf[0], *Y = v->buf[1], *Tm = v->buf[2], *S = v->buf[3];
  auto run = [&](const ConvLayer& L, const float* x, int T_in, int T_out, float slope, float* y, const float* res, float* sum,
                 int mode, int divide, int up) {
    return run_layer(L, v->hi + L.prep, v->lo + L.prep, W + L.b, v->valid, x, T_in, T_out, slope, y, res, sum, mode, divide,
                     up, s);
  };
  VOC_TRY(run(v->layers[li++], v->x0, T0, T0, 1.f, S, nullptr, nullptr, 0, 0, 1));   // conv_pre
  int U = 1;
  for (int i = 0; i < c.n_upsamples; ++i) {
    const int T_in = T0 * U, u = c.upsample_rates[i];
    U *= u;
    const int T = T0 * U;
    VOC_TRY(run(v->layers[li++], S, T_in, T, 0.1f, X, nullptr, nullptr, 0, 0, U));     // ups[i]
    for (int j = 0; j < nk; ++j) {
      const float* cur = X;
      for (int a = 0; a < 3; ++a) {
        const ConvLayer& c1 = v->layers[li++];
        const ConvLayer& c2 = v->layers[li++];
        VOC_TRY(run(c1, cur, T, T, 0.1f, Tm, nullptr, nullptr, 0, 0, U));
        if (a < 2) {
          VOC_TRY(run(c2, Tm, T, T, 0.1f, Y, cur, nullptr, 0, 0, U));
          cur = Y;
        } else {   // last conv of the ResBlock: add the residual, then into the running sum (and the mean at the end)
          VOC_TRY(run(c2, Tm, T, T, 0.1f, nullptr, cur, S, j == 0 ? 1 : 2, j == nk - 1 ? nk : 0, U));
        }
      }
    }
  }
  const int C = v->layers.back().Cout;
  dim3 grid((ldw + 255) / 256, B);
  post_kernel<<<grid, 256, 0, s>>>(S, C, W + v->t_post_w, W + v->t_post_b, v->starts, v->frames, U, B, wave, ldw);
  SK_LAUNCH_CHECK();
  return 0;
}

}  // namespace

extern "C" {

int sk_vocoder_create(const SkVocoderConfig* cfg, SkVocoder** out) {
  SK_REQUIRE(cfg && out, "sk_vocoder_create: null argument");
  const SkVocoderConfig& c = *cfg;
  SK_REQUIRE(c.num_embeddings > 0 && c.embedding_dim > 0 && c.embedding_dim % 4 == 0,
             "sk_vocoder_create: embedding_dim must be a positive multiple of 4");
  SK_REQUIRE(c.n_upsamples >= 1 && c.n_upsamples <= 8, "sk_vocoder_create: 1..8 upsampling stages");
  SK_REQUIRE(c.n_resblocks >= 1 && c.n_resblocks <= 4, "sk_vocoder_create: 1..4 ResBlocks per stage");
  SK_REQUIRE(c.max_rows >= 1 && c.max_frames >= 1, "sk_vocoder_create: max_rows and max_frames must be positive");
  const int in_dim = c.embedding_dim * (1 + (c.multispkr ? 1 : 0) + (c.multistyle ? 1 : 0));
  SK_REQUIRE(c.model_in_dim == in_dim, "sk_vocoder_create: model_in_dim %d != embedding_dim x (1 + multispkr + multistyle) = %d",
             c.model_in_dim, in_dim);
  SK_REQUIRE(c.upsample_initial_channel > 0 && c.upsample_initial_channel % (4 << c.n_upsamples) == 0,
             "sk_vocoder_create: every stage's channel count must be a multiple of 4");
  int U = 1;
  int G0 = 3;                               // conv_pre reach at frame resolution
  for (int i = 0; i < c.n_upsamples; ++i) {
    const int u = c.upsample_rates[i], k = c.upsample_kernel_sizes[i];
    SK_REQUIRE(u >= 1 && u <= MAX_TAPS && k >= u && k <= MAX_TAPS, "sk_vocoder_create: stage %d: need 1 <= rate <= kernel <= %d",
               i, MAX_TAPS);
    SK_REQUIRE((k - u) % 2 == 0, "sk_vocoder_create: stage %d: kernel - rate must be even (each frame must map to exactly "
               "rate samples)", i);
    G0 = std::max(G0, ((k + u - 1) / u + 1 + U - 1) / U);   // transposed-conv input reach at the stage's input resolution
    U *= u;
    const int ch = c.upsample_initial_channel >> (i + 1);
    int reach = 0;
    for (int j = 0; j < c.n_resblocks; ++j) {
      const int rk = c.resblock_kernel_sizes[j];
      SK_REQUIRE(rk % 2 == 1 && rk <= MAX_TAPS, "sk_vocoder_create: ResBlock kernels must be odd, <= %d", MAX_TAPS);
      for (int a = 0; a < 3; ++a) {
        const int dil = c.resblock_dilations[j][a];
        SK_REQUIRE(dil >= 1 && dil <= 1024, "sk_vocoder_create: dilations must be in [1, 1024]");
        const size_t smem = conv_smem_bytes((rk - 1) * dil, conv_nt(ch));
        SK_REQUIRE(smem <= CONV_SMEM_MAX, "sk_vocoder_create: stage %d: ResBlock kernel %d at dilation %d (%d channels) "
                   "needs %zu bytes of shared memory for its halo, more than %zu", i, rk, dil, ch, smem, CONV_SMEM_MAX);
        reach = std::max(reach, (rk - 1) * dil / 2);
      }
    }
    G0 = std::max(G0, (reach + U - 1) / U);
  }
  G0 = std::max(G0, (3 + U - 1) / U);       // conv_post
  SK_REQUIRE(!c.dur_predictor || (c.dur_kernel == 3 && c.dur_hidden >= 1 && c.dur_hidden <= 1024),
             "sk_vocoder_create: the duration predictor needs var_pred_kernel_size 3 (its second conv has padding 1) and "
             "var_pred_hidden_dim <= 1024");
  SK_REQUIRE(!c.dur_predictor || dur_smem_bytes(c.embedding_dim, c.dur_hidden) <= DUR_SMEM_MAX,
             "sk_vocoder_create: the duration predictor needs (5 x embedding_dim + 3 x var_pred_hidden_dim + 32) x 4 = %zu "
             "bytes of shared memory (embedding_dim %d, var_pred_hidden_dim %d), more than %zu",
             dur_smem_bytes(c.embedding_dim, c.dur_hidden), c.embedding_dim, c.dur_hidden, DUR_SMEM_MAX);
  SkVocoder* v = new (std::nothrow) SkVocoder();
  SK_REQUIRE(v, "sk_vocoder_create: out of host memory");
  v->cfg = c;
  v->in_dim = in_dim;
  v->G0 = G0;
  v->U_total = U;
  const int E = c.embedding_dim, H = c.dur_hidden;
  v->t_dict = add_tensor(v, "dict.weight", (int64_t)c.num_embeddings * E);
  if (c.multispkr) v->t_spk = add_tensor(v, "spkr.weight", (int64_t)c.num_speakers * E);
  if (c.multistyle) v->t_sty = add_tensor(v, "style.weight", (int64_t)c.num_styles * E);
  if (c.dur_predictor) {
    v->t_dur = add_tensor(v, "dur_predictor.conv1.0.weight", (int64_t)H * E * 3);
    add_tensor(v, "dur_predictor.conv1.0.bias", H);
    add_tensor(v, "dur_predictor.ln1.weight", H);
    add_tensor(v, "dur_predictor.ln1.bias", H);
    add_tensor(v, "dur_predictor.conv2.0.weight", (int64_t)H * H * 3);
    add_tensor(v, "dur_predictor.conv2.0.bias", H);
    add_tensor(v, "dur_predictor.ln2.weight", H);
    add_tensor(v, "dur_predictor.ln2.bias", H);
    add_tensor(v, "dur_predictor.proj.weight", H);
    add_tensor(v, "dur_predictor.proj.bias", 1);
  }
  const int C0 = c.upsample_initial_channel;
  add_conv(v, "conv_pre", C0, in_dim, 7, 0, 1, 1);
  char nm[64];
  int ch = C0;
  int64_t act = (int64_t)C0;   // conv_pre output per frame
  U = 1;
  for (int i = 0; i < c.n_upsamples; ++i) {
    snprintf(nm, sizeof nm, "ups.%d", i);
    add_conv(v, nm, ch / 2, ch, c.upsample_kernel_sizes[i], 1, c.upsample_rates[i], 1);
    ch /= 2;
    U *= c.upsample_rates[i];
    act = std::max(act, (int64_t)U * ch);
    for (int j = 0; j < c.n_resblocks; ++j)
      for (int a = 0; a < 3; ++a) {
        snprintf(nm, sizeof nm, "resblocks.%d.convs1.%d", i * c.n_resblocks + j, a);
        add_conv(v, nm, ch, ch, c.resblock_kernel_sizes[j], 0, 1, c.resblock_dilations[j][a]);
        snprintf(nm, sizeof nm, "resblocks.%d.convs2.%d", i * c.n_resblocks + j, a);
        add_conv(v, nm, ch, ch, c.resblock_kernel_sizes[j], 0, 1, 1);
      }
  }
  v->t_post_w = add_tensor(v, "conv_post.weight", (int64_t)ch * 7);
  v->t_post_b = add_tensor(v, "conv_post.bias", 1);
  v->T0_cap = (int64_t)c.max_frames + (int64_t)(c.max_rows + 1) * G0;
  v->act_elems = v->T0_cap * act;
  *out = v;
  return 0;
}

void sk_vocoder_destroy(SkVocoder* v) { delete v; }

int64_t sk_vocoder_param_count(const SkVocoder* v) { return v ? v->n_params : -1; }

int sk_vocoder_tensor_info(const SkVocoder* v, int idx, char* name_buf, int name_cap, int64_t* offset, int64_t* numel) {
  SK_REQUIRE(v, "sk_vocoder_tensor_info: null handle");
  if (idx < 0) return (int)v->tensors.size();
  SK_REQUIRE(idx < (int)v->tensors.size(), "sk_vocoder_tensor_info: index %d out of range", idx);
  const Tensor& t = v->tensors[idx];
  if (name_buf && name_cap > 0) snprintf(name_buf, name_cap, "%s", t.name);
  if (offset) *offset = t.off;
  if (numel) *numel = t.numel;
  return 0;
}

int sk_vocoder_gap(const SkVocoder* v) { return v ? v->G0 : -1; }
int sk_vocoder_upsampling(const SkVocoder* v) { return v ? v->U_total : -1; }

int64_t sk_vocoder_prepared_bytes(const SkVocoder* v) { return v ? 2 * v->prep_elems * (int64_t)sizeof(bf16) : -1; }

int64_t sk_vocoder_workspace_bytes(const SkVocoder* v) {
  if (!v) return -1;
  const int64_t R = v->cfg.max_rows, MU = v->cfg.max_frames;
  int64_t b = 0;
  b += 3 * align_up(R * MU * 4, 256);                 // units, dur, cum
  b += align_up(R * MU * 4, 256);                     // pre-rounding log-durations
  b += 3 * align_up((R + 1) * 4, 256) + 256;          // n_units, frames, starts, bad
  b += align_up(v->T0_cap, 256);                      // valid
  b += align_up(v->T0_cap * v->in_dim * 4, 256);      // x0
  b += 4 * align_up(v->act_elems * 4, 256);           // X, Y, T, S
  return b;
}

int sk_vocoder_bind(SkVocoder* v, const float* weights, void* prepared, int64_t prepared_bytes, void* workspace,
                    int64_t workspace_bytes, void* stream) {
  SK_REQUIRE(v && weights && prepared && workspace, "sk_vocoder_bind: null argument");
  SK_REQUIRE(prepared_bytes >= sk_vocoder_prepared_bytes(v), "sk_vocoder_bind: prepared buffer too small");
  SK_REQUIRE(workspace_bytes >= sk_vocoder_workspace_bytes(v), "sk_vocoder_bind: workspace too small");
  SK_REQUIRE(((uintptr_t)weights | (uintptr_t)prepared | (uintptr_t)workspace) % 256 == 0,
             "sk_vocoder_bind: buffers must be 256-byte aligned");
  cudaStream_t s = (cudaStream_t)stream;
  v->w = weights;
  v->hi = (bf16*)prepared;
  v->lo = v->hi + v->prep_elems;
  for (const auto& L : v->layers) VOC_TRY(prepare_layer(L, weights + L.w, v->hi + L.prep, v->lo + L.prep, s));
  const int64_t R = v->cfg.max_rows, MU = v->cfg.max_frames;
  unsigned char* p = (unsigned char*)workspace;
  auto take = [&](int64_t bytes) { unsigned char* r = p; p += align_up(bytes, 256); return r; };
  v->ws = (unsigned char*)workspace;
  v->units = (int32_t*)take(R * MU * 4);
  v->dur = (int32_t*)take(R * MU * 4);
  v->cum = (int32_t*)take(R * MU * 4);
  v->logd = (float*)take(R * MU * 4);
  v->n_units = (int32_t*)take((R + 1) * 4);
  v->frames = (int32_t*)take((R + 1) * 4);
  v->starts = (int32_t*)take((R + 1) * 4);
  v->bad = (int32_t*)take(256);
  v->valid = (uint8_t*)take(v->T0_cap);
  v->x0 = (float*)take(v->T0_cap * v->in_dim * 4);
  for (int i = 0; i < 4; ++i) v->buf[i] = (float*)take(v->act_elems * 4);
  return 0;
}

int sk_vocoder_durations(SkVocoder* v, const int64_t* codes, int ld, const int32_t* counts, int B, int32_t* dur,
                         float* log_dur, int32_t* frames, int32_t* status, void* stream) {
  SK_REQUIRE(v && v->ws, "sk_vocoder_durations: sk_vocoder_bind has not been called");
  SK_REQUIRE(B >= 0 && B <= v->cfg.max_rows, "sk_vocoder_durations: B = %d outside [0, max_rows = %d]", B, v->cfg.max_rows);
  SK_REQUIRE(ld >= 1 && ld <= v->cfg.max_frames, "sk_vocoder_durations: ld = %d outside [1, max_frames = %d]", ld,
             v->cfg.max_frames);
  SK_REQUIRE(codes && counts && frames && status, "sk_vocoder_durations: null argument");
  cudaStream_t s = (cudaStream_t)stream;
  SK_CUDA_CHECK(cudaMemsetAsync(v->bad, 0, 8, s));
  if (B > 0) {
    VOC_TRY(enqueue_durations(v, codes, ld, counts, B, s));
    const int64_t MU = v->cfg.max_frames;
    if (dur) SK_CUDA_CHECK(cudaMemcpy2DAsync(dur, ld * 4, v->dur, MU * 4, ld * 4, B, cudaMemcpyDeviceToDevice, s));
    if (log_dur && v->cfg.dur_predictor)
      SK_CUDA_CHECK(cudaMemcpy2DAsync(log_dur, ld * 4, v->logd, MU * 4, ld * 4, B, cudaMemcpyDeviceToDevice, s));
    SK_CUDA_CHECK(cudaMemcpyAsync(frames, v->frames, (size_t)B * 4, cudaMemcpyDeviceToDevice, s));
  }
  SK_CUDA_CHECK(cudaMemcpyAsync(status, v->bad, 8, cudaMemcpyDeviceToDevice, s));
  return 0;
}

int sk_vocoder_run(SkVocoder* v, const int64_t* codes, int ld, const int32_t* counts, int B, const int32_t* frames_host,
                   float* wave, int64_t ldw, void* stream) {
  SK_REQUIRE(v && v->ws, "sk_vocoder_run: sk_vocoder_bind has not been called");
  SK_REQUIRE(codes && counts && frames_host && wave, "sk_vocoder_run: null argument");
  SK_REQUIRE(ld >= 1 && ld <= v->cfg.max_frames, "sk_vocoder_run: ld = %d outside [1, max_frames = %d]", ld, v->cfg.max_frames);
  SK_REQUIRE(B >= 0, "sk_vocoder_run: negative B");
  cudaStream_t s = (cudaStream_t)stream;
  int64_t need = 0;
  for (int b = 0; b < B; ++b) {
    SK_REQUIRE(frames_host[b] >= 0 && frames_host[b] <= v->cfg.max_frames,
               "sk_vocoder_run: row %d has %d frames, more than max_frames = %d", b, frames_host[b], v->cfg.max_frames);
    need = std::max(need, (int64_t)frames_host[b] * v->U_total);
  }
  SK_REQUIRE(ldw >= need && ldw <= INT32_MAX, "sk_vocoder_run: ldw = %lld is smaller than the longest row (%lld samples)",
             (long long)ldw, (long long)need);
  // sub-batches of whole rows that fit the workspace
  for (int b0 = 0; b0 < B;) {
    int b1 = b0;
    int64_t fr = 0;
    while (b1 < B && b1 - b0 < v->cfg.max_rows && fr + frames_host[b1] <= v->cfg.max_frames) fr += frames_host[b1++];
    const int nb = b1 - b0;
    const int T0 = (int)(fr + (int64_t)(nb + 1) * v->G0);
    VOC_TRY(enqueue_durations(v, codes + (int64_t)b0 * ld, ld, counts + b0, nb, s));
    VOC_TRY(enqueue_network(v, nb, T0, wave + (int64_t)b0 * ldw, (int)ldw, s));
    b0 = b1;
  }
  return 0;
}

int sk_vocoder_conv(const SkVocoderConvDesc* desc, void* stream) {
  SK_REQUIRE(desc, "sk_vocoder_conv: null descriptor");
  const SkVocoderConvDesc& d = *desc;
  SK_REQUIRE(d.x && d.weight && d.bias && d.valid && d.prep, "sk_vocoder_conv: null x, weight, bias, valid or prep");
  SK_REQUIRE(d.T_in >= 1, "sk_vocoder_conv: T_in = %d must be positive", d.T_in);
  SK_REQUIRE(d.Cin > 0 && d.Cin % 4 == 0 && d.Cout > 0 && d.Cout % 4 == 0,
             "sk_vocoder_conv: Cin = %d and Cout = %d must be positive multiples of 4", d.Cin, d.Cout);
  SK_REQUIRE(d.k >= 1 && d.k <= MAX_TAPS, "sk_vocoder_conv: kernel %d outside [1, %d]", d.k, MAX_TAPS);
  if (d.transposed)
    SK_REQUIRE(d.rate >= 1 && d.rate <= d.k && (d.k - d.rate) % 2 == 0 && d.dilation == 1,
               "sk_vocoder_conv: a transposed conv needs 1 <= rate <= kernel, kernel - rate even and dilation 1 "
               "(rate %d, kernel %d, dilation %d)", d.rate, d.k, d.dilation);
  else
    SK_REQUIRE(d.rate == 1 && d.k % 2 == 1 && d.dilation >= 1 && d.dilation <= 1024,
               "sk_vocoder_conv: a conv needs rate 1, an odd kernel and a dilation in [1, 1024] (rate %d, kernel %d, "
               "dilation %d)", d.rate, d.k, d.dilation);
  const int64_t T_out = d.transposed ? (int64_t)d.T_in * d.rate : d.T_in;
  SK_REQUIRE(T_out <= INT32_MAX / 4, "sk_vocoder_conv: %lld output positions are too many", (long long)T_out);
  SK_REQUIRE(d.up >= 1 && T_out % d.up == 0, "sk_vocoder_conv: up = %d must divide T_out = %lld", d.up, (long long)T_out);
  SK_REQUIRE(d.mode >= 0 && d.mode <= 2 && d.divide >= 0, "sk_vocoder_conv: mode %d must be 0..2 and divide %d >= 0",
             d.mode, d.divide);
  SK_REQUIRE(d.mode == 0 ? (d.y && !d.divide) : d.sum != nullptr,
             "sk_vocoder_conv: mode 0 writes y (and does not divide); modes 1 and 2 write sum");
  SK_REQUIRE((uintptr_t)d.x % 16 == 0 && (uintptr_t)d.prep % 16 == 0 &&
                 ((uintptr_t)d.y | (uintptr_t)d.res | (uintptr_t)d.sum) % 8 == 0,
             "sk_vocoder_conv: x and prep must be 16-byte aligned, y, res and sum 8-byte aligned");
  const ConvLayer L = conv_layer(d.Cout, d.Cin, d.k, d.transposed, d.transposed ? d.rate : 1, d.dilation);
  const int64_t need = 2 * prep_elems(L) * (int64_t)sizeof(bf16);
  SK_REQUIRE(d.prep_bytes >= need, "sk_vocoder_conv: prep holds %lld bytes, the split weights need %lld",
             (long long)d.prep_bytes, (long long)need);
  const size_t smem = conv_smem_bytes(halo_span(L), conv_nt(d.Cout));
  SK_REQUIRE(smem <= CONV_SMEM_MAX, "sk_vocoder_conv: kernel %d at dilation %d needs %zu bytes of shared memory for its "
             "halo, more than %zu", d.k, d.dilation, smem, CONV_SMEM_MAX);
  cudaStream_t s = (cudaStream_t)stream;
  bf16* hi = (bf16*)d.prep;
  bf16* lo = hi + prep_elems(L);
  VOC_TRY(prepare_layer(L, d.weight, hi, lo, s));
  return run_layer(L, hi, lo, d.bias, d.valid, d.x, d.T_in, (int)T_out, d.slope, d.y, d.res, d.sum, d.mode, d.divide, d.up, s);
}

}  // extern "C"
