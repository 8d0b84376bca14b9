// Incremental decoding kernels of the causal LM (TokenLM.generate with a KV cache): the cache copy / append kernels,
// flash-decoding attention over the cache and on-device token selection (HF's logits processors + Philox sampling).
// The per-step orchestration (sk_lm_prefill / sk_lm_decode_step) lives in lm_step.cu.
//
// Every launch here is graph-safe: no allocation, no synchronisation, and launch parameters that depend only on the
// shapes (B, H, KVH, T_cache, V).  Step-varying values (positions, lengths, the step index) live in device memory.
#include "kernels.h"
#include "../../include/slamkit_b200.h"
#include <math.h>

namespace {

constexpr int DEC_CH = 64;        // keys per attention split (one CTA); the split count is ceil(T_cache / DEC_CH)
constexpr int DEC_THREADS = 128;
constexpr int DEC_MAX_G = 16;     // query heads per kv head served by one CTA
// smem row pitch of the K / V tiles: 144 B (bf16 cache) or 272 B (fp32 cache), conflict-free 16-byte row reads
template <typename KV> constexpr int dec_kpad() { return sizeof(KV) == 2 ? 72 : 68; }

// ---- KV cache ---------------------------------------------------------------------------------------------------
// cache layout per layer: [K|V][B][KVH][T_cache][64] of KV = bf16 (K after RoPE) or, for fp32 OPT inference, fp32
// (the value hi + lo of the split-bf16 projections: fp32-grade K / V).  `lo` (fp32 cache only) is the lo half of the
// projections, at the same offsets as their hi half.

// eight cache elements from the projections at src (+ lo)
SK_DEVINL void put8(bf16* dst, const bf16* src, const bf16*) { stg128(dst, ldg128(src)); }
SK_DEVINL void put8(float* dst, const bf16* src, const bf16* lo) {
  const uint4 h = ldg128(src), l = ldg128(lo);
  const uint32_t hw[4] = {h.x, h.y, h.z, h.w}, lw[4] = {l.x, l.y, l.z, l.w};
  float v[8];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const float2 a = unpack_bf16(hw[k]), b = unpack_bf16(lw[k]);
    v[2 * k] = a.x + b.x;
    v[2 * k + 1] = a.y + b.y;
  }
  reinterpret_cast<float4*>(dst)[0] = make_float4(v[0], v[1], v[2], v[3]);
  reinterpret_cast<float4*>(dst)[1] = make_float4(v[4], v[5], v[6], v[7]);
}

// prefill: copy K/V of positions t < lens[b] of every layer out of the fused projections [B*T, ldq] (layer stride
// `layer_stride` elements) into the cache.  grid (B*T, L)
template <typename KV>
__global__ void kv_prefill_kernel(const bf16* __restrict__ qkv, const bf16* __restrict__ qkv_lo, long layer_stride, int ldq,
                                  KV* __restrict__ cache, const int32_t* __restrict__ lens, int B, int T, int H, int KVH,
                                  int T_cache) {
  griddep_wait();
  const int row = blockIdx.x, l = blockIdx.y;
  const int b = row / T, t = row % T;
  if (t >= lens[b] || t >= T_cache) return;
  const size_t so = l * layer_stride + (size_t)row * ldq + (size_t)H * 64;
  const size_t plane = (size_t)B * KVH * T_cache * 64;
  KV* kc = cache + (size_t)l * 2 * plane;
  for (int i = threadIdx.x; i < 2 * KVH * 8; i += blockDim.x) {
    const int which = i / (KVH * 8), r = i % (KVH * 8), kvh = r / 8, c = r % 8;
    KV* dst = kc + which * plane + (((size_t)b * KVH + kvh) * T_cache + t) * 64 + c * 8;
    const size_t o = so + (size_t)(which * KVH + kvh) * 64 + c * 8;
    put8(dst, qkv + o, qkv_lo + o);
  }
}

// decode: append the K/V of the one new token of every row at pos[b] and publish lens[b] = pos[b] + 1.  grid B
template <typename KV>
__global__ void kv_append_kernel(const bf16* __restrict__ qkv, const bf16* __restrict__ qkv_lo, int ldq, KV* __restrict__ kc,
                                 KV* __restrict__ vc, const int32_t* __restrict__ pos, int32_t* __restrict__ lens, int H,
                                 int KVH, int T_cache) {
  griddep_wait();
  const int b = blockIdx.x;
  const int p = min(max(pos[b], 0), T_cache - 1);
  const size_t so = (size_t)b * ldq + (size_t)H * 64;
  for (int i = threadIdx.x; i < 2 * KVH * 8; i += blockDim.x) {
    const int which = i / (KVH * 8), r = i % (KVH * 8), kvh = r / 8, c = r % 8;
    KV* dst = (which ? vc : kc) + (((size_t)b * KVH + kvh) * T_cache + p) * 64 + c * 8;
    const size_t o = so + (size_t)(which * KVH + kvh) * 64 + c * 8;
    put8(dst, qkv + o, qkv_lo + o);
  }
  if (threadIdx.x == 0 && lens) lens[b] = p + 1;
}

// rows b*T + lens[b] - 1 of x [B*T, D] -> out [B, D].  grid B
__global__ void gather_last_kernel(const bf16* __restrict__ x, const int32_t* __restrict__ lens, bf16* __restrict__ out,
                                   int T, int D) {
  griddep_wait();
  const int b = blockIdx.x;
  const int t = min(max(lens[b], 1), T) - 1;
  for (int c = threadIdx.x; c < D / 8; c += blockDim.x)
    stg128(out + (size_t)b * D + c * 8, ldg128(x + ((size_t)b * T + t) * D + c * 8));
}

// ---- decode attention ------------------------------------------------------------------------------------------
// Flash-decoding: CTA (split s, kv head, row b) serves all G = H/KVH query heads of its group over keys
// [64 s, min(64 s + 64, lens[b])), so every K/V byte is read once.  Scores and the (unnormalised) P.V sum are fp32;
// the partial (o, m, l) per (row, head, split) goes to `partial` and sk_attn_decode's combine pass merges the splits in
// split order.  CTAs whose range starts at or past lens[b] exit before touching the cache.  An fp32 cache (KV = float)
// goes with a split-bf16 query: q = q_hi + q_lo.

// 16 bytes of a cache row (8 bf16 / 4 fp32 elements) at element i, and two elements as fp32
template <typename KV> SK_DEVINL uint4 cache16(const KV* p) { return ldg128_stream(reinterpret_cast<const bf16*>(p)); }
SK_DEVINL float2 two(const bf16* p) { return __bfloat1622float2(*reinterpret_cast<const bf162*>(p)); }
SK_DEVINL float2 two(const float* p) { return *reinterpret_cast<const float2*>(p); }

template <typename KV>
__global__ void __launch_bounds__(DEC_THREADS) attn_decode_split_kernel(
    const bf16* __restrict__ q, const bf16* __restrict__ q_lo, int ldq, const KV* __restrict__ kc, const KV* __restrict__ vc,
    const int32_t* __restrict__ lens, float* __restrict__ part_o, float2* __restrict__ part_ml, int H, int KVH,
    int T_cache, int S, float scale_log2) {
  constexpr int KPAD = dec_kpad<KV>();
  constexpr int EPV = 16 / sizeof(KV);   // cache elements per 16-byte vector
  extern __shared__ __align__(16) uint8_t dec_smem[];
  KV* sK = reinterpret_cast<KV*>(dec_smem);
  KV* sV = sK + DEC_CH * KPAD;
  float* sQ = reinterpret_cast<float*>(sV + DEC_CH * KPAD);   // [G][64], pre-scaled by scale * log2(e)
  float* sP = sQ + DEC_MAX_G * 64;                                  // [G][64] scores, then exp2(score - max)
  const int s = blockIdx.x, kvh = blockIdx.y, b = blockIdx.z;
  const int G = H / KVH;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  griddep_wait();
  const int len = lens[b];
  const int k0 = s * DEC_CH;
  if (k0 >= len) return;
  const int n = min(DEC_CH, len - k0);
  const size_t base = (((size_t)b * KVH + kvh) * T_cache + k0) * 64;
  for (int i = tid; i < n * (64 / EPV); i += DEC_THREADS) {
    const int r = i / (64 / EPV), c = i % (64 / EPV);
    *reinterpret_cast<uint4*>(sK + r * KPAD + c * EPV) = cache16(kc + base + (size_t)r * 64 + c * EPV);
    *reinterpret_cast<uint4*>(sV + r * KPAD + c * EPV) = cache16(vc + base + (size_t)r * 64 + c * EPV);
  }
  for (int i = tid; i < G * 8; i += DEC_THREADS) {
    const int g = i >> 3, c = i & 7;
    const size_t qo = (size_t)b * ldq + (size_t)(kvh * G + g) * 64 + c * 8;
    const uint4 v = ldg128(q + qo);
    const uint32_t u[4] = {v.x, v.y, v.z, v.w};
    uint32_t ul[4] = {0u, 0u, 0u, 0u};
    if constexpr (sizeof(KV) == 4) {
      const uint4 vl = ldg128(q_lo + qo);
      ul[0] = vl.x; ul[1] = vl.y; ul[2] = vl.z; ul[3] = vl.w;
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      float2 f = unpack_bf16(u[k]);
      if constexpr (sizeof(KV) == 4) {
        const float2 fl = unpack_bf16(ul[k]);
        f.x += fl.x;
        f.y += fl.y;
      }
      sQ[g * 64 + c * 8 + 2 * k] = f.x * scale_log2;
      sQ[g * 64 + c * 8 + 2 * k + 1] = f.y * scale_log2;
    }
  }
  __syncthreads();
  // scores: thread -> key j = tid % 64, heads tid / 64, +2, +4, ...
  {
    const int j = tid & 63;
    if (j < n) {
      float kf[64];
      if constexpr (sizeof(KV) == 2) {
#pragma unroll
        for (int c = 0; c < 8; ++c) {
          const uint4 v = *reinterpret_cast<const uint4*>(sK + j * KPAD + c * 8);
          const uint32_t u[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            const float2 f = unpack_bf16(u[k]);
            kf[c * 8 + 2 * k] = f.x;
            kf[c * 8 + 2 * k + 1] = f.y;
          }
        }
      } else {
#pragma unroll
        for (int c = 0; c < 16; ++c) {
          const float4 v = *reinterpret_cast<const float4*>(sK + j * KPAD + c * 4);
          kf[4 * c] = v.x;
          kf[4 * c + 1] = v.y;
          kf[4 * c + 2] = v.z;
          kf[4 * c + 3] = v.w;
        }
      }
      for (int g = tid >> 6; g < G; g += DEC_THREADS / 64) {
        const float4* qg = reinterpret_cast<const float4*>(sQ + g * 64);
        float acc = 0.f;
#pragma unroll
        for (int d = 0; d < 16; ++d) {
          const float4 qq = qg[d];
          acc = fmaf(qq.x, kf[4 * d], acc);
          acc = fmaf(qq.y, kf[4 * d + 1], acc);
          acc = fmaf(qq.z, kf[4 * d + 2], acc);
          acc = fmaf(qq.w, kf[4 * d + 3], acc);
        }
        sP[g * 64 + j] = acc;
      }
    } else {
      for (int g = tid >> 6; g < G; g += DEC_THREADS / 64) sP[g * 64 + j] = -INFINITY;
    }
  }
  __syncthreads();
  // per-head max / sum over the split: one warp per head
  for (int g = warp; g < G; g += DEC_THREADS / 32) {
    const float v0 = sP[g * 64 + lane], v1 = sP[g * 64 + lane + 32];
    const float mx = warp_max(fmaxf(v0, v1));
    const float e0 = exp2f(v0 - mx), e1 = exp2f(v1 - mx);
    sP[g * 64 + lane] = e0;
    sP[g * 64 + lane + 32] = e1;
    const float l = warp_sum(e0 + e1);
    if (lane == 0) part_ml[((size_t)b * H + kvh * G + g) * S + s] = make_float2(mx, l);
  }
  __syncthreads();
  // P.V: warp w -> heads w, w+4, w+8, w+12; lane -> dims 2*lane, 2*lane+1
  float2 acc[DEC_MAX_G / 4];
#pragma unroll
  for (int i = 0; i < DEC_MAX_G / 4; ++i) acc[i] = make_float2(0.f, 0.f);
  for (int j = 0; j < n; ++j) {
    const float2 v = two(sV + j * KPAD + 2 * lane);
#pragma unroll
    for (int i = 0; i < DEC_MAX_G / 4; ++i) {
      const int g = warp + 4 * i;
      if (g < G) {
        const float p = sP[g * 64 + j];
        acc[i].x = fmaf(p, v.x, acc[i].x);
        acc[i].y = fmaf(p, v.y, acc[i].y);
      }
    }
  }
#pragma unroll
  for (int i = 0; i < DEC_MAX_G / 4; ++i) {
    const int g = warp + 4 * i;
    if (g < G)
      *reinterpret_cast<float2*>(part_o + (((size_t)b * H + kvh * G + g) * S + s) * 64 + 2 * lane) = acc[i];
  }
}

// one warp per (row, head): merge the ceil(lens[b] / 64) valid splits in split order.  SPLIT_OUT: write the (hi, lo)
// pair of the fp32 result (o_lo) instead of its bf16 rounding
template <bool SPLIT_OUT>
__global__ void __launch_bounds__(128) attn_decode_combine_kernel(const float* __restrict__ part_o,
                                                                  const float2* __restrict__ part_ml,
                                                                  const int32_t* __restrict__ lens, bf16* __restrict__ o,
                                                                  bf16* __restrict__ o_lo, int ldo, int B, int H, int S) {
  griddep_wait();
  const int w = blockIdx.x * 4 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (w >= B * H) return;
  const int b = w / H, h = w % H;
  const int ns = min((lens[b] + DEC_CH - 1) / DEC_CH, S);
  const float2* ml = part_ml + (size_t)w * S;
  float M = -INFINITY;
  for (int s = 0; s < ns; ++s) M = fmaxf(M, ml[s].x);
  float L = 0.f;
  float2 acc = make_float2(0.f, 0.f);
  for (int s = 0; s < ns; ++s) {
    const float2 m = ml[s];
    const float f = exp2f(m.x - M);
    L = fmaf(f, m.y, L);
    const float2 v = *reinterpret_cast<const float2*>(part_o + ((size_t)w * S + s) * 64 + 2 * lane);
    acc.x = fmaf(f, v.x, acc.x);
    acc.y = fmaf(f, v.y, acc.y);
  }
  const float inv = ns > 0 ? 1.0f / L : 0.f;
  const size_t oo = (size_t)b * ldo + h * 64 + 2 * lane;
  if (SPLIT_OUT) {
    const float v0 = acc.x * inv, v1 = acc.y * inv, h0 = bf16_round(v0), h1 = bf16_round(v1);
    *reinterpret_cast<uint32_t*>(o + oo) = pack_bf16(h0, h1);
    *reinterpret_cast<uint32_t*>(o_lo + oo) = pack_bf16(v0 - h0, v1 - h1);
  } else {
    *reinterpret_cast<bf162*>(o + oo) = __floats2bfloat162_rn(acc.x * inv, acc.y * inv);
  }
}

// ---- token selection -------------------------------------------------------------------------------------------
constexpr int SEL_THREADS = 512;
constexpr int SEL_WARPS = SEL_THREADS / 32;

// order-preserving key of a score; -0.0 and +0.0 share the key of +0.0, as they compare equal in HF's argmax and warpers
SK_DEVINL uint32_t ordered_key(float f) {
  const uint32_t u = f == 0.f ? 0u : __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

// Philox4x32-10 (Salmon et al., SC'11), counter (step, row, 0, 0), key = seed
SK_DEVINL uint4 philox4x32_10(uint4 c, uint2 k) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t lo0 = 0xD2511F53u * c.x, hi0 = __umulhi(0xD2511F53u, c.x);
    const uint32_t lo1 = 0xCD9E8D57u * c.z, hi1 = __umulhi(0xCD9E8D57u, c.z);
    c = make_uint4(hi1 ^ c.y ^ k.x, lo1, hi0 ^ c.w ^ k.y, lo0);
    k.x += 0x9E3779B9u;
    k.y += 0xBB67AE85u;
  }
  return c;
}

// fixed-order block reductions (tree over the warps: the result does not depend on timing)
template <typename T, typename Op>
SK_DEVINL T block_reduce(T v, T* red, Op op) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = op(v, __shfl_xor_sync(0xffffffffu, v, o));
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  T r = red[0];
  for (int w = 1; w < SEL_WARPS; ++w) r = op(r, red[w]);
  return r;
}
// exclusive prefix over threads of a per-thread value (thread order = token order: each thread owns a contiguous
// chunk of the vocabulary); also returns the total
template <typename T>
SK_DEVINL T block_exclusive_scan(T v, T* red, T& total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  T inc = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const T n = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += n;
  }
  __syncthreads();
  if (lane == 31) red[warp] = inc;
  __syncthreads();
  T before = 0;
  total = 0;
  for (int w = 0; w < SEL_WARPS; ++w) {
    if (w < warp) before += red[w];
    total += red[w];
  }
  return before + inc - v;
}

SK_DEVINL float logit_at(const bf16* row, int i) { return __bfloat162float(row[i]); }
SK_DEVINL float logit_at(const float* row, int i) { return row[i]; }

// first index of the ascending a[0, n) whose value is >= x (n if none)
SK_DEVINL int lower_bound_i32(const int32_t* a, int n, int x) {
  int lo = 0, hi = n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (a[mid] < x) lo = mid + 1;
    else hi = mid;
  }
  return lo;
}

SK_DEVINL bool bit_set(const uint32_t* bits, int i) { return (bits[i >> 5] >> (i & 31)) & 1u; }

// RULES: the SkLogitRules processors of one row.  `dyn` holds this step's n-gram and min-length bans (NULL when there
// are none), `pres` the presence bitmap when the repetition penalty is on.  The penalty is one rounded multiply or divide
// and the temperature one rounded divide, as HF applies them one processor after the other.
template <typename LT, bool RULES>
struct SelRow {
  const LT* row;
  const uint32_t* ban;
  float temp;
  bool use_temp;
  const uint32_t* dyn;
  const uint32_t* pres;
  float penalty;
  SK_DEVINL float score(int i) const {
    if (ban && ((ban[i >> 5] >> (i & 31)) & 1u)) return -INFINITY;
    float x = logit_at(row, i);
    if constexpr (RULES) {
      if (dyn && bit_set(dyn, i)) return -INFINITY;
      if (pres && bit_set(pres, i)) x = x < 0.f ? __fmul_rn(x, penalty) : __fdiv_rn(x, penalty);
    }
    return use_temp ? __fdiv_rn(x, temp) : x;
  }
};

// appends the selected token (pad once finished) to the row's history and sets its presence bit
SK_DEVINL void rules_append(const SkLogitRules& r, int b, int step, int tok, int V) {
  const int c = r.prompt_len + step;
  if (c < r.hist_ld) r.history[(size_t)b * r.hist_ld + c] = tok;
  if (r.presence && tok >= 0 && tok < V) r.presence[(size_t)b * ((V + 31) >> 5) + (tok >> 5)] |= 1u << (tok & 31);
}

// this step's n-gram and min-length bans of row b into its scratch bitmap (all threads of the CTA); NULL if none apply
SK_DEVINL const uint32_t* rules_bans(const SkLogitRules& r, const SkSampling& cfg, int b, int step, int V) {
  const int cur = min(r.prompt_len + step, r.hist_ld), n = r.ngram;
  const bool ngram = n > 0 && cur + 1 >= n;
  const bool min_len = step < r.min_step && cfg.n_eos > 0;
  if (!ngram && !min_len) return nullptr;
  const int W = (V + 31) >> 5;
  uint32_t* d = r.scratch + (size_t)b * W;
  for (int w = threadIdx.x; w < W; w += blockDim.x) d[w] = 0u;
  __syncthreads();
  if (min_len && threadIdx.x == 0)
    for (int e = 0; e < cfg.n_eos && e < 8; ++e)
      if (cfg.eos[e] >= 0 && cfg.eos[e] < V) atomicOr(&d[cfg.eos[e] >> 5], 1u << (cfg.eos[e] & 31));
  if (ngram) {
    // HF's NoRepeatNGram: the n-grams h[j .. j+n-1], j <= cur - n, whose first n-1 tokens equal the last n-1 tokens
    // h[cur-n+1 .. cur-1] ban their last token
    const int64_t* h = r.history + (size_t)b * r.hist_ld;
    const int tail = cur - n + 1;
    for (int j = threadIdx.x; j <= cur - n; j += blockDim.x) {
      int m = 0;
      while (m < n - 1 && h[j + m] == h[tail + m]) ++m;
      if (m == n - 1) {
        const int64_t t = h[j + n - 1];
        if (t >= 0 && t < V) atomicOr(&d[t >> 5], 1u << (t & 31));
      }
    }
  }
  __syncthreads();
  return d;
}

// One CTA per row.  Order of HF's processors: bans -> (sampling only) temperature -> top-k -> top-p -> softmax -> draw;
// greedy = argmax of the banned scores, lowest id on ties.  Each thread owns the contiguous id range
// [tid * chunk, (tid + 1) * chunk), so per-thread partial sums are in token order and every sum is taken in a fixed order.
// LT: bf16 logits, or fp32 ones (fp32 OPT inference).  RULES: apply `rules` (sk_select_next_ex) and append to the
// history; without, `rules` is not read.  SUB (sk_select_next_sub): column c of the logits is token sub_ids[c] (ascending)
// and every other id is banned.  A thread then owns the columns whose ids fall in its id range, so each partial sum, scan
// and tie break sees the same values in the same order as the full-vocabulary kernel with those ids banned, and picks
// the same token.
template <typename LT, bool RULES, bool SUB>
SK_DEVINL void select_next_row(const LT* __restrict__ logits, int ldl, int V, const uint32_t* __restrict__ ban,
                               const SkSampling& cfg, const float* __restrict__ uniforms, const SkDecodeState& st,
                               const SkLogitRules& rules, const int32_t* __restrict__ sub_ids, int n_sub) {
  __shared__ float red_f[SEL_WARPS];
  __shared__ int red_i[SEL_WARPS];
  __shared__ unsigned long long red_u[SEL_WARPS];
  __shared__ int hist[256];
  __shared__ int s_step, s_tok;
  __shared__ uint32_t s_digit;
  const int b = blockIdx.x, tid = threadIdx.x;
  griddep_wait();
  if (tid == 0) s_step = st.step[0];
  __syncthreads();
  const int step = s_step;
  if (tid == 0) {
    // the last CTA to have read the step index advances it (all others have read it by then)
    __threadfence();
    if (atomicAdd(&st.step[1], 1) == (int)gridDim.x - 1) {
      st.step[1] = 0;
      st.step[0] = step + 1;
    }
  }
  const int p = st.pos[b];
  const bool fin = st.finished[b] != 0 || p + 1 >= cfg.max_length;
  if (fin) {
    if (tid == 0) {
      st.finished[b] = 1;
      if (step < st.max_new) st.out[(size_t)b * st.max_new + step] = cfg.pad_token_id;
      if constexpr (RULES) rules_append(rules, b, step, cfg.pad_token_id, V);
    }
    return;
  }
  const int chunk = (V + SEL_THREADS - 1) / SEL_THREADS;
  const int i0 = min(tid * chunk, V), i1 = min(i0 + chunk, V);
  // the thread's columns [c0, c1) and the id of a column
  int c0 = i0, c1 = i1;
  if constexpr (SUB) {
    c0 = lower_bound_i32(sub_ids, n_sub, i0);
    c1 = lower_bound_i32(sub_ids, n_sub, i1);
  }
  const int n_cols = SUB ? n_sub : V;
  SelRow<LT, RULES> R{logits + (size_t)b * ldl, ban, cfg.temperature, cfg.do_sample != 0 && cfg.temperature != 1.0f,
                      nullptr, nullptr, 1.f};
  if constexpr (RULES) {
    R.dyn = rules_bans(rules, cfg, b, step, V);
    if (rules.penalty != 1.f) {
      R.pres = rules.presence + (size_t)b * ((V + 31) >> 5);
      R.penalty = rules.penalty;
    }
  }
  int tok = 0;
  if (!cfg.do_sample) {
    // argmax, lowest id among equal maxima
    float bv = -INFINITY;
    int bi = 0x7fffffff;
    for (int c = c0; c < c1; ++c) {
      const float v = R.score(c);
      const int i = (SUB ? (int)sub_ids[c] : c);
      if (v > bv || (v == bv && i < bi)) { bv = v; bi = i; }
    }
    // pack (ordered value, inverted id) so that one max picks the largest value, then the smallest id
    unsigned long long key = ((unsigned long long)ordered_key(bv) << 32) | (uint32_t)(0x7fffffff - min(bi, 0x7fffffff));
    key = block_reduce(key, red_u, [](unsigned long long a, unsigned long long c) { return a > c ? a : c; });
    tok = 0x7fffffff - (int)(uint32_t)(key & 0xffffffffu);
    if (tok >= V) tok = 0;
  } else {
    // top-k: the k-th largest score by radix select on order-preserving keys (HF keeps every score >= it)
    // (SUB: with k >= n_sub the full kernel's k-th score is a banned -inf, which keeps every allowed id, as kth = 0 does)
    const int k = cfg.top_k > 0 ? min(cfg.top_k, n_cols) : n_cols;
    uint32_t kth = 0;
    if (k < n_cols) {
      uint32_t prefix = 0, mask = 0;
      int rank = k;
      for (int shift = 24; shift >= 0; shift -= 8) {
        for (int i = tid; i < 256; i += SEL_THREADS) hist[i] = 0;
        __syncthreads();
        for (int c = c0; c < c1; ++c) {
          const uint32_t key = ordered_key(R.score(c));
          if ((key & mask) == prefix) atomicAdd(&hist[(key >> shift) & 255u], 1);
        }
        __syncthreads();
        if (tid == 0) {
          int cum = 0;
          uint32_t d = 0;
          for (int dd = 255; dd >= 0; --dd) {
            if (cum + hist[dd] >= rank) { d = (uint32_t)dd; rank -= cum; break; }
            cum += hist[dd];
          }
          s_digit = d;
          hist[0] = rank;   // carried to the other threads below
        }
        __syncthreads();
        prefix |= s_digit << shift;
        mask |= 255u << shift;
        rank = hist[0];
        __syncthreads();
      }
      kth = prefix;
    }
    // softmax over the kept scores
    float mx = -INFINITY;
    for (int c = c0; c < c1; ++c) {
      const float v = R.score(c);
      if (ordered_key(v) >= kth) mx = fmaxf(mx, v);
    }
    mx = block_reduce(mx, red_f, [](float a, float c) { return fmaxf(a, c); });
    // top-p: HF sorts ascending and drops every token whose cumulative probability is <= 1 - top_p (keeping the most
    // likely one).  The dropped tokens are a prefix of the ascending order, so the cut is found by bisection on the
    // score key: K* = the smallest key whose mass of keys <= K* exceeds 1 - top_p.  Below K* everything goes; inside the
    // tie group at K* tokens go in id order (a stable sort) while the running sum stays <= 1 - top_p.
    uint32_t cut_key = kth;
    int cut_id = -1;   // ids <= cut_id with key == cut_key are dropped too
    if (cfg.top_p < 1.0) {
      const float thr = (float)(1.0 - cfg.top_p);
      float z = 0.f;
      for (int c = c0; c < c1; ++c) {
        const float v = R.score(c);
        if (ordered_key(v) >= kth) z += expf(v - mx);
      }
      float ztot;
      block_exclusive_scan(z, red_f, ztot);
      auto mass_le = [&](uint32_t K) {
        float m = 0.f;
        for (int c = c0; c < c1; ++c) {
          const float v = R.score(c);
          const uint32_t key = ordered_key(v);
          if (key >= kth && key <= K) m += expf(v - mx);
        }
        float tot;
        block_exclusive_scan(m, red_f, tot);
        return tot / ztot;
      };
      uint32_t lo = kth, hi = ordered_key(mx);
      while (lo < hi) {
        const uint32_t mid = lo + (hi - lo) / 2;
        if (mass_le(mid) > thr) hi = mid;
        else lo = mid + 1;
      }
      cut_key = lo;
      // the tie group at K*: count, and the mass strictly below it
      int cnt = 0, first_in_chunk = 0;
      float q = 0.f;
      for (int c = c0; c < c1; ++c) {
        const float v = R.score(c);
        if (ordered_key(v) == cut_key) { ++cnt; q = expf(v - mx); }
      }
      int cnt_tot;
      first_in_chunk = block_exclusive_scan(cnt, red_i, cnt_tot);
      const float below = lo > kth ? mass_le(lo - 1) : 0.f;
      q = block_reduce(q, red_f, [](float a, float c) { return fmaxf(a, c); }) / ztot;
      int drop = 0;
      float run = below;
      while (drop < cnt_tot - 1 && run + q <= thr) { run += q; ++drop; }
      if (drop > 0) {
        // id of the drop-th member of the group (1-based) in id order
        int id = -1, seen = first_in_chunk;
        if (seen < drop && seen + cnt >= drop) {
          for (int c = c0; c < c1; ++c) {
            if (ordered_key(R.score(c)) == cut_key && ++seen == drop) { id = (SUB ? (int)sub_ids[c] : c); break; }
          }
        }
        cut_id = block_reduce(id, red_i, [](int a, int c) { return a > c ? a : c; });
      }
    }
    auto kept = [&](int i, float v) {
      const uint32_t key = ordered_key(v);
      return key >= kth && (key > cut_key || (key == cut_key && i > cut_id)) && v > -INFINITY;
    };
    // draw: inverse CDF in token-id order at u
    float u;
    if (uniforms) {
      u = uniforms[b];
    } else {
      const uint4 r = philox4x32_10(make_uint4((uint32_t)step, (uint32_t)b, 0u, 0u),
                                    make_uint2((uint32_t)cfg.seed, (uint32_t)(cfg.seed >> 32)));
      u = (float)(r.x >> 8) * (1.0f / 16777216.0f);
    }
    float e = 0.f;
    int last = -1;
    for (int c = c0; c < c1; ++c) {
      const float v = R.score(c);
      const int i = (SUB ? (int)sub_ids[c] : c);
      if (kept(i, v)) { e += expf(v - mx); last = i; }
    }
    float etot;
    const float before = block_exclusive_scan(e, red_f, etot);
    const int last_kept = block_reduce(last, red_i, [](int a, int c) { return a > c ? a : c; });
    const float target = u * etot;
    if (tid == 0) s_tok = 0x7fffffff;
    __syncthreads();
    if (e > 0.f && before <= target && target < before + e) {
      float run = before;
      for (int c = c0; c < c1; ++c) {
        const float v = R.score(c);
        const int i = (SUB ? (int)sub_ids[c] : c);
        if (kept(i, v)) {
          run += expf(v - mx);
          if (run > target) { atomicMin(&s_tok, i); break; }
        }
      }
    }
    __syncthreads();
    tok = s_tok != 0x7fffffff ? s_tok : max(last_kept, 0);
  }
  if (tid == 0) {
    if (step < st.max_new) st.out[(size_t)b * st.max_new + step] = tok;
    st.n_gen[b] += 1;
    st.tokens[b] = tok;
    st.pos[b] = p + 1;
    bool eos = false;
    for (int e = 0; e < cfg.n_eos && e < 8; ++e) eos |= (tok == cfg.eos[e]);
    if (eos) st.finished[b] = 1;
    if constexpr (RULES) rules_append(rules, b, step, tok, V);
  }
}

template <typename LT, bool RULES>
__global__ void __launch_bounds__(SEL_THREADS) select_next_kernel(const LT* __restrict__ logits, int ldl, int V,
                                                                  const uint32_t* __restrict__ ban, SkSampling cfg,
                                                                  const float* __restrict__ uniforms, SkDecodeState st,
                                                                  SkLogitRules rules) {
  select_next_row<LT, RULES, false>(logits, ldl, V, ban, cfg, uniforms, st, rules, nullptr, 0);
}
__global__ void __launch_bounds__(SEL_THREADS) select_next_sub_kernel(const bf16* __restrict__ logits, int ld_sub, int V,
                                                                         SkSampling cfg, const float* __restrict__ uniforms,
                                                                         SkDecodeState st, const int32_t* __restrict__ ids,
                                                                         int n) {
  select_next_row<bf16, false, true>(logits, ld_sub, V, nullptr, cfg, uniforms, st, SkLogitRules{}, ids, n);
}

// presence[b] = bitmap of history[b, 0 .. T).  grid B
__global__ void presence_init_kernel(const int64_t* __restrict__ history, int hist_ld, int T, int V,
                                     uint32_t* __restrict__ presence) {
  griddep_wait();
  const int b = blockIdx.x, W = (V + 31) >> 5;
  uint32_t* p = presence + (size_t)b * W;
  for (int w = threadIdx.x; w < W; w += blockDim.x) p[w] = 0u;
  __syncthreads();
  for (int t = threadIdx.x; t < T; t += blockDim.x) {
    const int64_t id = history[(size_t)b * hist_ld + t];
    if (id >= 0 && id < V) atomicOr(&p[id >> 5], 1u << (id & 31));
  }
}

// compact head: row r < n of dst [n_pad, K] is row ids[r] of src [V, K] (zeros for an id outside [0, V)), rows
// n .. n_pad - 1 are zeros.  grid n_pad
__global__ void gather_rows_kernel(const bf16* __restrict__ src, const int32_t* __restrict__ ids, int n, int V, int K,
                                   bf16* __restrict__ dst) {
  const int r = blockIdx.x;
  const int id = r < n ? ids[r] : -1;
  const bool ok = id >= 0 && id < V;
  const uint4* s = reinterpret_cast<const uint4*>(src + (size_t)(ok ? id : 0) * K);
  uint4* d = reinterpret_cast<uint4*>(dst + (size_t)r * K);
  for (int c = threadIdx.x; c < K / 8; c += blockDim.x) d[c] = ok ? s[c] : make_uint4(0u, 0u, 0u, 0u);
}

// prompt fan-out: the first lens[b] rows of the [T_cache][row_bytes] plane of (layer | K/V, row b, kv head) go to rows
// b*k .. b*k+k-1 of the destination.  grid (B * KVH, 2 L)
__global__ void kv_fanout_kernel(const uint4* __restrict__ src, uint4* __restrict__ dst, const int32_t* __restrict__ lens,
                                 int B, int k, int KVH, int T_cache, int row16) {
  griddep_wait();
  const int b = blockIdx.x / KVH, kvh = blockIdx.x % KVH, lw = blockIdx.y;
  const int n = min(max(lens[b], 0), T_cache) * row16;
  const size_t plane = (size_t)T_cache * row16;
  const uint4* s = src + (((size_t)lw * B + b) * KVH + kvh) * plane;
  for (int j = 0; j < k; ++j) {
    uint4* d = dst + (((size_t)lw * B * k + (size_t)b * k + j) * KVH + kvh) * plane;
    for (int i = threadIdx.x; i < n; i += blockDim.x) d[i] = s[i];
  }
}

}  // namespace

int sk_kv_prefill_launch(const bf16* qkv, long layer_stride, int ldq, bf16* cache, const int32_t* lens, int L, int B, int T,
                         int H, int KVH, int T_cache, cudaStream_t s) {
  SK_REQUIRE(ldq % 8 == 0, "kv_prefill: ldq must be a multiple of 8");
  SK_CUDA_CHECK(sk_launch_pdl(kv_prefill_kernel<bf16>, dim3(B * T, L), dim3(64), (size_t)0, s, qkv, (const bf16*)nullptr,
                              layer_stride, ldq, cache, lens, B, T, H, KVH, T_cache));
  SK_LAUNCH_CHECK();
  return 0;
}
int sk_kv_prefill_f32_launch(const bf16* qkv_hi, const bf16* qkv_lo, int ldq, float* cache, const int32_t* lens, int B, int T,
                             int H, int T_cache, cudaStream_t s) {
  SK_REQUIRE(ldq % 8 == 0, "kv_prefill: ldq must be a multiple of 8");
  SK_CUDA_CHECK(sk_launch_pdl(kv_prefill_kernel<float>, dim3(B * T, 1), dim3(64), (size_t)0, s, qkv_hi, qkv_lo, 0L, ldq, cache,
                              lens, B, T, H, H, T_cache));
  SK_LAUNCH_CHECK();
  return 0;
}

int sk_kv_append_launch(const bf16* qkv, int ldq, bf16* kc, bf16* vc, const int32_t* pos, int32_t* lens, int B, int H,
                        int KVH, int T_cache, cudaStream_t s) {
  SK_CUDA_CHECK(sk_launch_pdl(kv_append_kernel<bf16>, dim3(B), dim3(64), (size_t)0, s, qkv, (const bf16*)nullptr, ldq, kc, vc,
                              pos, lens, H, KVH, T_cache));
  SK_LAUNCH_CHECK();
  return 0;
}
int sk_kv_append_f32_launch(const bf16* qkv_hi, const bf16* qkv_lo, int ldq, float* kc, float* vc, const int32_t* pos,
                            int32_t* lens, int B, int H, int T_cache, cudaStream_t s) {
  SK_CUDA_CHECK(sk_launch_pdl(kv_append_kernel<float>, dim3(B), dim3(64), (size_t)0, s, qkv_hi, qkv_lo, ldq, kc, vc, pos, lens,
                              H, H, T_cache));
  SK_LAUNCH_CHECK();
  return 0;
}

int sk_gather_last_launch(const bf16* x, const int32_t* lens, bf16* out, int B, int T, int D, cudaStream_t s) {
  SK_REQUIRE(D % 8 == 0, "gather_last: D must be a multiple of 8");
  SK_CUDA_CHECK(sk_launch_pdl(gather_last_kernel, dim3(B), dim3(128), (size_t)0, s, x, lens, out, T, D));
  SK_LAUNCH_CHECK();
  return 0;
}

int sk_kv_fanout_launch(const void* src, void* dst, const int32_t* lens, int L, int B, int k, int KVH, int T_cache,
                        int row_bytes, cudaStream_t s) {
  SK_REQUIRE(B > 0 && k > 0 && L > 0 && KVH > 0 && T_cache > 0 && row_bytes % 16 == 0, "kv_fanout: bad shape B=%d k=%d "
             "T_cache=%d row_bytes=%d", B, k, T_cache, row_bytes);
  SK_REQUIRE((((uintptr_t)src | (uintptr_t)dst) & 15) == 0, "kv_fanout: caches must be 16-byte aligned");
  SK_CUDA_CHECK(sk_launch_pdl(kv_fanout_kernel, dim3(B * KVH, 2 * L), dim3(256), (size_t)0, s,
                              reinterpret_cast<const uint4*>(src), reinterpret_cast<uint4*>(dst), lens, B, k, KVH, T_cache,
                              row_bytes / 16));
  SK_LAUNCH_CHECK();
  return 0;
}

int sk_attn_decode_splits(int T_cache) { return (T_cache + DEC_CH - 1) / DEC_CH; }

// KV = bf16: q, o bf16 (q_lo, o_lo unused); KV = float: q and o are (hi, lo) pairs
template <typename KV>
int attn_decode(const bf16* q, const bf16* q_lo, int ldq, const KV* kc, const KV* vc, const int32_t* lens, bf16* o, bf16* o_lo,
                int ldo, float* partial, int B, int H, int KVH, int T_cache, float scale, cudaStream_t s) {
  SK_REQUIRE(B > 0 && H > 0 && KVH > 0 && T_cache > 0 && H % KVH == 0 && H / KVH <= DEC_MAX_G,
             "attn_decode: bad shape B=%d H=%d KVH=%d T_cache=%d (H/KVH <= %d)", B, H, KVH, T_cache, DEC_MAX_G);
  SK_REQUIRE(ldq % 8 == 0 && ldo % 2 == 0, "attn_decode: ldq must be a multiple of 8 and ldo even");
  const int S = sk_attn_decode_splits(T_cache);
  float* part_o = partial;
  float2* part_ml = reinterpret_cast<float2*>(partial + (size_t)B * H * S * 64);
  const size_t smem = (size_t)2 * DEC_CH * dec_kpad<KV>() * sizeof(KV) + (size_t)2 * DEC_MAX_G * 64 * sizeof(float);
  constexpr bool split = sizeof(KV) == 4;
  sk_prof_begin(1, s);
  cudaError_t e = sk_launch_pdl(attn_decode_split_kernel<KV>, dim3(S, KVH, B), dim3(DEC_THREADS), smem, s, q, q_lo, ldq, kc, vc,
                                lens, part_o, part_ml, H, KVH, T_cache, S, scale * 1.4426950408889634f);
  if (e == cudaSuccess)
    e = sk_launch_pdl(attn_decode_combine_kernel<split>, dim3((B * H + 3) / 4), dim3(128), (size_t)0, s,
                      (const float*)part_o, (const float2*)part_ml, lens, o, o_lo, ldo, B, H, S);
  sk_prof_end(s);
  SK_CUDA_CHECK(e);
  SK_LAUNCH_CHECK();
  return 0;
}

int sk_attn_decode_launch(const bf16* q, int ldq, const bf16* kc, const bf16* vc, const int32_t* lens, bf16* o, int ldo,
                          float* partial, int B, int H, int KVH, int T_cache, float scale, cudaStream_t s) {
  return attn_decode<bf16>(q, nullptr, ldq, kc, vc, lens, o, nullptr, ldo, partial, B, H, KVH, T_cache, scale, s);
}
int sk_attn_decode_f32_launch(const bf16* q_hi, const bf16* q_lo, int ldq, const float* kc, const float* vc, const int32_t* lens,
                              bf16* o_hi, bf16* o_lo, int ldo, float* partial, int B, int H, int T_cache, float scale,
                              cudaStream_t s) {
  return attn_decode<float>(q_hi, q_lo, ldq, kc, vc, lens, o_hi, o_lo, ldo, partial, B, H, H, T_cache, scale, s);
}

template <typename LT>
int select_next(const LT* logits, int ldl, int V, int B, const uint32_t* ban, const SkSampling& cfg, const float* uniforms,
                const SkDecodeState& st, cudaStream_t s, const SkLogitRules* rules = nullptr) {
  SK_REQUIRE(B > 0 && V > 0 && ldl >= V, "select_next: bad shape B=%d V=%d ldl=%d", B, V, ldl);
  SK_REQUIRE(cfg.n_eos >= 0 && cfg.n_eos <= 8, "select_next: at most 8 eos ids");
  SK_REQUIRE(!cfg.do_sample || cfg.temperature > 0.f, "select_next: temperature must be > 0");
  SK_REQUIRE(st.tokens && st.pos && st.finished && st.n_gen && st.out && st.step && st.max_new > 0,
             "select_next: incomplete decode state");
  if (rules) {
    const SkLogitRules& r = *rules;
    SK_REQUIRE(r.history && r.prompt_len >= 0 && r.hist_ld >= r.prompt_len + st.max_new,
               "select_next_ex: history [B, hist_ld] with hist_ld >= prompt_len + max_new required (prompt_len=%d "
               "hist_ld=%d max_new=%d)", r.prompt_len, r.hist_ld, st.max_new);
    SK_REQUIRE(r.penalty > 0.f, "select_next_ex: repetition penalty must be > 0");
    SK_REQUIRE(r.penalty == 1.f || r.presence, "select_next_ex: the repetition penalty needs the presence bitmap");
    SK_REQUIRE(r.scratch || (r.ngram <= 0 && (r.min_step <= 0 || cfg.n_eos == 0)),
               "select_next_ex: n-gram and min-length bans need the scratch bitmap");
    SK_CUDA_CHECK(sk_launch_pdl(select_next_kernel<LT, true>, dim3(B), dim3(SEL_THREADS), (size_t)0, s, logits, ldl, V, ban,
                                cfg, uniforms, st, r));
  } else {
    SK_CUDA_CHECK(sk_launch_pdl(select_next_kernel<LT, false>, dim3(B), dim3(SEL_THREADS), (size_t)0, s, logits, ldl, V, ban,
                                cfg, uniforms, st, SkLogitRules{}));
  }
  SK_LAUNCH_CHECK();
  return 0;
}
int sk_select_next_launch(const bf16* logits, int ldl, int V, int B, const uint32_t* ban, const SkSampling& cfg,
                          const float* uniforms, const SkDecodeState& st, cudaStream_t s) {
  return select_next<bf16>(logits, ldl, V, B, ban, cfg, uniforms, st, s);
}

int sk_gather_rows_launch(const bf16* src, const int32_t* ids, int n, int n_pad, int V, int K, bf16* dst, cudaStream_t s) {
  SK_REQUIRE(src && ids && dst && n > 0 && n <= n_pad && K > 0 && K % 8 == 0, "gather_rows: bad arguments n=%d n_pad=%d K=%d",
             n, n_pad, K);
  SK_REQUIRE((((uintptr_t)src | (uintptr_t)dst) & 15) == 0, "gather_rows: rows must be 16-byte aligned");
  gather_rows_kernel<<<n_pad, 128, 0, s>>>(src, ids, n, V, K, dst);
  SK_LAUNCH_CHECK();
  return 0;
}

extern "C" {

int64_t sk_attn_decode_partial_bytes(int B, int H, int T_cache) {
  if (B <= 0 || H <= 0 || T_cache <= 0) return 0;
  return (int64_t)B * H * sk_attn_decode_splits(T_cache) * (64 + 2) * (int64_t)sizeof(float);
}

int sk_attn_decode(const void* q, int ldq, const void* k_cache, const void* v_cache, const int32_t* lens, void* o, int ldo,
                   float* partial, int B, int H, int KVH, int T_cache, float scale, void* stream) {
  SK_REQUIRE(q && k_cache && v_cache && lens && o && partial, "sk_attn_decode: null argument");
  return sk_attn_decode_launch(reinterpret_cast<const bf16*>(q), ldq, reinterpret_cast<const bf16*>(k_cache),
                               reinterpret_cast<const bf16*>(v_cache), lens, reinterpret_cast<bf16*>(o), ldo, partial, B, H,
                               KVH, T_cache, scale, (cudaStream_t)stream);
}

int sk_select_next(const void* logits, int ldl, int V, int B, const uint32_t* ban_bits, const SkSampling* cfg,
                   const float* uniforms, const SkDecodeState* state, void* stream) {
  SK_REQUIRE(logits && cfg && state, "sk_select_next: null argument");
  return sk_select_next_launch(reinterpret_cast<const bf16*>(logits), ldl, V, B, ban_bits, *cfg, uniforms, *state,
                               (cudaStream_t)stream);
}

int sk_select_next_f32(const float* logits, int ldl, int V, int B, const uint32_t* ban_bits, const SkSampling* cfg,
                       const float* uniforms, const SkDecodeState* state, void* stream) {
  SK_REQUIRE(logits && cfg && state, "sk_select_next_f32: null argument");
  SK_REQUIRE(((uintptr_t)logits & 15) == 0, "sk_select_next_f32: logits must be 16-byte aligned");
  return select_next<float>(logits, ldl, V, B, ban_bits, *cfg, uniforms, *state, (cudaStream_t)stream);
}

int sk_select_next_ex(const void* logits, int ldl, int V, int B, const uint32_t* ban_bits, const SkSampling* cfg,
                      const float* uniforms, const SkDecodeState* state, const SkLogitRules* rules, void* stream) {
  SK_REQUIRE(logits && cfg && state && rules, "sk_select_next_ex: null argument");
  return select_next<bf16>(reinterpret_cast<const bf16*>(logits), ldl, V, B, ban_bits, *cfg, uniforms, *state,
                           (cudaStream_t)stream, rules);
}

int sk_select_next_ex_f32(const float* logits, int ldl, int V, int B, const uint32_t* ban_bits, const SkSampling* cfg,
                          const float* uniforms, const SkDecodeState* state, const SkLogitRules* rules, void* stream) {
  SK_REQUIRE(logits && cfg && state && rules, "sk_select_next_ex_f32: null argument");
  SK_REQUIRE(((uintptr_t)logits & 15) == 0, "sk_select_next_ex_f32: logits must be 16-byte aligned");
  return select_next<float>(logits, ldl, V, B, ban_bits, *cfg, uniforms, *state, (cudaStream_t)stream, rules);
}

int sk_select_next_sub(const void* logits, int ld_sub, const int32_t* ids, int n, int V, int B, const SkSampling* cfg,
                       const float* uniforms, const SkDecodeState* state, void* stream) {
  SK_REQUIRE(logits && ids && cfg && state, "sk_select_next_sub: null argument");
  SK_REQUIRE(B > 0 && n > 0 && n <= V && ld_sub >= n, "sk_select_next_sub: bad shape B=%d n=%d V=%d ld_sub=%d", B, n, V,
             ld_sub);
  SK_REQUIRE(cfg->n_eos >= 0 && cfg->n_eos <= 8, "sk_select_next_sub: at most 8 eos ids");
  SK_REQUIRE(!cfg->do_sample || cfg->temperature > 0.f, "sk_select_next_sub: temperature must be > 0");
  const SkDecodeState& st = *state;
  SK_REQUIRE(st.tokens && st.pos && st.finished && st.n_gen && st.out && st.step && st.max_new > 0,
             "sk_select_next_sub: incomplete decode state");
  SK_CUDA_CHECK(sk_launch_pdl(select_next_sub_kernel, dim3(B), dim3(SEL_THREADS), (size_t)0, (cudaStream_t)stream,
                              reinterpret_cast<const bf16*>(logits), ld_sub, V, *cfg, uniforms, st, ids, n));
  SK_LAUNCH_CHECK();
  return 0;
}

int sk_presence_init(const int64_t* history, int hist_ld, int prompt_len, int B, int V, uint32_t* presence, void* stream) {
  SK_REQUIRE(history && presence, "sk_presence_init: null argument");
  SK_REQUIRE(B > 0 && V > 0 && prompt_len >= 0 && hist_ld >= prompt_len, "sk_presence_init: bad shape B=%d V=%d T=%d "
             "hist_ld=%d", B, V, prompt_len, hist_ld);
  SK_CUDA_CHECK(sk_launch_pdl(presence_init_kernel, dim3(B), dim3(256), (size_t)0, (cudaStream_t)stream, history, hist_ld,
                              prompt_len, V, presence));
  SK_LAUNCH_CHECK();
  return 0;
}

int sk_attn_decode_split(const void* q_hi, const void* q_lo, int ldq, const float* k_cache, const float* v_cache,
                         const int32_t* lens, void* o_hi, void* o_lo, int ldo, float* partial, int B, int H, int T_cache,
                         float scale, void* stream) {
  SK_REQUIRE(q_hi && q_lo && k_cache && v_cache && lens && o_hi && o_lo && partial, "sk_attn_decode_split: null argument");
  return sk_attn_decode_f32_launch(reinterpret_cast<const bf16*>(q_hi), reinterpret_cast<const bf16*>(q_lo), ldq, k_cache,
                                   v_cache, lens, reinterpret_cast<bf16*>(o_hi), reinterpret_cast<bf16*>(o_lo), ldo, partial,
                                   B, H, T_cache, scale, (cudaStream_t)stream);
}

}  // extern "C"
