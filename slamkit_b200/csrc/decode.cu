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
constexpr int DEC_KPAD = 72;      // smem row pitch of the K / V tiles (144 B: conflict-free 16-byte row reads)
constexpr int DEC_MAX_G = 16;     // query heads per kv head served by one CTA

// ---- KV cache ---------------------------------------------------------------------------------------------------
// cache layout per layer: [K|V][B][KVH][T_cache][64] bf16, K after RoPE

// prefill: copy K/V of positions t < lens[b] of every layer out of the fused projections [B*T, ldq] (layer stride
// `layer_stride` elements) into the cache.  grid (B*T, L)
__global__ void kv_prefill_kernel(const bf16* __restrict__ qkv, long layer_stride, int ldq, bf16* __restrict__ cache,
                                  const int32_t* __restrict__ lens, int B, int T, int H, int KVH, int T_cache) {
  griddep_wait();
  const int row = blockIdx.x, l = blockIdx.y;
  const int b = row / T, t = row % T;
  if (t >= lens[b] || t >= T_cache) return;
  const bf16* src = qkv + l * layer_stride + (size_t)row * ldq + (size_t)H * 64;
  const size_t plane = (size_t)B * KVH * T_cache * 64;
  bf16* kc = cache + (size_t)l * 2 * plane;
  for (int i = threadIdx.x; i < 2 * KVH * 8; i += blockDim.x) {
    const int which = i / (KVH * 8), r = i % (KVH * 8), kvh = r / 8, c = r % 8;
    bf16* dst = kc + which * plane + (((size_t)b * KVH + kvh) * T_cache + t) * 64 + c * 8;
    stg128(dst, ldg128(src + (size_t)(which * KVH + kvh) * 64 + c * 8));
  }
}

// decode: append the K/V of the one new token of every row at pos[b] and publish lens[b] = pos[b] + 1.  grid B
__global__ void kv_append_kernel(const bf16* __restrict__ qkv, int ldq, bf16* __restrict__ kc, bf16* __restrict__ vc,
                                 const int32_t* __restrict__ pos, int32_t* __restrict__ lens, int H, int KVH, int T_cache) {
  griddep_wait();
  const int b = blockIdx.x;
  const int p = min(max(pos[b], 0), T_cache - 1);
  const bf16* src = qkv + (size_t)b * ldq + (size_t)H * 64;
  for (int i = threadIdx.x; i < 2 * KVH * 8; i += blockDim.x) {
    const int which = i / (KVH * 8), r = i % (KVH * 8), kvh = r / 8, c = r % 8;
    bf16* dst = (which ? vc : kc) + (((size_t)b * KVH + kvh) * T_cache + p) * 64 + c * 8;
    stg128(dst, ldg128(src + (size_t)(which * KVH + kvh) * 64 + c * 8));
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
// split order.  CTAs whose range starts at or past lens[b] exit before touching the cache.
__global__ void __launch_bounds__(DEC_THREADS) attn_decode_split_kernel(
    const bf16* __restrict__ q, int ldq, const bf16* __restrict__ kc, const bf16* __restrict__ vc,
    const int32_t* __restrict__ lens, float* __restrict__ part_o, float2* __restrict__ part_ml, int H, int KVH,
    int T_cache, int S, float scale_log2) {
  extern __shared__ __align__(16) uint8_t dec_smem[];
  bf16* sK = reinterpret_cast<bf16*>(dec_smem);
  bf16* sV = sK + DEC_CH * DEC_KPAD;
  float* sQ = reinterpret_cast<float*>(sV + DEC_CH * DEC_KPAD);   // [G][64], pre-scaled by scale * log2(e)
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
  for (int i = tid; i < n * 8; i += DEC_THREADS) {
    const int r = i >> 3, c = i & 7;
    *reinterpret_cast<uint4*>(sK + r * DEC_KPAD + c * 8) = ldg128_stream(kc + base + (size_t)r * 64 + c * 8);
    *reinterpret_cast<uint4*>(sV + r * DEC_KPAD + c * 8) = ldg128_stream(vc + base + (size_t)r * 64 + c * 8);
  }
  for (int i = tid; i < G * 8; i += DEC_THREADS) {
    const int g = i >> 3, c = i & 7;
    const uint4 v = ldg128(q + (size_t)b * ldq + (size_t)(kvh * G + g) * 64 + c * 8);
    const uint32_t u[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float2 f = unpack_bf16(u[k]);
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
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        const uint4 v = *reinterpret_cast<const uint4*>(sK + j * DEC_KPAD + c * 8);
        const uint32_t u[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const float2 f = unpack_bf16(u[k]);
          kf[c * 8 + 2 * k] = f.x;
          kf[c * 8 + 2 * k + 1] = f.y;
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
    const float2 v = __bfloat1622float2(*reinterpret_cast<const bf162*>(sV + j * DEC_KPAD + 2 * lane));
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

// one warp per (row, head): merge the ceil(lens[b] / 64) valid splits in split order
__global__ void __launch_bounds__(128) attn_decode_combine_kernel(const float* __restrict__ part_o,
                                                                  const float2* __restrict__ part_ml,
                                                                  const int32_t* __restrict__ lens, bf16* __restrict__ o,
                                                                  int ldo, int B, int H, int S) {
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
  *reinterpret_cast<bf162*>(o + (size_t)b * ldo + h * 64 + 2 * lane) = __floats2bfloat162_rn(acc.x * inv, acc.y * inv);
}

// ---- token selection -------------------------------------------------------------------------------------------
constexpr int SEL_THREADS = 512;
constexpr int SEL_WARPS = SEL_THREADS / 32;

SK_DEVINL uint32_t ordered_key(float f) {
  const uint32_t u = __float_as_uint(f);
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

struct SelRow {
  const bf16* row;
  const uint32_t* ban;
  float temp;
  bool use_temp;
  SK_DEVINL float score(int i) const {
    if (ban && ((ban[i >> 5] >> (i & 31)) & 1u)) return -INFINITY;
    const float x = __bfloat162float(row[i]);
    return use_temp ? __fdiv_rn(x, temp) : x;
  }
};

// One CTA per row.  Order of HF's processors: bans -> (sampling only) temperature -> top-k -> top-p -> softmax -> draw;
// greedy = argmax of the banned scores, lowest id on ties.  Each thread owns the contiguous id range
// [tid * chunk, (tid + 1) * chunk), so per-thread partial sums are in token order and every sum is taken in a fixed order.
__global__ void __launch_bounds__(SEL_THREADS) select_next_kernel(const bf16* __restrict__ logits, int ldl, int V,
                                                                  const uint32_t* __restrict__ ban, SkSampling cfg,
                                                                  const float* __restrict__ uniforms, SkDecodeState st) {
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
    }
    return;
  }
  const int chunk = (V + SEL_THREADS - 1) / SEL_THREADS;
  const int i0 = min(tid * chunk, V), i1 = min(i0 + chunk, V);
  SelRow R{logits + (size_t)b * ldl, ban, cfg.temperature, cfg.do_sample != 0 && cfg.temperature != 1.0f};
  int tok = 0;
  if (!cfg.do_sample) {
    // argmax, lowest id among equal maxima
    float bv = -INFINITY;
    int bi = 0x7fffffff;
    for (int i = i0; i < i1; ++i) {
      const float v = R.score(i);
      if (v > bv || (v == bv && i < bi)) { bv = v; bi = i; }
    }
    // pack (ordered value, inverted id) so that one max picks the largest value, then the smallest id
    unsigned long long key = ((unsigned long long)ordered_key(bv) << 32) | (uint32_t)(0x7fffffff - min(bi, 0x7fffffff));
    key = block_reduce(key, red_u, [](unsigned long long a, unsigned long long c) { return a > c ? a : c; });
    tok = 0x7fffffff - (int)(uint32_t)(key & 0xffffffffu);
    if (tok >= V) tok = 0;
  } else {
    // top-k: the k-th largest score by radix select on order-preserving keys (HF keeps every score >= it)
    const int k = cfg.top_k > 0 ? min(cfg.top_k, V) : V;
    uint32_t kth = 0;
    if (k < V) {
      uint32_t prefix = 0, mask = 0;
      int rank = k;
      for (int shift = 24; shift >= 0; shift -= 8) {
        for (int i = tid; i < 256; i += SEL_THREADS) hist[i] = 0;
        __syncthreads();
        for (int i = i0; i < i1; ++i) {
          const uint32_t key = ordered_key(R.score(i));
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
    for (int i = i0; i < i1; ++i) {
      const float v = R.score(i);
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
      for (int i = i0; i < i1; ++i) {
        const float v = R.score(i);
        if (ordered_key(v) >= kth) z += expf(v - mx);
      }
      float ztot;
      block_exclusive_scan(z, red_f, ztot);
      auto mass_le = [&](uint32_t K) {
        float m = 0.f;
        for (int i = i0; i < i1; ++i) {
          const float v = R.score(i);
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
      for (int i = i0; i < i1; ++i) {
        const float v = R.score(i);
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
          for (int i = i0; i < i1; ++i) {
            if (ordered_key(R.score(i)) == cut_key && ++seen == drop) { id = i; break; }
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
    for (int i = i0; i < i1; ++i) {
      const float v = R.score(i);
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
      for (int i = i0; i < i1; ++i) {
        const float v = R.score(i);
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
  }
}

}  // namespace

int sk_kv_prefill_launch(const bf16* qkv, long layer_stride, int ldq, bf16* cache, const int32_t* lens, int L, int B, int T,
                         int H, int KVH, int T_cache, cudaStream_t s) {
  SK_REQUIRE(ldq % 8 == 0, "kv_prefill: ldq must be a multiple of 8");
  SK_CUDA_CHECK(sk_launch_pdl(kv_prefill_kernel, dim3(B * T, L), dim3(64), (size_t)0, s, qkv, layer_stride, ldq, cache, lens,
                              B, T, H, KVH, T_cache));
  SK_LAUNCH_CHECK();
  return 0;
}

int sk_kv_append_launch(const bf16* qkv, int ldq, bf16* kc, bf16* vc, const int32_t* pos, int32_t* lens, int B, int H,
                        int KVH, int T_cache, cudaStream_t s) {
  SK_CUDA_CHECK(sk_launch_pdl(kv_append_kernel, dim3(B), dim3(64), (size_t)0, s, qkv, ldq, kc, vc, pos, lens, H, KVH, T_cache));
  SK_LAUNCH_CHECK();
  return 0;
}

int sk_gather_last_launch(const bf16* x, const int32_t* lens, bf16* out, int B, int T, int D, cudaStream_t s) {
  SK_REQUIRE(D % 8 == 0, "gather_last: D must be a multiple of 8");
  SK_CUDA_CHECK(sk_launch_pdl(gather_last_kernel, dim3(B), dim3(128), (size_t)0, s, x, lens, out, T, D));
  SK_LAUNCH_CHECK();
  return 0;
}

int sk_attn_decode_splits(int T_cache) { return (T_cache + DEC_CH - 1) / DEC_CH; }

int sk_attn_decode_launch(const bf16* q, int ldq, const bf16* kc, const bf16* vc, const int32_t* lens, bf16* o, int ldo,
                          float* partial, int B, int H, int KVH, int T_cache, float scale, cudaStream_t s) {
  SK_REQUIRE(B > 0 && H > 0 && KVH > 0 && T_cache > 0 && H % KVH == 0 && H / KVH <= DEC_MAX_G,
             "attn_decode: bad shape B=%d H=%d KVH=%d T_cache=%d (H/KVH <= %d)", B, H, KVH, T_cache, DEC_MAX_G);
  SK_REQUIRE(ldq % 8 == 0 && ldo % 2 == 0, "attn_decode: ldq must be a multiple of 8 and ldo even");
  const int S = sk_attn_decode_splits(T_cache);
  float* part_o = partial;
  float2* part_ml = reinterpret_cast<float2*>(partial + (size_t)B * H * S * 64);
  const size_t smem = (size_t)2 * DEC_CH * DEC_KPAD * sizeof(bf16) + (size_t)2 * DEC_MAX_G * 64 * sizeof(float);
  sk_prof_begin(1, s);
  cudaError_t e = sk_launch_pdl(attn_decode_split_kernel, dim3(S, KVH, B), dim3(DEC_THREADS), smem, s, q, ldq, kc, vc, lens,
                                part_o, part_ml, H, KVH, T_cache, S, scale * 1.4426950408889634f);
  if (e == cudaSuccess)
    e = sk_launch_pdl(attn_decode_combine_kernel, dim3((B * H + 3) / 4), dim3(128), (size_t)0, s,
                      (const float*)part_o, (const float2*)part_ml, lens, o, ldo, B, H, S);
  sk_prof_end(s);
  SK_CUDA_CHECK(e);
  SK_LAUNCH_CHECK();
  return 0;
}

int sk_select_next_launch(const bf16* logits, int ldl, int V, int B, const uint32_t* ban, const SkSampling& cfg,
                          const float* uniforms, const SkDecodeState& st, cudaStream_t s) {
  SK_REQUIRE(B > 0 && V > 0 && ldl >= V, "select_next: bad shape B=%d V=%d ldl=%d", B, V, ldl);
  SK_REQUIRE(cfg.n_eos >= 0 && cfg.n_eos <= 8, "select_next: at most 8 eos ids");
  SK_REQUIRE(!cfg.do_sample || cfg.temperature > 0.f, "select_next: temperature must be > 0");
  SK_REQUIRE(st.tokens && st.pos && st.finished && st.n_gen && st.out && st.step && st.max_new > 0,
             "select_next: incomplete decode state");
  SK_CUDA_CHECK(sk_launch_pdl(select_next_kernel, dim3(B), dim3(SEL_THREADS), (size_t)0, s, logits, ldl, V, ban, cfg,
                              uniforms, st));
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

}  // extern "C"
