// Sequence scoring for the modelling metrics of cli/eval.py (sWUGGY, sBLIMP, StoryCloze, SALMon): the tail of
// UnitLM.log_likelihood (slamkit/model/unit_lm.py:184-194 -> calc_nll, slamkit/utils/calculation_utils.py:5-29) on the
// bf16 logits the forward pass leaves in the workspace, plus the unit-id -> token-id step of UnitTokeniser.tokenise.
//
// The reference model runs in bf16, so its numbers carry bf16 rounding at fixed points, and the metric's tie rule (0.5 for
// equal scores) sees them:
//   nll_t = -bf16((z_y - max) - log(sum exp(z - max)))       log_softmax in fp32, rounded to bf16 (torch's bf16 kernel)
//   seq   = bf16(sum_t nll_t)                                fp32 accumulation of the bf16 values, one rounding
//   mean  = bf16(seq / count)                                bf16 / int64 -> float division, one rounding
// Banned columns are -inf before the softmax; a target equal to the model's pad id is masked (0, not counted).
// An fp32 model (sk_seq_loglik_f32: fp32 OPT inference) is scored in fp32 throughout, as calc_nll does on fp32 logits:
// the same kernels on fp32 logits with every bf16 rounding above left out.
#include "kernels.h"
#include "../../include/slamkit_b200.h"

namespace {

constexpr float kLog2e = 1.4426950408889634f;
constexpr int kWarpRowMaxV = 8192;   // up to this many columns a warp scores a row; beyond it a 256-thread CTA does

SK_DEVINL float logit_at(const bf16* row, long i) { return __bfloat162float(row[i]); }
SK_DEVINL float logit_at(const float* row, long i) { return row[i]; }

// eight columns [c0, c0 + 8) of a logits row as fp32, -inf where banned or at/after V (those columns are not read)
SK_DEVINL void load8(const float* __restrict__ row, int c0, int V, const uint32_t* __restrict__ ban, float (&v)[8]) {
  const uint32_t bits = ban ? (__ldg(ban + (c0 >> 5)) >> (c0 & 31)) & 0xffu : 0u;
  if (c0 + 8 <= V) {
    const float4 a = __ldcs(reinterpret_cast<const float4*>(row + c0)), b = __ldcs(reinterpret_cast<const float4*>(row + c0 + 4));
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w;
    v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
  } else {
#pragma unroll
    for (int k = 0; k < 8; ++k) v[k] = (c0 + k < V) ? row[c0 + k] : -INFINITY;
  }
#pragma unroll
  for (int k = 0; k < 8; ++k)
    if ((bits >> k) & 1u) v[k] = -INFINITY;
}
SK_DEVINL void load8(const bf16* __restrict__ row, int c0, int V, const uint32_t* __restrict__ ban, float (&v)[8]) {
  const uint32_t bits = ban ? (__ldg(ban + (c0 >> 5)) >> (c0 & 31)) & 0xffu : 0u;
  if (c0 + 8 <= V) {
    const uint4 lv = ldg128_stream(row + c0);
    const uint32_t u[4] = {lv.x, lv.y, lv.z, lv.w};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float2 f = unpack_bf16(u[k]);
      v[2 * k] = f.x;
      v[2 * k + 1] = f.y;
    }
  } else {
#pragma unroll
    for (int k = 0; k < 8; ++k) v[k] = (c0 + k < V) ? __bfloat162float(row[c0 + k]) : -INFINITY;
  }
#pragma unroll
  for (int k = 0; k < 8; ++k)
    if ((bits >> k) & 1u) v[k] = -INFINITY;
}

// online (max, sum exp(z - max)) over one chunk
SK_DEVINL void ms_update(const float (&v)[8], float& m, float& s) {
  float cm = v[0];
#pragma unroll
  for (int k = 1; k < 8; ++k) cm = fmaxf(cm, v[k]);
  if (cm == -INFINITY) return;
  const float mn = fmaxf(m, cm);
  float acc = 0.f;
#pragma unroll
  for (int k = 0; k < 8; ++k) acc += ex2_approx((v[k] - mn) * kLog2e);
  s = s * ex2_approx((m - mn) * kLog2e) + acc;     // m == -inf: s is 0 and ex2(-inf) = 0
  m = mn;
}

SK_DEVINL void ms_combine(float& m, float& s, float m2, float s2) {
  const float mn = fmaxf(m, m2);
  if (mn > -INFINITY) s = s * ex2_approx((m - mn) * kLog2e) + s2 * ex2_approx((m2 - mn) * kLog2e);
  m = mn;
}

SK_DEVINL void ms_warp(float& m, float& s) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float m2 = __shfl_xor_sync(0xffffffffu, m, o), s2 = __shfl_xor_sync(0xffffffffu, s, o);
    ms_combine(m, s, m2, s2);
  }
}

// target logit of a row (-inf when banned): the same value the softmax saw
template <typename LT>
SK_DEVINL float target_logit(const LT* __restrict__ row, long y, const uint32_t* __restrict__ ban) {
  if (ban && ((__ldg(ban + (y >> 5)) >> (y & 31)) & 1u)) return -INFINITY;
  return logit_at(row, y);
}

// torch's log_softmax epilogue ((x - max) - log(sum)) in fp32, rounded to bf16 on a bf16 model, negated by nll_loss
template <bool ROUND>
SK_DEVINL float token_value(float zy, float m, float s) {
  const float lp = (zy - m) - logf(s);
  return -(ROUND ? bf16_round(lp) : lp);
}

// Scoring row r = b * (T - 1) + t: logits row b * T + t against target ids[b, t + 1].  A pad target is masked: its
// logits row is not read and its value is 0.  A target outside [0, V) gives NaN.
struct RowTarget {
  long y;
  int state;   // 0 score, 1 masked, 2 out of range
};
SK_DEVINL RowTarget row_target(const int64_t* __restrict__ ids, int r, int T, int V, int pad) {
  const int b = r / (T - 1), t = r % (T - 1);
  const long y = ids[(size_t)b * T + t + 1];
  return {y, y == pad ? 1 : (y < 0 || y >= V) ? 2 : 0};
}

template <typename LT, bool ROUND>
__global__ void __launch_bounds__(256)
seqll_warp_kernel(const LT* __restrict__ logits, int ldl, int V, const int64_t* __restrict__ ids, int R, int T, int pad,
                  const uint32_t* __restrict__ ban, float* __restrict__ token_nll) {
  const int r = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (r >= R) return;
  const RowTarget tg = row_target(ids, r, T, V, pad);
  if (tg.state != 0) {
    if (lane == 0) token_nll[r] = tg.state == 1 ? 0.f : __int_as_float(0x7fc00000);
    return;
  }
  const int b = r / (T - 1), t = r % (T - 1);
  const LT* row = logits + ((size_t)b * T + t) * ldl;
  float m = -INFINITY, s = 0.f;
  for (int c0 = lane * 8; c0 < V; c0 += 32 * 8) {
    float v[8];
    load8(row, c0, V, ban, v);
    ms_update(v, m, s);
  }
  ms_warp(m, s);
  if (lane == 0) token_nll[r] = token_value<ROUND>(target_logit(row, tg.y, ban), m, s);
}

template <typename LT, bool ROUND>
__global__ void __launch_bounds__(256)
seqll_cta_kernel(const LT* __restrict__ logits, int ldl, int V, const int64_t* __restrict__ ids, int T, int pad,
                 const uint32_t* __restrict__ ban, float* __restrict__ token_nll) {
  __shared__ float s_m[8], s_s[8];
  const int r = blockIdx.x;
  const RowTarget tg = row_target(ids, r, T, V, pad);
  if (tg.state != 0) {
    if (threadIdx.x == 0) token_nll[r] = tg.state == 1 ? 0.f : __int_as_float(0x7fc00000);
    return;
  }
  const int b = r / (T - 1), t = r % (T - 1);
  const LT* row = logits + ((size_t)b * T + t) * ldl;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float m = -INFINITY, s = 0.f;
  // four 16-byte loads in flight per thread before any of them is used
  constexpr int U = 4;
  for (int c0 = threadIdx.x * 8; c0 < V; c0 += U * 256 * 8) {
    float v[U][8];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int c = c0 + u * 256 * 8;
      if (c < V) load8(row, c, V, ban, v[u]);
    }
#pragma unroll
    for (int u = 0; u < U; ++u)
      if (c0 + u * 256 * 8 < V) ms_update(v[u], m, s);
  }
  ms_warp(m, s);
  if (lane == 0) { s_m[warp] = m; s_s[warp] = s; }
  __syncthreads();
  if (threadIdx.x == 0) {
    m = s_m[0];
    s = s_s[0];
#pragma unroll
    for (int i = 1; i < 8; ++i) ms_combine(m, s, s_m[i], s_s[i]);
    token_nll[r] = token_value<ROUND>(target_logit(row, tg.y, ban), m, s);
  }
}

// one warp per sequence: fixed-order fp32 sum of the token values (lane-strided partial sums, then a butterfly)
SK_DEVINL void store_ll(bf16* out, float v) { *out = __float2bfloat16_rn(v); }
SK_DEVINL void store_ll(float* out, float v) { *out = v; }
template <typename OT, bool ROUND>
__global__ void __launch_bounds__(256)
seqll_reduce_kernel(const int64_t* __restrict__ ids, const float* __restrict__ token_nll, int B, int T, int pad, int mean_nll,
                    OT* __restrict__ ll_out) {
  const int b = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (b >= B) return;
  float acc = 0.f;
  int cnt = 0;
  for (int t = lane; t < T - 1; t += 32) {
    if (ids[(size_t)b * T + t + 1] != pad) {
      acc += token_nll[(size_t)b * (T - 1) + t];
      ++cnt;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    acc += __shfl_xor_sync(0xffffffffu, acc, o);
    cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
  }
  if (lane == 0) {
    const float sum = ROUND ? bf16_round(acc) : acc;
    float v = sum;
    if (mean_nll) {   // count 0: 0 / 0 = NaN, as the reference
      v = __fdiv_rn(sum, (float)cnt);
      if (ROUND) v = bf16_round(v);
    }
    store_ll(ll_out + b, -v);
  }
}

__global__ void units_to_tokens_kernel(const int32_t* __restrict__ units, const int32_t* __restrict__ counts, int B,
                                       int T_units, int offset, int bos, int eos, int pad, int64_t* __restrict__ ids,
                                       int T_out) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long)B * T_out) return;
  const int b = (int)(i / T_out), t = (int)(i % T_out);
  const int n = min(max(counts[b], 0), T_units);
  long v;
  if (t == 0) v = bos;
  else if (t <= n) v = (long)units[(size_t)b * T_units + t - 1] + offset;
  else if (t == n + 1) v = eos;
  else v = pad;
  ids[i] = v;
}

// left-padded generation prompt of the interleaved tokeniser: row b = [pad..., prefix..., unit_id[u]..., marker] with the
// attention mask 0 on the pads, 1 elsewhere.  A unit outside [0, n_units) becomes pad (it has no id).
__global__ void units_to_prompt_kernel(const int32_t* __restrict__ units, const int32_t* __restrict__ counts, int B,
                                       int T_units, const int32_t* __restrict__ unit_id, int n_units,
                                       const int32_t* __restrict__ prefix, int n_prefix, int marker, int pad,
                                       int64_t* __restrict__ ids, int64_t* __restrict__ mask, int T_out) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long)B * T_out) return;
  const int b = (int)(i / T_out), t = (int)(i % T_out);
  const int n = min(max(counts[b], 0), T_units);
  const int start = T_out - (n_prefix + n + 1);
  const int j = t - start;
  long v;
  if (j < 0) v = pad;
  else if (j < n_prefix) v = prefix[j];
  else if (j < n_prefix + n) {
    const int u = units[(size_t)b * T_units + j - n_prefix];
    v = u >= 0 && u < n_units ? unit_id[u] : pad;
  } else v = marker;
  ids[i] = v;
  mask[i] = j >= 0 ? 1 : 0;
}

// LT: logits element type; OT: ll_out element type; ROUND: the bf16 model's roundings
template <typename LT, typename OT, bool ROUND>
int seq_loglik(const char* who, const void* logits, int ldl, int V, const int64_t* ids, int B, int T, int pad_id,
               const uint32_t* ban_bits, int mean_nll, float* token_nll, void* ll_out, cudaStream_t s) {
  SK_REQUIRE(logits && ids && token_nll && ll_out, "%s: null argument", who);
  SK_REQUIRE(B > 0 && T >= 1, "%s: bad shape B=%d T=%d", who, B, T);
  SK_REQUIRE(V >= 2 && V <= (1 << 20), "%s: V=%d outside [2, 2^20]", who, V);
  SK_REQUIRE(ldl >= V && ldl % 8 == 0, "%s: ldl must be >= V and a multiple of 8 (ldl=%d V=%d)", who, ldl, V);
  SK_REQUIRE(((uintptr_t)logits & 15) == 0, "%s: logits must be 16-byte aligned", who);
  SK_REQUIRE(((uintptr_t)ban_bits & 3) == 0, "%s: ban_bits must be 4-byte aligned", who);
  SK_REQUIRE(mean_nll == 0 || mean_nll == 1, "%s: mean_nll must be 0 or 1", who);
  SK_REQUIRE((long)B * T < (1L << 31), "%s: B*T=%ld too large", who, (long)B * T);
  const LT* lg = reinterpret_cast<const LT*>(logits);
  const int R = B * (T - 1);
  if (R > 0) {
    if (V <= kWarpRowMaxV)
      seqll_warp_kernel<LT, ROUND><<<(R + 7) / 8, 256, 0, s>>>(lg, ldl, V, ids, R, T, pad_id, ban_bits, token_nll);
    else
      seqll_cta_kernel<LT, ROUND><<<R, 256, 0, s>>>(lg, ldl, V, ids, T, pad_id, ban_bits, token_nll);
    SK_LAUNCH_CHECK();
  }
  seqll_reduce_kernel<OT, ROUND><<<(B + 7) / 8, 256, 0, s>>>(ids, token_nll, B, T, pad_id, mean_nll,
                                                            reinterpret_cast<OT*>(ll_out));
  SK_LAUNCH_CHECK();
  return 0;
}

}  // namespace

extern "C" {

int sk_seq_loglik(const void* logits, int ldl, int V, const int64_t* ids, int B, int T, int pad_id,
                  const uint32_t* ban_bits, int mean_nll, float* token_nll, void* ll_out, void* stream) {
  return seq_loglik<bf16, bf16, true>("sk_seq_loglik", logits, ldl, V, ids, B, T, pad_id, ban_bits, mean_nll, token_nll,
                                      ll_out, (cudaStream_t)stream);
}

int sk_seq_loglik_f32(const float* logits, int ldl, int V, const int64_t* ids, int B, int T, int pad_id,
                      const uint32_t* ban_bits, int mean_nll, float* token_nll, float* ll_out, void* stream) {
  return seq_loglik<float, float, false>("sk_seq_loglik_f32", logits, ldl, V, ids, B, T, pad_id, ban_bits, mean_nll,
                                         token_nll, ll_out, (cudaStream_t)stream);
}

int sk_units_to_tokens(const int32_t* units, const int32_t* counts, int B, int T_units, int offset, int bos, int eos,
                       int pad, int64_t* ids, int T_out, void* stream) {
  SK_REQUIRE(units && counts && ids, "sk_units_to_tokens: null argument");
  SK_REQUIRE(B > 0 && T_units >= 0 && T_out >= 2, "sk_units_to_tokens: bad shape B=%d T_units=%d T_out=%d", B, T_units,
             T_out);
  SK_REQUIRE((long)B * T_out < (1L << 31), "sk_units_to_tokens: B*T_out too large");
  const long n = (long)B * T_out;
  units_to_tokens_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(units, counts, B, T_units, offset, bos,
                                                                                          eos, pad, ids, T_out);
  SK_LAUNCH_CHECK();
  return 0;
}

int sk_units_to_prompt(const int32_t* units, const int32_t* counts, int B, int T_units, const int32_t* unit_id, int n_units,
                       const int32_t* prefix, int n_prefix, int marker, int pad, int64_t* ids, int64_t* mask, int T_out,
                       void* stream) {
  SK_REQUIRE(units && counts && unit_id && ids && mask && (prefix || n_prefix == 0), "sk_units_to_prompt: null argument");
  SK_REQUIRE(B > 0 && T_units >= 0 && n_units > 0 && n_prefix >= 0 && T_out >= n_prefix + 1,
             "sk_units_to_prompt: bad shape B=%d T_units=%d n_units=%d n_prefix=%d T_out=%d", B, T_units, n_units, n_prefix,
             T_out);
  SK_REQUIRE((long)B * T_out < (1L << 31), "sk_units_to_prompt: B*T_out too large");
  const long n = (long)B * T_out;
  units_to_prompt_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
      units, counts, B, T_units, unit_id, n_units, prefix, n_prefix, marker, pad, ids, mask, T_out);
  SK_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
