// HuBERT-25Hz unit extraction (hot path (i)) orchestration: waveform -> conv feature encoder -> projection ->
// positional conv -> `n_layers` post-LN transformer layers -> k-means labels (-> run-length dedup).
// Replaces HubertFeatureExtractor.extract + batch_cluster (slamkit/feature_extractor/hubert_feature_extractor.py:40-50,
// 73-81), i.e. HF HubertModel.forward (HF:models/hubert/modeling_hubert.py:45-231,262-470) and sklearn KMeans.predict
// (SK:cluster/_k_means_lloyd.pyx:168-213), with everything device-resident: the only D2H traffic is the int32 labels.
//
// All matrix products (7 strided convolutions as windowed GEMMs, projections, grouped positional conv, attention,
// FFN, k-means distances) run on the wgmma GEMM / wgmma attention kernels in split-bf16 (hi, lo) form, 3 passes,
// fp32 accumulation: the reference computes in fp32 and the unit ids have to agree with it.
#include "kernels.h"
#include "../../include/slamkit_b200.h"
#include <string>
#include <vector>
#include <string.h>
#include <math.h>
#include <stdlib.h>

namespace {
constexpr int64_t ALIGN_ELEMS = 64;
constexpr int GROUP_PAD = 64;   // positional-conv channel groups are padded to 64 channels (one 128-byte TMA row)

struct TensorDesc {
  std::string name;
  int64_t off;
  int rows, cols;
};
struct LayerOff {
  int64_t wqkv, bqkv, wo, bo, ln1g, ln1b, w1, b1, w2, b2, ln2g, ln2b;
};
struct WsLayout {
  int64_t stats, affine, act0, act1, lnc, x, xp, pc, h0, h1, qkv, ao, t1, ff, dot, n_frames, total;
};
int64_t align_up(int64_t v, int64_t a) { return (v + a - 1) / a * a; }
}  // namespace

struct SkHubert {
  SkHubertConfig cfg;
  int C, H, F, G, cg, Kpos, halo, U, Upad, nconv;
  std::vector<TensorDesc> tensors;
  int64_t n_params = 0;
  int64_t conv0_w, gn_g, gn_b, conv_w[8], fp_lng, fp_lnb, fp_w, fp_b, pos_w, pos_b, enc_lng, enc_lnb, km_c;
  std::vector<LayerOff> lo;
  const float* w32 = nullptr;   // flat fp32 weights (prepared layout)
  bf16* w_hi = nullptr;         // split copies
  bf16* w_lo = nullptr;
  float* csq = nullptr;
  uint8_t* ws = nullptr;
  int64_t ws_bytes = 0;
};

namespace {

int64_t add_tensor(SkHubert* h, const std::string& name, int rows, int cols) {
  const int64_t off = h->n_params;
  h->tensors.push_back({name, off, rows, cols});
  h->n_params = align_up(off + (int64_t)rows * cols, ALIGN_ELEMS);
  return off;
}

void frame_counts(const SkHubert* h, int S, int* T) {
  long L = (long)S + 2 * h->cfg.pad;
  for (int i = 0; i < h->nconv; ++i) {
    L = (L - h->cfg.conv_kernel[i]) / h->cfg.conv_stride[i] + 1;
    T[i] = (int)(L > 0 ? L : 0);
  }
}

WsLayout make_layout(const SkHubert* h, int B, int S) {
  int T[8];
  frame_counts(h, S, T);
  const int64_t Tf = T[h->nconv - 1];
  const int64_t M = (int64_t)B * Tf;
  WsLayout w;
  int64_t cur = 0;
  auto take = [&](int64_t bytes) {
    const int64_t o = cur;
    cur = align_up(cur + bytes, 256);
    return o;
  };
  auto hilo = [&](int64_t elems) { return take(2 * align_up(elems * 2, 256)); };  // hi then lo
  w.stats = take((int64_t)B * sk_conv0_nstat() * 8);
  w.affine = take((int64_t)B * h->C * 8);
  w.act0 = hilo((int64_t)B * T[0] * h->C);
  w.act1 = hilo((int64_t)B * (h->nconv > 1 ? T[1] : 1) * h->C);
  w.lnc = hilo(M * h->C);
  w.x = hilo(M * h->H);
  w.xp = hilo((int64_t)B * (Tf + 2 * h->halo) * h->G * GROUP_PAD);
  w.pc = hilo(M * h->H);
  w.h0 = hilo(M * h->H);
  w.h1 = hilo(M * h->H);
  w.qkv = hilo(M * 3 * h->H);
  w.ao = hilo(M * h->H);
  w.t1 = hilo(M * h->H);
  w.ff = hilo(M * h->F);
  w.dot = take(M * h->Upad * 4);
  w.n_frames = take((int64_t)B * 4);
  w.total = cur;
  return w;
}

struct HiLo {
  bf16* hi;
  bf16* lo;
};
HiLo hl(const SkHubert* h, int64_t off, int64_t elems) {
  HiLo r;
  r.hi = reinterpret_cast<bf16*>(h->ws + off);
  r.lo = reinterpret_cast<bf16*>(h->ws + off + align_up(elems * 2, 256));
  return r;
}

#define SK_TRY(expr)     \
  do {                   \
    int _rc = (expr);    \
    if (_rc) return _rc; \
  } while (0)

// y(hi,lo)[M,N] = act(x(hi,lo)[M,K] * W(hi,lo)[N,K]^T + bias) (+ residual(hi,lo)), split-bf16 3-pass
int linear_split(const SkHubert* h, int M, int N, int K, HiLo x, int64_t w_off, int64_t b_off, int act, const HiLo* res,
                 HiLo y, float* y_f32, int ldy, cudaStream_t s) {
  return sk_gemm_ex_launch(sk_gemm_linear_split(M, N, K, x.hi, x.lo, h->w_hi + w_off, h->w_lo + w_off,
                                                b_off >= 0 ? h->w32 + b_off : nullptr, act, res ? res->hi : nullptr,
                                                res ? res->lo : nullptr, y.hi, y.lo, y_f32, ldy),
                           s);
}

// dbg_stage (tests only): 100+i = output of conv layer i, 200 = projection, 201 = positional conv (post-GELU),
// 0..n_layers = hidden_states[stage], 300 + 10 l + j = intermediate j of encoder layer l (see the layer loop); the fp32
// stage tensor is written to feat_out and the pass stops there.
int forward_impl(SkHubert* h, const float* wav, const int64_t* lens, int B, int S, int32_t* ids, int32_t* n_frames,
                 float* feat_out, cudaStream_t s, int dbg_stage = -1) {
  SK_REQUIRE(h->w_hi && h->ws, "sk_hubert: sk_hubert_bind has not been called");
  SK_REQUIRE(B > 0 && S > 0, "sk_hubert: empty batch");
  const WsLayout w = make_layout(h, B, S);
  SK_REQUIRE(w.total <= h->ws_bytes, "sk_hubert: workspace too small: need %lld bytes, bound %lld", (long long)w.total,
             (long long)h->ws_bytes);
  int T[8];
  frame_counts(h, S, T);
  const int Tf = T[h->nconv - 1];
  SK_REQUIRE(Tf > 0, "sk_hubert: clip too short for the conv stack (S=%d)", S);
  const int M = B * Tf;
  const int C = h->C, H = h->H, F = h->F;
  const float eps = h->cfg.ln_eps;

  // conv0 + GroupNorm + GELU
  HiLo act[2] = {hl(h, w.act0, (int64_t)B * T[0] * C), hl(h, w.act1, (int64_t)B * (h->nconv > 1 ? T[1] : 1) * C)};
  SK_TRY(sk_conv0_launch(wav, h->w32 + h->conv0_w, h->w32 + h->gn_g, h->w32 + h->gn_b,
                         reinterpret_cast<double*>(h->ws + w.stats), reinterpret_cast<float2*>(h->ws + w.affine),
                         act[0].hi, act[0].lo, B, S, h->cfg.pad, T[0], C, h->cfg.conv_kernel[0], h->cfg.conv_stride[0],
                         1e-5f, s));
  if (dbg_stage == 100) return sk_hilo_to_f32_launch(act[0].hi, act[0].lo, feat_out, (long)B * T[0] * C, s);
  // conv 1..n-1 as strided-window GEMMs (+GELU)
  int cur = 0;
  for (int i = 1; i < h->nconv; ++i) {
    const int k = h->cfg.conv_kernel[i], st = h->cfg.conv_stride[i];
    SkGemmEx g = sk_gemm_base(T[i], C, k * C);
    g.batch = B; g.passes = 3;
    g.A = act[cur].hi; g.A_lo = act[cur].lo;
    g.a_inner = (long)k * C; g.a_rows = T[i]; g.a_row_stride = (long)st * C; g.a_batch_stride = (long)T[i - 1] * C;
    g.B = h->w_hi + h->conv_w[i]; g.B_lo = h->w_lo + h->conv_w[i]; g.ldb = k * C;
    // outputs of layer i alias buffer (cur^1); sizes shrink by ~2x per layer so ping-pong between act0/act1 fits
    HiLo out = act[cur ^ 1];
    if (i >= 2) out = hl(h, (cur ^ 1) == 0 ? w.act0 : w.act1, (int64_t)B * T[i] * C);
    g.C = out.hi; g.C_lo = out.lo; g.ldc = C;
    g.act = SK_ACT_GELU;
    SK_TRY(sk_gemm_ex_launch(g, s));
    act[cur ^ 1] = out;
    cur ^= 1;
    if (dbg_stage == 100 + i) return sk_hilo_to_f32_launch(out.hi, out.lo, feat_out, (long)B * T[i] * C, s);
  }
  // feature projection: LN(C) -> Linear(C->H)
  HiLo lnc = hl(h, w.lnc, (int64_t)M * C), x = hl(h, w.x, (int64_t)M * H);
  SK_TRY(sk_layernorm_hilo_launch(act[cur].hi, act[cur].lo, nullptr, nullptr, h->w32 + h->fp_lng, h->w32 + h->fp_lnb,
                                  lnc.hi, lnc.lo, nullptr, M, C, eps, s));
  SK_TRY(linear_split(h, M, H, C, lnc, h->fp_w, h->fp_b, SK_ACT_NONE, nullptr, x, nullptr, H, s));
  if (dbg_stage == 200) return sk_hilo_to_f32_launch(x.hi, x.lo, feat_out, (long)M * H, s);
  // positional conv (grouped, weight-norm folded on the host) + GELU, then x + pos -> LayerNorm
  const int Tp = Tf + 2 * h->halo, GP = h->G * GROUP_PAD;
  HiLo xp = hl(h, w.xp, (int64_t)B * Tp * GP), pc = hl(h, w.pc, (int64_t)M * H);
  SK_TRY(sk_regroup_pad_launch(x.hi, x.lo, xp.hi, xp.lo, B, Tf, h->halo, h->G, h->cg, GROUP_PAD, s));
  {
    SkGemmEx g = sk_gemm_base(Tf, GP, h->Kpos * GROUP_PAD);
    g.batch = B; g.passes = 3; g.a_mode = 1;
    g.A = xp.hi; g.A_lo = xp.lo;
    g.a_inner = GP; g.a_rows = Tp; g.a_row_stride = GP; g.a_batch_stride = (long)Tp * GP;
    g.B = h->w_hi + h->pos_w; g.B_lo = h->w_lo + h->pos_w; g.ldb = h->Kpos * GROUP_PAD;
    g.C = pc.hi; g.C_lo = pc.lo; g.ldc = H;
    g.bias = h->w32 + h->pos_b; g.bias_f32 = 1;
    g.act = SK_ACT_GELU;
    g.col_gin = GROUP_PAD; g.col_gout = h->cg;
    SK_TRY(sk_gemm_ex_launch(g, s));
  }
  if (dbg_stage == 201) return sk_hilo_to_f32_launch(pc.hi, pc.lo, feat_out, (long)M * H, s);
  HiLo hb[2] = {hl(h, w.h0, (int64_t)M * H), hl(h, w.h1, (int64_t)M * H)};
  SK_TRY(sk_layernorm_hilo_launch(x.hi, x.lo, pc.hi, pc.lo, h->w32 + h->enc_lng, h->w32 + h->enc_lnb, hb[0].hi, hb[0].lo,
                                  (h->cfg.n_layers == 0 || dbg_stage == 0) ? feat_out : nullptr, M, H, eps, s));
  if (dbg_stage == 0) return 0;
  // transformer layers (post-LN)
  HiLo qkv = hl(h, w.qkv, (int64_t)M * 3 * H), ao = hl(h, w.ao, (int64_t)M * H), t1 = hl(h, w.t1, (int64_t)M * H),
       ff = hl(h, w.ff, (int64_t)M * F);
  const float scale = 1.0f / sqrtf((float)(H / h->cfg.n_heads));
  // dbg_stage 300 + 10 l + j: intermediate j of layer l (0 qkv, 1 attention, 2 o-proj + residual, 3 LN1, 4 ff1 GELU,
  // 5 ff2 + residual)
  auto tap = [&](int l, int j, HiLo t, int cols) {
    return dbg_stage == 300 + 10 * l + j ? sk_hilo_to_f32_launch(t.hi, t.lo, feat_out, (long)M * cols, s) : -1;
  };
#define SK_TAP(l, j, t, cols)                  \
  do {                                         \
    const int _rc = tap(l, j, t, cols);        \
    if (_rc >= 0) return _rc;                  \
  } while (0)
  for (int l = 0; l < h->cfg.n_layers; ++l) {
    const LayerOff& o = h->lo[l];
    const bool last = (l == h->cfg.n_layers - 1) || (dbg_stage == l + 1);
    SK_TRY(linear_split(h, M, 3 * H, H, hb[0], o.wqkv, o.bqkv, SK_ACT_NONE, nullptr, qkv, nullptr, 3 * H, s));
    SK_TAP(l, 0, qkv, 3 * H);
    SK_TRY(sk_attn_tc_fwd_split_launch(qkv.hi, qkv.lo, ao.hi, ao.lo, B, Tf, h->cfg.n_heads, 3 * H, H, scale, s));
    SK_TAP(l, 1, ao, H);
    SK_TRY(linear_split(h, M, H, H, ao, o.wo, o.bo, SK_ACT_NONE, &hb[0], t1, nullptr, H, s));
    SK_TAP(l, 2, t1, H);
    SK_TRY(sk_layernorm_hilo_launch(t1.hi, t1.lo, nullptr, nullptr, h->w32 + o.ln1g, h->w32 + o.ln1b, hb[1].hi, hb[1].lo,
                                    nullptr, M, H, eps, s));
    SK_TAP(l, 3, hb[1], H);
    SK_TRY(linear_split(h, M, F, H, hb[1], o.w1, o.b1, SK_ACT_GELU, nullptr, ff, nullptr, F, s));
    SK_TAP(l, 4, ff, F);
    SK_TRY(linear_split(h, M, H, F, ff, o.w2, o.b2, SK_ACT_NONE, &hb[1], t1, nullptr, H, s));
    SK_TAP(l, 5, t1, H);
    SK_TRY(sk_layernorm_hilo_launch(t1.hi, t1.lo, nullptr, nullptr, h->w32 + o.ln2g, h->w32 + o.ln2b, hb[0].hi, hb[0].lo,
                                    last ? feat_out : nullptr, M, H, eps, s));
    if (dbg_stage == l + 1) return 0;
  }
#undef SK_TAP
  if (ids) {
    float* dot = reinterpret_cast<float*>(h->ws + w.dot);
    SK_TRY(linear_split(h, M, h->Upad, H, hb[0], h->km_c, -1, SK_ACT_NONE, nullptr, HiLo{nullptr, nullptr}, dot, h->Upad, s));
    SK_TRY(sk_kmeans_argmin_launch(dot, h->csq, ids, M, h->U, h->Upad, s));
  }
  if (n_frames) SK_TRY(sk_rel_len_launch(lens, n_frames, B, S, Tf, s));
  return 0;
}

}  // namespace

extern "C" {

int sk_hubert_create(const SkHubertConfig* cfg, SkHubert** out) {
  SK_REQUIRE(cfg && out, "sk_hubert_create: null argument");
  SK_REQUIRE(cfg->n_conv >= 1 && cfg->n_conv <= 8, "sk_hubert_create: n_conv must be in [1,8]");
  SK_REQUIRE(cfg->conv_dim % 64 == 0 && cfg->conv_dim <= 1024, "sk_hubert_create: conv_dim must be a multiple of 64, <= 1024");
  SK_REQUIRE(cfg->hidden % 64 == 0 && cfg->hidden <= 1024 && cfg->hidden / cfg->n_heads == 64,
             "sk_hubert_create: hidden must be a multiple of 64 (<= 1024) with head_dim 64");
  SK_REQUIRE(cfg->ffn % 8 == 0, "sk_hubert_create: ffn must be a multiple of 8");
  SK_REQUIRE(cfg->hidden % cfg->pos_conv_groups == 0, "sk_hubert_create: hidden must divide into pos_conv_groups");
  const int cg = cfg->hidden / cfg->pos_conv_groups;
  SK_REQUIRE(cg % 8 == 0 && cg <= GROUP_PAD, "sk_hubert_create: channels per positional-conv group must be a multiple of 8, <= 64");
  SK_REQUIRE(cfg->pos_conv_kernel % 2 == 0, "sk_hubert_create: only even positional-conv kernels (HF drops the last frame)");
  SkHubert* h = new SkHubert();
  h->cfg = *cfg;
  h->C = cfg->conv_dim; h->H = cfg->hidden; h->F = cfg->ffn;
  h->G = cfg->pos_conv_groups; h->cg = cg; h->Kpos = cfg->pos_conv_kernel; h->halo = cfg->pos_conv_kernel / 2;
  h->U = cfg->n_units; h->Upad = (cfg->n_units + 63) / 64 * 64;
  h->nconv = cfg->n_conv;
  h->conv0_w = add_tensor(h, "conv0.w", h->C, cfg->conv_kernel[0]);
  h->gn_g = add_tensor(h, "gn.g", 1, h->C);
  h->gn_b = add_tensor(h, "gn.b", 1, h->C);
  for (int i = 1; i < h->nconv; ++i)
    h->conv_w[i] = add_tensor(h, "conv" + std::to_string(i) + ".w", h->C, cfg->conv_kernel[i] * h->C);
  h->fp_lng = add_tensor(h, "fp.ln.g", 1, h->C);
  h->fp_lnb = add_tensor(h, "fp.ln.b", 1, h->C);
  h->fp_w = add_tensor(h, "fp.w", h->H, h->C);
  h->fp_b = add_tensor(h, "fp.b", 1, h->H);
  h->pos_w = add_tensor(h, "pos.w", h->G * GROUP_PAD, h->Kpos * GROUP_PAD);
  h->pos_b = add_tensor(h, "pos.b", 1, h->G * GROUP_PAD);
  h->enc_lng = add_tensor(h, "enc.ln.g", 1, h->H);
  h->enc_lnb = add_tensor(h, "enc.ln.b", 1, h->H);
  h->lo.resize(cfg->n_layers);
  for (int l = 0; l < cfg->n_layers; ++l) {
    const std::string p = "layers." + std::to_string(l) + ".";
    LayerOff& o = h->lo[l];
    o.wqkv = add_tensor(h, p + "wqkv", 3 * h->H, h->H);
    o.bqkv = add_tensor(h, p + "bqkv", 1, 3 * h->H);
    o.wo = add_tensor(h, p + "wo", h->H, h->H);
    o.bo = add_tensor(h, p + "bo", 1, h->H);
    o.ln1g = add_tensor(h, p + "ln1.g", 1, h->H);
    o.ln1b = add_tensor(h, p + "ln1.b", 1, h->H);
    o.w1 = add_tensor(h, p + "ff1.w", h->F, h->H);
    o.b1 = add_tensor(h, p + "ff1.b", 1, h->F);
    o.w2 = add_tensor(h, p + "ff2.w", h->H, h->F);
    o.b2 = add_tensor(h, p + "ff2.b", 1, h->H);
    o.ln2g = add_tensor(h, p + "ln2.g", 1, h->H);
    o.ln2b = add_tensor(h, p + "ln2.b", 1, h->H);
  }
  h->km_c = add_tensor(h, "km.centers", h->Upad, h->H);
  *out = h;
  return 0;
}

void sk_hubert_destroy(SkHubert* h) { delete h; }
int64_t sk_hubert_param_count(const SkHubert* h) { return h ? h->n_params : 0; }
int sk_hubert_tensor_info(const SkHubert* h, int idx, char* name_buf, int name_cap, int64_t* offset, int32_t* rows,
                          int32_t* cols) {
  SK_REQUIRE(h, "sk_hubert_tensor_info: null handle");
  if (idx < 0) return (int)h->tensors.size();
  SK_REQUIRE(idx < (int)h->tensors.size(), "sk_hubert_tensor_info: index %d out of range", idx);
  const TensorDesc& t = h->tensors[idx];
  if (name_buf && name_cap > 0) {
    strncpy(name_buf, t.name.c_str(), name_cap - 1);
    name_buf[name_cap - 1] = 0;
  }
  if (offset) *offset = t.off;
  if (rows) *rows = t.rows;
  if (cols) *cols = t.cols;
  return 0;
}
int sk_hubert_frames(const SkHubert* h, int S) {
  if (!h || S <= 0) return 0;
  int T[8];
  frame_counts(h, S, T);
  return T[h->nconv - 1];
}
int64_t sk_hubert_prepared_bytes(const SkHubert* h) {
  return h ? align_up(h->n_params * 2, 256) * 2 + align_up((int64_t)h->Upad * 4, 256) : 0;
}
int64_t sk_hubert_workspace_bytes(const SkHubert* h, int B, int S) {
  if (!h || B <= 0 || S <= 0) return 0;
  return make_layout(h, B, S).total;
}
int sk_hubert_bind(SkHubert* h, const float* weights, void* prepared, int64_t prepared_bytes, void* workspace,
                   int64_t workspace_bytes, void* stream) {
  SK_REQUIRE(h && weights && prepared && workspace, "sk_hubert_bind: null argument");
  SK_REQUIRE(prepared_bytes >= sk_hubert_prepared_bytes(h), "sk_hubert_bind: prepared buffer too small");
  SK_REQUIRE(((uintptr_t)weights & 127) == 0 && ((uintptr_t)prepared & 255) == 0 && ((uintptr_t)workspace & 255) == 0,
             "sk_hubert_bind: buffers must be 128/256-byte aligned");
  cudaStream_t s = (cudaStream_t)stream;
  h->w32 = weights;
  uint8_t* p = reinterpret_cast<uint8_t*>(prepared);
  h->w_hi = reinterpret_cast<bf16*>(p);
  h->w_lo = reinterpret_cast<bf16*>(p + align_up(h->n_params * 2, 256));
  h->csq = reinterpret_cast<float*>(p + 2 * align_up(h->n_params * 2, 256));
  h->ws = reinterpret_cast<uint8_t*>(workspace);
  h->ws_bytes = workspace_bytes;
  SK_TRY(sk_split_f32_launch(weights, h->w_hi, h->w_lo, h->n_params, s));
  SK_TRY(sk_row_sqnorm_launch(weights + h->km_c, h->csq, h->Upad, h->H, s));
  return 0;
}
int sk_hubert_units(SkHubert* h, const float* wav, const int64_t* lens, int B, int S, int32_t* ids, int32_t* n_frames,
                    void* stream) {
  SK_REQUIRE(h && wav && ids && n_frames, "sk_hubert_units: null argument");
  return forward_impl(h, wav, lens, B, S, ids, n_frames, nullptr, (cudaStream_t)stream);
}
int sk_hubert_features(SkHubert* h, const float* wav, int B, int S, float* feat, void* stream) {
  SK_REQUIRE(h && wav && feat, "sk_hubert_features: null argument");
  return forward_impl(h, wav, nullptr, B, S, nullptr, nullptr, feat, (cudaStream_t)stream);
}
int sk_hubert_debug_stage(SkHubert* h, const float* wav, int B, int S, int stage, float* out, void* stream) {
  SK_REQUIRE(h && wav && out, "sk_hubert_debug_stage: null argument");
  return forward_impl(h, wav, nullptr, B, S, nullptr, nullptr, out, (cudaStream_t)stream, stage);
}
int sk_rle(const int32_t* ids, const int32_t* n_frames, int32_t* units, int32_t* durations, int32_t* counts, int B, int T,
           void* stream) {
  SK_REQUIRE(ids && units && durations && counts, "sk_rle: null argument");
  return sk_rle_launch(ids, n_frames, units, durations, counts, B, T, (cudaStream_t)stream);
}
int sk_row_sqnorm(const float* x, float* out, int rows, int D, void* stream) {
  SK_REQUIRE(x && out, "sk_row_sqnorm: null argument");
  return sk_row_sqnorm_launch(x, out, rows, D, (cudaStream_t)stream);
}
int sk_kmeans_argmin(const float* dot, const float* centers_sqnorm, int32_t* labels, int M, int U, int ld, void* stream) {
  SK_REQUIRE(dot && centers_sqnorm && labels, "sk_kmeans_argmin: null argument");
  return sk_kmeans_argmin_launch(dot, centers_sqnorm, labels, M, U, ld, (cudaStream_t)stream);
}

}  // extern "C"
