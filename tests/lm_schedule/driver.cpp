// Runs every decoder variant of lm_step.cu through its C ABI with tiny shapes and prints what it launches.  Linked
// against the launcher stubs and runtime.cpp, so nothing runs on a device: the output is the launch schedule itself.
#include "../../include/slamkit_b200.h"
#include "trace.h"

#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <vector>

namespace {

enum Kind { QWEN2, OPT, NEOX };
enum Mode { BF16, MASTER, FP32 };

struct Variant {
  const char* name;
  Kind kind;
  Mode mode;
  const char* head_chunk;   // SK_HEAD_CHUNK while the handle is created (nullptr: unset)
  SkLmConfig q;
  SkOptConfig o;
  SkNeoxConfig n;
};

constexpr int B = 2, T = 16, BIG_T = 160, T_CACHE = 32, PROMPT_T = 8, FANOUT = 2;
void* const STREAM = (void*)0x1000;   // registered below; never dereferenced

void* halloc(const char* name, size_t bytes) {
  void* p = aligned_alloc(256, (bytes + 255) / 256 * 256 + 256);
  tr_register(name, p, bytes);
  return p;
}

#define CALL(expr)                                        \
  do {                                                    \
    tr_log("-- %s", #expr);                               \
    const int rc_ = (int)(expr);                          \
    if (rc_)                                              \
      tr_log("-> %d: %s", rc_, sk_last_error());          \
    else                                                  \
      tr_log("-> 0");                                     \
  } while (0)

SkLmConfig qwen2(int vocab, int tie, int bias) { return SkLmConfig{vocab, 128, 2, 2, 1, 64, 256, 256, 1e-6f, tie, bias}; }
SkOptConfig opt(int tie, int post_ln, int proj_dim) { return SkOptConfig{502, 128, 2, 2, 256, 256, 1e-5f, tie, post_ln, proj_dim}; }
SkNeoxConfig neox() { return SkNeoxConfig{502, 128, 2, 2, 512, 256, 16, 1e-5f}; }

int create(const Variant& v, SkLm** lm) {
  if (v.head_chunk)
    setenv("SK_HEAD_CHUNK", v.head_chunk, 1);
  else
    unsetenv("SK_HEAD_CHUNK");
  int rc = v.kind == QWEN2 ? sk_lm_create(&v.q, lm) : v.kind == OPT ? sk_lm_create_opt(&v.o, lm) : sk_lm_create_neox(&v.n, lm);
  unsetenv("SK_HEAD_CHUNK");
  return rc;
}

void run(const Variant& v) {
  tr_log("==== %s", v.name);
  SkLm* lm = nullptr;
  CALL(create(v, &lm));
  if (!lm) return;
  const int n_tensors = sk_lm_tensor_info(lm, -1, nullptr, 0, nullptr, nullptr, nullptr);
  for (int i = 0; i < n_tensors; ++i) {
    char name[64];
    int64_t off;
    int32_t rows, cols;
    sk_lm_tensor_info(lm, i, name, sizeof(name), &off, &rows, &cols);
    tr_log("tensor %s off=%lld [%d, %d]", name, (long long)off, rows, cols);
  }
  const int64_t n = sk_lm_param_count(lm);
  const int L = v.kind == QWEN2 ? v.q.n_layers : v.kind == OPT ? v.o.n_layers : v.n.n_layers;
  tr_log("param_count %lld", (long long)n);
  const size_t ws_bytes = 64 << 20;
  void* params = halloc("params", n * 2);
  void* grads = halloc("grads", n * 2);
  void* rope_cos = v.kind == OPT ? nullptr : halloc("rope_cos", 256 * 32 * 2);
  void* rope_sin = v.kind == OPT ? nullptr : halloc("rope_sin", 256 * 32 * 2);
  void* ws = halloc("ws", ws_bytes);
  CALL(sk_lm_bind(lm, params, grads, rope_cos, rope_sin, ws, ws_bytes));
  void* params32 = nullptr;
  void* grads32 = nullptr;
  void* prepared = nullptr;
  if (v.mode == MASTER) {
    params32 = halloc("params32", n * 4);
    grads32 = halloc("grads32", n * 4);
    CALL(sk_lm_set_master(lm, (float*)params32, (float*)grads32));
    std::vector<int64_t> cs(4096);
    std::vector<int32_t> cl(4096);
    const int nw = sk_lm_widen_chunks(lm, cs.data(), cl.data(), 4096);
    tr_log("widen_chunks %d", nw);
    for (int i = 0; i < nw; ++i) tr_log("  widen %lld %d", (long long)cs[i], cl[i]);
  }
  if (v.mode == FP32) {
    const int64_t pb = sk_lm_fp32_prepared_bytes(lm);
    tr_log("fp32_prepared_bytes %lld", (long long)pb);
    params32 = halloc("params32", n * 4);
    prepared = halloc("prepared", pb);
    CALL(sk_lm_set_fp32(lm, (const float*)params32, prepared, pb, STREAM));
  }
  tr_log("workspace_bytes(%d, %d) %lld  (1, 1) %lld  (%d, %d) %lld", B, T, (long long)sk_lm_workspace_bytes(lm, B, T),
         (long long)sk_lm_workspace_bytes(lm, 1, 1), B, BIG_T, (long long)sk_lm_workspace_bytes(lm, B, BIG_T));

  const int M = B * BIG_T;
  int64_t* ids = (int64_t*)halloc("ids", M * 8);
  int64_t* labels = (int64_t*)halloc("labels", M * 8);
  int32_t* pos_ids = (int32_t*)halloc("pos_ids", M * 4);
  float* stats = (float*)halloc("stats", 64);
  float* row_nll = (float*)halloc("row_nll", M * 4);
  float* row_weight = (float*)halloc("row_weight", B * 4);
  void* exp_avg = halloc("exp_avg", n * 4);
  void* exp_avg_sq = halloc("exp_avg_sq", n * 4);
  std::vector<char> ev(L + 1);
  tr_register("events", ev.data(), ev.size());
  std::vector<void*> events;
  for (int i = 0; i <= L; ++i) events.push_back(ev.data() + i);

  tr_log("## forward");
  CALL(sk_lm_forward(lm, ids, labels, nullptr, B, T, 20.f, stats, STREAM));
  CALL(sk_lm_forward(lm, ids, nullptr, nullptr, B, T, 0.f, nullptr, STREAM));
  CALL(sk_lm_forward(lm, ids, labels, pos_ids, B, T, 20.f, stats, STREAM));
  CALL(sk_lm_forward(lm, ids, labels, nullptr, B, 300, 20.f, stats, STREAM));
  tr_log("logits %s logits_f32 %s ld %d", tr_ptr(sk_lm_logits(lm)), tr_ptr(sk_lm_logits_f32(lm)), sk_lm_logits_ld(lm));
  tr_log("## training");
  CALL(sk_lm_forward_backward(lm, ids, labels, nullptr, B, T, 20.f, 0.5f, 0, stats, STREAM));
  CALL(sk_lm_forward_backward(lm, ids, labels, nullptr, B, T, 20.f, 0.5f, 1, stats, STREAM));
  CALL(sk_lm_forward_backward(lm, ids, labels, pos_ids, B, T, 20.f, 1.f, 0, stats, STREAM));
  const bool chunked = v.head_chunk || (v.kind == QWEN2 && v.q.vocab_size > 8192);
  if (chunked) CALL(sk_lm_forward_backward(lm, ids, labels, pos_ids, B, BIG_T, 300.f, 1.f, 1, stats, STREAM));   // 3 chunks
  CALL(sk_lm_forward_backward(lm, ids, labels, nullptr, B, T, 0.f, 1.f, 0, stats, STREAM));
  CALL(sk_lm_set_backward_events(lm, events.data(), L));
  CALL(sk_lm_set_backward_events(lm, events.data(), L + 1));
  CALL(sk_lm_forward_backward(lm, ids, labels, nullptr, B, T, 20.f, 1.f, 0, stats, STREAM));
  CALL(sk_lm_set_backward_events(lm, nullptr, 0));
  tr_log("## DPO rows");
  CALL(sk_lm_forward_rows(lm, ids, labels, pos_ids, B, T, row_nll, stats, STREAM));
  CALL(sk_lm_backward_weighted(lm, ids, labels, pos_ids, B, T, row_weight, 0, stats, STREAM));
  CALL(sk_lm_forward_rows(lm, ids, labels, nullptr, B, T, row_nll, stats, STREAM));
  CALL(sk_lm_backward_weighted(lm, ids, labels, nullptr, B, T, row_weight, 1, stats, STREAM));
  CALL(sk_lm_backward_weighted(lm, ids, labels, nullptr, 1, T, row_weight, 1, stats, STREAM));
  tr_log("## optimiser");
  CALL(sk_lm_optimizer_step(lm, exp_avg, exp_avg_sq, 1e-3f, 0.9f, 0.999f, 1e-8f, 0.f, 3, 1.f, 0, stats, STREAM));
  CALL(sk_lm_optimizer_step(lm, exp_avg, exp_avg_sq, 1e-3f, 0.9f, 0.999f, 1e-8f, 0.1f, 3, 1.f, 1, stats, STREAM));
  tr_log("## generation");
  const int64_t kv_bytes = sk_lm_kv_cache_bytes(lm, B, T_CACHE);
  const int64_t dws_bytes = sk_lm_decode_workspace_bytes(lm, B * FANOUT, T_CACHE);
  tr_log("kv_cache_bytes %lld decode_workspace_bytes %lld (B=%d) %lld (B=%d)", (long long)kv_bytes,
         (long long)sk_lm_decode_workspace_bytes(lm, B, T_CACHE), B, (long long)dws_bytes, B * FANOUT);
  void* kv = halloc("kv", kv_bytes);
  void* kv2 = halloc("kv_fanout", kv_bytes * FANOUT);
  void* dws = halloc("dws", dws_bytes);
  const int ldl = 1024 * 16;
  void* logits = halloc("logits_out", (size_t)B * FANOUT * ldl * 4);
  int32_t* lens = (int32_t*)halloc("lens", B * FANOUT * 4);
  int64_t* tokens = (int64_t*)halloc("tokens", B * FANOUT * 8);
  lens[0] = 5;
  lens[1] = PROMPT_T;
  CALL(sk_lm_prefill(lm, ids, lens, B, PROMPT_T, kv, T_CACHE, logits, ldl, dws, dws_bytes, STREAM));
  CALL(sk_lm_kv_fanout(lm, kv, B, FANOUT, kv2, T_CACHE, lens, STREAM));
  CALL(sk_lm_decode_step(lm, tokens, lens, B, kv, T_CACHE, logits, ldl, dws, dws_bytes, STREAM));
  CALL(sk_lm_decode_step(lm, tokens, lens, B, kv, T_CACHE, logits, ldl - 4, dws, dws_bytes, STREAM));
  CALL(sk_lm_prefill(lm, ids, lens, B, T_CACHE + 1, kv, T_CACHE, logits, ldl, dws, dws_bytes, STREAM));
  tr_log("## switching modes");   // refused except on a bf16 pre-LN OPT handle
  if (v.mode != FP32) CALL(sk_lm_set_fp32(lm, (const float*)ws, ws, 64 << 20, STREAM));
  if (v.mode != MASTER) CALL(sk_lm_set_master(lm, (float*)ws, (float*)ws));
  sk_lm_destroy(lm);
  for (void* p : {params, grads, rope_cos, rope_sin, ws, params32, grads32, prepared, (void*)ids, (void*)labels,
                  (void*)pos_ids, (void*)stats, (void*)row_nll, (void*)row_weight, exp_avg, exp_avg_sq, kv, kv2, dws,
                  logits, (void*)lens, (void*)tokens, (void*)ev.data()})
    if (p) tr_unregister(p);
}

}  // namespace

int main() {
  tr_register("stream", STREAM, 0);
  const SkLmConfig q0{};
  const SkOptConfig o0{};
  const SkNeoxConfig n0{};
  const Variant variants[] = {
      {"qwen2", QWEN2, BF16, nullptr, qwen2(502, 1, 1), o0, n0},
      {"qwen2 untied, no qkv bias", QWEN2, BF16, nullptr, qwen2(502, 0, 0), o0, n0},
      {"qwen2 chunked head (SK_HEAD_CHUNK)", QWEN2, BF16, "128", qwen2(502, 1, 1), o0, n0},
      {"qwen2 large vocabulary", QWEN2, BF16, nullptr, qwen2(9000, 1, 1), o0, n0},
      {"opt", OPT, BF16, nullptr, q0, opt(1, 0, 0), n0},
      {"opt untied", OPT, BF16, nullptr, q0, opt(0, 0, 0), n0},
      {"opt chunked head", OPT, BF16, "128", q0, opt(1, 0, 0), n0},
      {"opt master", OPT, MASTER, nullptr, q0, opt(1, 0, 0), n0},
      {"opt master untied", OPT, MASTER, nullptr, q0, opt(0, 0, 0), n0},
      {"opt master chunked head", OPT, MASTER, "128", q0, opt(1, 0, 0), n0},
      {"opt fp32", OPT, FP32, nullptr, q0, opt(1, 0, 0), n0},
      {"opt post-ln", OPT, BF16, nullptr, q0, opt(1, 1, 0), n0},
      {"opt post-ln chunked head", OPT, BF16, "128", q0, opt(1, 1, 0), n0},
      {"opt post-ln proj", OPT, BF16, nullptr, q0, opt(1, 1, 64), n0},
      {"opt post-ln proj chunked head", OPT, BF16, "128", q0, opt(1, 1, 64), n0},
      {"opt post-ln fp32", OPT, FP32, nullptr, q0, opt(1, 1, 0), n0},
      {"opt post-ln proj fp32", OPT, FP32, nullptr, q0, opt(1, 1, 64), n0},
      {"neox", NEOX, BF16, nullptr, q0, o0, neox()},
      {"neox chunked head", NEOX, BF16, "128", q0, o0, neox()},
  };
  for (const Variant& v : variants) run(v);

  tr_log("==== constructor refusals");
  SkLm* lm = nullptr;
  SkLmConfig q = qwen2(502, 1, 1);
  q.hidden = 256;   // n_heads * head_dim != hidden
  CALL(sk_lm_create(&q, &lm));
  q = qwen2(502, 1, 1);
  q.head_dim = 128;
  CALL(sk_lm_create(&q, &lm));
  q = qwen2(502, 1, 1);
  q.ffn = 200;
  CALL(sk_lm_create(&q, &lm));
  q = qwen2(0, 1, 1);
  CALL(sk_lm_create(&q, &lm));
  CALL(sk_lm_create(nullptr, &lm));
  SkOptConfig o = opt(1, 0, 64);
  CALL(sk_lm_create_opt(&o, &lm));
  o = opt(1, 1, 96);
  CALL(sk_lm_create_opt(&o, &lm));
  o = opt(1, 2, 0);
  CALL(sk_lm_create_opt(&o, &lm));
  o = opt(1, 0, 0);
  o.hidden = 4096;
  o.n_heads = 64;
  CALL(sk_lm_create_opt(&o, &lm));
  SkNeoxConfig nx = neox();
  nx.rot_dims = 8;
  CALL(sk_lm_create_neox(&nx, &lm));
  nx = neox();
  nx.ffn = 100;
  CALL(sk_lm_create_neox(&nx, &lm));
  tr_log("handle after refusals: %s", lm ? "set" : "null");
  return 0;
}
