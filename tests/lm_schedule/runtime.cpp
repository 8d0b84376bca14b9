// The CUDA runtime calls of lm_step.cu on host memory, the project's host hooks it links against, and the fixed answers
// of the kernel size queries.  Compiled with the host compiler: nvcc's device runtime header already declares several
// of these functions.
#include "trace.h"

#include <stdarg.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <map>
#include <string>

namespace {
struct Buf {
  std::string name;
  size_t bytes;
};
std::map<uintptr_t, Buf> g_bufs;
int g_dev = 0;
char g_err[2048];
}  // namespace

void tr_register(const char* name, const void* base, size_t bytes) { g_bufs[(uintptr_t)base] = {name, bytes}; }
void tr_unregister(const void* base) { g_bufs.erase((uintptr_t)base); }

const char* tr_ptr(const void* p) {
  static char ring[64][96];
  static int next = 0;
  char* out = ring[next];
  next = (next + 1) % 64;
  if (!p) return "null";
  const uintptr_t a = (uintptr_t)p;
  auto it = g_bufs.upper_bound(a);
  if (it != g_bufs.begin()) {
    --it;
    if (a < it->first + it->second.bytes || (a == it->first && it->second.bytes == 0)) {
      snprintf(out, 96, "%s+%llu", it->second.name.c_str(), (unsigned long long)(a - it->first));
      return out;
    }
  }
  return "?";
}

void tr_log(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vprintf(fmt, ap);
  va_end(ap);
  putchar('\n');
}

// ---- the CUDA runtime calls lm_step.cu makes (enum values as in driver_types.h)
struct CUstream_st;
struct CUevent_st;
extern "C" {
int cudaMalloc(void** p, size_t bytes) {
  *p = aligned_alloc(256, (bytes + 255) / 256 * 256 + 256);
  char name[32];
  snprintf(name, sizeof(name), "dev%d", g_dev++);
  tr_register(name, *p, bytes);
  return 0;
}
int cudaFree(void* p) {
  if (p) {
    tr_unregister(p);
    free(p);
  }
  return 0;
}
int cudaMemcpy(void* dst, const void* src, size_t bytes, int /*kind*/) {
  memcpy(dst, src, bytes);
  return 0;
}
int cudaMemset(void* p, int v, size_t bytes) {
  tr_log("cudaMemset(%s, %d, %zu)", tr_ptr(p), v, bytes);
  memset(p, v, bytes);
  return 0;
}
int cudaMemsetAsync(void* p, int v, size_t bytes, CUstream_st* s) {
  tr_log("cudaMemsetAsync(%s, %d, %zu, %s)", tr_ptr(p), v, bytes, tr_ptr(s));
  memset(p, v, bytes);
  return 0;
}
int cudaEventRecord(CUevent_st* e, CUstream_st* s) {
  tr_log("cudaEventRecord(%s, %s)", tr_ptr(e), tr_ptr(s));
  return 0;
}
int cudaDeviceSynchronize(void) { return 0; }
const char* cudaGetErrorString(int) { return "stub error"; }

void** __cudaRegisterFatBinary(void*) {
  static void* handle = nullptr;
  return &handle;
}
void __cudaRegisterFatBinaryEnd(void**) {}
void __cudaUnregisterFatBinary(void**) {}

// ---- size queries: fixed values, so the workspace plans are functions of the shapes alone
int sk_ce_blocks(int M) { return M < 64 ? M : 64; }
int sk_colsum_splits(void) { return 8; }
int sk_rmsnorm_bwd_blocks(void) { return 16; }
int sk_layernorm_bwd_blocks(void) { return 16; }
int64_t sk_attn_decode_partial_bytes(int B, int H, int T_cache) { return (int64_t)B * H * ((T_cache + 63) / 64) * 66 * 4; }

const char* sk_last_error(void) { return g_err; }
}  // extern "C"

size_t sk_gemm_ws_min_bytes(void) { return (size_t)1 << 20; }

// ---- host hooks of api.cu
void sk_set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
void sk_prof_begin(int cat, CUstream_st* s) { tr_log("sk_prof_begin(%d, %s)", cat, tr_ptr(s)); }
void sk_prof_end(CUstream_st* s) { tr_log("sk_prof_end(%s)", tr_ptr(s)); }
