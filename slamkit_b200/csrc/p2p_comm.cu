// Data-parallel gradient all-reduce over NVLink peer memory (SURVEY.md §8 e-ii / e-iii): replaces the NCCL all-reduce
// that accelerate's DDP wrapper issues per bucket (HF:trainer.py:1867-2014, config/training_args/default.yaml:18) on a
// single NVSwitch node.
//
// Why not NCCL here: with the element-wise work fused into GEMM epilogues the backward pass is wall-to-wall persistent
// CTAs that each own most of an SM's shared memory; NCCL's channel CTAs (hundreds of threads, tens of KB of shared
// memory) only get an SM when one of those exits.  The kernels below are built small instead -- 4 warps of <= 32 registers
// per thread and no shared memory -- so that they can find room next to those CTAs.  How much of the reduction actually
// overlaps the backward pass on an H100 depends on the resident kernels' register use and is not measured here.
//
// Algorithm (one launch per bucket, every rank runs the same code on its own copy of the flat bf16 gradient buffer; all
// buffers and flag arrays are mapped into every process with CUDA IPC):
//   signal   rank r stores `epoch` into READY[slot][r] of every peer once its own gradients of the bucket are final
//   reduce   rank r owns the r-th 1/W of the bucket: for each 16-byte chunk it loads the W copies (peer loads over
//            NVLink), adds them in fp32 in RANK ORDER (the same order on every rank: results are bit-identical
//            everywhere and run-to-run), rounds once to bf16 and stores the result into all W buffers
//            (reduce-scatter and all-gather in one pass, 2 (W-1)/W x bucket bytes over each GPU's links);
//            the last CTA to finish stores `epoch` into DONE[slot][r] of every peer
//   wait     rank r spins until DONE[slot][p] == epoch for all p (and a range of slots): every peer has read r's copy
//            and written its share
// Flags only ever grow (epoch = number of reductions so far), so nothing is reset between steps.  Spins give up after
// SK_P2P_TIMEOUT_NS and raise a flag in pinned host memory that the host checks after the step.
#include <cuda_runtime.h>
#include <cuda.h>
#include <cstdint>
#include <cstring>
#include <cstdlib>

#include "common.cuh"
#include "kernels.h"

namespace {

constexpr int P2P_MAX_WORLD = 8;
constexpr int P2P_SLOTS = 256;                       // buckets per reduction (flag rows)
constexpr int P2P_THREADS = 128;                     // 4 warps: one per SM sub-partition
constexpr uint64_t SK_P2P_TIMEOUT_NS = 60ull * 1000 * 1000 * 1000;   // a dead peer, not a slow one: ranks may be seconds apart at start-up

// flag array of one rank (uint32): READY[P2P_SLOTS][8] | DONE[P2P_SLOTS][8] | CTA counters[P2P_SLOTS]
constexpr size_t P2P_FLAG_WORDS = 2 * P2P_SLOTS * P2P_MAX_WORLD + P2P_SLOTS;

struct P2PPeers {
  bf16* buf[P2P_MAX_WORLD];
  uint32_t* flag[P2P_MAX_WORLD];
};

SK_DEVINL uint32_t ld_acquire_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
SK_DEVINL void st_release_sys(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
// the data loads follow an acquire of the producer's flag; volatile keeps them out of L1 and in program order
SK_DEVINL uint4 ld_peer128(const void* p) {
  uint4 v;
  asm volatile("ld.volatile.global.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p) : "memory");
  return v;
}
SK_DEVINL f32x2 bf2_to_f32x2(uint32_t v) {      // two packed bf16 -> two packed fp32 (bf16 is the high half of fp32)
  return pk2(__uint_as_float(v << 16), __uint_as_float(v & 0xffff0000u));
}
SK_DEVINL uint32_t f32x2_to_bf2(f32x2 v) {
  float x, y;
  upk2(v, x, y);
  return pack_bf16(x, y);
}
SK_DEVINL void st_peer128(void* p, uint4 v) {
  asm volatile("st.global.v4.u32 [%0], {%1, %2, %3, %4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}

// optional timeline (sk_p2p_set_trace): [slot][4] globaltimer stamps -- 0 READY signalled, 1 first CTA of the reduce
// kernel running, 2 peers ready, 3 last CTA done; row P2P_SLOTS: 0 wait kernel running, 1 all shares arrived
__device__ unsigned long long* g_p2p_trace = nullptr;

// true when the flag reached `epoch` (wrap-safe), false after the time-out
SK_DEVINL bool spin_until(const uint32_t* f, uint32_t epoch, int* err, int code) {
  const uint64_t t0 = globaltimer_ns();
  while ((int32_t)(ld_acquire_sys(f) - epoch) < 0) {
    __nanosleep(200);
    if (globaltimer_ns() - t0 > SK_P2P_TIMEOUT_NS) {
      if (err) *reinterpret_cast<volatile int*>(err) = code;
      return false;
    }
  }
  return true;
}

__global__ void __launch_bounds__(32) p2p_signal_kernel(P2PPeers pr, int rank, int world, int slot, uint32_t epoch) {
  const int p = threadIdx.x;
  uint32_t* f = nullptr;
#pragma unroll
  for (int q = 0; q < P2P_MAX_WORLD; ++q)
    if (q == p) f = pr.flag[q];                    // compile-time indices: the pointer table stays in the constant bank
  if (p < world && p != rank) {
    __threadfence_system();
    st_release_sys(f + slot * P2P_MAX_WORLD + rank, epoch);
  }
  if (p == 0 && g_p2p_trace) g_p2p_trace[slot * 4 + 0] = globaltimer_ns();
}

__global__ void __launch_bounds__(256) p2p_wait_kernel(const uint32_t* own_flags, int rank, int world, int slot_lo, int n_slots, uint32_t epoch, int* err) {
  if (threadIdx.x == 0 && g_p2p_trace) g_p2p_trace[P2P_SLOTS * 4 + 0] = globaltimer_ns();
  for (int t = threadIdx.x; t < n_slots * P2P_MAX_WORLD; t += blockDim.x) {
    const int slot = slot_lo + t / P2P_MAX_WORLD, p = t % P2P_MAX_WORLD;
    if (p < world && p != rank)
      spin_until(own_flags + (P2P_SLOTS + slot) * P2P_MAX_WORLD + p, epoch, err, 2);
  }
  __syncthreads();
  if (threadIdx.x == 0 && g_p2p_trace) g_p2p_trace[P2P_SLOTS * 4 + 1] = globaltimer_ns();
}

// W = compile-time world size (2, 4, 8) or 0 = run-time `world` (any size up to 8).
// Register budget: 32 per thread -- one warp then needs 1024 registers of its SM sub-partition, a small enough slice to
// fit next to the backward kernels.  Two 16-byte loads are in flight per thread; the memory-level parallelism
// comes from the number of resident warps instead.
template <int W>
__global__ void __launch_bounds__(P2P_THREADS, 16)
p2p_allreduce_kernel(P2PPeers pr, uint32_t* own_flags, int rank, int world, size_t off, uint32_t nchunks, int slot, uint32_t epoch,
                     int* err) {
  const int NW = W ? W : world;
  const int tid = threadIdx.x;
  if (g_p2p_trace && blockIdx.x == 0 && tid == 0) g_p2p_trace[slot * 4 + 1] = globaltimer_ns();
  // every peer's gradients of this bucket are final?
  if (tid < NW && tid != rank) spin_until(own_flags + slot * P2P_MAX_WORLD + tid, epoch, err, 1);
  __syncthreads();
  if (g_p2p_trace && blockIdx.x == 0 && tid == 0) g_p2p_trace[slot * 4 + 2] = globaltimer_ns();
  const uint32_t s1 = (uint32_t)((uint64_t)nchunks * (uint32_t)(rank + 1) / (uint32_t)NW);
  const uint32_t stride = gridDim.x * P2P_THREADS;
  for (uint32_t i = (uint32_t)((uint64_t)nchunks * (uint32_t)rank / (uint32_t)NW) + blockIdx.x * P2P_THREADS + tid; i < s1; i += stride) {
    const size_t e = off + (size_t)i * 8;
    f32x2 acc[4];
    {
      const uint4 a = ld_peer128(pr.buf[0] + e), b = ld_peer128(pr.buf[1] + e);
      acc[0] = add2(bf2_to_f32x2(a.x), bf2_to_f32x2(b.x));
      acc[1] = add2(bf2_to_f32x2(a.y), bf2_to_f32x2(b.y));
      acc[2] = add2(bf2_to_f32x2(a.z), bf2_to_f32x2(b.z));
      acc[3] = add2(bf2_to_f32x2(a.w), bf2_to_f32x2(b.w));
    }
#pragma unroll
    for (int p = 2; p < (W ? W : P2P_MAX_WORLD); ++p) {
      if (W || p < NW) {                                      // rank order: (.. + g_p) + g_{p+1}
        const uint4 a = ld_peer128(pr.buf[p] + e);
        acc[0] = add2(acc[0], bf2_to_f32x2(a.x));
        acc[1] = add2(acc[1], bf2_to_f32x2(a.y));
        acc[2] = add2(acc[2], bf2_to_f32x2(a.z));
        acc[3] = add2(acc[3], bf2_to_f32x2(a.w));
      }
    }
    uint4 o;
    o.x = f32x2_to_bf2(acc[0]);
    o.y = f32x2_to_bf2(acc[1]);
    o.z = f32x2_to_bf2(acc[2]);
    o.w = f32x2_to_bf2(acc[3]);
#pragma unroll
    for (int p = 0; p < (W ? W : P2P_MAX_WORLD); ++p)
      if (W || p < NW) st_peer128(pr.buf[p] + e, o);
  }
  // publish: all stores of this CTA are system-visible before it is counted; the last CTA tells the peers
  __threadfence_system();
  __syncthreads();
  if (tid == 0) {
    uint32_t* counter = own_flags + 2 * P2P_SLOTS * P2P_MAX_WORLD + slot;
    const uint32_t prev = atomicAdd(counter, 1u);
    if (prev == gridDim.x - 1) {
      *counter = 0u;                                   // next launch on this slot is stream-ordered after this one
      if (g_p2p_trace) g_p2p_trace[slot * 4 + 3] = globaltimer_ns();
      __threadfence_system();
#pragma unroll
      for (int p = 0; p < P2P_MAX_WORLD; ++p)
        if (p < NW && p != rank) st_release_sys(pr.flag[p] + (P2P_SLOTS + slot) * P2P_MAX_WORLD + rank, epoch);
    }
  }
}

// Stand-in with exactly the reduce kernel's footprint (128 threads, <= 32 registers, no shared memory) that just occupies
// its slot for `ns` nanoseconds: timing the backward kernels with and without it resident shows which of them share an SM
// with the reduce kernel.
__global__ void __launch_bounds__(P2P_THREADS, 16) p2p_hog_kernel(unsigned long long ns, unsigned* started, float* sink) {
  if (threadIdx.x == 0) atomicAdd(started, 1u);
  const uint64_t t0 = globaltimer_ns();
  float v[20];                                        // live values: the allocation is 32 registers like the reduce kernel's
#pragma unroll
  for (int i = 0; i < 20; ++i) v[i] = (float)(threadIdx.x + i);
  while (globaltimer_ns() - t0 < ns) {
    __nanosleep(1000);
#pragma unroll
    for (int i = 0; i < 20; ++i) v[i] = fmaf(v[i], 1.0001f, (float)i);
  }
  float t = 0.f;
#pragma unroll
  for (int i = 0; i < 20; ++i) t += v[i];
  if (t == 12345.678f) *sink = t;
}

// The GEMM / attention CTAs these kernels must share an SM with run under the maximum shared-memory carve-out; an SM
// cannot change its L1 / shared split while CTAs are resident, so a kernel that asks for the default (small) carve-out
// would wait for the SM to drain.  Ask for the same split (a hint the driver honours when it can).
int p2p_prepare() {
  static bool done = false;
  if (done) return 0;
  const int mx = cudaSharedmemCarveoutMaxShared;
  static const int on = [] { const char* e = getenv("SK_P2P_CARVEOUT"); return e ? atoi(e) : 1; }();
  if (on) {
    SK_CUDA_CHECK(cudaFuncSetAttribute(p2p_signal_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, mx));
    SK_CUDA_CHECK(cudaFuncSetAttribute(p2p_wait_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, mx));
    SK_CUDA_CHECK(cudaFuncSetAttribute(p2p_hog_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, mx));
    SK_CUDA_CHECK(cudaFuncSetAttribute(p2p_allreduce_kernel<0>, cudaFuncAttributePreferredSharedMemoryCarveout, mx));
    SK_CUDA_CHECK(cudaFuncSetAttribute(p2p_allreduce_kernel<2>, cudaFuncAttributePreferredSharedMemoryCarveout, mx));
    SK_CUDA_CHECK(cudaFuncSetAttribute(p2p_allreduce_kernel<4>, cudaFuncAttributePreferredSharedMemoryCarveout, mx));
    SK_CUDA_CHECK(cudaFuncSetAttribute(p2p_allreduce_kernel<8>, cudaFuncAttributePreferredSharedMemoryCarveout, mx));
  }
  done = true;
  return 0;
}

int fill_peers(P2PPeers& pr, void* const* bufs, void* const* flags, int rank, int world) {
  SK_REQUIRE(world >= 2 && world <= P2P_MAX_WORLD && rank >= 0 && rank < world, "p2p: world %d / rank %d out of range (2..%d ranks)",
             world, rank, P2P_MAX_WORLD);
  if (int rc = p2p_prepare()) return rc;
  memset(&pr, 0, sizeof(pr));
  for (int p = 0; p < world; ++p) {
    SK_REQUIRE(flags[p] != nullptr, "p2p: flag array of rank %d is not mapped", p);
    pr.flag[p] = reinterpret_cast<uint32_t*>(flags[p]);
    if (bufs) {
      SK_REQUIRE(bufs[p] != nullptr && (reinterpret_cast<uintptr_t>(bufs[p]) & 15) == 0, "p2p: buffer of rank %d missing or not 16-byte aligned", p);
      pr.buf[p] = reinterpret_cast<bf16*>(bufs[p]);
    }
  }
  return 0;
}

}  // namespace

int sk_p2p_hog_launch(int ctas, long long ns, unsigned* started, cudaStream_t s) {
  if (int rc = p2p_prepare()) return rc;
  SK_REQUIRE(ctas > 0 && ns > 0 && started, "p2p_hog: bad arguments");
  p2p_hog_kernel<<<ctas, P2P_THREADS, 0, s>>>((unsigned long long)ns, started, reinterpret_cast<float*>(started));
  SK_LAUNCH_CHECK();
  return 0;
}

int sk_p2p_set_trace_impl(void* buf) {
  unsigned long long* p = reinterpret_cast<unsigned long long*>(buf);
  SK_CUDA_CHECK(cudaMemcpyToSymbol(g_p2p_trace, &p, sizeof(p)));
  return 0;
}

size_t sk_p2p_flag_bytes_impl() { return P2P_FLAG_WORDS * sizeof(uint32_t); }

int sk_p2p_alloc_impl(size_t bytes, void** out) {
  SK_REQUIRE(out != nullptr && bytes > 0, "p2p_alloc: bad arguments");
  SK_CUDA_CHECK(cudaMalloc(out, bytes));
  SK_CUDA_CHECK(cudaMemset(*out, 0, bytes));
  SK_CUDA_CHECK(cudaDeviceSynchronize());
  return 0;
}

int sk_p2p_free_impl(void* p) {
  if (p) SK_CUDA_CHECK(cudaFree(p));
  return 0;
}

// IPC handle of the cudaMalloc allocation that contains `ptr` + the offset of `ptr` inside it
int sk_p2p_export_impl(const void* ptr, void* handle64, size_t* offset) {
  SK_REQUIRE(ptr && handle64 && offset, "p2p_export: null argument");
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
  typedef CUresult (*PFN_range)(CUdeviceptr*, size_t*, CUdeviceptr);
  static PFN_range fn_range = nullptr;
  if (!fn_range) {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult q;
    SK_CUDA_CHECK(cudaGetDriverEntryPoint("cuMemGetAddressRange", &fn, cudaEnableDefault, &q));
    SK_REQUIRE(q == cudaDriverEntryPointSuccess && fn, "p2p_export: cuMemGetAddressRange not available");
    fn_range = (PFN_range)fn;
  }
  CUdeviceptr base = 0;
  size_t size = 0;
  const CUresult r = fn_range(&base, &size, (CUdeviceptr)(uintptr_t)ptr);
  SK_REQUIRE(r == CUDA_SUCCESS, "p2p_export: cuMemGetAddressRange failed with CUresult %d", (int)r);
  cudaIpcMemHandle_t h;
  SK_CUDA_CHECK(cudaIpcGetMemHandle(&h, reinterpret_cast<void*>((uintptr_t)base)));
  memcpy(handle64, &h, sizeof(h));
  *offset = (size_t)((uintptr_t)ptr - (uintptr_t)base);
  return 0;
}

int sk_p2p_open_impl(const void* handle64, void** base) {
  SK_REQUIRE(handle64 && base, "p2p_open: null argument");
  cudaIpcMemHandle_t h;
  memcpy(&h, handle64, sizeof(h));
  SK_CUDA_CHECK(cudaIpcOpenMemHandle(base, h, cudaIpcMemLazyEnablePeerAccess));
  return 0;
}

int sk_p2p_close_impl(void* base) {
  if (base) SK_CUDA_CHECK(cudaIpcCloseMemHandle(base));
  return 0;
}

int sk_p2p_signal_launch(void* const* flags, int rank, int world, int slot, uint32_t epoch, cudaStream_t s) {
  P2PPeers pr;
  if (int rc = fill_peers(pr, nullptr, flags, rank, world)) return rc;
  SK_REQUIRE(slot >= 0 && slot < P2P_SLOTS, "p2p: slot %d out of range", slot);
  p2p_signal_kernel<<<1, 32, 0, s>>>(pr, rank, world, slot, epoch);
  SK_LAUNCH_CHECK();
  return 0;
}

int sk_p2p_wait_launch(void* const* flags, int rank, int world, int slot_lo, int n_slots, uint32_t epoch, int* err_flag, cudaStream_t s) {
  P2PPeers pr;
  if (int rc = fill_peers(pr, nullptr, flags, rank, world)) return rc;
  // (n_slots <= P2P_SLOTS - slot_lo: slot_lo + n_slots could overflow int and pass the bound)
  SK_REQUIRE(slot_lo >= 0 && slot_lo < P2P_SLOTS && n_slots >= 1 && n_slots <= P2P_SLOTS - slot_lo, "p2p: slots [%d, +%d) out of range",
             slot_lo, n_slots);
  p2p_wait_kernel<<<1, 256, 0, s>>>(pr.flag[rank], rank, world, slot_lo, n_slots, epoch, err_flag);
  SK_LAUNCH_CHECK();
  return 0;
}

int sk_p2p_allreduce_launch(void* const* bufs, void* const* flags, int rank, int world, size_t offset_elems, size_t n_elems,
                            int slot, uint32_t epoch, int ctas, int* err_flag, cudaStream_t s) {
  P2PPeers pr;
  if (int rc = fill_peers(pr, bufs, flags, rank, world)) return rc;
  SK_REQUIRE(slot >= 0 && slot < P2P_SLOTS, "p2p: slot %d out of range", slot);
  SK_REQUIRE(offset_elems % 8 == 0 && n_elems % 8 == 0 && n_elems > 0,
             "p2p_allreduce: range [%zu, +%zu) must be a non-empty multiple of 8 bf16 elements", offset_elems, n_elems);
  const size_t nchunks = n_elems / 8;
  SK_REQUIRE(nchunks < (1ull << 31), "p2p_allreduce: range too long (%zu elements)", n_elems);
  const size_t per_rank = (nchunks + world - 1) / world;
  size_t want = (per_rank + P2P_THREADS - 1) / P2P_THREADS;
  if (ctas < 1) ctas = 1;
  if ((size_t)ctas > want) ctas = (int)(want ? want : 1);
  switch (world) {
    case 2: p2p_allreduce_kernel<2><<<ctas, P2P_THREADS, 0, s>>>(pr, pr.flag[rank], rank, world, offset_elems, (uint32_t)nchunks, slot, epoch, err_flag); break;
    case 4: p2p_allreduce_kernel<4><<<ctas, P2P_THREADS, 0, s>>>(pr, pr.flag[rank], rank, world, offset_elems, (uint32_t)nchunks, slot, epoch, err_flag); break;
    case 8: p2p_allreduce_kernel<8><<<ctas, P2P_THREADS, 0, s>>>(pr, pr.flag[rank], rank, world, offset_elems, (uint32_t)nchunks, slot, epoch, err_flag); break;
    default: p2p_allreduce_kernel<0><<<ctas, P2P_THREADS, 0, s>>>(pr, pr.flag[rank], rank, world, offset_elems, (uint32_t)nchunks, slot, epoch, err_flag); break;
  }
  SK_LAUNCH_CHECK();
  return 0;
}
