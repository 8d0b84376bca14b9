"""Which kernels of the backward pass share an SM with the peer all-reduce kernel?  A stand-in with the reduce kernel's
exact footprint (128 threads, <= 32 registers, no shared memory; sk_p2p_debug_hog) is parked on every SM for 30 ms on a
high-priority side stream; each kernel is timed alone and while the stand-ins are resident.  A kernel that cannot
co-reside either waits for them (time jumps by milliseconds) or loses occupancy."""
import ctypes as C, os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from slamkit_b200 import _lib as L, ops

dev = "cuda:0"
lib = L.require_cuda()
side = torch.cuda.Stream(priority=-1)
started = torch.zeros(1, dtype=torch.int32, device=dev)
M = 8192
B, T, H, KVH = 8, 1024, 14, 2


def bf(*shape):
    return torch.randn(*shape, device=dev).to(torch.bfloat16)


x896, w_gu, wd = bf(M, 896), bf(9728, 896), bf(896, 4864)
dy, gu = bf(M, 896), bf(M, 9728)
a_t, b_t = bf(M, 9728), bf(M, 896)
qkv, d_o = bf(B * T, (H + 2 * KVH) * 64), bf(B * T, H * 64)
o, lse = ops.attn_tc_fwd(qkv, B, T, H, KVH, True, 0.125)
out1 = torch.empty(M, 9728, device=dev, dtype=torch.bfloat16)
cases = {
    "gemm 4 epilogue warps (gu_fwd shape)": lambda: ops.gemm(x896, w_gu, out=out1),
    "gemm stream-K wgrad (gu_wgrad shape)": lambda: ops.gemm(a_t, b_t, a_mn=True, b_mn=True, streamk=True),
    "gemm 8 epilogue warps (SwiGLU backward)": lambda: ops.linear_swiglu_bwd(dy, wd, gu),
    "attention forward": lambda: ops.attn_tc_fwd(qkv, B, T, H, KVH, True, 0.125),
    "attention backward (dq, dkdv, reduce)": lambda: ops.attn_tc_bwd(qkv, o, d_o, lse, B, T, H, KVH, True, 0.125),
}


def timed(fn, n=20):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(n):
        fn()
    e.record()
    e.synchronize()
    return s.elapsed_time(e) / n * 1e3


for ctas in (lib.sk_device_sm_count(), 48):
    print(f"--- {ctas} stand-in CTAs")
    for name, fn in cases.items():
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        alone = timed(fn)
        torch.cuda.synchronize()
        started.zero_()
        torch.cuda.synchronize()
        with torch.cuda.stream(side):
            L.check(lib.sk_p2p_debug_hog(ctas, C.c_int64(30_000_000), C.c_void_p(started.data_ptr()), C.c_void_p(side.cuda_stream)))
        time.sleep(0.002)                       # the stand-ins are resident before the timed launches start
        n0 = int(started.cpu())
        shared = timed(fn)
        torch.cuda.synchronize()
        print(f"{name:42s} alone {alone:8.1f} us   with stand-ins resident {shared:8.1f} us   ({n0}/{ctas} resident at start)", flush=True)
