"""Times the wgmma attention kernels (forward, backward) at the LM shape (B=8,H=14,KVH=2,T=1024)."""
import sys, os, math
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from slamkit_b200 import ops
dev = "cuda:0"
B, T, H, KVH = 8, 1024, 14, 2
qkv = torch.randn(B * T, (H + 2 * KVH) * 64, device=dev).to(torch.bfloat16)
d_o = torch.randn(B * T, H * 64, device=dev).to(torch.bfloat16)
scale = 0.125
def timeit(fn, n=20):
    for _ in range(3): fn()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize(); s.record()
    for _ in range(n): fn()
    e.record(); torch.cuda.synchronize()
    return s.elapsed_time(e) / n * 1e3
fl_fwd = 4 * B * H * T * T * 64 / 2
o, lse = ops.attn_tc_fwd(qkv, B, T, H, KVH, True, scale)
t = timeit(lambda: ops.attn_tc_fwd(qkv, B, T, H, KVH, True, scale)); print(f"fwd {t:8.1f} us {fl_fwd/t/1e6:7.1f} TF/s")
t = timeit(lambda: ops.attn_tc_bwd(qkv, o, d_o, lse, B, T, H, KVH, True, scale)); print(f"bwd {t:8.1f} us {2.5*fl_fwd/t/1e6:7.1f} TF/s (5 GEMM-equivalents)")
