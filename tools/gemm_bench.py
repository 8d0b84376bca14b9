"""Micro-benchmark of the wgmma GEMM on the LM shapes (CUDA events, L2 flushed between iterations).
Prints one line per shape: our TFLOP/s per tile width (bn0 = the planner's choice), with the scratch buffer (sk: split-K /
stream-K where the planner takes them), torch.matmul (cuBLAS) for context, and the schedule the planner picks with scratch."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from slamkit_b200 import ops

dev = "cuda:0"
flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)


def timeit(fn, iters=10):
    for _ in range(3):
        fn()
    ts = []
    for _ in range(iters):
        flush.zero_()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record(); fn(); e.record()
        torch.cuda.synchronize()
        ts.append(s.elapsed_time(e))
    ts.sort()
    return ts[len(ts) // 2]


M = 8192
shapes = [  # (name, M, N, K, a_mn, b_mn)
    ("qkv_fwd", M, 1152, 896, 0, 0), ("o_fwd", M, 896, 896, 0, 0), ("gu_fwd", M, 9728, 896, 0, 0),
    ("down_fwd", M, 896, 4864, 0, 0), ("head_fwd", M, 512, 896, 0, 0),
    ("gu_dgrad", M, 896, 9728, 0, 1), ("down_dgrad", M, 4864, 896, 0, 1),
    ("gu_wgrad", 9728, 896, M, 1, 1), ("down_wgrad", 896, 4864, M, 1, 1), ("qkv_wgrad", 1152, 896, M, 1, 1),
    ("qkv_dgrad", M, 896, 1152, 0, 1), ("o_dgrad", M, 896, 896, 0, 1), ("o_wgrad", 896, 896, M, 1, 1),
    ("head_dgrad", M, 896, 512, 0, 1), ("head_wgrad", 512, 896, M, 1, 1),
]
_only = os.environ.get('GEMM_SHAPES')
for name, m, n, k, a_mn, b_mn in shapes:
    if _only and name not in _only.split(','):
        continue
    a = torch.randn((k, m) if a_mn else (m, k), device=dev).to(torch.bfloat16)
    b = torch.randn((k, n) if b_mn else (n, k), device=dev).to(torch.bfloat16)
    out = torch.empty((m, n), device=dev, dtype=torch.bfloat16)
    flops = 2.0 * m * n * k
    res = []
    for bn in (0, 128, 192, 224, 256):
        t = timeit(lambda: ops.gemm(a, b, a_mn=bool(a_mn), b_mn=bool(b_mn), out=out, force_bn=bn))
        res.append(f"bn{bn}: {flops / t / 1e9:7.1f} TF/s ({t * 1e3:7.1f} us)")
    for bn in (0, 224, 256):   # with the scratch buffer: split-K / stream-K balancing
        t = timeit(lambda: ops.gemm(a, b, a_mn=bool(a_mn), b_mn=bool(b_mn), out=out, force_bn=bn, streamk=True))
        res.append(f"sk{bn}: {flops / t / 1e9:7.1f} TF/s ({t * 1e3:7.1f} us)")
    A = a.t() if a_mn else a
    Bt = b if b_mn else b.t()
    t = timeit(lambda: torch.matmul(A, Bt, out=out))
    pl = ops.gemm_plan(a, b, a_mn=bool(a_mn), b_mn=bool(b_mn), out=out, streamk=True)
    sched = (f"splitk{pl['splits']}" if pl["splits"] > 1 else
             (f"streamk-{'cols' if pl['sk_colunits'] else 'rows'} {pl['sk_units']}u/{pl['sk_groups']}g" if pl["sk_units"] else "tiles"))
    print(f"{name:11s} M{m} N{n} K{k} | " + " | ".join(res) + f" | cublas {flops / t / 1e9:7.1f} TF/s ({t*1e3:7.1f} us)"
          f" | plan bn{pl['bn']} {sched}", flush=True)
