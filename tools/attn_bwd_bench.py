"""Per-kernel time of the causal attention forward and backward at the LM step's shapes.

Shapes (H = 14 query heads, KVH = 2 kv heads, head_dim 64, RoPE tables as in the LM step):
  cfg2: B = 8,  T = 1024        cfg5: B = 16, T = 1024        cfg4: one 8192-token row packed with 512..2048-token documents

For each shape the backward call (sk_attn_tc_bwd, then the inverse RoPE of dq / dk with sk_rope, as the LM step runs
it) is timed with CUDA events over `--iters` launches, and a separate torch.profiler run splits forward and backward
into their kernels: attn_fwd_kernel, attn_delta_kernel, attn_bwd_kernel (dK/dV and dQ tiles in one grid; libraries
before it ran attn_bwd_dkdv_kernel and attn_bwd_dq_kernel) and rope_kernel.  TFLOP/s counts the matmul FLOPs a kernel
executes on the causal half (forward 2, dK/dV 4, dQ 3, dK/dV + dQ 7 products of 2*T*T/2*64 per head; the packed row's
masks are not subtracted).

  python tools/attn_bwd_bench.py [--shapes cfg2,cfg5,cfg4] [--iters 50] [--json out.jsonl] [--tag name]
"""
import argparse
import json
import os
import subprocess
import sys
from collections import defaultdict

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from slamkit_b200 import _lib as L  # noqa: E402
from slamkit_b200 import ops  # noqa: E402

DEV = "cuda:0"
H, KVH, HD = 14, 2, 64
SHAPES = {"cfg2": (8, 1024, False), "cfg5": (16, 1024, False), "cfg4": (1, 8192, True)}
KERNELS = ["attn_fwd_kernel", "attn_delta_kernel", "attn_bwd_kernel", "attn_bwd_dkdv_kernel", "attn_bwd_dq_kernel",
           "rope_kernel"]
PRODUCTS = {"attn_fwd_kernel": 2, "attn_bwd_kernel": 7, "attn_bwd_dkdv_kernel": 4, "attn_bwd_dq_kernel": 3}


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"{torch.cuda.get_device_name(0)} (power limit unknown: {e})"


def packed_docs(T, seed=0):
    g = torch.Generator().manual_seed(seed)
    docs, t = [], 0
    while t < T:
        n = int(torch.randint(512, 2049, (1,), generator=g))
        n = T - t if T - t < 1024 else min(n, T - t - 512)
        docs.append(n)
        t += n
    return docs


class Case:
    def __init__(self, lib, name):
        B, T, packed = SHAPES[name]
        self.lib, self.name, self.B, self.T = lib, name, B, T
        g = torch.Generator().manual_seed(1)
        self.qkv = (torch.randn(B * T, (H + 2 * KVH) * HD, generator=g) * 0.5).to(torch.bfloat16).to(DEV)
        self.do = (torch.randn(B * T, H * HD, generator=g) * 0.1).to(torch.bfloat16).to(DEV)
        self.seg = self.seg_end = self.pos = None
        if packed:
            pos = torch.cat([torch.arange(n) for n in packed_docs(T)])[None].expand(B, T).contiguous()
            self.pos = pos.reshape(-1).to(torch.int32).to(DEV)
            self.seg, self.seg_end = ops.seg_bounds(pos.to(DEV))
        inv = 1.0 / (1e6 ** (torch.arange(0, HD, 2, dtype=torch.float32) / HD))
        ang = torch.outer(torch.arange(max(T, 1024), dtype=torch.float32), inv)
        self.cos = ang.cos().to(torch.bfloat16).to(DEV)
        self.sin = ang.sin().to(torch.bfloat16).to(DEV)
        self.o, self.lse = ops.attn_tc_fwd(self.qkv, B, T, H, KVH, True, 0.125, self.seg)
        self.dqkv = torch.empty_like(self.qkv)
        self.delta = torch.empty_like(self.lse)

    def fwd(self):
        ops.attn_tc_fwd(self.qkv, self.B, self.T, H, KVH, True, 0.125, self.seg)

    def bwd(self):
        lib, B, T, p = self.lib, self.B, self.T, L.ptr
        ld = self.qkv.stride(0)
        L.check(lib.sk_attn_tc_bwd(p(self.qkv), p(self.o), p(self.do), p(self.lse), p(self.delta), None, p(self.dqkv),
                                   B, T, H, KVH, ld, self.o.stride(0), ld, 1, L.f32(0.125), p(self.seg),
                                   p(self.seg_end), L.stream_ptr()))
        L.check(lib.sk_rope(p(self.dqkv), p(self.cos), p(self.sin), p(self.pos), B * T, T, ld, H + KVH, HD, 1,
                            self.cos.shape[0], L.stream_ptr()))

    def flops(self, products):
        return products * 2.0 * self.B * H * (self.T * self.T / 2) * HD


def event_us(fn, iters):
    for _ in range(5):
        fn()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters * 1e3


def kernel_us(fn, iters):
    from torch.profiler import ProfilerActivity, profile
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            fn()
        torch.cuda.synchronize()
    tot = defaultdict(float)
    for ev in prof.events():
        if ev.device_type.name != "CUDA":
            continue
        for k in KERNELS:
            if k in ev.name:
                tot[k] += ev.device_time
    return {k: v / iters for k, v in tot.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="cfg2,cfg5,cfg4")
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--json", default=None, help="append one JSON line per shape here")
    ap.add_argument("--tag", default="")
    a = ap.parse_args()
    lib = L.require_cuda()
    dev = card()
    print(f"# {dev}  tag={a.tag}")
    for name in a.shapes.split(","):
        c = Case(lib, name)
        bwd_us = event_us(c.bwd, a.iters)
        per = kernel_us(lambda: (c.fwd(), c.bwd()), a.iters)
        row = {"tag": a.tag, "card": dev, "shape": name, "bwd_call_us": round(bwd_us, 1),
               "kernels_us": {k: round(v, 1) for k, v in per.items()}}
        print(f"{name}: backward call {bwd_us:8.1f} us (events)")
        for k in KERNELS:
            if k in per:
                tf = f"{c.flops(PRODUCTS[k]) / per[k] / 1e6:7.1f} TFLOP/s" if k in PRODUCTS else ""
                print(f"    {k:24s} {per[k]:8.1f} us {tf}")
        if a.json:
            with open(a.json, "a") as fh:
                fh.write(json.dumps(row) + "\n")
        del c
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
