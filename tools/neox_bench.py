"""GPT-NeoX train-step benchmark: this package's step (forward + backward + clip + AdamW) against HF
`GPTNeoXForCausalLM` (bf16 parameters, bf16 autocast, sdpa attention, fused AdamW) on the same card and the same
batches, in one call.  Prints one JSON line per shape with the card name and power limit.

    python tools/neox_bench.py [--steps 20] [--warmup 5] [--shapes 160m,410m,410m-scale] [--no-hf]
                               [--profile] [--generate] [--epilogue]

Shapes: pythia-160m / -410m geometry with the 502-unit vocabulary at [8, 1024], and the interleaving-scaling recipe's
shape: pythia-410m, packed [4, 2048] rows (512-token documents), a 50 816-row interleaved vocabulary, untied head.  At
the packed shape this package runs block-diagonal attention over the 512-token documents; HF's sdpa path has no varlen
kernel, so the baseline runs causal attention over the whole 2048-token rows (more attention work than ours).

--profile   a separate run per shape: torch.profiler kernel time per step, split GEMM / attention / LayerNorm / other
--generate  cached greedy generate at pythia-160m geometry, 64-token prompts, 256 new tokens, B = 1 and 64
--epilogue  the GELU' backward epilogue (dense_4h_to_h's input gradient) against the same GEMM without it, at [8192, F]"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SHAPES = {
    "160m": dict(hidden=768, n_layers=12, n_heads=12, vocab=502, B=8, T=1024, packed=False),
    "410m": dict(hidden=1024, n_layers=24, n_heads=16, vocab=502, B=8, T=1024, packed=False),
    "410m-scale": dict(hidden=1024, n_layers=24, n_heads=16, vocab=50816, B=4, T=2048, packed=True),
}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=20).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in out.split(",")]
        return name, power
    except Exception:   # noqa: BLE001
        return torch.cuda.get_device_name(0), "unknown"


def batches(s, n, seed=0):
    g = torch.Generator().manual_seed(seed)
    out = []
    for _ in range(n):
        ids = torch.randint(2, s["vocab"], (s["B"], s["T"]), generator=g)
        pos = (torch.arange(s["T"]) % 512)[None].expand(s["B"], -1).contiguous() if s["packed"] else None
        out.append((ids, ids.clone(), pos))
    return out


def timed(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(steps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    ts.sort()
    return ts[len(ts) // 2], ts[0], ts[-1]


def bench_ours(s, data, steps, warmup):
    from slamkit_b200.lm import B200AdamW, B200UnitLM, NeoxLMConfig
    cfg = NeoxLMConfig(vocab_size=s["vocab"], hidden=s["hidden"], n_layers=s["n_layers"], n_heads=s["n_heads"],
                       ffn=4 * s["hidden"], max_positions=2048, rot_dims=16)
    m = B200UnitLM(cfg, device="cuda:0", max_batch=s["B"], max_seq=s["T"], seed=0)
    opt = B200AdamW(m, lr=1e-4, max_grad_norm=1.0)
    dev = [(i.cuda(), l.cuda(), p.cuda() if p is not None else None) for i, l, p in data]
    it = [0]

    def step():
        ids, labels, pos = dev[it[0] % len(dev)]
        it[0] += 1
        m.forward_backward(ids, labels, position_ids=pos, num_items_in_batch=float(labels.numel()))
        opt.step()
    r = timed(step, steps, warmup)
    del m, opt
    torch.cuda.empty_cache()
    return r


def bench_hf(s, data, steps, warmup):
    from transformers import GPTNeoXConfig, GPTNeoXForCausalLM
    cfg = GPTNeoXConfig(vocab_size=s["vocab"], hidden_size=s["hidden"], num_hidden_layers=s["n_layers"],
                        num_attention_heads=s["n_heads"], intermediate_size=4 * s["hidden"], max_position_embeddings=2048,
                        tie_word_embeddings=False, attn_implementation="sdpa",
                        rope_parameters={"rope_theta": 10000.0, "partial_rotary_factor": 0.25, "rope_type": "default"})
    torch.manual_seed(0)
    m = GPTNeoXForCausalLM(cfg).to(device="cuda:0", dtype=torch.bfloat16)
    m.train()
    opt = torch.optim.AdamW(m.parameters(), lr=1e-4, fused=True)
    dev = [(i.cuda(), l.cuda(), p.cuda() if p is not None else None) for i, l, p in data]
    it = [0]

    def step():
        ids, labels, pos = dev[it[0] % len(dev)]
        it[0] += 1
        with torch.autocast("cuda", dtype=torch.bfloat16):
            # packed rows: HF's sdpa path has no varlen kernel, so it attends causally over the whole row (more work)
            out = m(input_ids=ids, labels=labels)
        out.loss.backward()
        torch.nn.utils.clip_grad_norm_(m.parameters(), 1.0)
        opt.step()
        opt.zero_grad(set_to_none=True)
    r = timed(step, steps, warmup)
    del m, opt
    torch.cuda.empty_cache()
    return r


def profile_ours(s, data, steps=3):
    """Kernel time per step by category from torch.profiler (its own run: the profiler perturbs the timing above)."""
    from torch.profiler import ProfilerActivity, profile
    from slamkit_b200.lm import B200AdamW, B200UnitLM, NeoxLMConfig
    cfg = NeoxLMConfig(vocab_size=s["vocab"], hidden=s["hidden"], n_layers=s["n_layers"], n_heads=s["n_heads"],
                       ffn=4 * s["hidden"], max_positions=2048, rot_dims=16)
    m = B200UnitLM(cfg, device="cuda:0", max_batch=s["B"], max_seq=s["T"], seed=0)
    opt = B200AdamW(m, lr=1e-4, max_grad_norm=1.0)
    ids, labels, pos = (t.cuda() if t is not None else None for t in data[0])
    for _ in range(2):
        m.forward_backward(ids, labels, position_ids=pos, num_items_in_batch=float(labels.numel()))
        opt.step()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA], acc_events=True) as prof:
        for _ in range(steps):
            m.forward_backward(ids, labels, position_ids=pos, num_items_in_batch=float(labels.numel()))
            opt.step()
        torch.cuda.synchronize()
    split = {"gemm": 0.0, "attention": 0.0, "layernorm": 0.0, "other": 0.0}
    for e in prof.key_averages():
        if str(getattr(e, "device_type", "")).split(".")[-1] != "CUDA":
            continue                       # kernels only: host-side ops would count their kernels a second time
        t = getattr(e, "self_device_time_total", None) or getattr(e, "self_cuda_time_total", 0.0)
        n = e.key.lower()
        k = "gemm" if "gemm" in n or "splitk" in n else "attention" if "attn" in n else "layernorm" if "layernorm" in n \
            else "other"
        split[k] += t / 1e3 / steps
    del m, opt
    torch.cuda.empty_cache()
    return {k: round(v, 3) for k, v in split.items()}


def bench_generate(B, steps_new=256, prompt=64):
    from slamkit_b200.lm import B200UnitLM, NeoxLMConfig
    s = SHAPES["160m"]
    cfg = NeoxLMConfig(vocab_size=502, hidden=s["hidden"], n_layers=s["n_layers"], n_heads=s["n_heads"], ffn=4 * s["hidden"],
                       max_positions=2048, rot_dims=16)
    m = B200UnitLM(cfg, device="cuda:0", max_batch=B, max_seq=prompt, trainable=False, seed=0)
    ids = torch.randint(2, 502, (B, prompt), generator=torch.Generator().manual_seed(0))
    m.generate(ids, max_new_tokens=8, do_sample=False, eos_token_id=None)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = m.generate(ids, max_new_tokens=steps_new, do_sample=False, eos_token_id=None)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    del m
    torch.cuda.empty_cache()
    return {"B": B, "new_tokens": int(out.shape[1] - prompt), "s": round(dt, 4),
            "tokens_per_s": round(B * (out.shape[1] - prompt) / dt), "ms_per_step": round(dt / steps_new * 1e3, 3)}


def bench_gelu_bwd_epilogue(M, N, F, steps=50):
    """sk_linear_gelu_bwd (d_pre from the GEMM epilogue) against the plain dgrad GEMM of the same shape: the difference is
    what the epilogue costs; a separate GELU' pass would have to move 3 x M x F bf16 values through HBM."""
    import ctypes as C
    from slamkit_b200 import _lib as L
    lib = L.require_cuda()
    dy = torch.randn(M, N, device="cuda:0").to(torch.bfloat16)
    w2 = (torch.randn(N, F, device="cuda:0") * 0.02).to(torch.bfloat16)
    pre = torch.randn(M, F, device="cuda:0").to(torch.bfloat16)
    out = torch.empty(M, F, device="cuda:0", dtype=torch.bfloat16)
    fused = lambda: L.check(lib.sk_linear_gelu_bwd(M, N, F, L.ptr(dy), L.ptr(w2), L.ptr(pre), L.ptr(out), L.stream_ptr()))  # noqa: E731
    plain = lambda: L.check(lib.sk_gemm_bf16(M, F, N, L.ptr(dy), N, 0, L.ptr(w2), F, 1, L.ptr(out), F, 0, None, None, 0,  # noqa: E731
                                             0, 0, 0, L.stream_ptr()))
    r = {}
    for name, fn in (("plain", plain), ("fused", fused), ("plain2", plain), ("fused2", fused)):
        r[name] = timed(lambda: [fn() for _ in range(10)], steps // 10, 2)[0] / 10 * 1e3
    f, p = min(r["fused"], r["fused2"]), min(r["plain"], r["plain2"])
    return {"M": M, "N": N, "F": F, "fused_us": round(f, 1), "plain_dgrad_us": round(p, 1), "epilogue_us": round(f - p, 1),
            "separate_pass_hbm_floor_us": round(3 * M * F * 2 / 3.35e12 * 1e6, 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--shapes", default="160m,410m,410m-scale")
    ap.add_argument("--no-hf", action="store_true")
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--generate", action="store_true")
    ap.add_argument("--epilogue", action="store_true")
    a = ap.parse_args()
    name, power = card()
    if a.epilogue:
        for N, F in ((768, 3072), (1024, 4096)):
            print(json.dumps({"gelu_bwd_epilogue": bench_gelu_bwd_epilogue(8192, N, F), "card": name, "power_limit": power}),
                  flush=True)
    if a.generate:
        for B in (1, 64):
            print(json.dumps({"generate": bench_generate(B), "card": name, "power_limit": power}), flush=True)
    if a.profile:
        for key in a.shapes.split(","):
            print(json.dumps({"shape": key, "kernel_split_ms_per_step": profile_ours(SHAPES[key], batches(SHAPES[key], 1)),
                              "card": name, "power_limit": power}), flush=True)
    if a.profile or a.generate or a.epilogue:
        return
    for key in a.shapes.split(","):
        s = SHAPES[key]
        data = batches(s, 4)
        ours = bench_ours(s, data, a.steps, a.warmup)
        hf = None if a.no_hf else bench_hf(s, data, a.steps, a.warmup)
        tok = s["B"] * s["T"]
        print(json.dumps({"shape": key, "B": s["B"], "T": s["T"], "vocab": s["vocab"], "card": name, "power_limit": power,
                          "ours_ms": round(ours[0], 3), "ours_min_max_ms": [round(ours[1], 3), round(ours[2], 3)],
                          "ours_tok_s": round(tok / ours[0] * 1e3),
                          "hf_ms": None if hf is None else round(hf[0], 3),
                          "hf_min_max_ms": None if hf is None else [round(hf[1], 3), round(hf[2], 3)],
                          "time": time.strftime("%Y-%m-%dT%H:%M:%S")}), flush=True)


if __name__ == "__main__":
    main()
