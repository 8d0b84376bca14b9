"""OPT decoder on the GPU path: train-step throughput at facebook/opt-125m geometry with the 502-unit vocabulary, its
device-time split (GEMM / attention / LayerNorm / other, from torch.profiler kernel names in a separate profiled step),
the model-FLOP rate against 989 TFLOP/s dense bf16, HF OPTForCausalLM (bf16 autocast, sdpa, fused AdamW) on the same
batches and card, and cached greedy generate at B = 1 and 64.  Prints one JSON line per measurement, the card's name
and power limit first.

    python tools/opt_bench.py [--steps 20] [--warmup 5] [--out results.jsonl]

Shapes: [8, 512] is config/model/default.yaml's context_len with config/training_args/default.yaml's per-device batch;
[8, 1024] doubles the context."""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle.opt_oracle import OracleOptConfig, flops_per_token  # noqa: E402
from slamkit_b200.lm import B200AdamW, B200UnitLM, OptLMConfig  # noqa: E402

PEAK_BF16 = 989e12
DEV = "cuda:0"


def emit(rec, out):
    line = json.dumps(rec)
    print(line, flush=True)
    if out:
        with open(out, "a") as f:
            f.write(line + "\n")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def batch(B, T, seed):
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(2, 502, (B, T), generator=g)
    ids[:, 0] = 1
    return ids.to(DEV), ids.clone().to(DEV)


def time_steps(step, steps, warmup):
    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        step()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


def split(step):
    """Device time of one step by kernel class, from a profiled step.  Run in a process of its own with SK_PDL=0: with
    programmatic dependent launch a kernel starts while its predecessor drains and waits inside, so kernel spans
    overlap and would not add up to the step."""
    from torch.profiler import ProfilerActivity, profile
    step()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        step()
        torch.cuda.synchronize()
    out = {"gemm": 0.0, "attention": 0.0, "layernorm": 0.0, "relu_bwd": 0.0, "other": 0.0}
    for e in prof.key_averages():
        us = getattr(e, "self_device_time_total", None)
        if us is None:
            us = e.self_cuda_time_total
        if us <= 0 or e.key.startswith("cuda") or e.key.startswith("Memset") or e.key.startswith("Memcpy"):
            continue
        k = e.key.lower()
        cat = ("gemm" if "gemm" in k or "splitk" in k else "attention" if "attn" in k else
               "layernorm" if "layernorm" in k else "relu_bwd" if "relu_bwd" in k else "other")
        out[cat] += us / 1e3
    out["total"] = sum(out.values())
    return {k: round(v, 3) for k, v in out.items()}


def bench_train(B, T, steps, warmup, out):
    cfg = OptLMConfig()
    m = B200UnitLM(cfg, device=DEV, max_batch=B, max_seq=T, seed=0)
    opt = B200AdamW(m, lr=1e-4, max_grad_norm=0.5)
    ids, labels = batch(B, T, T)
    n = float(B * T)

    def step():
        m.forward_backward(ids, labels, num_items_in_batch=n)
        opt.step()
    ms = time_steps(step, steps, warmup)
    toks = B * T / (ms / 1e3)
    fl = flops_per_token(OracleOptConfig(), T) * toks
    rec = {"what": "opt125m_train_step", "impl": "sk", "B": B, "T": T, "ms": round(ms, 3), "tokens_per_s": round(toks),
           "model_tflops": round(fl / 1e12, 1), "mfu_vs_989": round(fl / PEAK_BF16, 4), "loss": float(m.stats[0])}
    if os.environ.get("SK_PDL") == "0":
        rec = {"what": "opt125m_train_step_split", "impl": "sk_no_pdl", "B": B, "T": T, "ms": round(ms, 3),
               "kernel_ms": split(step)}
    emit(rec, out)
    del m, opt
    torch.cuda.empty_cache()
    return rec


def bench_hf(B, T, steps, warmup, out):
    from transformers import OPTConfig, OPTForCausalLM
    torch.manual_seed(0)
    hf = OPTForCausalLM(OPTConfig(vocab_size=502, dropout=0.0, attention_dropout=0.0, layerdrop=0.0, pad_token_id=0,
                                  bos_token_id=1, eos_token_id=1, attn_implementation="sdpa")).to(DEV).train()
    opt = torch.optim.AdamW(hf.parameters(), lr=1e-4, fused=True)
    ids, labels = batch(B, T, T)

    def step():
        with torch.autocast("cuda", dtype=torch.bfloat16):
            logits = hf(input_ids=ids).logits
        loss = torch.nn.functional.cross_entropy(logits.float()[:, :-1].reshape(-1, 502), labels[:, 1:].reshape(-1),
                                                 reduction="sum") / float(B * T)
        loss.backward()
        torch.nn.utils.clip_grad_norm_(hf.parameters(), 0.5)
        opt.step()
        opt.zero_grad(set_to_none=True)
    ms = time_steps(step, steps, warmup)
    toks = B * T / (ms / 1e3)
    fl = flops_per_token(OracleOptConfig(), T) * toks
    emit({"what": "opt125m_train_step", "impl": "hf_sdpa_autocast_bf16", "B": B, "T": T, "ms": round(ms, 3),
          "tokens_per_s": round(toks), "model_tflops": round(fl / 1e12, 1), "mfu_vs_989": round(fl / PEAK_BF16, 4)}, out)
    del hf, opt
    torch.cuda.empty_cache()


def bench_generate(B, prompt, new, out):
    m = B200UnitLM(OptLMConfig(), device=DEV, max_batch=B, max_seq=prompt, trainable=False, seed=0)
    ids = batch(B, prompt, 5)[0]
    kw = dict(max_new_tokens=new, do_sample=False, eos_token_id=None)
    m.generate(ids, **kw)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    reps = 3
    for _ in range(reps):
        m.generate(ids, **kw)
    torch.cuda.synchronize()
    s = (time.perf_counter() - t0) / reps
    emit({"what": "opt125m_generate", "impl": "sk", "B": B, "prompt": prompt, "new_tokens": new, "s": round(s, 4),
          "new_tokens_per_s": round(B * new / s), "ms_per_step": round(s / new * 1e3, 3)}, out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=None)
    ap.add_argument("--split-only", action="store_true", help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.split_only:
        for T in (512, 1024):
            bench_train(8, T, a.steps, a.warmup, a.out)
        return
    if not torch.cuda.is_available():
        raise SystemExit("opt_bench needs a CUDA device: there is nothing to measure on the CPU")
    emit({"what": "card", "name_power_limit_max_sm_clock": card()}, a.out)
    for T in (512, 1024):
        bench_train(8, T, a.steps, a.warmup, a.out)
        bench_hf(8, T, a.steps, a.warmup, a.out)
    subprocess.run([sys.executable, os.path.abspath(__file__), "--split-only", "--steps", "3", "--warmup", "2"] +
                   (["--out", a.out] if a.out else []), env={**os.environ, "SK_PDL": "0"}, check=True)
    for B in (1, 64):
        bench_generate(B, 64, 256, a.out)


if __name__ == "__main__":
    main()
