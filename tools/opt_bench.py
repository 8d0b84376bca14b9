"""OPT decoder on the GPU path: train-step throughput at facebook/opt-125m geometry with the 502-unit vocabulary, its
device-time split (GEMM / attention / LayerNorm / other, from torch.profiler kernel names in a separate profiled step),
the model-FLOP rate against 989 TFLOP/s dense bf16, HF OPTForCausalLM (bf16 autocast, sdpa, fused AdamW) on the same
batches and card, and cached greedy generate at B = 1 and 64.  Prints one JSON line per measurement, the card's name
and power limit first.

    python tools/opt_bench.py [--steps 20] [--warmup 5] [--out results.jsonl]
    python tools/opt_bench.py --master [--steps 20] [--warmup 5] [--rounds 3]
    python tools/opt_bench.py --geometry opt-350m [--steps 20] [--warmup 5]

--geometry opt-350m runs the same train / HF / split / generate measurements on the post-LayerNorm facebook/opt-350m
geometry (hidden 1024, 24 layers, 16 heads, ffn 4096, project_in / project_out to a 512-wide tied head).

--master times bf16 parameters against fp32 master weights (the reference's default recipe: fp32 parameters,
gradients and AdamW moments under bf16 autocast) on the same batches, alternating the two in rounds, and reports each
mode's median step; then each mode's kernel split with the master-weight element-wise kernels and the optimiser named.

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

from oracle import opt_oracle, opt_postln_oracle  # noqa: E402
from slamkit_b200.lm import B200AdamW, B200UnitLM, OptLMConfig, OptPostLnLMConfig  # noqa: E402

PEAK_BF16 = 989e12
DEV = "cuda:0"
# per geometry: the model's config, the oracle config whose FLOPs are counted, the HF OPTConfig fields, the record prefix
GEOMETRIES = {
    "opt-125m": (OptLMConfig, opt_oracle.OracleOptConfig, opt_oracle.flops_per_token, {}, "opt125m"),
    "opt-350m": (OptPostLnLMConfig, lambda: opt_postln_oracle.OraclePostLnConfig(hidden=1024, n_layers=24, n_heads=16,
                                                                                  ffn=4096, proj_dim=512),
                 opt_postln_oracle.flops_per_token,
                 dict(hidden_size=1024, num_hidden_layers=24, num_attention_heads=16, ffn_dim=4096, word_embed_proj_dim=512,
                      do_layer_norm_before=False), "opt350m"),
}
GEOM = GEOMETRIES["opt-125m"]


def OptConfig():
    return GEOM[0]()


def flops_per_token(T):
    return GEOM[2](GEOM[1](), T)


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


SPLIT = (("gemm", ("gemm", "splitk")), ("attention", ("attn",)), ("layernorm", ("layernorm",)), ("relu_bwd", ("relu_bwd",)))
# the master-weight element-wise kernels and the optimiser by name (checked in this order, before SPLIT's classes)
SPLIT_MASTER = (("add_layernorm_f32", ("add_layernorm_f32",)), ("layernorm_bwd_f32", ("layernorm_bwd_f32",)),
                ("widen_grads", ("widen_grads",)), ("adamw", ("adamw",)), ("grad_norm", ("sumsq", "gradnorm")),
                ("embedding_fwd_bwd", ("embed", "scatter", "add_fix"))) + SPLIT


def split(step, classes=SPLIT):
    """Device time of one step by kernel class, from a profiled step.  Run in a process of its own with SK_PDL=0: with
    programmatic dependent launch a kernel starts while its predecessor drains and waits inside, so kernel spans
    overlap and would not add up to the step."""
    from torch.profiler import ProfilerActivity, profile
    step()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        step()
        torch.cuda.synchronize()
    out = {name: 0.0 for name, _ in classes}
    out["other"] = 0.0
    for e in prof.key_averages():
        us = getattr(e, "self_device_time_total", None)
        if us is None:
            us = e.self_cuda_time_total
        if us <= 0 or e.key.startswith("cuda") or e.key.startswith("Memset") or e.key.startswith("Memcpy"):
            continue
        k = e.key.lower()
        cat = next((name for name, keys in classes if any(x in k for x in keys)), "other")
        out[cat] += us / 1e3
    out["total"] = sum(out.values())
    return {k: round(v, 3) for k, v in out.items()}


def bench_train(B, T, steps, warmup, out):
    cfg = OptConfig()
    m = B200UnitLM(cfg, device=DEV, max_batch=B, max_seq=T, seed=0)
    opt = B200AdamW(m, lr=1e-4, max_grad_norm=0.5)
    ids, labels = batch(B, T, T)
    n = float(B * T)

    def step():
        m.forward_backward(ids, labels, num_items_in_batch=n)
        opt.step()
    ms = time_steps(step, steps, warmup)
    toks = B * T / (ms / 1e3)
    fl = flops_per_token(T) * toks
    rec = {"what": f"{GEOM[4]}_train_step", "impl": "sk", "B": B, "T": T, "ms": round(ms, 3), "tokens_per_s": round(toks),
           "model_tflops": round(fl / 1e12, 1), "mfu_vs_989": round(fl / PEAK_BF16, 4), "loss": float(m.stats[0])}
    if os.environ.get("SK_PDL") == "0":
        rec = {"what": f"{GEOM[4]}_train_step_split", "impl": "sk_no_pdl", "B": B, "T": T, "ms": round(ms, 3),
               "kernel_ms": split(step)}
    emit(rec, out)
    del m, opt
    torch.cuda.empty_cache()
    return rec


def bench_master(B, T, steps, warmup, rounds, out, profile_only=False):
    """bf16 parameters against fp32 master weights at opt-125m geometry: both models on the same batch, timed in
    alternating rounds (each round: `warmup` untimed steps, then `steps` steps timed one by one with device events), the
    median step of each mode over all rounds."""
    import statistics
    ids, labels = batch(B, T, T)
    n = float(B * T)
    models = {}
    for mode in ("bf16", "master"):
        m = B200UnitLM(OptLMConfig(), device=DEV, max_batch=B, max_seq=T, seed=0, master_weights=mode == "master")
        models[mode] = (m, B200AdamW(m, lr=1e-4, max_grad_norm=0.5))

    def stepper(mode):
        m, opt = models[mode]

        def step():
            m.forward_backward(ids, labels, num_items_in_batch=n)
            opt.step()
        return step
    if profile_only:
        for mode in models:
            emit({"what": "opt125m_train_step_split", "impl": f"sk_{mode}_no_pdl", "B": B, "T": T,
                  "kernel_ms": split(stepper(mode), SPLIT_MASTER)}, out)
    else:
        times = {mode: [] for mode in models}
        for _ in range(rounds):
            for mode in models:
                step = stepper(mode)
                for _ in range(warmup):
                    step()
                ev = [torch.cuda.Event(enable_timing=True) for _ in range(steps + 1)]
                ev[0].record()
                for i in range(steps):
                    step()
                    ev[i + 1].record()
                torch.cuda.synchronize()
                times[mode] += [ev[i].elapsed_time(ev[i + 1]) for i in range(steps)]
        med = {mode: statistics.median(t) for mode, t in times.items()}
        for mode, t in times.items():
            emit({"what": "opt125m_train_step", "impl": f"sk_{mode}", "B": B, "T": T, "median_ms": round(med[mode], 3),
                  "min_ms": round(min(t), 3), "max_ms": round(max(t), 3), "steps_timed": len(t),
                  "loss": float(models[mode][0].stats[0])}, out)
        emit({"what": "opt125m_master_overhead", "B": B, "T": T,
              "master_over_bf16": round(med["master"] / med["bf16"] - 1.0, 4)}, out)
    del models
    torch.cuda.empty_cache()


def bench_hf(B, T, steps, warmup, out):
    from transformers import OPTConfig, OPTForCausalLM
    torch.manual_seed(0)
    hf = OPTForCausalLM(OPTConfig(vocab_size=502, dropout=0.0, attention_dropout=0.0, layerdrop=0.0, pad_token_id=0,
                                  bos_token_id=1, eos_token_id=1, attn_implementation="sdpa", **GEOM[3])).to(DEV).train()
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
    fl = flops_per_token(T) * toks
    emit({"what": f"{GEOM[4]}_train_step", "impl": "hf_sdpa_autocast_bf16", "B": B, "T": T, "ms": round(ms, 3),
          "tokens_per_s": round(toks), "model_tflops": round(fl / 1e12, 1), "mfu_vs_989": round(fl / PEAK_BF16, 4)}, out)
    del hf, opt
    torch.cuda.empty_cache()


def bench_generate(B, prompt, new, out):
    m = B200UnitLM(OptConfig(), device=DEV, max_batch=B, max_seq=prompt, trainable=False, seed=0)
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
    emit({"what": f"{GEOM[4]}_generate", "impl": "sk", "B": B, "prompt": prompt, "new_tokens": new, "s": round(s, 4),
          "new_tokens_per_s": round(B * new / s), "ms_per_step": round(s / new * 1e3, 3)}, out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=None)
    ap.add_argument("--split-only", action="store_true", help=argparse.SUPPRESS)
    ap.add_argument("--master", action="store_true", help="bf16 parameters vs fp32 master weights, alternating")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--geometry", choices=sorted(GEOMETRIES), default="opt-125m")
    a = ap.parse_args()
    global GEOM
    GEOM = GEOMETRIES[a.geometry]
    if a.master and a.geometry != "opt-125m":
        raise SystemExit("--master measures the pre-LayerNorm opt-125m geometry only (post-LN OPT trains bf16 parameters)")
    if a.master and a.split_only:
        for T in (512, 1024):
            bench_master(8, T, a.steps, a.warmup, 1, a.out, profile_only=True)
        return
    if a.master:
        if not torch.cuda.is_available():
            raise SystemExit("opt_bench needs a CUDA device: there is nothing to measure on the CPU")
        emit({"what": "card", "name_power_limit_max_sm_clock": card()}, a.out)
        for T in (512, 1024):
            bench_master(8, T, a.steps, a.warmup, a.rounds, a.out)
        subprocess.run([sys.executable, os.path.abspath(__file__), "--master", "--split-only"] + (["--out", a.out] if a.out else []),
                       env={**os.environ, "SK_PDL": "0"}, check=True)
        return
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
    subprocess.run([sys.executable, os.path.abspath(__file__), "--split-only", "--steps", "3", "--warmup", "2",
                    "--geometry", a.geometry] +
                   (["--out", a.out] if a.out else []), env={**os.environ, "SK_PDL": "0"}, check=True)
    for B in (1, 64):
        bench_generate(B, 64, 256, a.out)


if __name__ == "__main__":
    main()
