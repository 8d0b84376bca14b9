"""bf16 vs fp32 OPT inference at the opt-125m geometry (502-unit vocabulary), in one process, alternating the two models:
the scoring forward (`sequence_log_likelihood`) at [32, 256] and [8, 1024], and cached greedy `generate` at B = 1 and 64.
Both models carry the same seeded fp32 weights (the bf16 one rounded).  Prints the card name and power limit first, then
one JSON line per measurement (median over rounds of CUDA-event times).

    python tools/opt_fp32_bench.py [--rounds 5] [--out results.jsonl] [--geometry opt-350m]

--geometry opt-350m: the post-LayerNorm facebook/opt-350m geometry (hidden 1024, 24 layers, project_in / project_out to
a 512-wide tied head) instead.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() or "unknown"


def emit(rec, out):
    line = json.dumps(rec)
    print(line, flush=True)
    if out:
        with open(out, "a") as f:
            f.write(line + "\n")


def timed(fn, reps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def main():
    from oracle import opt_oracle as O
    from oracle import opt_postln_oracle as OP
    from slamkit_b200.lm import B200UnitLM, OptLMConfig, OptPostLnLMConfig
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    ap.add_argument("--geometry", choices=("opt-125m", "opt-350m"), default="opt-125m")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("opt_fp32_bench needs a CUDA device")
    emit({"what": "card", "name_power_limit_max_sm_clock": card()}, a.out)
    if a.geometry == "opt-350m":
        c = OP.OraclePostLnConfig(hidden=1024, n_layers=24, n_heads=16, ffn=4096, proj_dim=512)
        p = OP.init_params(c, seed=0, dtype=torch.float32)
        lc = OptPostLnLMConfig()
    else:
        c = O.OracleOptConfig()
        p = O.init_params(c, seed=0, dtype=torch.float32)
        lc = OptLMConfig()
    models = {}
    for mode in ("bf16", "fp32"):
        # sized for 8192 rows (both scoring shapes); the workspace grows on demand.  A [64, 1024] bf16 workspace would
        # take ~40 GB at the opt-350m geometry
        m = B200UnitLM(lc, device="cuda:0", max_batch=32, max_seq=256, trainable=False, fp32_inference=mode == "fp32")
        m.load_hf_state_dict(p)
        models[mode] = m
    g = torch.Generator().manual_seed(1)
    for B, T in ((32, 256), (8, 1024)):
        ids = torch.randint(2, 502, (B, T), generator=g).cuda()
        ids[:, 0] = 1
        ms = {k: [] for k in models}
        for r in range(a.rounds + 1):
            for mode, m in models.items():
                t = timed(lambda: m.sequence_log_likelihood(ids, mean_nll=True), 10)
                if r:
                    ms[mode].append(t)
        rec = {"what": "score", "geometry": a.geometry, "B": B, "T": T}
        rec.update({f"{k}_ms": round(statistics.median(v), 3) for k, v in ms.items()})
        rec["fp32_over_bf16"] = round(rec["fp32_ms"] / rec["bf16_ms"], 3)
        emit(rec, a.out)
    prompt_len, new = 32, 128
    for B in (1, 64):
        prompt = torch.randint(2, 502, (B, prompt_len), generator=g)
        prompt[:, 0] = 1
        ms = {k: [] for k in models}
        for r in range(a.rounds + 1):
            for mode, m in models.items():
                t = timed(lambda: m.generate(prompt, max_new_tokens=new, do_sample=False, eos_token_id=[]), 1)
                if r:
                    ms[mode].append(t)
        rec = {"what": "generate", "geometry": a.geometry, "B": B, "prompt": prompt_len, "new_tokens": new}
        rec.update({f"{k}_ms": round(statistics.median(v), 3) for k, v in ms.items()})
        rec["fp32_over_bf16"] = round(rec["fp32_ms"] / rec["bf16_ms"], 3)
        emit(rec, a.out)


if __name__ == "__main__":
    main()
