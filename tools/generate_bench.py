"""Cached batched decoding (`B200UnitLM.generate`) on the cfg-2 shape (Qwen2.5-0.5B body, 502 units, seeded random
weights) with the generate metric's settings (config/metric/generate.yaml: temperature 0.8, top_k 25, 150 new tokens) after
a 75-token prompt (3 s of 25 Hz units).  For B in {1, 8, 64} it reports the prefill time, the decode-step time (eager and
replayed from a CUDA graph, device events after warm-up), end-to-end tokens/s of `generate`, and the graph step time
against its HBM bound (weight bytes + KV bytes read) / 3.35 TB/s; then a per-kernel split of one step (torch.profiler, a
separate run), the same rows for the cfg-4 text+unit vocabulary (152,167 ids), decode attention alone, and the
uncached per-row path the cached one replaced, timed at B=1 with 32 new tokens.  Prints one line per measurement and a
final JSON line.

    python tools/generate_bench.py [--batches 1,8,64] [--skip-cfg4]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch  # noqa: E402

from slamkit_b200 import _lib as L  # noqa: E402
from slamkit_b200.generation import generate_tokens  # noqa: E402
from slamkit_b200.lm import B200UnitLM, DecodeSession, LMConfig  # noqa: E402

HBM_BPS = 3.35e12          # H100 SXM data sheet, HBM3 (a ceiling, not a measured rate)
PROMPT, NEW = 75, 150


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=60).stdout.strip()
    except Exception as e:   # noqa: BLE001
        q = f"unavailable ({e})"
    return name, q


def events_ms(fn, n):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / n


def sampling_cfg(T_cache, seed=0):
    return L.SkSampling(seed=seed, top_p=1.0, temperature=0.8, do_sample=1, top_k=25, n_eos=0, pad_token_id=0,
                        max_length=T_cache)


def prompts(B, V, seed=0):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(2, min(V, 502), (B, PROMPT), generator=g) + (V - 502 if V > 502 else 0)


def kv_bytes_per_pos(c: LMConfig):
    return c.n_layers * 2 * c.n_kv_heads * c.head_dim * 2


def bench_batch(m: B200UnitLM, B: int):
    c = m.config
    T_cache = PROMPT + NEW
    ids = prompts(B, c.vocab_size)
    lens = torch.full((B,), PROMPT)
    cfg = sampling_cfg(T_cache)
    r = {"B": B}
    # prefill (+ first token selection)
    sess = DecodeSession(m, B, T_cache, NEW)

    def prefill():
        sess.step_ctr.zero_()
        sess.finished.zero_()
        sess.prefill(ids, lens)
        sess.select(cfg)
    prefill()
    torch.cuda.synchronize()
    r["prefill_ms"] = events_ms(prefill, 5)

    # eager steps over positions 75 .. 75+n-1 (the cache is refilled by a new prefill before each timed window)
    def step():
        sess.step()
        sess.select(cfg)
    n_eager = 64
    prefill()
    for _ in range(3):
        step()
    prefill()
    torch.cuda.synchronize()
    r["step_eager_ms"] = events_ms(step, n_eager)
    # graph replay over the same positions
    prefill()
    step()
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gr):
        step()
    prefill()
    torch.cuda.synchronize()
    r["step_graph_ms"] = events_ms(gr.replay, n_eager)
    mean_len = PROMPT + (n_eager + 1) / 2
    weight_b = m.n_params * 2
    kv_b = B * mean_len * kv_bytes_per_pos(c)
    bound_ms = (weight_b + kv_b) / HBM_BPS * 1e3
    r.update(weight_mb=weight_b / 1e6, kv_mb=kv_b / 1e6, hbm_bound_ms=bound_ms,
             hbm_bound_share_graph=bound_ms / r["step_graph_ms"])
    del gr
    # end to end: generate() as a user calls it (left-padded prompts, graph capture included)
    kw = dict(max_new_tokens=NEW, do_sample=True, temperature=0.8, top_k=25, eos_token_id=None)
    mask = torch.ones(B, PROMPT, dtype=torch.long)
    m.generate(ids, attention_mask=mask, **kw)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = m.generate(ids, attention_mask=mask, **kw)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    assert out.shape == (B, PROMPT + NEW)
    r["generate_s"] = dt
    r["tokens_per_s"] = B * NEW / dt
    return r, sess


def kernel_split(m: B200UnitLM, sess: DecodeSession, B: int, n=10):
    """Per-step device time by kernel family, from torch.profiler over n eager steps.  Runs in a process of its own with
    programmatic dependent launch off (SK_PDL=0): with it on, a kernel is resident while it waits for its predecessor and
    the trace would charge it that wait."""
    from torch.profiler import ProfilerActivity, profile
    cfg = sampling_cfg(sess.T_cache)
    sess.step_ctr.zero_()
    sess.finished.zero_()
    sess.prefill(prompts(B, m.config.vocab_size), torch.full((B,), PROMPT))
    sess.select(cfg)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(n):
            sess.step()
            sess.select(cfg)
        torch.cuda.synchronize()
    fam = {}
    for e in prof.key_averages():
        name = e.key
        t = getattr(e, "device_time_total", None)
        if t is None:
            t = e.cuda_time_total
        if t <= 0:
            continue
        if "gemm_wgmma" in name or "splitk_reduce" in name:
            k = "gemm"
        elif "attn_decode" in name:
            k = "decode_attention"
        elif "select_next" in name:
            k = "sampler"
        elif "rmsnorm" in name:
            k = "rmsnorm"
        elif "kv_append" in name:
            k = "kv_append"
        elif "embed" in name:
            k = "embed"
        else:
            k = "other"
        fam[k] = fam.get(k, 0.0) + t / 1e3 / n
    return {k: round(v, 4) for k, v in sorted(fam.items(), key=lambda kv: -kv[1])}


def attention_alone(B=64, H=14, KVH=2, n_pos=1024, T_cache=2048):
    lib = L.require_cuda()
    g = torch.Generator(device="cuda").manual_seed(0)
    k = torch.randn(B, KVH, T_cache, 64, device="cuda", generator=g).to(torch.bfloat16)
    v = torch.randn_like(k)
    q = torch.randn(B, H * 64, device="cuda", generator=g).to(torch.bfloat16)
    o = torch.empty_like(q)
    lens = torch.full((B,), n_pos, dtype=torch.int32, device="cuda")
    part = torch.empty(int(lib.sk_attn_decode_partial_bytes(B, H, T_cache)) // 4, device="cuda", dtype=torch.float32)

    def run():
        L.check(lib.sk_attn_decode(L.ptr(q), H * 64, L.ptr(k), L.ptr(v), L.ptr(lens), L.ptr(o), H * 64, L.ptr(part), B, H, KVH,
                                   T_cache, L.f32(0.125), L.stream_ptr()))
    for _ in range(10):
        run()
    torch.cuda.synchronize()
    ms = events_ms(run, 200)
    byts = 2 * B * KVH * n_pos * 64 * 2
    return {"B": B, "H": H, "KVH": KVH, "cached_positions": n_pos, "us": ms * 1e3, "gb_s": byts / ms / 1e6,
            "hbm_share": byts / (ms * 1e-3) / HBM_BPS}


def uncached_path(m: B200UnitLM, n_new=32):
    """The previous generate body: one row at a time, a full forward over the prefix for every token, selection on the CPU."""
    V = m.config.vocab_size
    ids = prompts(1, V)

    def next_logits(x):
        return m.forward(x).logits[0, -1, :V].float().cpu()
    kw = dict(max_new_tokens=n_new, do_sample=True, temperature=0.8, top_k=25, eos_token_id=None,
              max_positions=m.config.max_positions)
    generate_tokens(next_logits, ids, **dict(kw, max_new_tokens=4))
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    generate_tokens(next_logits, ids, **kw)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    return {"B": 1, "new_tokens": n_new, "s": dt, "ms_per_token": dt / n_new * 1e3, "tokens_per_s": n_new / dt}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="1,8,64")
    ap.add_argument("--skip-cfg4", action="store_true")
    ap.add_argument("--profile-vocab", type=int, default=0, help=argparse.SUPPRESS)   # internal: the profiler run
    a = ap.parse_args()
    batches = [int(x) for x in a.batches.split(",")]
    L.require_cuda()
    if a.profile_vocab:
        m = B200UnitLM(LMConfig(vocab_size=a.profile_vocab), device="cuda:0", max_batch=max(batches), max_seq=PROMPT,
                       trainable=False, seed=0)
        print(json.dumps({B: kernel_split(m, DecodeSession(m, B, PROMPT + NEW, NEW), B) for B in batches}))
        return
    name, limits = card()
    print(f"card: {name}; power.limit, clocks.max.sm: {limits}")
    res = {"card": name, "power_limit_and_max_sm_clock": limits, "cfg2": [], "cfg4": []}
    for tag, V in (("cfg2", 502), ("cfg4", 152167)):
        if tag == "cfg4" and a.skip_cfg4:
            continue
        q = subprocess.run([sys.executable, os.path.abspath(__file__), "--profile-vocab", str(V), "--batches", a.batches],
                           capture_output=True, text=True, env=dict(os.environ, SK_PDL="0"), check=True)
        prof = json.loads(q.stdout.strip().splitlines()[-1])
        m = B200UnitLM(LMConfig(vocab_size=V), device="cuda:0", max_batch=max(batches), max_seq=PROMPT, trainable=False,
                       seed=0)
        for B in batches:
            r, sess = bench_batch(m, B)
            del sess
            r["kernels_ms_per_step"] = prof[str(B)]
            res[tag].append(r)
            print(f"{tag} B={B}: prefill {r['prefill_ms']:.3f} ms; step eager {r['step_eager_ms']:.3f} ms, graph "
                  f"{r['step_graph_ms']:.3f} ms; HBM bound {r['hbm_bound_ms']:.3f} ms ({r['weight_mb']:.1f} MB weights + "
                  f"{r['kv_mb']:.1f} MB KV) = {100 * r['hbm_bound_share_graph']:.1f} % of the graph step; generate "
                  f"{NEW} tokens: {r['generate_s']:.3f} s = {r['tokens_per_s']:.0f} tokens/s; per-kernel ms/step (eager, no PDL) "
                  f"{r['kernels_ms_per_step']}")
            torch.cuda.empty_cache()
        if tag == "cfg2":
            u = uncached_path(m)
            res["uncached_b1"] = u
            print(f"uncached per-row path (previous generate), B=1, {u['new_tokens']} new tokens: {u['ms_per_token']:.2f} ms/token "
                  f"= {u['tokens_per_s']:.1f} tokens/s; rows run one after another, so B rows x {NEW} tokens cost about "
                  f"B x {NEW} x {u['ms_per_token']:.2f} ms (scaled, not run)")
        del m
        torch.cuda.empty_cache()
    att = attention_alone()
    res["decode_attention"] = att
    print(f"decode attention alone B={att['B']} {att['H']}:{att['KVH']} heads, {att['cached_positions']} cached positions: "
          f"{att['us']:.1f} us, {att['gb_s']:.0f} GB/s = {100 * att['hbm_share']:.1f} % of 3.35 TB/s")
    print(json.dumps(res))


if __name__ == "__main__":
    main()
