"""Speech-LM evaluation (cli/eval.py's modelling metrics) on one GPU:

  1. end-to-end pairs/s of `B200SpeechLM.log_likelihood` over synthetic pair sets -- sBLIMP-like (1-4 s clips) and
     sStoryCloze-like (10-20 s clips) -- at batch_size 8 and 32, positives and negatives as separate batches as the metric
     runs them, with random-init mHuBERT-25Hz geometry and the cfg-2 LM (Qwen2.5-0.5B body, 502 units).  Audio is
     already on the device (file decoding is not timed).  The HuBERT + tokens, LM-forward and scoring shares come from
     CUDA events around each phase (per pass, averaged over 5 passes);
  2. `sk_seq_loglik` alone against the reference's torch formula (bf16 -inf fill, cross_entropy(reduction='none') on bf16,
     mask, bf16 sum, division) at V = 502 and V = 152,167, as bytes of logits read (B*T*V*2) per kernel time, against the
     3.35 TB/s HBM3 ceiling of the H100 SXM data sheet.

Prints the card name and power limit, one line per measurement and a final JSON line.

    python tools/eval_bench.py [--pairs 64] [--skip-e2e]
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
import torch.nn.functional as F  # noqa: E402

from slamkit_b200 import _lib as L  # noqa: E402
from slamkit_b200.lm import B200UnitLM, LMConfig  # noqa: E402

HBM_BPS = 3.35e12
DEV = "cuda:0"


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
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


def calibrated_ms(fn, window_ms=250.0):
    """Mean time of `fn` over a window of about `window_ms` (the count comes from one short probe)."""
    probe = events_ms(fn, 3)
    return events_ms(fn, max(3, int(window_ms / max(probe, 1e-3))))


def kernel_bench(V, B=8, T=512):
    lib = L.require_cuda()
    g = torch.Generator(device=DEV).manual_seed(0)
    ldl = (V + 127) // 128 * 128
    logits = (torch.randn(B * T, ldl, device=DEV, generator=g) * 2).to(torch.bfloat16)
    ids = torch.randint(2, V, (B, T), device=DEV, generator=g)
    ids[:, 0] = 1
    tok = torch.empty(B * (T - 1), device=DEV)
    ll = torch.empty(B, device=DEV, dtype=torch.bfloat16)

    def kern():
        L.check(lib.sk_seq_loglik(L.ptr(logits), ldl, V, L.ptr(ids), B, T, 0, None, 1, L.ptr(tok), L.ptr(ll),
                                  L.stream_ptr()))

    z = logits.view(B, T, ldl)[:, :, :V]

    def torch_formula():
        x = ids[:, 1:].clone()
        x[x == 0] = -100
        nll = F.cross_entropy(z[:, :-1].reshape(-1, V), x.reshape(-1), reduction="none").view(x.shape)
        mask = x.ne(-100)
        return -((nll * mask).sum(-1) / mask.sum(-1))

    kern()
    torch_formula()
    torch.cuda.synchronize()
    k_ms = calibrated_ms(kern)
    t_ms = calibrated_ms(torch_formula)
    read = B * T * V * 2
    r = {"V": V, "B": B, "T": T, "rows": B * (T - 1), "kernel_ms": round(k_ms, 4), "torch_ms": round(t_ms, 4),
         "kernel_TBps": round(read / k_ms / 1e9, 3), "kernel_frac_of_3.35TBps": round(read / (k_ms * 1e-3) / HBM_BPS, 3),
         "torch_TBps": round(read / t_ms / 1e9, 3)}
    print(f"sk_seq_loglik V={V} rows={B * (T - 1)}: {k_ms:.3f} ms = {r['kernel_TBps']} TB/s "
          f"({100 * r['kernel_frac_of_3.35TBps']:.1f} % of 3.35); torch formula {t_ms:.3f} ms ({r['torch_TBps']} TB/s)")
    return r


def synthetic_pairs(n, lo_s, hi_s, seed):
    g = torch.Generator().manual_seed(seed)
    out = []
    for _ in range(2 * n):
        k = int(torch.randint(int(lo_s * 16000), int(hi_s * 16000) + 1, (1,), generator=g))
        out.append(0.1 * torch.randn(k, generator=g))
    return out[0::2], out[1::2]


def pad(wavs):
    lens = torch.tensor([len(w) for w in wavs])
    x = torch.zeros(len(wavs), int(lens.max()))
    for i, w in enumerate(wavs):
        x[i, :len(w)] = w
    return x.to(DEV), lens.to(DEV)


def e2e_bench(name, pos, neg, bs, tok, lm, reps=5):
    """One untimed pass, then `reps` timed passes with events around tokens / forward / scoring of every batch."""
    batches = []
    for i in range(0, len(pos), bs):
        batches.append(pad(pos[i:i + bs]))
        batches.append(pad(neg[i:i + bs]))

    def run():
        evs = []
        for w, n in batches:
            e = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
            e[0].record()
            ids, _ = tok.tokenise_device(w, n)
            e[1].record()
            lm.forward(ids)
            e[2].record()
            lm.score_last_forward(ids, True)
            e[3].record()
            evs.append(e)
        torch.cuda.synchronize()
        return evs

    run()
    t0 = time.perf_counter()
    evs = [e for _ in range(reps) for e in run()]
    wall = (time.perf_counter() - t0) / reps
    hub = sum(e[0].elapsed_time(e[1]) for e in evs) / reps
    fwd = sum(e[1].elapsed_time(e[2]) for e in evs) / reps
    sc = sum(e[2].elapsed_time(e[3]) for e in evs) / reps
    tot = hub + fwd + sc
    r = {"set": name, "batch_size": bs, "pairs": len(pos), "pairs_per_s": round(len(pos) / wall, 1),
         "wall_s": round(wall, 4), "hubert_tokens_ms": round(hub, 2), "lm_forward_ms": round(fwd, 2),
         "scoring_ms": round(sc, 3), "shares": [round(x / tot, 4) for x in (hub, fwd, sc)]}
    print(f"{name} bs={bs}: {r['pairs_per_s']} pairs/s; device time HuBERT+tokens {hub:.1f} ms, LM forward {fwd:.1f} ms, "
          f"scoring {sc:.2f} ms (shares {r['shares']})")
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=64)
    ap.add_argument("--skip-e2e", action="store_true")
    a = ap.parse_args()
    torch.cuda.set_device(DEV)
    name, limit = card()
    print(f"card: {name}; power.limit: {limit}")
    res = {"card": name, "power_limit": limit, "kernel": [], "e2e": []}
    with torch.inference_mode():
        for V in (502, 152167):
            res["kernel"].append(kernel_bench(V))
            torch.cuda.empty_cache()
        if not a.skip_e2e:
            from slamkit_b200.feature_extractor import HubertB200Config, HubertB200FeatureExtractor, random_params
            from slamkit_b200.tokeniser import B200UnitTokeniser
            hc = HubertB200Config()
            fe = HubertB200FeatureExtractor(hc, random_params(hc, seed=0), device=DEV, max_batch=32, max_samples=16000 * 20)
            tok = B200UnitTokeniser(fe)
            lm = B200UnitLM(LMConfig(), device=DEV, max_batch=32, max_seq=512, trainable=False, seed=0)
            sets = {"sBLIMP-like 1-4 s": synthetic_pairs(a.pairs, 1, 4, 1),
                    "sSC-like 10-20 s": synthetic_pairs(a.pairs // 2, 10, 20, 2)}
            for nm, (pos, neg) in sets.items():
                for bs in (8, 32):
                    res["e2e"].append(e2e_bench(nm, pos, neg, bs, tok, lm))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
