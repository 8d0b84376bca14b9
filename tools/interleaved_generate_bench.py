"""Speech continuation with an interleaved speech-text model: `B200UnitLM.generate` on the cfg-2 body (Qwen2.5-0.5B
shape, seeded random weights) with the 152,167-id text+unit vocabulary, 75-token prompts and 150 new tokens sampled as
config/metric/generate.yaml does (temperature 0.8, top_k 25).  For B in {1, 8, 64} it times three calls, alternating,
median of 5 rounds: the compact head (`allowed_token_ids` = the 500 units + bos / eos), the same continuation through
`bad_words_ids` (the full 152 k head every step) and the 502-id unit model as the floor.  Every generated row runs all
150 steps (no eos), so the per-step call time is the call time / 150; for the full path it includes turning the
151,665-entry ban list into a bitmask on the host once per call.  The device step alone (decode step + selection
replayed from a CUDA graph, CUDA events over 140 replays) is timed as well, with the ban bitmask built beforehand.
Prints the card and its power limit, one line per B and a final JSON line.

    python tools/interleaved_generate_bench.py [--batches 1,8,64] [--rounds 5]
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
from slamkit_b200.generation import ban_bitmask  # noqa: E402
from slamkit_b200.lm import B200UnitLM, DecodeSession, LMConfig  # noqa: E402

PROMPT, NEW = 75, 150
V_INTER, V_UNIT = 152167, 502


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=60).stdout.strip()
    except Exception as e:   # noqa: BLE001
        q = f"unavailable ({e})"
    return name, q


def model(V, max_batch):
    cfg = LMConfig(vocab_size=V, hidden=896, n_layers=24, n_heads=14, n_kv_heads=2, head_dim=64, ffn=4864,
                   max_positions=PROMPT + NEW + 8)
    m = B200UnitLM(cfg, device="cuda:0", max_batch=max_batch, max_seq=PROMPT, trainable=False)
    m.init_weights(0, std=0.02)
    return m


def timed(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t, out


def graph_step_ms(m, ids, allowed=None, banned=None, reps=NEW):
    """Device time of one decode step + sampled selection, replayed from a CUDA graph (prompt prefilled first)."""
    B, T = ids.shape
    sess = DecodeSession(m, B, T + reps + 8, reps + 8, 0, allowed)
    ban = ban_bitmask(banned, m.config.vocab_size).to(m.device) if banned else None
    cfg = L.SkSampling(seed=1, top_p=1.0, temperature=0.8, do_sample=1, top_k=25, n_eos=0, pad_token_id=0,
                       max_length=T + reps + 8)
    sess.prefill(ids, torch.full((B,), T))
    sess.select(cfg, ban)

    def step():
        sess.step()
        sess.select(cfg, ban)
    step()
    g, side = torch.cuda.CUDAGraph(), torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        g.capture_begin()
        step()
        g.capture_end()
    torch.cuda.current_stream().wait_stream(side)
    for _ in range(5):
        g.replay()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps - 10):
        g.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / (reps - 10)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="1,8,64")
    ap.add_argument("--rounds", type=int, default=5)
    a = ap.parse_args()
    batches = [int(b) for b in a.batches.split(",")]
    name, power = card()
    print(f"card: {name}; power.limit, clocks.max.sm: {power}", flush=True)
    inter, unit = model(V_INTER, max(batches)), model(V_UNIT, max(batches))
    allowed = [0, 1] + list(range(V_INTER - 502, V_INTER - 2))        # bos / eos + the 500 units
    keep = set(allowed)
    bad = [[i] for i in range(V_INTER) if i not in keep]
    kw = dict(max_new_tokens=NEW, do_sample=True, temperature=0.8, top_k=25, eos_token_id=None, pad_token_id=0)
    rows = []
    for B in batches:
        g = torch.Generator().manual_seed(B)
        ids_i = torch.randint(V_INTER - 500, V_INTER - 2, (B, PROMPT), generator=g)
        ids_u = torch.randint(2, V_UNIT, (B, PROMPT), generator=g)
        calls = {
            "compact": lambda: inter.generate(ids_i, allowed_token_ids=allowed, generator=torch.Generator().manual_seed(1),
                                              **kw),
            "full": lambda: inter.generate(ids_i, bad_words_ids=bad, generator=torch.Generator().manual_seed(1), **kw),
            "unit502": lambda: unit.generate(ids_u, generator=torch.Generator().manual_seed(1), **kw),
        }
        outs = {k: f() for k, f in calls.items()}                         # warm-up (and the outputs compared below)
        same = bool(torch.equal(outs["compact"], outs["full"]))
        times = {k: [] for k in calls}
        for _ in range(a.rounds):
            for k, f in calls.items():
                times[k].append(timed(f)[0])
        med = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
        dev = {"compact": graph_step_ms(inter, ids_i, allowed=torch.tensor(allowed)),
               "full": graph_step_ms(inter, ids_i, banned=[b[0] for b in bad]),
               "unit502": graph_step_ms(unit, ids_u)}
        row = {"B": B, **{f"{k}_ms_per_step": round(1e3 * v / NEW, 3) for k, v in med.items()},
               **{f"{k}_graph_step_ms": round(v, 3) for k, v in dev.items()}, "compact_equals_full": same}
        rows.append(row)
        print(" ".join(f"{k}={v}" for k, v in row.items()), flush=True)
    print(json.dumps({"card": name, "power": power, "prompt": PROMPT, "new_tokens": NEW, "rows": rows}))


if __name__ == "__main__":
    main()
