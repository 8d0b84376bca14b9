"""Cost of the history-dependent generation rules and of the prompt fan-out of num_return_sequences, on a Qwen2 decoder
at the SLAM geometry (hidden 896, 24 layers, 14 / 2 heads; random weights).

  * decode step (sk_lm_decode_step + token selection) with rules off and on (repetition_penalty 1.3,
    no_repeat_ngram_size 3, min_new_tokens past the step), greedy and sampled, at B = 1 / 64 and V = 502 / 152,167, with a
    256-token history; CUDA events over 200 steps replayed as one captured CUDA graph, median of 5 rounds;
  * prefill of B = 8 prompts of 256 tokens fanned out to B*k rows (sk_lm_kv_fanout) against prefilling the expanded
    batch of B*k rows, at k = 4 / 8, median of 5 rounds.

Prints one JSON line per measurement, preceded by the card's name and power limit."""
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from slamkit_b200 import _lib as L  # noqa: E402
from slamkit_b200.lm import B200UnitLM, DecodeSession, LMConfig  # noqa: E402

DEV = "cuda:0"
T, STEPS, ROUNDS = 256, 200, 5


def _model(V, max_batch):
    return B200UnitLM(LMConfig(vocab_size=V), device=DEV, max_batch=max_batch, max_seq=T, trainable=False, seed=0)


def _time(fn, n):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(n):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / n


def decode_step(m, B, rules, do_sample):
    V = m.config.vocab_size
    g = torch.Generator().manual_seed(B)
    ids = torch.randint(0, min(V, 502), (B, T), generator=g)
    sess = DecodeSession(m, B, T + STEPS + 8, STEPS + 8)
    if rules:
        sess.set_rules(ids, penalty=1.3, ngram=3, min_step=STEPS + 8)
    cfg = L.SkSampling(seed=1, top_p=0.95 if do_sample else 1.0, temperature=0.8, do_sample=int(do_sample),
                       top_k=25 if do_sample else 0, n_eos=1, pad_token_id=0, max_length=1 << 30)
    cfg.eos[0] = 1
    sess.prefill(ids, torch.full((B,), T))
    sess.select(cfg)
    sess.step()
    sess.select(cfg)
    gr, side = torch.cuda.CUDAGraph(), torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        gr.capture_begin()
        sess.step()
        sess.select(cfg)
        gr.capture_end()
    torch.cuda.current_stream().wait_stream(side)
    state = [t.clone() for t in (sess.tokens, sess.pos, sess.step_ctr)]
    ms = []
    for _ in range(ROUNDS):
        for t, t0 in zip((sess.tokens, sess.pos, sess.step_ctr), state):
            t.copy_(t0)                            # every round decodes the same steps
        ms.append(_time(gr.replay, STEPS))
    return statistics.median(ms)


def prefill(m, B, k, fanout):
    g = torch.Generator().manual_seed(k)
    ids = torch.randint(2, 502, (B, T), generator=g)
    lens = torch.full((B,), T)

    def run():
        sess = DecodeSession(m, B * k, T + 8, 8)
        if fanout:
            sess.prefill(ids, lens, k)
        else:
            sess.prefill(ids.repeat_interleave(k, 0), lens.repeat_interleave(k))
    run()
    torch.cuda.synchronize()
    return statistics.median(_time(run, 3) for _ in range(ROUNDS))


def main():
    L.require_cuda()
    info = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    print(json.dumps({"gpu": info}))
    with torch.inference_mode():
        for V in (502, 152167):
            m = _model(V, 64)
            for B in (1, 64):
                for do_sample in (False, True):
                    off = decode_step(m, B, False, do_sample)
                    on = decode_step(m, B, True, do_sample)
                    print(json.dumps({"bench": "decode_step", "V": V, "B": B, "do_sample": do_sample, "history": T,
                                      "rules_off_ms": round(off, 4), "rules_on_ms": round(on, 4),
                                      "overhead_pct": round(100 * (on / off - 1), 1)}), flush=True)
            del m
            torch.cuda.empty_cache()
        m = _model(502, 64)
        for k in (4, 8):
            fan = prefill(m, 8, k, True)
            full = prefill(m, 8, k, False)
            print(json.dumps({"bench": "prefill", "B": 8, "k": k, "T": T, "fanout_ms": round(fan, 3),
                              "expanded_ms": round(full, 3), "speedup": round(full / fan, 2)}), flush=True)


if __name__ == "__main__":
    main()
