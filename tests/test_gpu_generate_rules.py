"""GPU tests of the history-dependent generation rules (`sk_select_next_ex`, `sk_presence_init`) and the prompt KV fan-out
of num_return_sequences (`sk_lm_kv_fanout`): exact tokens on constructed rows against slamkit_b200.generation's CPU rules,
the device history and presence bitmap after several steps, `generate` with each key on every decoder against
`generate_tokens` driven by the same model's per-step logits, the fan-out's cache rows and group behaviour, and the
`generate` metric of cli/eval.py with several continuations per prompt."""
import ctypes as C

import pytest
import torch

from decode_ref import FILL, expected_token, spread
from slamkit_b200 import generation as G

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _lib():
    from slamkit_b200 import _lib as L
    return L, L.require_cuda()


# ---------------------------------------------------------------------------------------------- 1. exact selection
class Sel:
    """One selection launch over given rows: logits fp32 [B, V] (bf16 values), the padded prompts plus `step` generated
    tokens as history, and the decode state with the step index set to `step`."""

    def __init__(self, logits, prompts, gen, step, dtype, penalty=1.0, ngram=0, min_step=0, eos=(), do_sample=False,
                 temperature=1.0, top_k=0, top_p=1.0, uniforms=None, max_new=8):
        L, lib = _lib()
        B, V = logits.shape
        T = prompts.shape[1]
        ldl = (V + 63) // 64 * 64 + 64
        dl = torch.full((B, ldl), float("nan"), dtype=dtype)           # NaN guard columns past V
        dl[:, :V] = logits.to(dtype)
        self.dl = dl.to(DEV)
        hist = torch.full((B, T + max_new), -7, dtype=torch.long)
        hist[:, :T] = prompts
        if step:
            hist[:, T:T + step] = gen
        self.hist = hist.to(DEV)
        W = (V + 31) // 32
        self.pres = torch.empty(B, W, dtype=torch.int32, device=DEV)
        self.scratch = torch.empty(B, W, dtype=torch.int32, device=DEV)
        self.rules = L.SkLogitRules(self.hist.data_ptr(), self.pres.data_ptr(), self.scratch.data_ptr(), float(penalty),
                                    int(ngram), int(min_step), T, T + max_new, 0)
        L.check(lib.sk_presence_init(L.ptr(self.hist), T + max_new, T + step, B, V, L.ptr(self.pres), L.stream_ptr()))
        self.cfg = L.SkSampling(seed=5, top_p=float(top_p), temperature=float(temperature), do_sample=int(do_sample),
                                top_k=int(top_k), n_eos=len(eos), pad_token_id=0, max_length=1 << 30)
        for i, e in enumerate(eos):
            self.cfg.eos[i] = e
        z = lambda: torch.zeros(B, dtype=torch.int32, device=DEV)
        self.pos, self.fin, self.ngen = z(), z(), z()
        self.tokens = torch.zeros(B, dtype=torch.long, device=DEV)
        self.out = torch.full((B, max_new), -1, dtype=torch.long, device=DEV)
        self.step = torch.tensor([step, 0], dtype=torch.int32, device=DEV)
        self.state = L.SkDecodeState(self.tokens.data_ptr(), self.pos.data_ptr(), self.fin.data_ptr(), self.ngen.data_ptr(),
                                     self.out.data_ptr(), self.step.data_ptr(), max_new, 0)
        self.ud = uniforms.to(DEV) if uniforms is not None else None
        self.L, self.lib, self.V, self.B, self.ldl, self.dtype = L, lib, V, B, ldl, dtype

    def run(self):
        fn = self.lib.sk_select_next_ex_f32 if self.dtype == torch.float32 else self.lib.sk_select_next_ex
        self.L.check(fn(self.L.ptr(self.dl), self.ldl, self.V, self.B, None, C.byref(self.cfg), self.L.ptr(self.ud),
                        C.byref(self.state), C.byref(self.rules), self.L.stream_ptr()))
        torch.cuda.synchronize()
        return self


def _expected(logits, history, T, do_sample, temperature=1.0, top_k=0, top_p=1.0, u=0.5, **rules):
    s = G.apply_rules(logits.float().clone(), history=history, prompt_len=T, **rules)
    return expected_token(s, do_sample, temperature, top_k or None, top_p if top_p < 1.0 else None, [], u)


VOCABS = [2, 37, 502, 8193, 152167]


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("V", VOCABS)
def test_constructed_rows_exact(V, dtype):
    """Each case is built so that its rule decides the token; the expected token comes from the CPU rules with no
    tolerance (power-of-two penalties and temperatures on bf16 values, equal kept scores, u on exact CDF steps)."""
    ids = spread(V, min(V, 4))
    a, b = ids[0], ids[-1]
    T = 4
    cases = []
    # penalty 2 halves a present positive maximum below an absent one; a present negative score doubles
    x = torch.full((V,), FILL)
    x[a], x[b] = 4.0, 3.0
    cases.append((x, [a, a, a, a], [], dict(repetition_penalty=2.0), False, {}))
    x = torch.full((V,), FILL)
    x[a], x[b] = -1.0, -1.5
    cases.append((x, [a] * 4, [], dict(repetition_penalty=2.0), False, {}))
    # penalty 0.5 doubles a present score; temperature 2 then makes it equal to the absent maximum: u = 0.25 of two
    # equal scores picks the lower id
    x = torch.full((V,), FILL)
    x[a], x[b] = 1.0, 2.0
    cases.append((x, [a] * 4, [], dict(repetition_penalty=0.5), True, dict(temperature=2.0, u=0.25)))
    cases.append((x, [a] * 4, [], dict(repetition_penalty=0.5), True, dict(temperature=2.0, u=0.75)))
    # forced n-gram bans: history (a, b, a) -> a was followed by b: b banned at n = 2; at n = 1 every present id
    x = torch.full((V,), FILL)
    x[b], x[a] = 5.0, 1.0
    for n in (1, 2, 3):
        cases.append((x, [a, b, a, b], [a], dict(no_repeat_ngram_size=n), False, {}))
    # eos masked until the bound: step 2 with min_new_tokens 2 / 3
    x = torch.full((V,), FILL)
    x[b], x[a] = 5.0, 1.0
    for mn in (2, 3):
        cases.append((x, [a] * 4, [a, a], dict(eos=[b], min_new_tokens=mn), False, {}))
        cases.append((x, [a] * 4, [a, a], dict(eos=[b], min_new_tokens=mn), True, dict(top_k=1, u=0.5)))
    for logits, prompt, gen, rules, do_sample, samp in cases:
        if V == 2 and a == b:
            continue
        u = samp.get("u", 0.5)
        step = len(gen)
        eos = rules.get("eos", [])
        bound = G.min_step(T, None, rules.get("min_new_tokens"))
        s = Sel(logits[None], torch.tensor([prompt]), torch.tensor([gen], dtype=torch.long) if gen else None, step, dtype,
                penalty=rules.get("repetition_penalty", 1.0), ngram=rules.get("no_repeat_ngram_size", 0),
                min_step=bound, eos=eos, do_sample=do_sample, temperature=samp.get("temperature", 1.0),
                top_k=samp.get("top_k", 0), uniforms=torch.tensor([u])).run()
        want, _ = _expected(logits, prompt + gen, T, do_sample, samp.get("temperature", 1.0), samp.get("top_k", 0), 1.0, u,
                            **rules)
        got = int(s.out[0, step])
        assert got == want, (V, rules, samp, got, want)
        hist = s.hist[0].cpu()
        assert int(hist[T + step]) == got and int(s.tokens[0]) == got


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("V", [502, 152167])
@pytest.mark.parametrize("do_sample", [False, True])
def test_random_rows_and_device_state(V, dtype, do_sample):
    """48 rows over several steps with all rules on: every token equals the CPU rules at the given uniform (rows whose
    u lies within 1e-6 of a CDF step are skipped), and the history and presence bitmap equal a CPU recomputation."""
    B, T, steps = 48, 12, 6
    g = torch.Generator().manual_seed(V + int(do_sample))
    prompts = torch.randint(0, 40, (B, T), generator=g)
    prompts[:, :3] = 0                                                 # left pads
    rules = dict(repetition_penalty=1.5, no_repeat_ngram_size=2, eos=[3], min_new_tokens=3)
    s = Sel(torch.zeros(B, V), prompts, None, 0, dtype, penalty=1.5, ngram=2, min_step=3, eos=[3], do_sample=do_sample,
            temperature=0.7, top_k=30, top_p=0.95, uniforms=torch.zeros(B))
    gen = torch.zeros(B, 0, dtype=torch.long)
    fin = torch.zeros(B, dtype=torch.bool)
    skipped = 0
    for step in range(steps):
        logits = torch.randn(B, V, generator=g) * 3.0
        logits[:, :40] += 4.0                                         # keep the history ids in play
        logits = logits.to(torch.bfloat16).float()                    # values both entry points see exactly
        u = torch.rand(B, generator=g)
        s.dl[:, :V] = logits.to(dtype).to(DEV)
        s.ud.copy_(u.to(DEV))
        s.run()
        got = s.out[:, step].cpu()
        for r in range(B):
            if fin[r]:
                assert int(got[r]) == 0                               # finished rows append the pad id
                continue
            want, dist = _expected(logits[r], prompts[r].tolist() + gen[r].tolist(), T, do_sample, 0.7, 30, 0.95,
                                   float(u[r]), **rules)
            if do_sample and dist < 1e-6:
                skipped += 1
                continue
            assert int(got[r]) == want, (step, r, int(got[r]), want)
        fin |= got == 3
        gen = torch.cat([gen, got[:, None]], 1)
        full = torch.cat([prompts, gen], 1)
        assert torch.equal(s.hist[:, :T + step + 1].cpu(), full)
        bits = torch.zeros(B, (V + 31) // 32 * 32, dtype=torch.bool)
        bits.scatter_(1, full, True)
        words = (bits.view(B, -1, 32).long() << torch.arange(32)).sum(-1)
        assert torch.equal(s.pres.cpu().long() & 0xFFFFFFFF, words), step
    assert skipped <= 4


# ---------------------------------------------------------------------------------------------- 2. generate end to end
def _model(arch):
    from slamkit_b200.lm import B200UnitLM
    if arch == "qwen2":
        from oracle import lm_oracle as O
        from slamkit_b200.lm import LMConfig
        c = O.OracleLMConfig(vocab_size=502, hidden=128, n_layers=2, n_heads=2, n_kv_heads=1, head_dim=64, ffn=256)
        cfg = LMConfig(vocab_size=502, hidden=128, n_layers=2, n_heads=2, n_kv_heads=1, head_dim=64, ffn=256,
                       max_positions=256)
        p, kw = O.init_params(c, seed=3), {}
    elif arch in ("opt", "opt-fp32"):
        from oracle import opt_oracle as O
        from slamkit_b200.lm import OptLMConfig
        c = O.OracleOptConfig(vocab_size=502, hidden=128, n_layers=2, n_heads=2, ffn=256, max_positions=256)
        cfg = OptLMConfig(vocab_size=502, hidden=128, n_layers=2, n_heads=2, ffn=256, max_positions=256)
        fp32 = arch == "opt-fp32"
        p = O.init_params(c, seed=3, dtype=torch.float32 if fp32 else torch.bfloat16)
        kw = dict(fp32_inference=fp32)
    elif arch == "opt-postln":
        from oracle import opt_postln_oracle as O
        from slamkit_b200.lm import OptPostLnLMConfig
        c = O.OraclePostLnConfig(vocab_size=502, hidden=128, n_layers=2, n_heads=2, ffn=256, max_positions=256, proj_dim=64)
        cfg = OptPostLnLMConfig(vocab_size=502, hidden=128, n_layers=2, n_heads=2, ffn=256, max_positions=256, proj_dim=64)
        p, kw = O.init_params(c, seed=3), {}
    else:
        from oracle import neox_oracle as O
        from slamkit_b200.lm import NeoxLMConfig
        c = O.OracleNeoxConfig(vocab_size=502, hidden=128, n_layers=2, n_heads=2, ffn=256, max_positions=256)
        cfg = NeoxLMConfig(vocab_size=502, hidden=128, n_layers=2, n_heads=2, ffn=256, max_positions=256, rot_dims=c.rot_dims)
        p, kw = O.init_params(c, seed=3), {}
    m = B200UnitLM(cfg, device=DEV, max_batch=8, max_seq=64, trainable=False, **kw)
    m.load_hf_state_dict(p)
    return m


def _left_padded(lengths, T, V, seed):
    g = torch.Generator().manual_seed(seed)
    ids, mask = torch.zeros(len(lengths), T, dtype=torch.long), torch.zeros(len(lengths), T, dtype=torch.long)
    for r, n in enumerate(lengths):
        ids[r, T - n:], mask[r, T - n:] = torch.randint(2, 40, (n,), generator=g), 1   # small ids: many repeats
    return ids, mask


def _teacher_logits(m, ids, mask, out):
    """The per-step logits `generate` saw: a session of the same shape fed the generated tokens."""
    from slamkit_b200.lm import DecodeSession
    B, T = ids.shape
    lens = mask.sum(1)
    n_new = out.shape[1] - T
    right = torch.zeros(B, int(lens.max()), dtype=torch.long)
    for r in range(B):
        right[r, :int(lens[r])] = ids[r, T - int(lens[r]):]
    sess = DecodeSession(m, B, int(lens.max()) + n_new, n_new)
    table = {}
    lg = sess.prefill(right, lens)
    for s in range(n_new):
        for r in range(B):
            key = tuple(right[r, :int(lens[r])].tolist() + out[r, T:T + s].tolist())
            table[key] = lg[r].float().cpu()
        if s + 1 < n_new:
            lg = sess.step(out[:, T + s].to(DEV), (lens + s).to(torch.int32).to(DEV))
    return lambda x: table[tuple(x[0].tolist())]


ARCHS = ["qwen2", "opt", "opt-postln", "neox", "opt-fp32"]
KEYS = {
    "penalty": dict(repetition_penalty=1.6),
    "ngram2": dict(no_repeat_ngram_size=2),
    "ngram1-penalty0.7": dict(no_repeat_ngram_size=1, repetition_penalty=0.7),
    "min_new_tokens": dict(min_new_tokens=5),
    "min_length": dict(min_length=20),
}


@pytest.mark.parametrize("key", list(KEYS))
@pytest.mark.parametrize("arch", ARCHS)
def test_generate_equals_generate_tokens(arch, key):
    """Greedy `generate` (40 steps: the CUDA graph path) equals `generate_tokens` with the same keys driven by the
    model's own per-step logits; eos is the first greedy token of row 0, so the min-length keys decide."""
    m = _model(arch)
    ids, mask = _left_padded([5, 14, 9, 1], 14, 502, 7)
    plain = m.generate(ids, attention_mask=mask, max_new_tokens=40, eos_token_id=None)
    kw = dict(KEYS[key])
    eos = int(plain[0, 14]) if key.startswith("min") else None
    out = m.generate(ids, attention_mask=mask, max_new_tokens=40, eos_token_id=eos, pad_token_id=0, **kw)
    want = G.generate_tokens(_teacher_logits(m, ids, mask, out), ids, attention_mask=mask, max_new_tokens=40,
                             eos_token_id=eos, pad_token_id=0, **kw)
    assert torch.equal(out.cpu(), want), (arch, key)
    if eos is not None:
        assert eos not in out[0, 14:14 + G.min_step(14, kw.get("min_length"), kw.get("min_new_tokens"))].tolist()
    if key == "ngram2":
        for r in range(4):                      # no generated token repeats a bigram of the row (pads included)
            row = out[r].tolist()
            for j in range(14, len(row)):
                assert tuple(row[j - 1:j + 1]) not in {tuple(row[i - 1:i + 1]) for i in range(1, j)}, (r, j)


def test_neutral_keys_are_bit_identical_with_the_same_launches():
    _, lib = _lib()
    m = _model("qwen2")
    ids, mask = _left_padded([5, 14, 9], 14, 502, 2)
    runs = []
    for kw in ({}, dict(repetition_penalty=1.0, no_repeat_ngram_size=0, num_return_sequences=1, min_length=0)):
        torch.manual_seed(0)
        n0 = lib.sk_launch_count()
        out = m.generate(ids, attention_mask=mask, max_new_tokens=24, do_sample=True, eos_token_id=None, **kw)
        torch.cuda.synchronize()
        runs.append((out, lib.sk_launch_count() - n0))
    assert torch.equal(runs[0][0], runs[1][0]) and runs[0][1] == runs[1][1], runs


# ---------------------------------------------------------------------------------------------- 3. fan-out
@pytest.mark.parametrize("arch", ["qwen2", "opt-fp32"])
def test_kv_fanout_rows_equal_source(arch):
    from slamkit_b200.lm import DecodeSession
    m = _model(arch)
    lengths, k, T_cache = [3, 11, 7], 3, 20
    right = torch.zeros(3, 11, dtype=torch.long)
    g = torch.Generator().manual_seed(1)
    for r, n in enumerate(lengths):
        right[r, :n] = torch.randint(2, 502, (n,), generator=g)
    lens = torch.tensor(lengths)
    one = DecodeSession(m, 3, T_cache, 4)
    one.prefill(right, lens)
    fan = DecodeSession(m, 3 * k, T_cache, 4)
    fan.kv.fill_(0xA5)                                               # guard bytes
    fan.prefill(right, lens, k)
    torch.cuda.synchronize()
    esz = 4 if arch == "opt-fp32" else 2
    KVH = 1 if arch == "qwen2" else 2
    src = one.kv.view(2 * 2, 3, KVH, T_cache, 64 * esz)             # [L*2][B][KVH][T_cache][row bytes]
    dst = fan.kv.view(2 * 2, 3 * k, KVH, T_cache, 64 * esz)
    for b, n in enumerate(lengths):
        for j in range(k):
            assert torch.equal(dst[:, b * k + j, :, :n], src[:, b, :, :n]), (b, j)
            assert bool((dst[:, b * k + j, :, n:] == 0xA5).all()), (b, j)
    assert torch.equal(fan.logits, one.logits.repeat_interleave(k, 0))
    assert torch.equal(fan.tokens, one.tokens.repeat_interleave(k)) and torch.equal(fan.pos, one.pos.repeat_interleave(k))


@pytest.mark.parametrize("arch", ["qwen2", "opt-fp32"])
def test_fanout_groups(arch):
    """With equal uniforms a group's k rows equal each other and the k = 1 run of the prompt (rules on); Philox rows
    differ; greedy with k > 1 raises."""
    from slamkit_b200 import _lib as L
    from slamkit_b200.lm import DecodeSession
    m = _model(arch)
    ids, mask = _left_padded([6, 12], 12, 502, 3)
    lens = mask.sum(1)
    right = torch.zeros(2, 12, dtype=torch.long)
    for r in range(2):
        right[r, :int(lens[r])] = ids[r, 12 - int(lens[r]):]
    k, steps = 4, 12
    cfg = L.SkSampling(seed=9, top_p=0.9, temperature=0.8, do_sample=1, top_k=25, n_eos=0, pad_token_id=0,
                       max_length=12 + steps)
    g = torch.Generator().manual_seed(4)
    us = [torch.rand(2, generator=g) for _ in range(steps)]
    outs = []
    for kk in (1, k):
        sess = DecodeSession(m, 2 * kk, 12 + steps, steps)
        sess.set_rules(ids.repeat_interleave(kk, 0), penalty=1.3, ngram=2)
        sess.prefill(right, lens, kk)
        for s in range(steps):
            if s:
                sess.step()
            sess.select(cfg, uniforms=us[s].repeat_interleave(kk).to(DEV))
        outs.append(sess.out.cpu())
    assert torch.equal(outs[1], outs[0].repeat_interleave(k, 0))
    torch.manual_seed(0)
    out = m.generate(ids, attention_mask=mask, do_sample=True, max_new_tokens=16, num_return_sequences=k,
                     eos_token_id=None, repetition_penalty=1.2)
    assert out.shape == (2 * k, 28) and torch.equal(out[:, :12].cpu(), ids.repeat_interleave(k, 0))
    for b in range(2):
        grp = out[b * k:(b + 1) * k, 12:]
        assert len({tuple(r.tolist()) for r in grp}) > 1, b
    with pytest.raises(ValueError, match="num_return_sequences"):
        m.generate(ids, attention_mask=mask, do_sample=False, num_return_sequences=2)


# ---------------------------------------------------------------------------------------------- 4. CLI
def test_cli_generate_num_return_sequences(tmp_path):
    """`cli/eval.py metric=generate` with two sampled continuations per prompt and a repetition penalty writes one file
    per continuation, numbered in result order."""
    import os
    from flac_writer import write_flac
    from test_gpu_vocoder import _textless_checkpoint
    import cli.eval as E
    from slamkit_b200.lm import B200UnitLM, LMConfig

    ck = tmp_path / "ck"
    lm = B200UnitLM(LMConfig(vocab_size=502, hidden=128, n_layers=2, n_heads=2, n_kv_heads=1, head_dim=64, ffn=256),
                    device=DEV, max_batch=4, max_seq=128, trainable=False)
    lm.init_weights(5, std=0.05)
    lm.save_pretrained(str(ck))
    g = torch.Generator().manual_seed(21)
    data = tmp_path / "prompts"
    data.mkdir()
    for i, n in enumerate((36000, 20000, 52000, 41000)):
        pcm = (0.2 * torch.randn(n, generator=g).clamp(-4, 4) / 4 * 32767).round().long().numpy()[:, None]
        write_flac(str(data / f"p{i}.flac"), pcm)
    mp, cp = _textless_checkpoint(tmp_path)
    out = tmp_path / "gen"
    res = E.main([f"model.pretrained_model={ck}", "+synthetic_weights=true", "batch_size=3", "num_workers=2",
                  "metric=generate", "vocoder=vocoder_hubert_25", f"vocoder.model_path={mp}", f"vocoder.config_path={cp}",
                  f"metric.data_path={data}/*.flac", "metric.prompt_length=2", f"metric.out_path={out}",
                  "metric.generate_kwargs.max_new_tokens=24", "+metric.generate_kwargs.num_return_sequences=2",
                  "+metric.generate_kwargs.repetition_penalty=1.3", "+metric.generate_kwargs.min_new_tokens=8"])
    gens = res["generate"]
    assert len(gens) == 8 and all(w.numel() > 0 for w in gens)
    assert sorted(os.listdir(out)) == sorted(f"generate_{i}.wav" for i in range(8))
