"""Batched KV-cache decoding behind `B200UnitLM.generate`: decode attention against fp32 math, prefill + decode steps against
the full forward and the fp32 oracle, cached greedy generation against the oracle's argmax, the device sampler against the
CPU statement of HF's selection rules (tests/decode_ref.py), the Philox draw distribution, reproducibility and CUDA
graph replay, and the 152 k text+unit vocabulary."""
import ctypes as C
import math

import pytest
import torch

from decode_ref import expected_token
from helpers import rel_err

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _lib():
    from slamkit_b200 import _lib as L
    return L, L.require_cuda()


def _mk_lm(cfg_o, seed, max_batch=8, max_seq=256, max_positions=2048):
    from oracle import lm_oracle as O
    from slamkit_b200.lm import B200UnitLM, LMConfig
    p = O.init_params(cfg_o, seed=seed)
    cfg = LMConfig(vocab_size=cfg_o.vocab_size, hidden=cfg_o.hidden, n_layers=cfg_o.n_layers, n_heads=cfg_o.n_heads,
                   n_kv_heads=cfg_o.n_kv_heads, head_dim=cfg_o.head_dim, ffn=cfg_o.ffn, rms_eps=cfg_o.rms_eps,
                   rope_theta=cfg_o.rope_theta, tie_embeddings=cfg_o.tie_embeddings, max_positions=max_positions)
    m = B200UnitLM(cfg, device=DEV, max_batch=max_batch, max_seq=max_seq, trainable=False)
    m.load_hf_state_dict(p)
    return m, p


def _tiny(vocab=502):
    from oracle import lm_oracle as O
    return O.OracleLMConfig(vocab_size=vocab, hidden=128, n_layers=2, n_heads=2, n_kv_heads=1, head_dim=64, ffn=256)


def _cpus():
    import bench
    return bench.usable_cpus()


def _left_padded(lengths, T, V, seed):
    g = torch.Generator().manual_seed(seed)
    ids, mask = torch.zeros(len(lengths), T, dtype=torch.long), torch.zeros(len(lengths), T, dtype=torch.long)
    prompts = []
    for r, n in enumerate(lengths):
        a = torch.randint(2, V, (n,), generator=g)
        ids[r, T - n:], mask[r, T - n:] = a, 1
        prompts.append(a)
    return ids, mask, prompts


# ---------------------------------------------------------------------------------------------- 1. decode attention
@pytest.mark.parametrize("H,KVH", [(14, 2), (2, 1), (12, 12)])
@pytest.mark.parametrize("B", [1, 5, 64])
def test_decode_attention_vs_fp32(H, KVH, B):
    L, lib = _lib()
    T_cache = 2048
    g = torch.Generator(device=DEV).manual_seed(H * 100 + B)
    choices = [1, 63, 64, 65, 257, 2048]
    lens = torch.tensor([choices[(b * 5 + H) % len(choices)] for b in range(B)], dtype=torch.int32, device=DEV)
    k = torch.randn(B, KVH, T_cache, 64, device=DEV, generator=g).to(torch.bfloat16)
    v = torch.randn(B, KVH, T_cache, 64, device=DEV, generator=g).to(torch.bfloat16)
    for b in range(B):                                     # never read: the output stays finite
        k[b, :, int(lens[b]):] = float("nan")
        v[b, :, int(lens[b]):] = float("nan")
    ldq = (H + 2 * KVH) * 64                               # q as a column slice of a fused projection
    qkv = torch.randn(B, ldq, device=DEV, generator=g).to(torch.bfloat16)
    scale = 0.125
    partial = torch.empty(int(lib.sk_attn_decode_partial_bytes(B, H, T_cache)) // 4, device=DEV, dtype=torch.float32)
    outs = []
    for _ in range(2):
        o = torch.full((B, H * 64), 7.0, device=DEV, dtype=torch.bfloat16)
        L.check(lib.sk_attn_decode(L.ptr(qkv), ldq, L.ptr(k), L.ptr(v), L.ptr(lens), L.ptr(o), H * 64, L.ptr(partial), B, H,
                                   KVH, T_cache, L.f32(scale), L.stream_ptr()))
        outs.append(o)
    torch.cuda.synchronize()
    assert torch.equal(outs[0], outs[1]), "decode attention is not bit-identical run to run"
    o = outs[0].float()
    assert torch.isfinite(o).all()
    G = H // KVH
    worst = 0.0
    for b in range(B):
        n = int(lens[b])
        q = qkv[b, :H * 64].float().view(H, 64)
        kk = k[b, :, :n].float().repeat_interleave(G, dim=0)       # [H, n, 64]
        vv = v[b, :, :n].float().repeat_interleave(G, dim=0)
        p = torch.softmax(torch.einsum("hd,hnd->hn", q, kk) * scale, dim=-1)
        ref = torch.einsum("hn,hnd->hd", p, vv).reshape(-1)
        err = rel_err(o[b], ref)
        worst = max(worst, err)
        assert err < 4e-3, (b, n, err)
    print(f"decode attention H={H} KVH={KVH} B={B}: worst relative error vs fp32 {worst:.2e}")


# ---------------------------------------------------------------------------------------------- 2. prefill + decode
@pytest.mark.parametrize("width", ["tiny", "cfg2-3layers"])
def test_prefill_decode_equal_full_forward(width):
    from oracle import lm_oracle as O
    from slamkit_b200.lm import DecodeSession
    torch.set_num_threads(_cpus())
    cfg_o = _tiny() if width == "tiny" else O.OracleLMConfig(n_layers=3)
    m, p = _mk_lm(cfg_o, 3, max_batch=4, max_seq=256)
    lengths, steps = [1, 7, 64, 130], 32
    T = max(lengths)
    g = torch.Generator().manual_seed(7)
    seqs = [torch.randint(2, 502, (n + steps,), generator=g) for n in lengths]
    ids = torch.zeros(4, T, dtype=torch.long)
    for r, n in enumerate(lengths):
        ids[r, :n] = seqs[r][:n]
    lens = torch.tensor(lengths)
    sess = DecodeSession(m, 4, T + steps, steps)
    dec = [sess.prefill(ids, lens).float().cpu()]          # logits at position lens-1
    for s in range(steps):
        tok = torch.stack([seqs[r][lengths[r] + s] for r in range(4)]).to(DEV)
        pos = (lens + s).to(torch.int32).to(DEV)
        dec.append(sess.step(tok, pos).float().cpu())
    dec = torch.stack(dec, 1)                               # [4, steps+1, V]: logits at positions lens-1 .. lens-1+steps
    p32 = {k: v.float() for k, v in p.items()}
    for r, n in enumerate(lengths):
        full = m.forward(seqs[r][None]).logits[0].float().cpu()[n - 1:n + steps]
        e = rel_err(dec[r], full)
        per_step = max(rel_err(dec[r, s], full[s]) for s in range(steps + 1))
        ref32 = O.forward_logits(p32, cfg_o, seqs[r][None])[0][n - 1:n + steps]
        e_dec, e_fwd = rel_err(dec[r], ref32), rel_err(full, ref32)
        print(f"{width} row {r} (prompt {n}): decode vs full forward {e:.2e} (worst step {per_step:.2e}); vs fp32 oracle "
              f"decode {e_dec:.2e}, full forward {e_fwd:.2e}")
        # the logits bar between two bf16 paths: 8e-3 at the tiny widths; at cfg-2 widths two correct bf16 paths differ by
        # their independent rounding noise (~1e-2 after a few layers), so the bar is test_lm_true_width_vs_oracle's
        pair_bar = 8e-3 if width == "tiny" else 2.0 * e_fwd + 4e-3
        assert e < pair_bar, (r, e, pair_bar)
        assert e_dec < 1.3 * e_fwd + 1e-3, (r, e_dec, e_fwd)
        # every single step: within that bar of the full forward, or at least as close to the fp32 answer as the full
        # forward is (two independently rounded paths can differ by ~sqrt(2) x their own error)
        for s in range(steps + 1):
            d, d32, f32 = rel_err(dec[r, s], full[s]), rel_err(dec[r, s], ref32[s]), rel_err(full[s], ref32[s])
            assert d < pair_bar or d32 < 1.3 * f32 + 1e-3, (r, s, d, d32, f32)


# ---------------------------------------------------------------------------------------------- 3. cached greedy generate
def _assert_oracle_argmax(p, cfg_o, prompt, new_tokens, margin=0.02):
    from oracle import lm_oracle as O
    seq = torch.cat([prompt, torch.tensor(new_tokens, dtype=torch.long)])
    lo = O.forward_logits(p, cfg_o, seq[None])[0].float()
    n = len(prompt)
    for i, tok in enumerate(new_tokens):
        row = lo[n - 1 + i]
        assert float(row[tok]) >= float(row.max()) - margin * float(row.max() - row.min()), (n, i, tok, int(row.argmax()))


def test_cached_greedy_generate_follows_the_oracle():
    torch.set_num_threads(_cpus())
    cfg_o = _tiny()
    m, p = _mk_lm(cfg_o, 5)
    lengths = [3, 17, 9, 1, 40, 25, 12, 33]
    T = max(lengths)
    ids, mask, prompts = _left_padded(lengths, T, 502, 11)
    out = m.generate(ids, attention_mask=mask, max_new_tokens=48, do_sample=False, eos_token_id=None)
    assert out.shape == (8, T + 48) and torch.equal(out[:, :T], ids)
    for r in range(8):
        _assert_oracle_argmax(p, cfg_o, prompts[r], out[r, T:].tolist())
    # batch independence: a row's logits alone and inside the batch
    from slamkit_b200.lm import DecodeSession
    right = torch.zeros(8, T, dtype=torch.long)
    for r, n in enumerate(lengths):
        right[r, :n] = prompts[r]
    both = DecodeSession(m, 8, T + 8, 8)
    one = DecodeSession(m, 1, lengths[4] + 8, 8)
    la, lb = [both.prefill(right, torch.tensor(lengths)).float().cpu()[4]], [one.prefill(right[4:5, :lengths[4]], torch.tensor(lengths[4:5])).float().cpu()[0]]
    for s in range(8):
        toks = out[:, T + s].to(DEV)
        la.append(both.step(toks, (torch.tensor(lengths) + s).int().to(DEV)).float().cpu()[4])
        lb.append(one.step(toks[4:5], torch.tensor([lengths[4] + s], dtype=torch.int32, device=DEV)).float().cpu()[0])
    assert rel_err(torch.stack(la), torch.stack(lb)) < 8e-3


def test_generate_eos_max_length_max_positions_and_bans():
    cfg_o = _tiny()
    m, p = _mk_lm(cfg_o, 6, max_positions=40)
    ids, mask, prompts = _left_padded([5, 12, 30], 30, 502, 3)
    base = m.generate(ids, attention_mask=mask, max_new_tokens=20, eos_token_id=None)
    # max_positions = 40 stops every row at 40 tokens: rows of 5, 12, 30 real tokens get 20, 20, 10 new ones
    assert base.shape == (3, 50)
    assert base[2, 40:].tolist() == [m.config.pad_token_id] * 10
    first = int(base[0, 30])
    out = m.generate(ids, attention_mask=mask, max_new_tokens=6, eos_token_id=first, pad_token_id=7)
    assert int(out[0, 30]) == first and out[0, 31:].tolist() == [7] * (out.shape[1] - 31)
    for r in (1, 2):                     # the other rows follow the same greedy path up to their own eos, then pad
        want = base[r, 30:36].tolist()
        if first in want:
            k = want.index(first) + 1
            want = want[:k] + [7] * (6 - k)
        assert out[r, 30:].tolist() == want[:out.shape[1] - 30], r
    out2 = m.generate(ids, attention_mask=mask, max_length=34, eos_token_id=None)
    assert out2.shape == (3, 34) and torch.equal(out2, base[:, :34])
    g = torch.Generator().manual_seed(0)
    banned = torch.randperm(502, generator=g)[:400].tolist()
    for kw in ({"do_sample": False}, {"do_sample": True, "temperature": 0.8, "top_k": 25}, {"do_sample": True, "top_p": 0.9}):
        out3 = m.generate(ids, attention_mask=mask, max_new_tokens=10, eos_token_id=None, bad_words_ids=[[b] for b in banned], **kw)
        assert not (set(out3[:, 30:].flatten().tolist()) & set(banned)), kw
    with pytest.raises(NotImplementedError):
        m.generate(ids, attention_mask=mask, num_beams=2)
    with pytest.raises(NotImplementedError):
        m.generate(ids, attention_mask=mask, max_new_tokens=2, bad_words_ids=[[3, 4]])
    m.generate(ids, attention_mask=mask, max_new_tokens=2, use_cache=False)


# ---------------------------------------------------------------------------------------------- 4. sampler vs CPU rules
SAMPLER_CASES = {
    "greedy": dict(do_sample=False),
    "temp0.8-top_k25": dict(do_sample=True, temperature=0.8, top_k=25),
    "top_p0.9": dict(do_sample=True, top_p=0.9),
    "top_k50-top_p0.7": dict(do_sample=True, top_k=50, top_p=0.7),
    "top_k>V": dict(do_sample=True, top_k=1_000_000),
    "bans-temp1.3-top_k40": dict(do_sample=True, temperature=1.3, top_k=40, bans=True),
    "bans-greedy": dict(do_sample=False, bans=True),
}


@pytest.mark.parametrize("V", [502, 152167])
@pytest.mark.parametrize("case", list(SAMPLER_CASES))
def test_sampler_matches_cpu_rules(V, case):
    from slamkit_b200 import _lib as L
    from slamkit_b200.generation import ban_bitmask
    lib = L.require_cuda()
    c = dict(SAMPLER_CASES[case])
    bans = c.pop("bans", False)
    B = 48
    g = torch.Generator().manual_seed(V + len(case))
    logits = (torch.randn(B, V, generator=g) * 3.0).to(torch.bfloat16)
    logits[0, 5] = logits[0, 9] = logits[0].max() + 1           # tied maxima: greedy takes the lower id
    banned = torch.randperm(V, generator=g)[:V // 3].tolist() if bans else []
    if bans:
        logits[1, banned[0]] = 100.0                             # a banned id with the largest logit
    u = torch.rand(B, generator=g)
    ldl = (V + 63) // 64 * 64
    dl = torch.zeros(B, ldl, dtype=torch.bfloat16)
    dl[:, :V] = logits
    dl = dl.to(DEV)
    cfg = L.SkSampling(seed=1, top_p=float(c.get("top_p", 1.0)), temperature=float(c.get("temperature", 1.0)),
                       do_sample=int(c["do_sample"]), top_k=int(c.get("top_k", 0)), n_eos=0, pad_token_id=0,
                       max_length=1 << 30)
    st = {k: torch.zeros(B, dtype=torch.int32, device=DEV) for k in ("pos", "finished", "n_gen")}
    tokens, out, step = torch.zeros(B, dtype=torch.long, device=DEV), torch.full((B, 1), -1, dtype=torch.long, device=DEV), \
        torch.zeros(2, dtype=torch.int32, device=DEV)
    state = L.SkDecodeState(tokens.data_ptr(), st["pos"].data_ptr(), st["finished"].data_ptr(), st["n_gen"].data_ptr(),
                            out.data_ptr(), step.data_ptr(), 1, 0)
    ban = ban_bitmask(banned, V).to(DEV) if banned else None
    ud = u.to(DEV)
    L.check(lib.sk_select_next(L.ptr(dl), ldl, V, B, L.ptr(ban), C.byref(cfg), L.ptr(ud), C.byref(state), L.stream_ptr()))
    got = out[:, 0].cpu().tolist()
    assert int(step[0]) == 1 and tokens.cpu().tolist() == got and st["pos"].cpu().tolist() == [1] * B
    skipped = 0
    for b in range(B):
        want, dist = expected_token(logits[b], c["do_sample"], c.get("temperature", 1.0), c.get("top_k"), c.get("top_p"),
                                    banned, float(u[b]))
        if dist < 1e-6:
            skipped += 1
            continue
        assert got[b] == want, (b, got[b], want)
    if not c["do_sample"]:
        assert got[0] == 5
    if banned:
        assert not (set(got) & set(banned))
    assert skipped <= 2, skipped


# ---------------------------------------------------------------------------------------------- 5. sampling distribution
def test_philox_draws_follow_the_filtered_distribution():
    from scipy.stats import chi2
    from slamkit_b200 import _lib as L
    from slamkit_b200.generation import process_logits
    lib = L.require_cuda()
    V, B, steps = 64, 5000, 10
    g = torch.Generator().manual_seed(3)
    row = (torch.randn(V, generator=g) * 1.5).to(torch.bfloat16)
    s = process_logits(row, 0.8, 10, None, None)
    probs = torch.softmax(s.double(), -1)
    support = torch.nonzero(probs > 0)[:, 0]
    assert len(support) == 10
    dl = row[None].repeat(B, 1).to(DEV)
    cfg = L.SkSampling(seed=1234, top_p=1.0, temperature=0.8, do_sample=1, top_k=10, n_eos=0, pad_token_id=0,
                       max_length=1 << 30)
    z = lambda dt: torch.zeros(B, dtype=dt, device=DEV)
    tokens, pos, fin, ngen = z(torch.long), z(torch.int32), z(torch.int32), z(torch.int32)
    out, step = torch.zeros(B, steps, dtype=torch.long, device=DEV), torch.zeros(2, dtype=torch.int32, device=DEV)
    state = L.SkDecodeState(tokens.data_ptr(), pos.data_ptr(), fin.data_ptr(), ngen.data_ptr(), out.data_ptr(),
                            step.data_ptr(), steps, 0)
    for _ in range(steps):
        L.check(lib.sk_select_next(L.ptr(dl), V, V, B, None, C.byref(cfg), None, C.byref(state), L.stream_ptr()))
    draws = out.flatten().cpu()
    assert set(draws.tolist()) <= set(support.tolist())
    counts = torch.bincount(draws, minlength=V)[support].double()
    expect = probs[support] * draws.numel()
    stat = float(((counts - expect) ** 2 / expect).sum())
    q = chi2.ppf(0.999, len(support) - 1)
    print(f"chi-square {stat:.2f} (0.999 quantile {q:.2f}) over {draws.numel()} draws")
    assert stat < q


# ---------------------------------------------------------------------------------------------- 6. reproducibility, graphs
def test_sampling_reproducible_and_graph_replay_equals_eager():
    from slamkit_b200 import _lib as L
    from slamkit_b200.lm import DecodeSession
    cfg_o = _tiny()
    m, _ = _mk_lm(cfg_o, 8)
    ids, mask, prompts = _left_padded([4, 20, 11, 30], 30, 502, 5)
    kw = dict(attention_mask=mask, max_new_tokens=40, do_sample=True, temperature=0.8, top_k=25, eos_token_id=None)
    torch.manual_seed(0)
    a = m.generate(ids, **kw)
    torch.manual_seed(0)
    b = m.generate(ids, **kw)
    c = m.generate(ids, **kw, generator=torch.Generator().manual_seed(0))
    assert torch.equal(a, b) and a.shape == (4, 70)
    assert not torch.equal(a, m.generate(ids, **kw))                   # the default generator moved on
    assert c.shape == a.shape
    # eager steps vs one captured step replayed: same tokens and the same final logits, bit for bit
    lens = torch.tensor([4, 20, 11, 30])
    right = torch.zeros(4, 30, dtype=torch.long)
    for r, n in enumerate(lens.tolist()):
        right[r, :n] = prompts[r]
    cfg = L.SkSampling(seed=99, top_p=0.9, temperature=0.8, do_sample=1, top_k=25, n_eos=0, pad_token_id=0, max_length=60)
    runs = []
    for use_graph in (False, True):
        sess = DecodeSession(m, 4, 60, 24)
        sess.prefill(right, lens)
        sess.select(cfg)
        sess.step()
        sess.select(cfg)
        if use_graph:
            gr = torch.cuda.CUDAGraph()
            with torch.cuda.graph(gr):
                sess.step()
                sess.select(cfg)
            for _ in range(22):
                gr.replay()
        else:
            for _ in range(22):
                sess.step()
                sess.select(cfg)
        torch.cuda.synchronize()
        runs.append((sess.out.clone(), sess.logits.clone()))
    assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])


def test_text_unit_vocabulary():
    """cfg-4 vocabulary (152,167 ids): one decode step matches the full forward, and with every non-unit id banned only unit
    ids come out (here the units are the last 502 ids)."""
    from slamkit_b200.lm import DecodeSession
    V = 152167
    cfg_o = _tiny(V)
    m, _ = _mk_lm(cfg_o, 9, max_batch=2, max_seq=64)
    ids, mask, prompts = _left_padded([6, 19], 19, V, 4)
    right = torch.zeros(2, 19, dtype=torch.long)
    for r, pr in enumerate(prompts):
        right[r, :len(pr)] = pr
    sess = DecodeSession(m, 2, 24, 2)
    sess.prefill(right, torch.tensor([6, 19]))
    nxt = torch.tensor([1000, 151900], device=DEV)
    got = sess.step(nxt, torch.tensor([6, 19], dtype=torch.int32, device=DEV)).float().cpu()
    for r, pr in enumerate(prompts):
        seq = torch.cat([pr, nxt[r:r + 1].cpu()])
        full = m.forward(seq[None]).logits[0, -1].float().cpu()
        assert rel_err(got[r], full) < 8e-3
    units = set(range(V - 502, V))
    banned = [[i] for i in range(V - 502)]
    for kw in ({"do_sample": False}, {"do_sample": True, "temperature": 0.8, "top_k": 25}, {"do_sample": True, "top_p": 0.95}):
        out = m.generate(ids, attention_mask=mask, max_new_tokens=8, eos_token_id=None, bad_words_ids=banned, **kw)
        assert set(out[:, 19:].flatten().tolist()) <= units, kw
