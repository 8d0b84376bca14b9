"""GPU parity of the GPT-NeoX decoder (the Pythia bases of the interleaving-scaling recipe) through the same `sk_lm_*`
handle as Qwen2 and OPT: against tests/golden/neox_tiny.npz (the reference's own UnitLM over HF GPTNeoXForCausalLM) with
the tolerances of tests/test_gpu_opt.py, against oracle/neox_oracle.py at mid-size shapes, plus exact checks of the new
kernels: the partial-RoPE, GELU-forward, GELU'-backward and two-residual GEMM epilogues, an exhaustive sweep of every
finite bf16 pre-activation through the GELU epilogues, and the dual LayerNorm."""
import ctypes as C
import json
import os

import numpy as np
import pytest
import torch

from helpers import rel_err, u16_to_bf16
from oracle import neox_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _lib():
    from slamkit_b200 import _lib as L
    return L, L.require_cuda()


def _lm_cfg(c: "O.OracleNeoxConfig"):
    from slamkit_b200.lm import NeoxLMConfig
    return NeoxLMConfig(vocab_size=c.vocab_size, hidden=c.hidden, n_layers=c.n_layers, n_heads=c.n_heads, ffn=c.ffn,
                        max_positions=c.max_positions, rot_dims=c.rot_dims, rope_theta=c.rope_theta, ln_eps=c.ln_eps)


def _mk(c, seed, max_batch, max_seq, trainable=True):
    from slamkit_b200.lm import B200UnitLM
    p = O.init_params(c, seed=seed)
    m = B200UnitLM(_lm_cfg(c), device=DEV, max_batch=max_batch, max_seq=max_seq, trainable=trainable)
    m.load_hf_state_dict(p)
    return m, p


def _golden(golden_dir):
    z = np.load(os.path.join(golden_dir, "neox_tiny.npz"))
    c = z["cfg"]
    cfg = O.OracleNeoxConfig(vocab_size=int(c[0]), hidden=int(c[1]), n_layers=int(c[2]), n_heads=int(c[3]), ffn=int(c[4]),
                             max_positions=int(c[5]), rot_dims=int(c[6]))
    return z, cfg, int(c[7])


def _fp32_grads(p, c, *args, **kw):
    return O.forward_backward({k: v.float() for k, v in p.items()}, c, *args, **kw)[2]


def _check_grads(sd_g, grads_ref, grads_fp32, keys, tol=2e-2):
    """Every gradient within `tol` of the bf16 reference, or at least as close to the fp32 gradient as the reference's
    own bf16 autograd is (the allowance of tests/test_gpu_opt.py)."""
    bad = []
    for k in keys:
        got = sd_g[k].cpu()
        e_ref = rel_err(got, grads_ref[k])
        if e_ref < tol:
            continue
        e_ours, e_theirs = rel_err(got, grads_fp32[k]), rel_err(grads_ref[k], grads_fp32[k])
        if e_ours > 1.25 * e_theirs + 5e-3:
            bad.append((k, round(e_ref, 4), round(e_ours, 4), round(e_theirs, 4)))
    assert not bad, bad


# ---- the model against the reference and the oracle ----------------------------------------------------------------

def test_neox_matches_reference_golden(golden_dir):
    """Loss, logits, every gradient, the clip norm and one AdamW step against the reference's UnitLM (Trainer path)."""
    from slamkit_b200.lm import B200AdamW
    z, c, seed = _golden(golden_dir)
    ids, labels = torch.from_numpy(z["train/ids"]), torch.from_numpy(z["train/labels"])
    B, T = ids.shape
    m, p = _mk(c, seed, B, T)
    out = m.forward_backward(ids, labels, num_items_in_batch=float(z["train/num_items"]))
    loss = float(out.loss)
    assert abs(loss - float(z["train/loss"])) < 1e-3 * abs(float(z["train/loss"])), (loss, float(z["train/loss"]))
    valid = ids != 0
    assert rel_err(m.logits_view(B, T).cpu()[valid], O.golden_masked_logits(z)[valid]) < 8e-3
    ref_g = O.golden_grads(z, p, c)
    g32 = _fp32_grads(p, c, ids, labels, float(z["train/num_items"]))
    _check_grads(m.state_dict_hf(grads=True), ref_g, g32, p)
    opt = B200AdamW(m, lr=1e-3, max_grad_norm=0.5)
    opt.step()
    assert abs(float(opt.stats[0]) - float(z["train/total_norm"])) < 0.01 * float(z["train/total_norm"])
    sd_p = m.state_dict_hf()
    for k in p:
        upd = sd_p[k].cpu().float() - p[k].float()
        ref_sign = torch.from_numpy(z["upd_sign/" + k]).float().view_as(upd)
        ref_size = float(z["upd_absmean/" + k])
        assert abs(float(upd.abs().mean()) - ref_size) <= 0.2 * ref_size + 1e-9, k
        agree = (torch.sign(upd) == ref_sign).float().mean()
        if agree < 0.9:
            want = -torch.sign(g32[k])
            ours, theirs = (torch.sign(upd) == want).float().mean(), (ref_sign == want).float().mean()
            assert ours >= theirs - 0.03, (k, float(agree), float(ours), float(theirs))


def test_neox_pure_causal_logits_match_oracle_bitwise_reference(golden_dir):
    """The unmasked path: the device logits against the fixture (which the CPU oracle reproduces bit for bit)."""
    z, c, seed = _golden(golden_dir)
    ids = torch.from_numpy(z["train/ids"])
    m, _ = _mk(c, seed, *ids.shape, trainable=False)
    out = m.forward(ids)
    assert rel_err(out.logits.cpu(), u16_to_bf16(z["nomask/logits_u16"])) < 8e-3


def test_neox_packed_row_and_loglik_match_reference(golden_dir):
    z, c, seed = _golden(golden_dir)
    ids, pos, labels = (torch.from_numpy(z["packed/" + k]) for k in ("ids", "position_ids", "labels"))
    m, _ = _mk(c, seed, 1, ids.shape[1], trainable=False)
    out = m.forward(ids, position_ids=pos, labels=labels, num_items_in_batch=float(z["packed/num_items"]))
    assert rel_err(out.logits.cpu(), u16_to_bf16(z["packed/logits_u16"])) < 8e-3
    assert abs(float(out.loss) - float(z["packed/loss"])) < 1e-3 * abs(float(z["packed/loss"]))
    m, _ = _mk(c, int(z["loglik/seed_params"]), 3, 40, trainable=False)
    tokens = torch.from_numpy(z["loglik/tokens"])
    for mean, key in ((False, "loglik/sum"), (True, "loglik/mean")):
        ll = m.sequence_log_likelihood(tokens, mean_nll=mean).float().cpu()
        ref = torch.from_numpy(z[key])
        assert bool(((ll - ref).abs() <= 0.02 * ref.abs()).all()), (mean, ll.tolist(), ref.tolist())


def _batch(B, T, seed, V=502, pad_last=17):
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(2, V, (B, T), generator=g)
    ids[:, 0] = 1
    if pad_last:
        ids[-1, T - pad_last:] = 0
    labels = ids.clone()
    labels[ids == 0] = -100
    return ids, labels


@pytest.mark.parametrize("rot", [16, 32, 64])
def test_neox_mid_size_against_oracle(rot):
    """Forward / backward at hidden 256 (4 heads, 2 layers, ffn 1024) against the fp32 oracle, for each rotary width."""
    c = O.OracleNeoxConfig(vocab_size=502, hidden=256, n_layers=2, n_heads=4, ffn=1024, max_positions=256, rot_dims=rot)
    ids, labels = _batch(2, 192, 3)
    m, p = _mk(c, 11, 2, 192)
    ni = float((labels != -100).sum())
    out = m.forward_backward(ids, labels, num_items_in_batch=ni)
    loss32, logits32, g32 = O.forward_backward({k: v.float() for k, v in p.items()}, c, ids, labels, ni)
    assert abs(float(out.loss) - float(loss32)) < 3e-3 * abs(float(loss32))
    assert rel_err(m.logits_view(2, 192).cpu(), logits32) < 1e-2
    sd = m.state_dict_hf(grads=True)
    errs = {k: rel_err(sd[k].cpu(), g32[k]) for k in p}
    assert max(errs.values()) < 4e-2, sorted(errs.items(), key=lambda kv: -kv[1])[:4]


def test_neox_packed_rows_with_accumulation():
    """Two packed micro-batches accumulated equal the oracle's summed gradients."""
    c = O.OracleNeoxConfig(vocab_size=502, hidden=256, n_layers=2, n_heads=4, ffn=1024, max_positions=128, rot_dims=16)
    m, p = _mk(c, 5, 1, 256)
    g = torch.Generator().manual_seed(4)
    tot = None
    for i, lens in enumerate(([100, 1, 91, 64], [128, 128])):
        ids = torch.randint(2, 502, (1, sum(lens)), generator=g)
        pos = torch.cat([torch.arange(n) for n in lens])[None]
        labels = ids.clone()
        for a in np.cumsum([0] + lens[:-1]):
            labels[0, a] = -100
        m.forward_backward(ids, labels, position_ids=pos, num_items_in_batch=400.0, accumulate=i > 0)
        _, _, g32 = O.forward_backward({k: v.float() for k, v in p.items()}, c, ids, labels, 400.0, pos, packed=True)
        tot = g32 if tot is None else {k: tot[k] + g32[k] for k in tot}
    sd = m.state_dict_hf(grads=True)
    errs = {k: rel_err(sd[k].cpu(), tot[k]) for k in p}
    assert max(errs.values()) < 4e-2, sorted(errs.items(), key=lambda kv: -kv[1])[:4]


def test_neox_five_step_trajectory():
    """Five clip + AdamW steps follow the oracle trainer's losses."""
    from slamkit_b200.lm import B200AdamW
    c = O.OracleNeoxConfig(vocab_size=502, hidden=128, n_layers=2, n_heads=2, ffn=512, max_positions=128, rot_dims=16)
    m, p = _mk(c, 2, 2, 96)
    opt = B200AdamW(m, lr=1e-3, max_grad_norm=0.5)
    ref = O.OracleNeoxTrainer(p, c)
    for s in range(5):
        ids, labels = _batch(2, 96, 100 + s)
        out = m.forward_backward(ids, labels, num_items_in_batch=float((labels != -100).sum()))
        lo = float(out.loss)
        opt.step()
        lr_ = ref.train_step(ids, labels)
        assert abs(lo - lr_) < 5e-3 * abs(lr_), (s, lo, lr_)


@pytest.mark.parametrize("geom", ["pythia-160m", "pythia-410m"])
def test_neox_pythia_geometry_deterministic(geom):
    """Pythia-160m / -410m shapes: finite, and two identical steps give bit-identical loss and gradients."""
    d, L, H = {"pythia-160m": (768, 12, 12), "pythia-410m": (1024, 24, 16)}[geom]
    c = O.OracleNeoxConfig(vocab_size=502, hidden=d, n_layers=L, n_heads=H, ffn=4 * d, max_positions=2048, rot_dims=16)
    from slamkit_b200.lm import B200UnitLM
    m = B200UnitLM(_lm_cfg(c), device=DEV, max_batch=2, max_seq=512, seed=0)
    ids, labels = _batch(2, 512, 8)
    outs = []
    for _ in range(2):
        o = m.forward_backward(ids, labels, num_items_in_batch=float((labels != -100).sum()))
        outs.append((float(o.loss), m.grads.clone()))
    assert np.isfinite(outs[0][0]) and bool(torch.isfinite(outs[0][1].float()).all())
    assert outs[0][0] == outs[1][0] and torch.equal(outs[0][1], outs[1][1])


def test_neox_generate_follows_oracle_and_graph_replay_equals_eager():
    """Cached greedy generate: each new token is the oracle's argmax up to bf16 near-ties; the graph-replayed decode steps
    give the same logits as eager steps."""
    from slamkit_b200.lm import DecodeSession
    c = O.OracleNeoxConfig(vocab_size=502, hidden=128, n_layers=2, n_heads=2, ffn=512, max_positions=64, rot_dims=16)
    m, p = _mk(c, 4, 2, 64, trainable=False)
    g = torch.Generator().manual_seed(1)
    prompt = torch.randint(2, 502, (2, 8), generator=g)
    mask = torch.ones(2, 8, dtype=torch.long)
    mask[1, :3] = 0
    out = m.generate(prompt, attention_mask=mask, max_new_tokens=12, do_sample=False, eos_token_id=None)
    assert out.shape == (2, 20)
    for r, start in enumerate((0, 3)):
        seq = out[r:r + 1, start:].cpu()
        lo = O.forward_logits(p, c, seq)[0].float()
        for t in range(8 - start, seq.shape[1]):
            pred = lo[t - 1]
            assert pred[seq[0, t]] >= pred.max() - 0.05 * pred.abs().max(), (r, t)
    # eager vs graph replay of the same decode step
    ids = prompt.clone()
    lens = torch.full((2,), 8)
    s1, s2 = DecodeSession(m, 2, 32, 8), DecodeSession(m, 2, 32, 8)
    s1.prefill(ids, lens)
    s2.prefill(ids, lens)
    tok = torch.tensor([5, 7], device=DEV)
    pos = torch.tensor([8, 8], dtype=torch.int32, device=DEV)
    eager = s1.step(tok, pos).clone()
    s2.step(tok, pos)                        # one eager call first (kernel attributes), then capture the same call
    s2b = DecodeSession(m, 2, 32, 8)
    s2b.prefill(ids, lens)
    graph = torch.cuda.CUDAGraph()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        graph.capture_begin()
        s2b.step(tok, pos)
        graph.capture_end()
    torch.cuda.current_stream().wait_stream(side)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(s2b.logits, eager)


def test_neox_dpo_entry_points():
    """sk_lm_forward_rows + sk_lm_backward_weighted on a NeoX handle: the row-weighted gradient of the oracle."""
    from slamkit_b200 import _lib as L
    c = O.OracleNeoxConfig(vocab_size=502, hidden=128, n_layers=2, n_heads=2, ffn=512, max_positions=64, rot_dims=16)
    m, p = _mk(c, 6, 2, 48)
    ids, labels = _batch(2, 48, 21, pad_last=0)
    B, T = ids.shape
    idd, lab = ids.to(DEV), labels.to(DEV)
    nll = torch.zeros(B * T, device=DEV)
    L.check(m.lib.sk_lm_forward_rows(m._h, L.ptr(idd), L.ptr(lab), None, B, T, L.ptr(nll), L.ptr(m.stats), L.stream_ptr()))
    w = torch.tensor([0.7, -0.3], device=DEV)
    row_w = w[:, None].expand(B, T).contiguous().view(-1)     # one weight per logits row, as slamkit_b200/dpo.py passes
    L.check(m.lib.sk_lm_backward_weighted(m._h, L.ptr(idd), L.ptr(lab), None, B, T, L.ptr(row_w), 0, L.ptr(m.stats),
                                          L.stream_ptr()))
    _, _, g32 = O.forward_backward({k: v.float() for k, v in p.items()}, c, ids, labels, row_weight=w.cpu())
    sd = m.state_dict_hf(grads=True)
    errs = {k: rel_err(sd[k].cpu(), g32[k]) for k in p}
    assert max(errs.values()) < 5e-2, sorted(errs.items(), key=lambda kv: -kv[1])[:4]


def test_neox_bind_and_entry_point_guards():
    from slamkit_b200 import _lib as L
    from slamkit_b200.lm import NeoxLMConfig
    lib = L.require_cuda()
    h = C.c_void_p()
    for bad in (dict(rot_dims=8), dict(rot_dims=48), dict(hidden=96, n_heads=2), dict(ffn=1000), dict(hidden=4096, n_heads=64)):
        kw = dict(vocab_size=502, hidden=128, n_layers=1, n_heads=2, ffn=512, max_positions=64, rot_dims=16, ln_eps=1e-5)
        kw.update(bad)
        cfg = L.SkNeoxConfig(*[kw[k] for k in ("vocab_size", "hidden", "n_layers", "n_heads", "ffn", "max_positions",
                                               "rot_dims", "ln_eps")])
        assert lib.sk_lm_create_neox(C.byref(cfg), C.byref(h)) != 0, bad
    cfg = L.SkNeoxConfig(502, 128, 1, 2, 512, 64, 16, 1e-5)
    assert lib.sk_lm_create_neox(C.byref(cfg), C.byref(h)) == 0
    try:
        params = torch.zeros(int(lib.sk_lm_param_count(h)), device=DEV, dtype=torch.bfloat16)
        ws = torch.zeros(int(lib.sk_lm_workspace_bytes(h, 1, 16)), device=DEV, dtype=torch.uint8)
        rc = lib.sk_lm_bind(h, L.ptr(params), None, None, None, L.ptr(ws), C.c_int64(ws.numel()))
        assert rc != 0 and b"RoPE" in lib.sk_last_error()
        names = []
        buf = C.create_string_buffer(64)
        for i in range(lib.sk_lm_tensor_info(h, -1, None, 0, None, None, None)):
            L.check(lib.sk_lm_tensor_info(h, i, buf, 64, None, None, None))
            names.append(buf.value.decode())
        assert names[:12] == [f"layers.0.{n}" for n in ("ln1", "ln1_b", "ln2", "ln2_b", "wqkv", "bqkv", "wo", "bo", "w1", "b1",
                                                         "w2", "b2")]
        assert names[12:] == ["final_norm", "final_norm_b", "embed", "lm_head"]
    finally:
        lib.sk_lm_destroy(h)
    NeoxLMConfig()   # the dataclass defaults are a valid pythia-160m shape


def test_neox_qkv_permutation_round_trip():
    """HF's per-head [q|k|v] fused weight and bias load into [Q;K;V] and save back unchanged."""
    c = O.OracleNeoxConfig(vocab_size=502, hidden=192, n_layers=1, n_heads=3, ffn=256, max_positions=64, rot_dims=16)
    m, p = _mk(c, 9, 1, 16, trainable=False)
    sd = m.state_dict_hf()
    for k in p:
        assert torch.equal(sd[k].cpu(), p[k]), k
    W = p["lm.gpt_neox.layers.0.attention.query_key_value.weight"]
    flat = m.tensor("layers.0.wqkv").cpu()
    for h in range(3):
        for j in range(3):
            assert torch.equal(flat[j * 192 + h * 64: j * 192 + h * 64 + 64], W[h * 192 + j * 64: h * 192 + j * 64 + 64])


def test_neox_chunked_head_untied_50k_vocab():
    """At a 50 k-row untied vocabulary the lm_head + CE runs in row chunks: loss and the embed_out / embed_in gradients
    against a torch restatement."""
    c = O.OracleNeoxConfig(vocab_size=50304, hidden=128, n_layers=1, n_heads=2, ffn=512, max_positions=512, rot_dims=16)
    m, p = _mk(c, 13, 2, 2560)
    assert m.lib is not None
    ids, labels = _batch(2, 2560, 31, V=50304, pad_last=100)
    ni = float((labels != -100).sum())
    pos = torch.arange(2560)[None].expand(2, -1) % 512        # rows of five 512-token documents
    out = m.forward_backward(ids, labels, position_ids=pos, num_items_in_batch=ni)
    loss32, _, g32 = O.forward_backward({k: v.float() for k, v in p.items()}, c, ids, labels, ni, pos, packed=True)
    assert abs(float(out.loss) - float(loss32)) < 3e-3 * abs(float(loss32))
    sd = m.state_dict_hf(grads=True)
    for k in ("lm.embed_out.weight", "lm.gpt_neox.embed_in.weight", "lm.gpt_neox.final_layer_norm.weight"):
        assert rel_err(sd[k].cpu(), g32[k]) < 4e-2, k


# ---- kernels ---------------------------------------------------------------------------------------------------------

def _int_operands(M, N, K, seed, lo=-3, hi=4):
    """Small-integer bf16 operands: every product and partial sum is an exact fp32 integer."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randint(lo, hi, (M, K), generator=g).to(torch.bfloat16)
    w = torch.randint(lo, hi, (N, K), generator=g).to(torch.bfloat16)
    b = torch.randint(-8, 9, (N,), generator=g).to(torch.bfloat16)
    return x, w, b


def _rope_ref(pre, cos, sin, pos, rot, rope_cols):
    """The partial-RoPE epilogue on CPU at its rounding points: bf16 products, their bf16 sum."""
    out = pre.clone()
    h = rot // 2
    c, s = cos[pos].float(), sin[pos].float()
    for c0 in range(0, rope_cols, 64):
        x1, x2 = pre[:, c0:c0 + h].float(), pre[:, c0 + h:c0 + rot].float()
        r = lambda t: t.to(torch.bfloat16).float()   # noqa: E731
        out[:, c0:c0 + h] = (r(x1 * c) + r(-x2 * s)).to(torch.bfloat16)
        out[:, c0 + h:c0 + rot] = (r(x2 * c) + r(x1 * s)).to(torch.bfloat16)
    return out


# (M, N, K): the q|k|v projection of pythia-160m / -410m at training and decode sizes
QKV_SHAPES = [(m, n, k) for (n, k) in ((2304, 768), (3072, 1024)) for m in (1, 7, 64, 129, 1000)] + [(8192, 2304, 768)]


@pytest.mark.parametrize("rot", [16, 32])
@pytest.mark.parametrize("M,N,K", QKV_SHAPES)
def test_partial_rope_epilogue_exact(rot, M, N, K):
    from slamkit_b200.lm import rope_tables
    L, lib = _lib()
    x, w, b = _int_operands(M, N, K, M + N + rot)
    maxpos = 300
    cos, sin = rope_tables(10000.0, rot, maxpos)
    pos = (torch.arange(M, dtype=torch.int32) * 7) % maxpos
    xd, wd, bd = x.to(DEV), w.to(DEV), b.to(DEV)
    out = torch.full((M, N), float("nan"), device=DEV, dtype=torch.bfloat16)
    rope_cols = N // 3 * 2
    cd, sd, pd = cos.to(DEV), sin.to(DEV), pos.to(DEV)     # named: a temporary's memory could be reused by the next copy
    L.check(lib.sk_linear_rope_partial(M, N, K, L.ptr(xd), L.ptr(wd), L.ptr(bd), L.ptr(out), L.ptr(cd), L.ptr(sd), L.ptr(pd),
                                       1, rope_cols, maxpos, rot, L.stream_ptr()))
    pre = (x.float() @ w.float().T + b.float()).to(torch.bfloat16)
    ref = _rope_ref(pre, cos, sin, pos.long(), rot, rope_cols)
    got = out.cpu()
    bad = (got.view(torch.int16) != ref.view(torch.int16))
    assert not bool(bad.any()), (int(bad.sum()), bad.nonzero()[:5].tolist())


@pytest.mark.parametrize("M", [1, 37, 129, 2048])
def test_partial_rope_width64_equals_full_rope(M):
    from slamkit_b200.lm import rope_tables
    L, lib = _lib()
    N, K = 2304, 768
    g = torch.Generator().manual_seed(M)
    x = (torch.randn(M, K, generator=g)).to(torch.bfloat16).to(DEV)
    w = (torch.randn(N, K, generator=g) * 0.05).to(torch.bfloat16).to(DEV)
    b = (torch.randn(N, generator=g) * 0.1).to(torch.bfloat16).to(DEV)
    cos, sin = (t.to(DEV) for t in rope_tables(10000.0, 64, 4096))
    outs = []
    for fn in ("full", "partial"):
        o = torch.empty(M, N, device=DEV, dtype=torch.bfloat16)
        if fn == "full":
            L.check(lib.sk_linear_rope(M, N, K, L.ptr(x), L.ptr(w), L.ptr(b), L.ptr(o), L.ptr(cos), L.ptr(sin), None, 512,
                                       1536, 4096, L.stream_ptr()))
        else:
            L.check(lib.sk_linear_rope_partial(M, N, K, L.ptr(x), L.ptr(w), L.ptr(b), L.ptr(o), L.ptr(cos), L.ptr(sin), None,
                                               512, 1536, 4096, 64, L.stream_ptr()))
        outs.append(o)
    assert torch.equal(outs[0], outs[1])


@pytest.mark.parametrize("rot", [16, 32, 64])
def test_inverse_partial_rope_is_the_transpose(rot):
    """sk_rope_partial(inverse) undoes the forward rotation up to bf16 rounding and leaves columns >= rot untouched."""
    from slamkit_b200.lm import rope_tables
    L, lib = _lib()
    M, H = 300, 6
    cos, sin = (t.to(DEV) for t in rope_tables(10000.0, rot, 512))
    x = torch.randn(M, 3 * H * 64, device=DEV).to(torch.bfloat16)
    y = x.clone()
    L.check(lib.sk_rope_partial(L.ptr(y), L.ptr(cos), L.ptr(sin), None, M, 100, 3 * H * 64, 2 * H, 64, rot, 0, 512,
                                L.stream_ptr()))
    hv = y.view(M, 3 * H, 64)
    assert torch.equal(hv[:, :, rot:], x.view(M, 3 * H, 64)[:, :, rot:])
    assert torch.equal(hv[:, 2 * H:], x.view(M, 3 * H, 64)[:, 2 * H:])
    L.check(lib.sk_rope_partial(L.ptr(y), L.ptr(cos), L.ptr(sin), None, M, 100, 3 * H * 64, 2 * H, 64, rot, 1, 512,
                                L.stream_ptr()))
    assert rel_err(y.cpu(), x.cpu()) < 1e-2
    assert lib.sk_rope_partial(L.ptr(y), L.ptr(cos), L.ptr(sin), None, M, 100, 3 * H * 64, 2 * H, 64, 24, 1, 512,
                               L.stream_ptr()) != 0


def _gelu_fwd(M, F, K, x, w, b):
    L, lib = _lib()
    pre = torch.full((M, F), float("nan"), device=DEV, dtype=torch.bfloat16)
    act = torch.full((M, F), float("nan"), device=DEV, dtype=torch.bfloat16)
    L.check(lib.sk_linear_gelu_fwd(M, F, K, L.ptr(x), L.ptr(w), L.ptr(b), L.ptr(pre), L.ptr(act), L.stream_ptr()))
    return pre, act


def _gelu_bwd(M, N, F, dy, w2, pre):
    L, lib = _lib()
    dpre = torch.full((M, F), float("nan"), device=DEV, dtype=torch.bfloat16)
    L.check(lib.sk_linear_gelu_bwd(M, N, F, L.ptr(dy), L.ptr(w2), L.ptr(pre), L.ptr(dpre), L.stream_ptr()))
    return dpre


@pytest.mark.parametrize("M,F,K", [(m, f, k) for (f, k) in ((3072, 768), (4096, 1024)) for m in (1, 5, 64, 129, 1000)]
                         + [(8192, 3072, 768)])
def test_gelu_forward_epilogue_exact(M, F, K):
    """pre = bf16(acc + bias) exactly, act = gelu(pre) as torch computes it on the device."""
    x, w, b = _int_operands(M, F, K, M + F)
    xd, wd, bd = x.to(DEV), w.to(DEV), b.to(DEV)
    pre, act = _gelu_fwd(M, F, K, xd, wd, bd)
    ref_pre = (x.float() @ w.float().T + b.float()).to(torch.bfloat16)
    assert torch.equal(pre.cpu().view(torch.int16), ref_pre.view(torch.int16))
    ref_act = torch.nn.functional.gelu(pre)
    d = (act.view(torch.int16).int() - ref_act.view(torch.int16).int()).abs()
    assert int(d.max()) <= 1


@pytest.mark.parametrize("M,N,F", [(m, n, f) for (n, f) in ((768, 3072), (1024, 4096)) for m in (1, 5, 64, 129, 1000)]
                         + [(8192, 768, 3072)])
def test_gelu_backward_epilogue_exact(M, N, F):
    """d_pre = bf16(bf16(dy W2) * gelu'(pre)) against torch autograd of gelu on the exact bf16 d_act."""
    g = torch.Generator().manual_seed(M + F)
    dy = torch.randint(-3, 4, (M, N), generator=g).to(torch.bfloat16)
    w2 = torch.randint(-3, 4, (N, F), generator=g).to(torch.bfloat16)
    pre = (torch.randn(M, F, generator=g) * 2).to(torch.bfloat16)
    dyd, w2d, pred = dy.to(DEV), w2.to(DEV), pre.to(DEV)
    dpre = _gelu_bwd(M, N, F, dyd, w2d, pred)
    dact = (dy.float() @ w2.float()).to(torch.bfloat16).to(DEV)
    pr = pre.to(DEV).requires_grad_(True)
    torch.nn.functional.gelu(pr).backward(dact)
    d = (dpre.view(torch.int16).int() - pr.grad.view(torch.int16).int()).abs()
    assert int(d.max()) <= 1


def _all_finite_bf16():
    u = torch.arange(65536, dtype=torch.int32).to(torch.int16).view(torch.bfloat16)
    return u[torch.isfinite(u.float())]


def _ulp_diff(a, b):
    """|a - b| in bf16 ulps on the ordered integer line (+0 and -0 coincide)."""
    def key(t):
        i = t.view(torch.int16).int()
        return torch.where(i < 0, -(i & 0x7FFF), i)
    return (key(a) - key(b)).abs()


def test_gelu_epilogues_exhaustive_bf16_sweep(capsys):
    """Every finite bf16 pre-activation through the GELU forward and GELU' backward epilogues via an identity weight (the
    accumulator is exact), against torch.nn.functional.gelu and its autograd on the device: at most 1 ulp."""
    v = _all_finite_bf16()
    n = v.numel()
    K = 64
    M = (n + K - 1) // K
    x = torch.zeros(M * K, dtype=torch.bfloat16)
    x[:n] = v
    x = x.view(M, K).to(DEV)
    eye = torch.eye(K, dtype=torch.bfloat16, device=DEV)
    pre, act = _gelu_fwd(M, K, K, x, eye, torch.zeros(K, dtype=torch.bfloat16, device=DEV))
    assert torch.equal(pre, x)
    ref = torch.nn.functional.gelu(x)
    df = _ulp_diff(act, ref).view(-1)[:n]
    assert int(df.max()) <= 1
    ones = torch.ones(M, K, dtype=torch.bfloat16, device=DEV)
    dpre = _gelu_bwd(M, K, K, ones, eye, x)
    xr = x.clone().requires_grad_(True)
    torch.nn.functional.gelu(xr).backward(ones)
    db = _ulp_diff(dpre, xr.grad).view(-1)[:n]
    assert int(db.max()) <= 1
    with capsys.disabled():
        print(f"\nGELU sweep over {n} finite bf16 values: forward {int((df == 1).sum())} differ by 1 ulp, "
              f"backward {int((db == 1).sum())} differ by 1 ulp")


@pytest.mark.parametrize("with_ws", [0, 1])
@pytest.mark.parametrize("M,N,K", [(m, n, k) for (n, k) in ((768, 3072), (1024, 4096)) for m in (1, 5, 64, 129, 1000)]
                         + [(8192, 768, 3072)])
def test_two_residual_epilogue_exact(M, N, K, with_ws):
    """bf16(bf16(bf16(acc + bias) + attn) + x), also with the stream-K scratch and written over x in place."""
    L, lib = _lib()
    a, w, b = _int_operands(M, N, K, M + N + K, lo=-2, hi=3)
    g = torch.Generator().manual_seed(M)
    attn = (torch.randn(M, N, generator=g) * 4).to(torch.bfloat16)
    x = (torch.randn(M, N, generator=g) * 8).to(torch.bfloat16)
    ws = torch.zeros(int(lib.sk_gemm_ws_bytes()), device=DEV, dtype=torch.uint8) if with_ws else None
    xd, ad, wd, bd, attd = x.to(DEV), a.to(DEV), w.to(DEV), b.to(DEV), attn.to(DEV)
    L.check(lib.sk_linear_res2(M, N, K, L.ptr(ad), L.ptr(wd), L.ptr(bd), L.ptr(attd), L.ptr(xd), L.ptr(xd), L.ptr(ws),
                               C.c_int64(ws.numel() if ws is not None else 0), L.stream_ptr()))
    mlp = (a.float() @ w.float().T + b.float()).to(torch.bfloat16)
    ref = ((mlp.float() + attn.float()).to(torch.bfloat16).float() + x.float()).to(torch.bfloat16)
    assert torch.equal(xd.cpu().view(torch.int16), ref.view(torch.int16))


def test_neox_gemm_plans_and_argument_checks():
    """The new epilogues run on whole 64-column tiles of the existing widths (no 192 / 224 for the GELU pair), and the
    launchers refuse what they cannot do."""
    L, lib = _lib()
    plan = L.SkGemmPlan()
    for kind, (M, N, K) in ((1, (8192, 3072, 768)), (2, (8192, 3072, 768)), (1, (4, 4096, 1024))):
        L.check(lib.sk_neox_gemm_plan(kind, M, N, K, 0, C.byref(plan)))
        assert plan.bn in (64, 128, 256) and plan.tma_store == 1
    L.check(lib.sk_neox_gemm_plan(0, 8192, 2304, 768, 0, C.byref(plan)))
    assert plan.bn % 64 == 0
    L.check(lib.sk_neox_gemm_plan(3, 8, 768, 3072, 1, C.byref(plan)))
    assert plan.splits == 1
    t = torch.zeros(64, 64, device=DEV, dtype=torch.bfloat16)
    # GELU forward needs N % 64 == 0
    assert lib.sk_linear_gelu_fwd(64, 40, 64, L.ptr(t), L.ptr(t), None, L.ptr(t), L.ptr(t), L.stream_ptr()) != 0
    assert lib.sk_linear_rope_partial(64, 192, 64, L.ptr(t), L.ptr(t), None, L.ptr(t), L.ptr(t), L.ptr(t), None, 1, 128, 8,
                                      48, L.stream_ptr()) != 0
    assert b"rot_dims" in lib.sk_last_error()


@pytest.mark.parametrize("D", [128, 768, 1024, 2048])
@pytest.mark.parametrize("M", [1, 37, 1000])
def test_dual_layernorm(D, M):
    """Forward: each output bit-identical to a single-LN launch, shared mean / rstd equal.  Backward: dx and the four
    parameter gradients against fp64 per element."""
    L, lib = _lib()
    g = torch.Generator().manual_seed(D + M)
    x = (torch.randn(M, D, generator=g) * 2 + 0.3).to(torch.bfloat16).to(DEV)
    w1, w2 = ((1 + 0.2 * torch.randn(D, generator=g)).to(torch.bfloat16).to(DEV) for _ in range(2))
    b1, b2 = ((0.1 * torch.randn(D, generator=g)).to(torch.bfloat16).to(DEV) for _ in range(2))
    y1, y2, s1, s2 = (torch.empty(M, D, device=DEV, dtype=torch.bfloat16) for _ in range(4))
    mean, rstd, m1, r1 = (torch.empty(M, device=DEV) for _ in range(4))
    eps = L.f32(1e-5)
    L.check(lib.sk_layernorm2_fwd(L.ptr(x), L.ptr(w1), L.ptr(b1), L.ptr(w2), L.ptr(b2), L.ptr(y1), L.ptr(y2), L.ptr(mean),
                                  L.ptr(rstd), M, D, eps, L.stream_ptr()))
    L.check(lib.sk_layernorm_fwd(L.ptr(x), L.ptr(w1), L.ptr(b1), L.ptr(s1), L.ptr(m1), L.ptr(r1), M, D, eps, L.stream_ptr()))
    L.check(lib.sk_layernorm_fwd(L.ptr(x), L.ptr(w2), L.ptr(b2), L.ptr(s2), None, None, M, D, eps, L.stream_ptr()))
    assert torch.equal(y1, s1) and torch.equal(y2, s2) and torch.equal(mean, m1) and torch.equal(rstd, r1)

    dy1, dy2, dres = ((torch.randn(M, D, generator=g)).to(torch.bfloat16).to(DEV) for _ in range(3))
    dx = torch.empty(M, D, device=DEV, dtype=torch.bfloat16)
    grads = [torch.empty(D, device=DEV, dtype=torch.bfloat16) for _ in range(4)]
    part = torch.empty(4 * int(lib.sk_layernorm_bwd_blocks()) * D, device=DEV)
    L.check(lib.sk_layernorm2_bwd(L.ptr(dy1), L.ptr(dy2), L.ptr(x), L.ptr(w1), L.ptr(w2), L.ptr(mean), L.ptr(rstd),
                                  L.ptr(dres), L.ptr(dx), *[L.ptr(t) for t in grads], L.ptr(part), M, D, 0, L.stream_ptr()))
    xd = x.cpu().double().requires_grad_(True)
    W1, W2, B1, B2 = (t.cpu().double().requires_grad_(True) for t in (w1, w2, b1, b2))
    o1 = torch.nn.functional.layer_norm(xd, (D,), W1, B1, 1e-5)
    o2 = torch.nn.functional.layer_norm(xd, (D,), W2, B2, 1e-5)
    ((o1 * dy1.cpu().double()).sum() + (o2 * dy2.cpu().double()).sum() + (xd * dres.cpu().double()).sum()).backward()
    refs = [xd.grad, W1.grad, B1.grad, W2.grad, B2.grad]
    for got, ref in zip([dx] + grads, refs):
        got = got.cpu().double()
        # bf16 output rounding plus fp32 summation: 2^-8 relative per element, plus an fp32 accumulation term
        tol = ref.abs() * 2 ** -8 + 1e-4 * (ref.abs().max() + 1e-30) * max(1.0, (M / 64) ** 0.5)
        bad = (got - ref).abs() > tol
        assert not bool(bad.any()), (int(bad.sum()), float((got - ref).abs().max()))
    # accumulate adds onto the bf16 gradients
    prev = [t.clone() for t in grads]
    L.check(lib.sk_layernorm2_bwd(L.ptr(dy1), L.ptr(dy2), L.ptr(x), L.ptr(w1), L.ptr(w2), L.ptr(mean), L.ptr(rstd),
                                  None, L.ptr(dx), *[L.ptr(t) for t in grads], L.ptr(part), M, D, 1, L.stream_ptr()))
    for a, b in zip(grads, prev):
        assert rel_err(a.cpu(), 2 * b.cpu()) < 1e-2


# ---- CLIs ----------------------------------------------------------------------------------------------------------
def _tiny_neox_dir(path, twist: bool):
    """A tiny Pythia-style GPTNeoXForCausalLM (head_dim 64, partial_rotary_factor 0.25, untied) in `path`: weights when
    `twist`, the config only otherwise."""
    from transformers import GPTNeoXConfig, GPTNeoXForCausalLM
    cfg = GPTNeoXConfig(hidden_size=128, intermediate_size=512, num_hidden_layers=2, num_attention_heads=2,
                        max_position_embeddings=256, vocab_size=600, tie_word_embeddings=False,
                        rope_parameters={"rope_theta": 10000.0, "partial_rotary_factor": 0.25, "rope_type": "default"})
    if twist:
        torch.manual_seed(0)
        GPTNeoXForCausalLM(cfg).save_pretrained(str(path))
    else:
        cfg.save_pretrained(str(path))
    return str(path)


def test_cli_train_neox_packed_trains_saves_and_resumes(tmp_path):
    """cli/train.py with a GPT-NeoX base, model.tlm_type=b200, torch_dtype=bfloat16 and packed rows (the
    train_inter_scale recipe's data.packing=true): the loss falls, the checkpoint is a gpt_neox UnitLM, and a run resumed
    from checkpoint-4 ends with the same losses and the same weights."""
    import shutil
    from safetensors.torch import load_file
    from cli import train
    from test_gpu_round2 import _write_tokens
    base = _tiny_neox_dir(tmp_path / "base", twist=False)
    tok = str(tmp_path / "tok.jsonl")
    _write_tokens(tok, 40, 1)
    common = [f"data.train_path={tok}", f"data.val_path={tok}", "model=gslm", "model.tlm_type=b200",
              "model.context_len=64", f"model.config_args.base_model_name={base}", "model.config_args.torch_dtype=bfloat16",
              "data.packing=true", "training_args.per_device_train_batch_size=4", "+training_args.logging_steps=1",
              "training_args.warmup_steps=2", "training_args.warmup_ratio=0", "+training_args.save_steps=4",
              "+training_args.max_steps=8"]
    log_a = train.main(common + [f"training_args.output_dir={tmp_path}/a"])
    la = [r for r in log_a if "loss" in r]
    assert len(la) == 8 and la[-1]["loss"] < la[0]["loss"]
    c = json.load(open(tmp_path / "a" / "config.json"))
    assert c["base_config"]["model_type"] == "gpt_neox" and c["base_model_name"] == base
    assert c["base_config"]["rope_parameters"]["partial_rotary_factor"] == 0.25
    os.makedirs(tmp_path / "b")
    shutil.copytree(tmp_path / "a" / "checkpoint-4", tmp_path / "b" / "checkpoint-4")
    log_b = train.main(common + ["cont_training=true", f"training_args.output_dir={tmp_path}/b"])
    lb = [r for r in log_b if "loss" in r]
    assert [r["loss"] for r in la][-4:] == [r["loss"] for r in lb][-4:]
    a, b = load_file(str(tmp_path / "a" / "model.safetensors")), load_file(str(tmp_path / "b" / "model.safetensors"))
    assert set(a) == set(b) and all(torch.equal(a[k], b[k]) for k in a)
    # fp32 master weights are not implemented: the run stops instead of silently training bf16
    with pytest.raises(ValueError, match="torch_dtype"):
        train.main([x for x in common if "torch_dtype" not in x] + [f"training_args.output_dir={tmp_path}/c"])


def test_twist_init_neox_loads_hf_weights_and_eval_scores_it(tmp_path):
    """twist_init=true from a tiny random HF GPTNeoXForCausalLM: after the vocabulary resize the flat parameters equal
    HF's (the fused query_key_value round-trips through the [Q;K;V] permutation) and the logits follow HF's bf16 forward;
    the saved checkpoint is scored by cli/eval.py."""
    from transformers import GPTNeoXForCausalLM
    from slamkit_b200.integration import tlm_b200_from_cfg
    import cli.eval as E
    from test_gpu_eval import _write_clips
    base = _tiny_neox_dir(tmp_path / "hf", twist=True)
    cfg = {"context_len": 64, "config_args": {"base_model_name": base, "vocab_size": 502, "twist_init": True,
                                              "torch_dtype": "bfloat16", "pad_token_id": 0, "bos_token_id": 1,
                                              "eos_token_id": 1}}
    m = tlm_b200_from_cfg(cfg, device=DEV, max_batch=2, max_seq=64)
    assert m.is_neox and m.config.rot_dims == 16
    hf = GPTNeoXForCausalLM.from_pretrained(base, dtype=torch.bfloat16)
    hf.resize_token_embeddings(502)
    want = {"lm." + k: v for k, v in hf.state_dict().items()}
    got = m.state_dict_hf()
    assert set(got) == set(want)
    for k, v in want.items():
        assert torch.equal(got[k].cpu(), v), k
    ids, _ = _batch(2, 64, 17, pad_last=0)
    with torch.no_grad():
        ref = hf(input_ids=ids).logits
    assert rel_err(m.forward(ids).logits.cpu(), ref) < 8e-3
    ck = tmp_path / "ck"
    m.save_pretrained(str(ck), base_model_name=base)
    g = torch.Generator().manual_seed(13)
    sw = tmp_path / "swuggy"
    _write_clips(sw, [f"{d}/{i}_w.wav" for d in ("a", "b") for i in range(4)], g)
    res = E.main([f"model.pretrained_model={ck}", "+synthetic_weights=true", "batch_size=2", "num_workers=2",
                  "metric=swuggy_inter", f"metric.data_path={sw}"])
    assert set(res) == {"sWUGGY"} and 0.0 <= res["sWUGGY"] <= 1.0


def _res2_exact(M, N, K, ws):
    L, lib = _lib()
    a, w, b = _int_operands(M, N, K, M, lo=-2, hi=3)
    g = torch.Generator().manual_seed(M)
    attn = (torch.randn(M, N, generator=g) * 4).to(torch.bfloat16)
    x = (torch.randn(M, N, generator=g) * 8).to(torch.bfloat16)
    xd, ad, wd, bd, attd = x.to(DEV), a.to(DEV), w.to(DEV), b.to(DEV), attn.to(DEV)
    L.check(lib.sk_linear_res2(M, N, K, L.ptr(ad), L.ptr(wd), L.ptr(bd), L.ptr(attd), L.ptr(xd), L.ptr(xd), L.ptr(ws),
                               C.c_int64(ws.numel()), L.stream_ptr()))
    mlp = (a.float() @ w.float().T + b.float()).to(torch.bfloat16)
    ref = ((mlp.float() + attn.float()).to(torch.bfloat16).float() + x.float()).to(torch.bfloat16)
    assert torch.equal(xd.cpu().view(torch.int16), ref.view(torch.int16)), M


@pytest.mark.parametrize("M,N,K", [(8192, 768, 3072), (4096, 768, 3072), (5120, 1024, 4096)])
def test_two_residual_epilogue_on_stream_k(M, N, K):
    """With the scratch these shapes plan stream-K (the epilogue then runs in the owner CTA's fix-up path after the
    partial tiles are added): exact."""
    L, lib = _lib()
    plan = L.SkGemmPlan()
    L.check(lib.sk_neox_gemm_plan(3, M, N, K, 1, C.byref(plan)))
    assert plan.sk_units > 0 and plan.bn == 256, (plan.sk_units, plan.bn)
    _res2_exact(M, N, K, torch.zeros(int(lib.sk_gemm_ws_bytes()), device=DEV, dtype=torch.uint8))


def test_two_residual_exact_over_decode_range():
    """dense_4h_to_h at every decode size M = 1..129 (pythia-160m) with the decode step's scratch: exact.  (At these
    sizes the planner prefers 128-wide whole tiles, so no stream-K runs here; see the test above for that arm.)"""
    L, lib = _lib()
    N, K = 768, 3072
    ws = torch.zeros(int(lib.sk_gemm_ws_bytes()), device=DEV, dtype=torch.uint8)
    for M in range(1, 130):
        _res2_exact(M, N, K, ws)


def test_rope_and_gelu_epilogues_exact_over_decode_range():
    """The partial-RoPE q|k|v projection and the GELU forward / backward epilogues at every decode size M = 1..129."""
    from slamkit_b200.lm import rope_tables
    L, lib = _lib()
    cos, sin = rope_tables(10000.0, 16, 2048)
    cd, sd = cos.to(DEV), sin.to(DEV)
    for M in range(1, 130):
        N, K = 2304, 768
        x, w, b = _int_operands(M, N, K, 7 * M)
        pos = ((torch.arange(M, dtype=torch.int32) * 13 + M) % 2048)
        xd, wd, bd, pd = x.to(DEV), w.to(DEV), b.to(DEV), pos.to(DEV)
        out = torch.full((M, N), float("nan"), device=DEV, dtype=torch.bfloat16)
        L.check(lib.sk_linear_rope_partial(M, N, K, L.ptr(xd), L.ptr(wd), L.ptr(bd), L.ptr(out), L.ptr(cd), L.ptr(sd),
                                           L.ptr(pd), 1, 1536, 2048, 16, L.stream_ptr()))
        pre = (x.float() @ w.float().T + b.float()).to(torch.bfloat16)
        assert torch.equal(out.cpu().view(torch.int16), _rope_ref(pre, cos, sin, pos.long(), 16, 1536).view(torch.int16)), M
        F_, K2 = 3072, 768
        x, w, b = _int_operands(M, F_, K2, 11 * M)
        xd, wd, bd = x.to(DEV), w.to(DEV), b.to(DEV)
        pre_d, act = _gelu_fwd(M, F_, K2, xd, wd, bd)
        assert torch.equal(pre_d.cpu(), (x.float() @ w.float().T + b.float()).to(torch.bfloat16)), M
        assert int(_ulp_diff(act, torch.nn.functional.gelu(pre_d)).max()) <= 1, M
        dy = torch.randint(-3, 4, (M, K2), generator=torch.Generator().manual_seed(M)).to(torch.bfloat16).to(DEV)
        w2 = torch.randint(-3, 4, (K2, F_), generator=torch.Generator().manual_seed(M + 1)).to(torch.bfloat16).to(DEV)
        dpre = _gelu_bwd(M, K2, F_, dy, w2, pre_d)
        pr = pre_d.clone().requires_grad_(True)
        torch.nn.functional.gelu(pr).backward((dy.float() @ w2.float()).to(torch.bfloat16))
        assert int(_ulp_diff(dpre, pr.grad).max()) <= 1, M


def test_neox_decode_with_ffn_narrower_than_hidden():
    """A NeoX handle with ffn < hidden: the decode step's logits equal the forward pass's last-row logits (the decode
    workspace holds the pre-activation and ln2's output side by side for any ffn)."""
    from slamkit_b200.lm import DecodeSession
    c = O.OracleNeoxConfig(vocab_size=502, hidden=256, n_layers=2, n_heads=4, ffn=64, max_positions=64, rot_dims=32)
    m, p = _mk(c, 3, 2, 16, trainable=False)
    ids, _ = _batch(2, 9, 5, pad_last=0)
    sess = DecodeSession(m, 2, 16, 4)
    sess.prefill(ids[:, :8], torch.full((2,), 8))
    got = sess.step(ids[:, 8].to(DEV), torch.full((2,), 8, dtype=torch.int32, device=DEV)).clone()
    want = m.forward(ids).logits[:, -1]
    assert rel_err(got.cpu(), want.cpu()) < 1e-2
    ref = O.forward_logits(p, c, ids)[:, -1]
    assert rel_err(got.cpu(), ref) < 1e-2
