"""OPT with fp32 master weights on the GPU (`B200UnitLM(..., master_weights=True)`, `sk_lm_set_master`): the reference's
default TWIST / GSLM precision -- fp32 parameters, gradients and AdamW moments under bf16 autocast -- against the
autocast oracle (oracle/opt_amp_oracle.py, pinned to the reference by tests/golden/opt_amp_tiny.npz), the new kernels on
their own, determinism, resume, the refusals and the training CLI."""
import ctypes as C
import json
import os

import numpy as np
import pytest
import torch

from helpers import rel_err
from oracle import opt_amp_oracle as A
from oracle import opt_oracle as O
from oracle.lm_oracle import adamw_step_, clip_grad_norm_

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SKIP = ("k_proj.bias",)   # softmax is invariant to the key bias: its true gradient is 0, both sides hold rounding noise


def _lm_cfg(c):
    from slamkit_b200.lm import OptLMConfig
    return OptLMConfig(vocab_size=c.vocab_size, hidden=c.hidden, n_layers=c.n_layers, n_heads=c.n_heads, ffn=c.ffn,
                       max_positions=c.max_positions, ln_eps=c.ln_eps, tie_embeddings=c.tie_embeddings)


def _mk(c, p, B, T, master=True, trainable=True):
    from slamkit_b200.lm import B200UnitLM
    m = B200UnitLM(_lm_cfg(c), device=DEV, max_batch=B, max_seq=T, trainable=trainable, master_weights=master)
    m.load_hf_state_dict(p)
    return m


def _batch(B, T, seed, pad_last=17):
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(2, 502, (B, T), generator=g)
    ids[:, 0] = 1
    if B > 1 and pad_last:
        ids[-1, T - pad_last:] = 0
    labels = ids.clone()
    labels[ids == 0] = -100
    return ids, labels


def _grad_errors(m, ref_g):
    sd = m.state_dict_hf(grads=True)
    return {k: rel_err(sd[k].float().cpu(), ref_g[k]) for k in ref_g if not k.endswith(SKIP)}


# Bounds of the master path against the autocast oracle.  Both run bf16 GEMMs on the same bf16 weights over the same fp32
# residual and differ in summation order only, but at these widths a flipped bf16 rounding in attention or a GEMM output
# carries through the backward pass: single gradient tensors sit up to ~5 % away (GRAD_TOL per tensor).  The bf16 path
# (bf16 parameters, embeddings and residual) is further from the same oracle, and the tests assert that gap: the master
# path's logit error and mean gradient error are at most GAP of the bf16 path's (measured on an H100: 0.58-0.66).
GRAD_TOL = 8e-2
GAP = 0.8


@pytest.mark.parametrize("B,T,layers", [(3, 200, 2), (1, 333, 1), (2, 130, 3)])
def test_master_forward_backward_vs_amp_oracle(B, T, layers):
    c = O.OracleOptConfig(vocab_size=502, hidden=256, n_layers=layers, n_heads=4, ffn=1024, max_positions=512)
    p = A.init_params_fp32(c, seed=5)
    ids, labels = _batch(B, T, B * 1000 + T)
    n = float((labels != -100).sum())
    ref_loss, ref_logits, ref_g = A.forward_backward_amp(p, c, ids, labels, n)
    m = _mk(c, p, B, T)
    out = m.forward_backward(ids, labels, num_items_in_batch=n)
    valid = ids != 0
    e_loss = abs(float(out.loss) - float(ref_loss)) / abs(float(ref_loss))
    e_logits = rel_err(m.logits_view(B, T).cpu()[valid], ref_logits[valid])
    errs = _grad_errors(m, ref_g)
    assert all(m.tensor(k, grad=True).dtype == torch.float32 for k in ("embed", "layers.0.ln1", "layers.0.w1"))
    b = _mk(c, p, B, T, master=False)
    ob = b.forward_backward(ids, labels, num_items_in_batch=n)
    b_logits = rel_err(b.logits_view(B, T).cpu()[valid], ref_logits[valid])
    b_errs = _grad_errors(b, ref_g)
    report = {"loss": e_loss, "logits": e_logits, "bf16_logits": b_logits, "grad_max": max(errs.values()),
              "grad_mean": float(np.mean(list(errs.values()))), "bf16_grad_mean": float(np.mean(list(b_errs.values()))),
              "bf16_loss": abs(float(ob.loss) - float(ref_loss)) / abs(float(ref_loss))}
    print("master vs amp oracle", B, T, layers, json.dumps(report))
    assert e_loss < 1e-4, report
    assert e_logits < 6e-3, report
    bad = {k: v for k, v in errs.items() if v > GRAD_TOL}
    assert not bad, (bad, report)
    # the mode changes the numerics: the bf16 path is measurably further from the same oracle
    assert e_logits <= GAP * b_logits and report["grad_mean"] <= GAP * report["bf16_grad_mean"], report


def test_master_packed_rows_and_two_micro_batches_vs_amp_oracle():
    c = O.OracleOptConfig(vocab_size=502, hidden=256, n_layers=2, n_heads=4, ffn=1024, max_positions=512)
    p = A.init_params_fp32(c, seed=6)
    g = torch.Generator().manual_seed(3)
    ids = torch.randint(2, 502, (2, 160), generator=g)
    pos = torch.cat([torch.cat([torch.arange(n) for n in (50, 1, 109)])[None],
                     torch.cat([torch.arange(n) for n in (160,)])[None]])
    labels = ids.clone()
    labels[pos == 0] = -100
    ids2, labels2 = _batch(2, 160, 77)
    n = float((labels[:, 1:] != -100).sum() + (labels2[:, 1:] != -100).sum())
    tr = A.OracleOptAmpTrainer(p, c)
    ref_g = tr.accumulate([(ids, labels, pos, True), (ids2, labels2)], n)
    m = _mk(c, p, 2, 160)
    o1 = float(m.forward_backward(ids, labels, position_ids=pos, num_items_in_batch=n).loss)
    o2 = float(m.forward_backward(ids2, labels2, num_items_in_batch=n, accumulate=True).loss)
    for ours, ref in zip((o1, o2), tr.losses):
        assert abs(ours - ref) < 2e-4 * abs(ref), (ours, ref)
    errs = _grad_errors(m, ref_g)
    print("packed + 2 micro-batches, gradient errors:", json.dumps({k: round(v, 4) for k, v in errs.items()}))
    bad = {k: v for k, v in errs.items() if v > GRAD_TOL}
    assert not bad, bad


def test_master_five_step_trajectory_and_shadow():
    """5 clip + AdamW steps: the fp32 masters follow the oracle's; after every step the bf16 shadow is bf16(master)."""
    from slamkit_b200.lm import B200AdamW
    c = O.OracleOptConfig(vocab_size=502, hidden=128, n_layers=2, n_heads=2, ffn=512, max_positions=256)
    p = A.init_params_fp32(c, seed=9)
    m = _mk(c, p, 2, 96)
    tr = A.OracleOptAmpTrainer(p, c, lr=1e-3, max_grad_norm=0.5)
    opt = B200AdamW(m, lr=1e-3, max_grad_norm=0.5)
    assert opt.exp_avg.dtype == torch.float32 and opt.exp_avg.numel() == m.n_params
    for s in range(5):
        ids, labels = _batch(2, 96, 100 + s)
        ref = tr.train_step(ids, labels)
        out = m.forward_backward(ids, labels, num_items_in_batch=float((labels != -100).sum()))
        opt.step()
        assert abs(float(out.loss) - ref) < 1e-3 * abs(ref), (s, float(out.loss), ref)
        assert abs(float(opt.stats[0]) - float(tr.last_total_norm)) < 5e-3 * float(tr.last_total_norm), s
        assert torch.equal(m.params, m.params32.to(torch.bfloat16)), s
    sd = m.state_dict_hf()
    # the 5-step update of every tensor (up to 5 lr per element) against the oracle's: Adam's sign-like steps turn the
    # gradients' few-% noise into ~10 % on the update (elements with near-zero gradients may step the other way; measured
    # on an H100: mean 0.10, max 0.19 over the tensors)
    errs = {k: rel_err(sd[k].cpu() - p[k], tr.p[k] - p[k]) for k in p if not k.endswith(SKIP)}
    print("5-step update errors:", json.dumps({k: round(v, 4) for k, v in errs.items()}))
    assert all(sd[k].dtype == torch.float32 for k in p)
    assert max(errs.values()) < 0.3 and float(np.mean(list(errs.values()))) < 0.15, errs


def test_master_keeps_learning_where_bf16_rounds_updates_away():
    """lr = 5e-5 (the recipe's min_lr) on trained-scale weights (std 0.05, LayerNorm gains near 1): every master element
    with a gradient moves, while the bf16 path leaves most weights and every LayerNorm gain where they were (an update
    below half a bf16 ulp rounds away)."""
    from slamkit_b200.lm import B200AdamW
    c = O.OracleOptConfig(vocab_size=502, hidden=256, n_layers=2, n_heads=4, ffn=1024, max_positions=256)
    p = A.init_params_fp32(c, seed=11, std=0.05)
    ids, labels = _batch(4, 128, 5)
    n = float((labels != -100).sum())
    moved = {}
    for master in (True, False):
        m = _mk(c, p, 4, 128, master=master)
        before = m.state_dict_hf()
        m.forward_backward(ids, labels, num_items_in_batch=n)
        grads = m.state_dict_hf(grads=True)
        B200AdamW(m, lr=5e-5, max_grad_norm=0.5).step()
        after = m.state_dict_hf()
        w_keys = [k for k in p if ".layers." in k and k.endswith("weight")]
        ln = [k for k in w_keys if "layer_norm" in k]
        lin = [k for k in w_keys if "layer_norm" not in k]
        has_g = {k: grads[k] != 0 for k in w_keys}
        frac = lambda ks: float(sum(int(((after[k] != before[k]) & has_g[k]).sum()) for k in ks) /
                                sum(int(has_g[k].sum()) for k in ks))
        moved[master] = (frac(lin), frac(ln))
    print("moved fraction (linear, layernorm): master", moved[True], "bf16", moved[False])
    assert moved[True][0] > 0.99 and moved[True][1] > 0.99, moved
    assert moved[False][0] < 0.5 and moved[False][1] == 0.0, moved


# ---- kernels on their own --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("D", [128, 768, 2048])
@pytest.mark.parametrize("M", [1, 37, 1000])
def test_add_layernorm_and_backward_f32_vs_fp64(D, M):
    from slamkit_b200 import _lib as L
    lib = L.require_cuda()
    g = torch.Generator(device="cpu").manual_seed(D + M)
    x = (torch.randn(M, D, generator=g) * 2 + 0.5).to(DEV)
    y = torch.randn(M, D, generator=g).bfloat16().to(DEV)
    w = (1 + 0.2 * torch.randn(D, generator=g)).to(DEV)
    b = (0.1 * torch.randn(D, generator=g)).to(DEV)
    xo = torch.empty_like(x)
    h = torch.empty(M, D, device=DEV, dtype=torch.bfloat16)
    mean, rstd = torch.empty(M, device=DEV), torch.empty(M, device=DEV)
    s = L.stream_ptr()
    L.check(lib.sk_add_layernorm_f32(L.ptr(x), L.ptr(y), L.ptr(w), L.ptr(b), L.ptr(xo), L.ptr(h), L.ptr(mean), L.ptr(rstd),
                                     M, D, L.f32(1e-5), s))
    assert torch.equal(xo, x + y.float())                 # fp32 + bf16 -> fp32, one rounding
    xd = xo.double()
    mu, var = xd.mean(-1, keepdim=True), xd.var(-1, unbiased=False, keepdim=True)
    xhat = (xd - mu) / torch.sqrt(var + 1e-5)
    ref = xhat * w.double() + b.double()
    # one bf16 rounding of the fp32 result: within one bf16 ulp of the fp64 value
    assert float(((h.double() - ref).abs() / ref.abs().clamp_min(1e-3)).max()) < 2 ** -7
    assert rel_err(mean.cpu(), mu.flatten().cpu()) < 1e-6 and rel_err(rstd.cpu(), (1 / torch.sqrt(var + 1e-5)).flatten().cpu()) < 1e-5
    h0 = torch.empty_like(h)                              # without y: LayerNorm of x itself
    L.check(lib.sk_add_layernorm_f32(L.ptr(xo), None, L.ptr(w), L.ptr(b), None, L.ptr(h0), None, None, M, D, L.f32(1e-5), s))
    assert torch.equal(h0, h)
    dy = torch.randn(M, D, generator=g).bfloat16().to(DEV)
    dres = torch.randn(M, D, generator=g).to(DEV)
    part = torch.empty(2 * lib.sk_layernorm_bwd_blocks() * D, device=DEV)

    def bwd(dres_in, dres_out, dw, db, acc):
        d16 = torch.empty(M, D, device=DEV, dtype=torch.bfloat16)
        L.check(lib.sk_layernorm_bwd_f32(L.ptr(dy), L.ptr(xo), L.ptr(w), L.ptr(mean), L.ptr(rstd), L.ptr(dres_in), L.ptr(dres_out),
                                         L.ptr(d16), L.ptr(dw), L.ptr(db), L.ptr(part), M, D, int(acc), s))
        return d16
    out = torch.empty_like(dres)
    dw, db = torch.zeros(D, device=DEV), torch.zeros(D, device=DEV)
    d16 = bwd(dres, out, dw, db, False)
    gd = dy.double() * w.double()
    r = 1 / torch.sqrt(var + 1e-5)
    dx_ref = r * (gd - gd.mean(-1, keepdim=True) - xhat * (gd * xhat).mean(-1, keepdim=True)) + dres.double()
    assert rel_err(out, dx_ref) < 1e-5
    assert torch.equal(d16, out.to(torch.bfloat16))
    assert rel_err(dw, (dy.double() * xhat).sum(0)) < 2e-5 and rel_err(db, dy.double().sum(0)) < 2e-5
    dw2, db2 = dw.clone(), db.clone()
    inplace = dres.clone()
    bwd(inplace, inplace, dw2, db2, True)                 # in place on dres, accumulating dw / db
    assert torch.equal(inplace, out)
    assert torch.equal(dw2, 2 * dw) and torch.equal(db2, 2 * db)   # same fixed-order sums, added once
    z = torch.empty_like(dres)
    bwd(None, z, torch.zeros_like(dw), torch.zeros_like(db), False)
    assert rel_err(z, dx_ref - dres.double()) < 1e-5


def _adamw_strict(p, g, m, v, *, lr, beta1, beta2, eps, weight_decay, step):
    """adamw_step_'s fp32 arithmetic in numpy, one IEEE operation at a time (numpy's float32 sqrt is correctly rounded;
    torch's vectorised CPU sqrt is not on every CPU, so adamw_step_ itself can differ from this in the last bit)."""
    F = np.float32
    p, g, m, v = (t.numpy().astype(np.float32) for t in (p, g, m, v))
    bc1 = 1 - beta1 ** step
    p = p - F(lr * weight_decay) * p
    m = m + F(1 - beta1) * (g - m)
    v = F(beta2) * v + (F(1 - beta2) * g) * g
    den = np.sqrt(v) / F(np.sqrt(1 - beta2 ** step)) + F(eps)
    return p - (F(lr / bc1) * m) / den, m, v


def test_master_adamw_is_bit_identical_to_the_oracle():
    """sk_adamw_master_step on fp32 tensors, with a clip coefficient, weight decay and a step > 1: bit for bit equal to
    oracle/lm_oracle.adamw_step_'s arithmetic rounded one IEEE operation at a time; against adamw_step_ itself the
    moments are bit-identical and the parameters within one ulp (torch's CPU sqrt).  The hyperparameters are fp32 values
    (the C ABI passes fp32) given to the oracle as Python floats, so both form 1 - beta, lr * wd, lr / bc1 and sqrt(bc2)
    in double from the same numbers."""
    from slamkit_b200 import _lib as L
    lib = L.require_cuda()
    g = torch.Generator().manual_seed(1)
    n = 100_000
    p = torch.randn(n, generator=g) * 0.05
    gr = torch.randn(n, generator=g) * 1e-3
    m = torch.randn(n, generator=g) * 1e-4
    v = torch.rand(n, generator=g) * 1e-6
    f = lambda x: float(np.float32(x))
    hp = dict(lr=f(3e-4), beta1=f(0.9), beta2=f(0.999), eps=f(1e-8), weight_decay=f(0.01), step=3)
    coef = f(0.7)
    pd, gd, md, vd = (t.clone().to(DEV) for t in (p, gr, m, v))
    shadow = torch.empty(n, device=DEV, dtype=torch.bfloat16)
    stats = torch.tensor([1.0, coef, 1.0], device=DEV)
    L.check(lib.sk_adamw_master_step(L.ptr(pd), L.ptr(shadow), L.ptr(gd), L.ptr(md), L.ptr(vd), C.c_int64(n), L.f32(hp["lr"]),
                                     L.f32(hp["beta1"]), L.f32(hp["beta2"]), L.f32(hp["eps"]), L.f32(hp["weight_decay"]),
                                     hp["step"], L.ptr(stats), L.stream_ptr()))
    g2 = gr * torch.tensor(coef)                           # clip_grad_norm_'s in-place scale, fp32
    sp, sm, sv = _adamw_strict(p, g2, m, v, **hp)
    assert np.array_equal(pd.cpu().numpy(), sp) and np.array_equal(md.cpu().numpy(), sm) and np.array_equal(vd.cpu().numpy(), sv)
    assert torch.equal(shadow.cpu(), pd.cpu().to(torch.bfloat16))
    adamw_step_(p, g2, m, v, **hp)
    assert torch.equal(md.cpu(), m) and torch.equal(vd.cpu(), v)
    big = torch.maximum(p.abs(), torch.tensor(hp["lr"]))
    assert bool(((pd.cpu() - p).abs() <= torch.nextafter(big, torch.tensor(float("inf"))) - big).all())


def test_fp32_grad_norm_vs_clip_grad_norm():
    from slamkit_b200 import _lib as L
    lib = L.require_cuda()
    g = torch.Generator().manual_seed(2)
    sizes, chunk = (100_000, 768, 50_048, 8), 16384
    offs, o = [], 0
    for sz in sizes:
        offs.append(o)
        o = (o + sz + 63) // 64 * 64
    flat = torch.zeros(o)
    parts = []
    for off, sz in zip(offs, sizes):
        t = torch.randn(sz, generator=g) * (0.1 + off % 7)
        flat[off:off + sz] = t
        parts.append(t.clone())
    cs, cl, tb = [], [], []
    for off, sz in zip(offs, sizes):
        tb.append(len(cs))
        for s in range(0, sz, chunk):
            cs.append(off + s)
            cl.append(min(chunk, sz - s))
    tb.append(len(cs))
    dev = lambda x, dt: torch.tensor(x, dtype=dt, device=DEV)
    cs_d, cl_d, tb_d = dev(cs, torch.int64), dev(cl, torch.int32), dev(tb, torch.int32)
    part = torch.empty(len(cs), device=DEV)
    stats = torch.empty(3, device=DEV)
    flat_d = flat.to(DEV)
    L.check(lib.sk_grad_norm_f32(L.ptr(flat_d), L.ptr(cs_d), L.ptr(cl_d), len(cs), L.ptr(tb_d), len(sizes), L.ptr(part),
                                 L.f32(0.5), L.ptr(stats), L.stream_ptr()))
    total = clip_grad_norm_(parts, 0.5)
    assert abs(float(stats[0]) - float(total)) <= 2e-6 * float(total)
    assert abs(float(stats[1]) - float(torch.clamp(0.5 / (total + 1e-6), max=1.0))) <= 2e-6 * float(stats[1])


# ---- determinism, resume, refusals ------------------------------------------------------------------------------------
def test_master_runs_are_bit_identical():
    c = O.OracleOptConfig(vocab_size=502, hidden=256, n_layers=2, n_heads=4, ffn=1024, max_positions=512)
    m = _mk(c, A.init_params_fp32(c, seed=3), 4, 300)
    ids, labels = _batch(4, 300, 8, pad_last=40)
    n = float((labels != -100).sum())
    runs = []
    for _ in range(2):
        out = m.forward_backward(ids, labels, num_items_in_batch=n)
        torch.cuda.synchronize()
        runs.append((float(out.loss), m.grads32.clone(), m.logits_view(4, 300).clone()))
    assert runs[0][0] == runs[1][0] and torch.equal(runs[0][1], runs[1][1]) and torch.equal(runs[0][2], runs[1][2])
    assert bool(torch.isfinite(runs[0][1]).all())


def test_master_resume_is_bit_identical(tmp_path):
    """4 trainer steps (2 micro-batches each) in one go, and 2 + save + reload (fp32 checkpoint, fp32 moments) + 2:
    the same fp32 masters, moments and shadow bit for bit."""
    from slamkit_b200.lm import B200UnitLM
    from slamkit_b200.trainer import B200Trainer
    c = O.OracleOptConfig(vocab_size=502, hidden=128, n_layers=2, n_heads=2, ffn=512, max_positions=256)
    p = A.init_params_fp32(c, seed=4)
    batches = [[dict(zip(("input_ids", "labels"), _batch(2, 64, 10 * s + i))) for i in range(2)] for s in range(4)]
    kw = dict(lr=1e-3, min_lr=5e-5, warmup_steps=1, total_steps=4, grad_accum=2)
    a = _mk(c, p, 2, 64)
    ta = B200Trainer(a, **kw)
    for mb in batches:
        ta.train_step(mb)
    b = _mk(c, p, 2, 64)
    tb = B200Trainer(b, **kw)
    for mb in batches[:2]:
        tb.train_step(mb)
    b.save_pretrained(str(tmp_path / "ck"))
    st = {k: (v.cpu() if torch.is_tensor(v) else v) for k, v in tb.state_dict().items()}
    assert st["exp_avg"].dtype == torch.float32
    del b, tb
    r = B200UnitLM.from_pretrained(str(tmp_path / "ck"), device=DEV, max_batch=2, max_seq=64, master_weights=True)
    tr = B200Trainer(r, **kw)
    tr.load_state_dict(st)
    for mb in batches[2:]:
        tr.train_step(mb)
    assert torch.equal(r.params32, a.params32) and torch.equal(r.params, a.params)
    assert torch.equal(tr.opt.exp_avg, ta.opt.exp_avg) and torch.equal(tr.opt.exp_avg_sq, ta.opt.exp_avg_sq)


def test_master_refusals_launch_nothing():
    from slamkit_b200 import _lib as L
    from slamkit_b200.dpo import B200DPOTrainer
    from slamkit_b200.hf_module import B200UnitLMModule
    from slamkit_b200.lm import B200UnitLM, DecodeSession, LMConfig, NeoxLMConfig
    c = O.OracleOptConfig(vocab_size=502, hidden=128, n_layers=1, n_heads=2, ffn=256, max_positions=64)
    m = _mk(c, A.init_params_fp32(c, seed=1), 2, 32)
    lib = m.lib
    q = B200UnitLM(LMConfig(vocab_size=502, hidden=128, n_layers=1, n_heads=2, n_kv_heads=1, ffn=256), device=DEV,
                   max_batch=1, max_seq=16)
    x = B200UnitLM(NeoxLMConfig(vocab_size=502, hidden=128, n_layers=1, n_heads=2, ffn=512, max_positions=64), device=DEV,
                   max_batch=1, max_seq=16)
    buf = torch.zeros(max(q.n_params, x.n_params), device=DEV)
    sess = DecodeSession(m, 2, 16, 4)
    torch.cuda.synchronize()
    n0 = lib.sk_launch_count()
    with pytest.raises(L.SkError, match="master weights"):
        sess.prefill(torch.ones(2, 4, dtype=torch.long), torch.tensor([4, 3]))
    with pytest.raises(L.SkError, match="master weights"):
        sess.step()
    with pytest.raises(NotImplementedError, match="master weights"):
        m.generate(torch.ones(1, 4, dtype=torch.long), max_new_tokens=3)
    for h in (q, x):
        assert lib.sk_lm_set_master(h._h, L.ptr(buf), L.ptr(buf)) == -1
        assert b"OPT decoder only" in lib.sk_last_error()
    assert lib.sk_launch_count() == n0, "a refused call launched a kernel"
    with pytest.raises(ValueError, match="OPT decoder only"):
        B200UnitLM(LMConfig(vocab_size=502, hidden=128, n_layers=1, n_heads=2, n_kv_heads=1, ffn=256), device=DEV,
                   max_batch=1, max_seq=16, master_weights=True)
    with pytest.raises(NotImplementedError):
        B200UnitLMModule(m)
    with pytest.raises(NotImplementedError):
        B200DPOTrainer(m, m)


# ---- CLI ---------------------------------------------------------------------------------------------------------------
def test_cli_train_gslm_float32_trains_saves_resumes_and_eval_scores(tmp_path):
    import shutil
    from safetensors.torch import load_file
    import cli.eval as E
    from cli import train
    from test_gpu_eval import _write_clips
    from test_gpu_opt import _opt_train_args, _tiny_opt_dir
    from test_gpu_round2 import _write_tokens
    base = _tiny_opt_dir(tmp_path / "base", twist=False)
    tok = str(tmp_path / "tok.jsonl")
    _write_tokens(tok, 40, 1)
    args = [a.replace("torch_dtype=bfloat16", "torch_dtype=float32") for a in _opt_train_args(base, False)]
    common = [f"data.train_path={tok}", f"data.val_path={tok}", *args, "+training_args.save_steps=4",
              "+training_args.max_steps=8"]
    with pytest.raises(ValueError, match=r"training_args\.bf16"):
        train.main(common + ["training_args.bf16=false", f"training_args.output_dir={tmp_path}/x"])
    log_a = train.main(common + [f"training_args.output_dir={tmp_path}/a"])
    la = [r for r in log_a if "loss" in r]
    assert len(la) == 8 and la[-1]["loss"] < la[0]["loss"]
    c = json.load(open(tmp_path / "a" / "config.json"))
    assert c["torch_dtype"] == "float32" and c["base_config"]["torch_dtype"] == "float32"
    sd = load_file(str(tmp_path / "a" / "model.safetensors"))
    assert all(v.dtype == torch.float32 for v in sd.values())
    opt = torch.load(str(tmp_path / "a" / "checkpoint-4" / "optimizer.pt"))
    assert opt["exp_avg"].dtype == torch.float32
    os.makedirs(tmp_path / "b")
    shutil.copytree(tmp_path / "a" / "checkpoint-4", tmp_path / "b" / "checkpoint-4")
    log_b = train.main(common + ["cont_training=true", f"training_args.output_dir={tmp_path}/b"])
    lb = [r for r in log_b if "loss" in r]
    assert [r["loss"] for r in la][-4:] == [r["loss"] for r in lb][-4:]
    b = load_file(str(tmp_path / "b" / "model.safetensors"))
    assert set(sd) == set(b) and all(torch.equal(sd[k], b[k]) for k in sd)
    g = torch.Generator().manual_seed(13)
    sw = tmp_path / "swuggy"
    _write_clips(sw, [f"{d}/{i}_w.wav" for d in ("a", "b") for i in range(4)], g)
    res = E.main([f"model.pretrained_model={tmp_path / 'a'}", "+synthetic_weights=true", "batch_size=2", "num_workers=2",
                  "metric=swuggy_inter", f"metric.data_path={sw}"])
    assert set(res) == {"sWUGGY"} and 0.0 <= res["sWUGGY"] <= 1.0
