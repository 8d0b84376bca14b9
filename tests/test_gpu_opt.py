"""GPU parity of the OPT decoder (the reference's default TWIST / GSLM base) through the same `sk_lm_*` handle as Qwen2:
against tests/golden/opt_tiny.npz (the reference's own UnitLM over HF OPTForCausalLM) with the tolerances of
tests/test_gpu_lm.py, against oracle/opt_oracle.py at mid-size shapes, plus the new kernels on their own (LayerNorm,
the ReLU GEMM epilogue, the position-table gradient), the DPO entry points, cached generation and the CLIs."""
import json
import os

import numpy as np
import pytest
import torch

from helpers import rel_err, u16_to_bf16
from oracle import opt_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _lm_cfg(c: "O.OracleOptConfig"):
    from slamkit_b200.lm import OptLMConfig
    return OptLMConfig(vocab_size=c.vocab_size, hidden=c.hidden, n_layers=c.n_layers, n_heads=c.n_heads, ffn=c.ffn,
                       max_positions=c.max_positions, ln_eps=c.ln_eps, tie_embeddings=c.tie_embeddings)


def _mk(c, seed, max_batch, max_seq, trainable=True):
    from slamkit_b200.lm import B200UnitLM
    p = O.init_params(c, seed=seed)
    m = B200UnitLM(_lm_cfg(c), device=DEV, max_batch=max_batch, max_seq=max_seq, trainable=trainable)
    m.load_hf_state_dict(p)
    return m, p


def _golden(golden_dir):
    z = np.load(os.path.join(golden_dir, "opt_tiny.npz"))
    c = z["cfg"]
    cfg = O.OracleOptConfig(vocab_size=int(c[0]), hidden=int(c[1]), n_layers=int(c[2]), n_heads=int(c[3]), ffn=int(c[4]),
                            max_positions=int(c[5]))
    return z, cfg, int(c[6])


def _fp32_grads(p, c, *args, **kw):
    """The oracle's gradients with fp32 parameters and activations: the value both bf16 implementations approximate."""
    return O.forward_backward({k: v.float() for k, v in p.items()}, c, *args, **kw)[2]


def _check_grads(sd_g, grads_ref, grads_fp32, keys, tol=2e-2):
    """Every gradient within `tol` of the bf16 reference -- or, where the reference's own bf16 autograd noise exceeds that
    (at these tiny widths a few LayerNorm / projection gradients of the bf16 reference are 5-9 % away from fp32), at
    least as close to the fp32 gradient as the reference is.  The key biases are skipped: softmax is invariant to them,
    their true gradient is 0 and both sides hold rounding noise."""
    bad = []
    for k in keys:
        if k.endswith("k_proj.bias"):
            continue
        got = sd_g[k].cpu()
        e_ref = rel_err(got, grads_ref[k])
        if e_ref < tol:
            continue
        e_ours, e_theirs = rel_err(got, grads_fp32[k]), rel_err(grads_ref[k], grads_fp32[k])
        if e_ours > 1.25 * e_theirs + 5e-3:
            bad.append((k, round(e_ref, 4), round(e_ours, 4), round(e_theirs, 4)))
    assert not bad, bad


def test_opt_matches_reference_golden(golden_dir):
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
    ref_g = {k: u16_to_bf16(z["grad/" + k]).view_as(p[k]) for k in p}
    g32 = _fp32_grads(p, c, ids, labels, float(z["train/num_items"]))
    _check_grads(m.state_dict_hf(grads=True), ref_g, g32, p)
    opt = B200AdamW(m, lr=1e-3, max_grad_norm=0.5)
    opt.step()
    assert abs(float(opt.stats[0]) - float(z["train/total_norm"])) < 0.01 * float(z["train/total_norm"])
    sd_p = m.state_dict_hf()
    for k in p:
        if k.endswith("k_proj.bias"):
            continue
        # a first AdamW step moves each element by about lr * sign(grad): the update's direction element by element and
        # its mean size per tensor against the reference's
        upd = sd_p[k].cpu().float() - p[k].float()
        ref_sign = torch.from_numpy(z["upd_sign/" + k]).float().view_as(upd)
        ref_size = float(z["upd_absmean/" + k])
        assert abs(float(upd.abs().mean()) - ref_size) <= 0.2 * ref_size + 1e-9, k
        agree = (torch.sign(upd) == ref_sign).float().mean()
        if agree < 0.9:
            # the two part only where bf16 gradient noise flips the sign of a near-zero gradient: ours must point the
            # fp32 gradient's way about as often as the reference's does
            want = -torch.sign(g32[k])
            ours, theirs = (torch.sign(upd) == want).float().mean(), (ref_sign == want).float().mean()
            assert ours >= theirs - 0.03, (k, float(agree), float(ours), float(theirs))


def test_opt_packed_row_and_loglik_match_reference(golden_dir):
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
        ll2 = m.log_likelihood(tokens, mean_nll=mean).float().cpu()
        assert bool(((ll2 - ref).abs() <= 0.02 * ref.abs()).all())


def _batch(B, T, seed, pad_last=17):
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(2, 502, (B, T), generator=g)
    ids[:, 0] = 1
    if B > 1 and pad_last:
        ids[-1, T - pad_last:] = 0
    labels = ids.clone()
    labels[ids == 0] = -100
    return ids, labels


@pytest.mark.parametrize("B,T,layers", [(3, 200, 2), (1, 333, 1), (2, 130, 3)])
def test_opt_forward_backward_vs_oracle(B, T, layers):
    """Mid-size shapes (ragged T, right-padded rows): loss / logits / every gradient against the CPU oracle."""
    c = O.OracleOptConfig(vocab_size=502, hidden=256, n_layers=layers, n_heads=4, ffn=1024, max_positions=512)
    m, p = _mk(c, 5, B, T)
    ids, labels = _batch(B, T, B * 1000 + T)
    n = float((labels != -100).sum())
    ref_loss, ref_logits, ref_g = O.forward_backward(p, c, ids, labels, n)
    out = m.forward_backward(ids, labels, num_items_in_batch=n)
    assert abs(float(out.loss) - float(ref_loss)) < 1e-3 * abs(float(ref_loss))
    valid = ids != 0
    assert rel_err(m.logits_view(B, T).cpu()[valid], ref_logits[valid]) < 8e-3
    _check_grads(m.state_dict_hf(grads=True), ref_g, _fp32_grads(p, c, ids, labels, n), p)


def test_opt_packed_rows_and_accumulation_vs_oracle():
    """Packed rows (position_ids restart per document: block-diagonal attention, positions from pos_ids) against the
    oracle, and gradient accumulation: the same micro-batch twice gives twice the gradient."""
    c = O.OracleOptConfig(vocab_size=502, hidden=256, n_layers=2, n_heads=4, ffn=1024, max_positions=512)
    m, p = _mk(c, 6, 2, 160)
    g = torch.Generator().manual_seed(3)
    ids = torch.randint(2, 502, (2, 160), generator=g)
    pos = torch.cat([torch.cat([torch.arange(n) for n in (50, 1, 109)])[None],
                     torch.cat([torch.arange(n) for n in (160,)])[None]])
    labels = ids.clone()
    labels[pos == 0] = -100
    n = float((labels[:, 1:] != -100).sum())
    ref_loss, ref_logits, ref_g = O.forward_backward(p, c, ids, labels, n, position_ids=pos, packed=True)
    out = m.forward_backward(ids, labels, position_ids=pos, num_items_in_batch=n)
    assert abs(float(out.loss) - float(ref_loss)) < 1e-3 * abs(float(ref_loss))
    assert rel_err(m.logits_view(2, 160).cpu(), ref_logits) < 8e-3
    _check_grads(m.state_dict_hf(grads=True), ref_g, _fp32_grads(p, c, ids, labels, n, position_ids=pos, packed=True), p)
    one = m.grads.clone()
    m.forward_backward(ids, labels, position_ids=pos, num_items_in_batch=n, accumulate=True)
    assert rel_err(m.grads.float(), 2 * one.float()) < 1e-2


def test_opt_five_step_trajectory_vs_oracle():
    from slamkit_b200.lm import B200AdamW
    c = O.OracleOptConfig(vocab_size=502, hidden=128, n_layers=2, n_heads=2, ffn=512, max_positions=256)
    m, p = _mk(c, 9, 2, 96)
    tr = O.OracleOptTrainer(p, c, lr=1e-3, max_grad_norm=0.5)
    opt = B200AdamW(m, lr=1e-3, max_grad_norm=0.5)
    for s in range(5):
        ids, labels = _batch(2, 96, 100 + s)
        ref = tr.train_step(ids, labels)
        out = m.forward_backward(ids, labels, num_items_in_batch=float((labels != -100).sum()))
        opt.step()
        assert abs(float(out.loss) - ref) < 3e-3 * abs(ref), (s, float(out.loss), ref)
        assert abs(float(opt.stats[0]) - float(tr.last_total_norm)) < 0.02 * float(tr.last_total_norm), s


def test_opt_125m_geometry_is_finite_and_deterministic():
    """facebook/opt-125m geometry with the unit vocabulary at [8, 1024]: finite, and bit-identical run to run (loss,
    every gradient -- including the fixed-point position-table gradient -- and the logits)."""
    from slamkit_b200.lm import B200UnitLM, OptLMConfig
    m = B200UnitLM(OptLMConfig(), device=DEV, max_batch=8, max_seq=1024, seed=0)
    ids, labels = _batch(8, 1024, 1, pad_last=300)
    n = float((labels != -100).sum())
    runs = []
    for _ in range(2):
        out = m.forward_backward(ids, labels, num_items_in_batch=n)
        torch.cuda.synchronize()
        runs.append((float(out.loss), m.grads.clone(), m.logits_view(8, 1024).clone()))
    assert np.isfinite(runs[0][0]) and bool(torch.isfinite(runs[0][1].float()).all())
    assert runs[0][0] == runs[1][0]
    assert torch.equal(runs[0][1], runs[1][1]) and torch.equal(runs[0][2], runs[1][2])
    pos_g = m.tensor("pos_embed", grad=True)
    # positions 0..1022 get gradient; the last position feeds nothing (no target, no later query), nor do unused rows
    assert float(pos_g[2:2 + 1023].float().abs().sum(1).min()) > 0 and float(pos_g[2 + 1023:].float().abs().max()) == 0


@pytest.mark.parametrize("D", [128, 768, 2048])
@pytest.mark.parametrize("M", [1, 37, 1000])
def test_layernorm_vs_fp64(D, M):
    from slamkit_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(D + M)
    x = (torch.randn(M, D, generator=g) * 2 + 0.5).bfloat16().to(DEV)
    w = (1 + 0.2 * torch.randn(D, generator=g)).bfloat16().to(DEV)
    b = (0.1 * torch.randn(D, generator=g)).bfloat16().to(DEV)
    y, mean, rstd = ops.layernorm_fwd(x, w, b, 1e-5)
    xd = x.double()
    mu, var = xd.mean(-1, keepdim=True), xd.var(-1, unbiased=False, keepdim=True)
    xhat = (xd - mu) / torch.sqrt(var + 1e-5)
    ref = xhat * w.double() + b.double()
    # one bf16 rounding of the fp32 result: within one bf16 ulp of the fp64 value
    assert float(((y.double() - ref).abs() / ref.abs().clamp_min(1e-3)).max()) < 2 ** -7
    assert rel_err(mean.cpu(), mu.flatten().cpu()) < 1e-6 and rel_err(rstd.cpu(), (1 / torch.sqrt(var + 1e-5)).flatten().cpu()) < 1e-5
    dy = torch.randn(M, D, generator=g).bfloat16().to(DEV)
    dres = torch.randn(M, D, generator=g).bfloat16().to(DEV)
    dw = torch.zeros(D, device=DEV, dtype=torch.bfloat16)
    db = torch.zeros(D, device=DEV, dtype=torch.bfloat16)
    dx = ops.layernorm_bwd(dy, x, w, mean, rstd, dres, dw, db, False)
    gd = dy.double() * w.double()
    r = 1 / torch.sqrt(var + 1e-5)
    dx_ref = r * (gd - gd.mean(-1, keepdim=True) - xhat * (gd * xhat).mean(-1, keepdim=True)) + dres.double()
    assert rel_err(dx, dx_ref) < 5e-3
    assert rel_err(dw, (dy.double() * xhat).sum(0)) < 5e-3
    assert rel_err(db, dy.double().sum(0)) < 5e-3
    dw2, db2 = dw.clone(), db.clone()
    dx2 = ops.layernorm_bwd(dy, x, w, mean, rstd, dres, dw2, db2, True)       # accumulate: adds, bit-identical dx
    assert torch.equal(dx, dx2)
    assert rel_err(dw2, 2 * dw.double()) < 1e-2 and rel_err(db2, 2 * db.double()) < 1e-2
    dw3, db3 = torch.zeros_like(dw), torch.zeros_like(db)
    ops.layernorm_bwd(dy, x, w, mean, rstd, dres, dw3, db3, False)
    assert torch.equal(dw3, dw) and torch.equal(db3, db)                        # fixed-order partials: deterministic


@pytest.mark.parametrize("M,N,K,streamk", [(130, 3072, 768, False), (1, 768, 3072, True), (8192, 3072, 768, False),
                                           (64, 768, 3072, True), (300, 256, 128, False)])
def test_relu_epilogue_exact(M, N, K, streamk):
    """act = 2: out = bf16(relu(acc + bias)) bit for bit on integer operands (exact fp32 accumulator), with and without
    a residual; reports the schedule each case runs."""
    import gemm_ref as R
    from slamkit_b200 import ops
    a = R.int_operand(M, K, 3, seed=M + N, device=DEV)
    b = R.int_operand(N, K, 3, seed=K, device=DEV)
    bias = R.real_operand((N,), R.acc_scale(K, 3), seed=N, device=DEV)
    acc = R.exact_acc(a, b)
    plan = ops.gemm_plan(a, b, bias=bias, act=2, streamk=streamk)
    print(f"relu M={M} N={N} K={K}: {R.schedule_kind(plan, K)} {plan}")
    out = ops.gemm(a, b, bias=bias, act=2, streamk=streamk)
    want = R.bf16_round(torch.clamp_min(acc.float() + bias.float(), 0.0))
    err = R.mismatch_exact(out, want, plan["bn"], "relu")
    assert err is None, err
    # bias + ReLU must match act = 0 followed by a ReLU exactly (the rounding commutes)
    plain = ops.gemm(a, b, bias=bias, act=0, streamk=streamk)
    assert torch.equal(out, torch.relu(plain))


def test_position_gradient_is_deterministic_and_ordered():
    """The position table's gradient (64-bit fixed point, order-independent): bit-identical run to run, equal to the
    oracle's, and with positions from pos_ids it lands on row position + 2."""
    c = O.OracleOptConfig(vocab_size=502, hidden=128, n_layers=1, n_heads=2, ffn=256, max_positions=128)
    m, p = _mk(c, 4, 4, 100)
    ids, labels = _batch(4, 100, 8)
    n = float((labels != -100).sum())
    gs = []
    for _ in range(3):
        m.forward_backward(ids, labels, num_items_in_batch=n)
        gs.append(m.tensor("pos_embed", grad=True).clone())
    assert torch.equal(gs[0], gs[1]) and torch.equal(gs[0], gs[2])
    _, _, ref_g = O.forward_backward(p, c, ids, labels, n)
    k = "lm.model.decoder.embed_positions.weight"
    _check_grads({k: gs[0]}, ref_g, _fp32_grads(p, c, ids, labels, n), [k])
    pos = torch.arange(100).repeat(4, 1) + 7
    m.forward_backward(ids, labels, position_ids=pos, num_items_in_batch=n)
    g = m.tensor("pos_embed", grad=True).float()
    assert float(g[:9].abs().max()) == 0 and float(g[9:9 + 99].abs().sum(1).min()) > 0 and float(g[9 + 99:].abs().max()) == 0


def test_opt_dpo_entry_points_vs_oracle_autograd():
    """sk_lm_forward_rows / sk_lm_backward_weighted (the DPO path) against oracle autograd with per-row weights."""
    from slamkit_b200 import _lib as L
    c = O.OracleOptConfig(vocab_size=502, hidden=128, n_layers=2, n_heads=2, ffn=256, max_positions=256)
    m, p = _mk(c, 12, 4, 64)
    ids, labels = _batch(4, 64, 21)
    w = torch.tensor([0.7, -0.3, 0.25, -1.1])
    ids_d, lab_d = ids.to(DEV), labels.to(DEV)
    row_nll = torch.empty(4 * 64, device=DEV)
    L.check(m.lib.sk_lm_forward_rows(m._h, L.ptr(ids_d), L.ptr(lab_d), None, 4, 64, L.ptr(row_nll), L.ptr(m.stats),
                                     L.stream_ptr()))
    ref_loss, ref_logits, ref_g = O.forward_backward(p, c, ids, labels, row_weight=w)
    ref_nll = torch.nn.functional.cross_entropy(ref_logits.float()[:, :-1].reshape(-1, 502), labels[:, 1:].reshape(-1),
                                                reduction="none", ignore_index=-100).view(4, 63).sum(-1)
    assert rel_err(row_nll.view(4, 64).sum(-1).cpu(), ref_nll) < 2e-3
    rw = w.to(DEV).repeat_interleave(64).contiguous()
    L.check(m.lib.sk_lm_backward_weighted(m._h, L.ptr(ids_d), L.ptr(lab_d), None, 4, 64, L.ptr(rw), 0, L.ptr(m.stats),
                                          L.stream_ptr()))
    _check_grads(m.state_dict_hf(grads=True), ref_g, _fp32_grads(p, c, ids, labels, row_weight=w), p, tol=3e-2)


def test_opt_cached_generate_follows_oracle_and_graph_replay_equals_eager():
    from slamkit_b200 import _lib as L
    from slamkit_b200.lm import DecodeSession
    c = O.OracleOptConfig(vocab_size=502, hidden=128, n_layers=2, n_heads=2, ffn=256, max_positions=64)
    m, p = _mk(c, 2, 3, 64, trainable=False)
    g = torch.Generator().manual_seed(4)
    prompt = torch.randint(2, 502, (3, 10), generator=g)
    mask = torch.ones(3, 10, dtype=torch.long)
    mask[1, :4] = 0
    mask[2, :9] = 0
    out = m.generate(prompt, attention_mask=mask, max_new_tokens=20, do_sample=False, eos_token_id=None)
    assert out.shape == (3, 30)
    for r, start in enumerate((0, 4, 9)):
        lo = O.forward_logits(p, c, out[r:r + 1, start:].cpu())[0].float()
        for i, tok in enumerate(out[r, 10:].tolist()):
            row = lo[10 - start - 1 + i]
            assert float(row[tok]) >= float(row.max()) - 0.02 * float(row.max() - row.min()), (r, i)
    # each row alone gives the same continuation (batch invariance of the decode path)
    for r in range(3):
        alone = m.generate(prompt[r:r + 1], attention_mask=mask[r:r + 1], max_new_tokens=20, do_sample=False,
                           eos_token_id=None)
        assert torch.equal(alone[0, 10:], out[r, 10:].to(alone.device)), r
    with pytest.raises(ValueError, match="learned positions"):
        m.generate(prompt, attention_mask=mask, max_new_tokens=60, do_sample=False, eos_token_id=None)
    lens = mask.sum(1)
    right = torch.zeros(3, 10, dtype=torch.long)
    for r, n in enumerate(lens.tolist()):
        right[r, :n] = prompt[r, 10 - n:]
    cfg = L.SkSampling(seed=5, top_p=1.0, temperature=1.0, do_sample=0, top_k=0, n_eos=0, pad_token_id=0, max_length=40)
    runs = []
    for use_graph in (False, True):
        sess = DecodeSession(m, 3, 40, 24)
        sess.prefill(right, lens)
        sess.select(cfg)
        sess.step()
        sess.select(cfg)
        if use_graph:
            gr = torch.cuda.CUDAGraph()
            with torch.cuda.graph(gr):
                sess.step()
                sess.select(cfg)
            for _ in range(20):
                gr.replay()
        else:
            for _ in range(20):
                sess.step()
                sess.select(cfg)
        torch.cuda.synchronize()
        runs.append((sess.out.clone(), sess.logits.clone()))
    assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])


def test_opt_bind_and_entry_point_guards():
    """An OPT handle binds without RoPE tables and reports its own flat layout; a Qwen2 handle still needs them."""
    import ctypes as C
    from slamkit_b200 import _lib as L
    from slamkit_b200.lm import B200UnitLM, LMConfig
    c = O.OracleOptConfig(vocab_size=502, hidden=128, n_layers=1, n_heads=2, ffn=256, max_positions=100)
    m, _ = _mk(c, 1, 1, 16)
    assert m.tensors["pos_embed"][1:] == (102, 128) and "ln1_b" in "".join(m.tensors)
    q = B200UnitLM(LMConfig(vocab_size=502, hidden=128, n_layers=1, n_heads=2, n_kv_heads=1, ffn=256), device=DEV,
                   max_batch=1, max_seq=16)
    assert m.lib.sk_lm_bind(q._h, L.ptr(q.params), L.ptr(q.grads), None, None, L.ptr(q.workspace),
                            C.c_int64(q.workspace.numel())) == -1
    bad = L.SkOptConfig(502, 96, 1, 2, 256, 100, 1e-5, 1)                   # head_dim 48
    h = C.c_void_p()
    assert m.lib.sk_lm_create_opt(C.byref(bad), C.byref(h)) == -1
    assert b"head_dim" in m.lib.sk_last_error()


# ---- CLIs ----------------------------------------------------------------------------------------------------------
def _tiny_opt_dir(path, twist: bool):
    from transformers import OPTConfig, OPTForCausalLM
    cfg = OPTConfig(hidden_size=128, ffn_dim=256, num_hidden_layers=2, num_attention_heads=2, word_embed_proj_dim=128,
                    max_position_embeddings=256, vocab_size=600)
    if twist:
        torch.manual_seed(0)
        OPTForCausalLM(cfg).save_pretrained(str(path))
    else:
        cfg.save_pretrained(str(path))
    return str(path)


def _opt_train_args(base, twist):
    return ["model=gslm" if not twist else "model=twist", "model.tlm_type=b200", "model.context_len=64",
            f"model.config_args.base_model_name={base}", "model.config_args.torch_dtype=bfloat16",
            "training_args.per_device_train_batch_size=4", "+training_args.logging_steps=1",
            "training_args.warmup_steps=2", "training_args.warmup_ratio=0"]


def test_cli_train_gslm_opt_trains_saves_and_resumes(tmp_path):
    import shutil
    from safetensors.torch import load_file
    from cli import train
    from test_gpu_round2 import _write_tokens
    base = _tiny_opt_dir(tmp_path / "base", twist=False)
    tok = str(tmp_path / "tok.jsonl")
    _write_tokens(tok, 40, 1)
    common = [f"data.train_path={tok}", f"data.val_path={tok}", *_opt_train_args(base, False),
              "+training_args.save_steps=4", "+training_args.max_steps=8"]
    log_a = train.main(common + [f"training_args.output_dir={tmp_path}/a"])
    la = [r for r in log_a if "loss" in r]
    assert len(la) == 8 and la[-1]["loss"] < la[0]["loss"]
    c = json.load(open(tmp_path / "a" / "config.json"))
    assert c["base_config"]["model_type"] == "opt" and c["base_model_name"] == base
    os.makedirs(tmp_path / "b")
    shutil.copytree(tmp_path / "a" / "checkpoint-4", tmp_path / "b" / "checkpoint-4")
    log_b = train.main(common + ["cont_training=true", f"training_args.output_dir={tmp_path}/b"])
    lb = [r for r in log_b if "loss" in r]
    assert [r["loss"] for r in la][-4:] == [r["loss"] for r in lb][-4:]
    a, b = load_file(str(tmp_path / "a" / "model.safetensors")), load_file(str(tmp_path / "b" / "model.safetensors"))
    assert set(a) == set(b) and all(torch.equal(a[k], b[k]) for k in a)


def test_twist_init_opt_loads_hf_weights_and_eval_scores_it(tmp_path):
    """twist_init=true from a tiny random HF OPTForCausalLM: the flat parameters equal HF's after the vocabulary resize;
    the saved checkpoint is scored by cli/eval.py."""
    from transformers import OPTForCausalLM
    from slamkit_b200.integration import tlm_b200_from_cfg
    import cli.eval as E
    from test_gpu_eval import _write_clips
    base = _tiny_opt_dir(tmp_path / "hf", twist=True)
    cfg = {"context_len": 64, "config_args": {"base_model_name": base, "vocab_size": 502, "twist_init": True,
                                              "dropout": 0.0, "attention_dropout": 0.0, "layerdrop": 0.0,
                                              "torch_dtype": "bfloat16", "pad_token_id": 0, "bos_token_id": 1,
                                              "eos_token_id": 1}}
    m = tlm_b200_from_cfg(cfg, device=DEV, max_batch=2, max_seq=64)
    hf = OPTForCausalLM.from_pretrained(base, dtype=torch.bfloat16)
    hf.resize_token_embeddings(502)
    want = {"lm." + k: v for k, v in hf.state_dict().items()}
    got = m.state_dict_hf()
    assert set(got) == set(want)
    for k, v in want.items():
        assert torch.equal(got[k].cpu(), v), k
    ck = tmp_path / "ck"
    m.save_pretrained(str(ck), base_model_name=base)
    g = torch.Generator().manual_seed(13)
    sw = tmp_path / "swuggy"
    _write_clips(sw, [f"{d}/{i}_w.wav" for d in ("a", "b") for i in range(4)], g)
    res = E.main([f"model.pretrained_model={ck}", "+synthetic_weights=true", "batch_size=2", "num_workers=2",
                  "metric=swuggy_inter", f"metric.data_path={sw}"])
    assert set(res) == {"sWUGGY"} and 0.0 <= res["sWUGGY"] <= 1.0
