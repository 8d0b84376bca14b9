"""GPU parity of the post-LayerNorm OPT decoder (facebook/opt-350m layout: LayerNorm after each residual add, no final
LayerNorm, bias-free project_in / project_out around a 512-wide tied head) through the same `sk_lm_*` handle as the other
decoders: against tests/golden/opt_postln_tiny.npz (the reference's own UnitLM) with the bounds of tests/test_gpu_opt.py
and tests/test_gpu_opt_fp32.py, against oracle/opt_postln_oracle.py at mid-size shapes and at the opt-350m geometry, the
DPO entry points, cached generation, the refusals and the CLIs."""
import json
import os

import numpy as np
import pytest
import torch

from helpers import rel_err, u16_to_bf16
from oracle import opt_postln_oracle as O
from test_gpu_opt import _batch, _check_grads

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
MID = dict(vocab_size=502, hidden=256, n_heads=4, ffn=1024, max_positions=512, proj_dim=128)
C350 = dict(vocab_size=502, hidden=1024, n_layers=24, n_heads=16, ffn=4096, max_positions=2048, proj_dim=512)


def _lm_cfg(c: "O.OraclePostLnConfig"):
    from slamkit_b200.lm import OptPostLnLMConfig
    return OptPostLnLMConfig(vocab_size=c.vocab_size, hidden=c.hidden, n_layers=c.n_layers, n_heads=c.n_heads, ffn=c.ffn,
                             max_positions=c.max_positions, ln_eps=c.ln_eps, tie_embeddings=c.tie_embeddings,
                             proj_dim=c.proj_dim)


def _mk(c, seed, max_batch, max_seq, trainable=True, fp32=False, std=0.02):
    from slamkit_b200.lm import B200UnitLM
    p = O.init_params(c, seed=seed, std=std, dtype=torch.float32 if fp32 else torch.bfloat16)
    m = B200UnitLM(_lm_cfg(c), device=DEV, max_batch=max_batch, max_seq=max_seq, trainable=trainable and not fp32,
                   fp32_inference=fp32)
    m.load_hf_state_dict(p)
    return m, p


def _fp32_grads(p, c, *args, **kw):
    return O.forward_backward({k: v.float() for k, v in p.items()}, c, *args, **kw)[2]


# ---- bf16 against the reference fixture ----------------------------------------------------------------------------
def test_post_ln_matches_reference_golden(golden_dir):
    """Loss, logits, every gradient (project_in / project_out and the tied 64-wide table included), the clip norm and
    one AdamW step against the reference's UnitLM in bf16; the packed row."""
    from test_opt_postln_cpu import golden
    from slamkit_b200.lm import B200AdamW
    z, c, seed = golden(golden_dir)
    ids, labels = torch.from_numpy(z["train/ids"]), torch.from_numpy(z["train/labels"])
    B, T = ids.shape
    m, p = _mk(c, seed, B, T)
    assert m.tensors["embed"][2] == 64 and m.tensors["proj_in"][1:] == (128, 64) and m.tensors["proj_out"][1:] == (64, 128)
    assert "final_norm" not in m.tensors
    out = m.forward_backward(ids, labels, num_items_in_batch=float(z["train/num_items"]))
    loss = float(out.loss)
    assert abs(loss - float(z["train/loss"])) < 1e-3 * abs(float(z["train/loss"])), (loss, float(z["train/loss"]))
    valid = ids != 0
    assert rel_err(m.logits_view(B, T).cpu()[valid], u16_to_bf16(z["train/logits_u16"])[valid]) < 8e-3
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
        upd = sd_p[k].cpu().float() - p[k].float()
        ref_sign = torch.from_numpy(z["upd_sign/" + k]).float().view_as(upd)
        ref_size = float(z["upd_absmean/" + k])
        assert abs(float(upd.abs().mean()) - ref_size) <= 0.2 * ref_size + 1e-9, k
        agree = (torch.sign(upd) == ref_sign).float().mean()
        if agree < 0.9:
            want = -torch.sign(g32[k])
            ours, theirs = (torch.sign(upd) == want).float().mean(), (ref_sign == want).float().mean()
            assert ours >= theirs - 0.03, (k, float(agree), float(ours), float(theirs))
    ids, pos, labels = (torch.from_numpy(z["packed/" + k]) for k in ("ids", "position_ids", "labels"))
    m, _ = _mk(c, seed, 1, ids.shape[1], trainable=False)
    out = m.forward(ids, position_ids=pos, labels=labels, num_items_in_batch=float(z["packed/num_items"]))
    assert rel_err(out.logits.cpu(), u16_to_bf16(z["packed/logits_u16"])) < 8e-3
    assert abs(float(out.loss) - float(z["packed/loss"])) < 1e-3 * abs(float(z["packed/loss"]))


# ---- bf16 against the oracle ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,T,layers", [(3, 200, 2), (1, 333, 1), (2, 130, 3)])
def test_post_ln_forward_backward_vs_oracle(B, T, layers):
    c = O.OraclePostLnConfig(n_layers=layers, **MID)
    m, p = _mk(c, 5, B, T)
    ids, labels = _batch(B, T, B * 1000 + T)
    n = float((labels != -100).sum())
    ref_loss, ref_logits, ref_g = O.forward_backward(p, c, ids, labels, n)
    out = m.forward_backward(ids, labels, num_items_in_batch=n)
    assert abs(float(out.loss) - float(ref_loss)) < 1e-3 * abs(float(ref_loss))
    valid = ids != 0
    assert rel_err(m.logits_view(B, T).cpu()[valid], ref_logits[valid]) < 8e-3
    _check_grads(m.state_dict_hf(grads=True), ref_g, _fp32_grads(p, c, ids, labels, n), p)


def test_post_ln_without_projections_packed_rows_and_accumulation():
    """post-LN with word_embed_proj_dim = hidden (no projections) on packed rows against the oracle; accumulating the
    same micro-batch twice gives twice the gradient."""
    c = O.OraclePostLnConfig(n_layers=2, **{**MID, "proj_dim": 0})
    m, p = _mk(c, 6, 2, 160)
    assert "proj_in" not in m.tensors and m.tensors["embed"][2] == 256
    g = torch.Generator().manual_seed(3)
    ids = torch.randint(2, 502, (2, 160), generator=g)
    pos = torch.cat([torch.cat([torch.arange(n) for n in (50, 1, 109)])[None], torch.arange(160)[None]])
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


def test_post_ln_accumulation_log_likelihood_and_five_step_trajectory():
    from slamkit_b200.lm import B200AdamW
    c = O.OraclePostLnConfig(vocab_size=502, hidden=128, n_layers=2, n_heads=2, ffn=512, max_positions=256, proj_dim=64)
    m, p = _mk(c, 9, 3, 96)
    ids, labels = _batch(2, 96, 77)
    n = float((labels != -100).sum())
    m.forward_backward(ids, labels, num_items_in_batch=n)
    one = m.grads.clone()
    m.forward_backward(ids, labels, num_items_in_batch=n, accumulate=True)
    assert rel_err(m.grads.float(), 2 * one.float()) < 1e-2
    tokens, _ = _batch(3, 40, 11, pad_last=9)
    lo = O.forward_logits(p, c, tokens).float()
    lp = torch.log_softmax(lo[:, :-1], -1).gather(-1, tokens[:, 1:, None])[..., 0]
    mask = tokens[:, 1:] != 0
    for mean in (False, True):
        want = (lp * mask).sum(-1) / (mask.sum(-1) if mean else 1)
        ll = m.sequence_log_likelihood(tokens, mean_nll=mean).float().cpu()
        assert bool(((ll - want).abs() <= 0.02 * want.abs()).all()), (mean, ll.tolist(), want.tolist())
    tr = O.OraclePostLnTrainer(p, c, lr=1e-3, max_grad_norm=0.5)
    opt = B200AdamW(m, lr=1e-3, max_grad_norm=0.5)
    for s in range(5):
        ids, labels = _batch(2, 96, 100 + s)
        ref = tr.train_step(ids, labels)
        out = m.forward_backward(ids, labels, num_items_in_batch=float((labels != -100).sum()))
        opt.step()
        assert abs(float(out.loss) - ref) < 3e-3 * abs(ref), (s, float(out.loss), ref)
        assert abs(float(opt.stats[0]) - float(tr.last_total_norm)) < 0.02 * float(tr.last_total_norm), s


def test_post_ln_dpo_entry_points_vs_oracle_autograd():
    from slamkit_b200 import _lib as L
    c = O.OraclePostLnConfig(vocab_size=502, hidden=128, n_layers=2, n_heads=2, ffn=256, max_positions=256, proj_dim=64)
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


def test_opt350m_geometry_is_finite_and_deterministic():
    """facebook/opt-350m geometry with the unit vocabulary at [8, 512]: finite, and bit-identical run to run (loss, every
    gradient -- the fixed-point table gradients included -- and the logits)."""
    from slamkit_b200.lm import B200UnitLM, OptPostLnLMConfig
    m = B200UnitLM(OptPostLnLMConfig(), device=DEV, max_batch=8, max_seq=512, seed=0)
    ids, labels = _batch(8, 512, 1, pad_last=100)
    n = float((labels != -100).sum())
    runs = []
    for _ in range(2):
        out = m.forward_backward(ids, labels, num_items_in_batch=n)
        torch.cuda.synchronize()
        runs.append((float(out.loss), m.grads.clone(), m.logits_view(8, 512).clone()))
    assert np.isfinite(runs[0][0]) and bool(torch.isfinite(runs[0][1].float()).all())
    assert runs[0][0] == runs[1][0]
    assert torch.equal(runs[0][1], runs[1][1]) and torch.equal(runs[0][2], runs[1][2])
    for name in ("proj_in", "proj_out", "embed", "pos_embed"):
        assert float(m.tensor(name, grad=True).float().abs().sum()) > 0, name


def test_post_ln_cached_generate_follows_oracle_and_graph_replay_equals_eager():
    from slamkit_b200 import _lib as L
    from slamkit_b200.lm import DecodeSession
    c = O.OraclePostLnConfig(vocab_size=502, hidden=128, n_layers=2, n_heads=2, ffn=256, max_positions=64, proj_dim=64)
    m, p = _mk(c, 2, 3, 64, trainable=False, std=0.1)
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
    for r in range(3):
        alone = m.generate(prompt[r:r + 1], attention_mask=mask[r:r + 1], max_new_tokens=20, do_sample=False,
                           eos_token_id=None)
        assert torch.equal(alone[0, 10:], out[r, 10:].to(alone.device)), r
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


# ---- fp32 inference ------------------------------------------------------------------------------------------------
def _fp64_logits(p, c, ids):
    p64 = {k: v.to(DEV, torch.float64) for k, v in p.items()}
    with torch.no_grad():
        return O.forward_logits(p64, c, ids.to(DEV))


def test_fp32_reference_golden(golden_dir):
    """The bounds of tests/test_gpu_opt_fp32.py::test_reference_golden."""
    from test_opt_postln_cpu import fp32_golden
    from slamkit_b200.lm import B200UnitLM
    z, c, p = fp32_golden(golden_dir)
    m = B200UnitLM(_lm_cfg(c), device=DEV, max_batch=4, max_seq=c.max_positions, trainable=False, fp32_inference=True)
    m.load_hf_state_dict(p)
    want = torch.from_numpy(z["f32/logits"]).to(DEV)
    got = m.forward(torch.from_numpy(z["f32/ids"]).to(DEV)).logits
    rel = float((got.double() - want.double()).norm() / want.double().norm())
    tokens = torch.from_numpy(z["f32/loglik_tokens"])
    ignore = z["f32/loglik_ignore"].tolist()
    errs = {}
    for key, mean_nll, ign in (("sum", False, None), ("mean", True, None), ("sum_ign", False, ignore),
                               ("mean_ign", True, ignore)):
        ll = m.sequence_log_likelihood(tokens, mean_nll, ign)
        assert ll.dtype == torch.float32
        errs[key] = float((ll.cpu().double() - torch.from_numpy(z["f32/loglik_" + key]).double()).abs().max())
    print(f"post-LN golden: logits rel-L2 {rel:.3e}, log-likelihood errors {errs}")
    assert rel < 1e-4
    n = int((tokens[:, 1:] != 0).sum(-1).max())
    for key, e in errs.items():
        assert e < (1e-4 if key.startswith("mean") else 1e-4 * n), key
    prompt = torch.from_numpy(z["f32/gen_prompt"])
    want_seq = torch.from_numpy(z["f32/gen_out"])[0]
    margin = torch.from_numpy(z["f32/gen_margin"])
    out = m.generate(prompt, max_new_tokens=len(margin), do_sample=False)[0].cpu()
    P = prompt.shape[1]
    for i in range(len(margin)):
        if float(margin[i]) <= 1e-4:
            break
        assert int(out[P + i]) == int(want_seq[P + i]), i


def test_opt350m_fp32_token_nll_vs_fp64_and_bf16_gap():
    """opt-350m geometry on [8, 512]: the fp32 path's logits and per-token NLL against an fp64 restatement, with the
    bounds of the opt-125m test, and a hundredfold gap to the bf16 path."""
    from test_gpu_opt_fp32 import NLL_BOUND, _fp64_token_nll, _right_padded
    from slamkit_b200.lm import B200UnitLM
    c = O.OraclePostLnConfig(**C350)
    B, T = 8, 512
    m, p = _mk(c, 3, B, T, fp32=True)
    m16 = B200UnitLM(_lm_cfg(c), device=DEV, max_batch=B, max_seq=T, trainable=False)
    m16.load_hf_state_dict(p)
    ids, lens = _right_padded(B, T, c.vocab_size, 4)
    ids_d = ids.to(DEV)
    ref = _fp64_logits(p, c, ids)
    want, mask = _fp64_token_nll(ref, ids)
    ll, tok = m.sequence_log_likelihood(ids_d, mean_nll=False, return_token_nll=True)
    logits = m.forward(ids_d).logits
    valid = torch.arange(T, device=DEV)[None] < lens.to(DEV)[:, None]
    zerr = (logits.double() - ref)[valid].norm() / ref[valid].norm()
    err32 = (tok.double() - want).abs()[mask]
    _, tok16 = m16.sequence_log_likelihood(ids_d, mean_nll=False, return_token_nll=True)
    err16 = (tok16.double() - want).abs()[mask]
    print(f"opt-350m fp32 path: logits rel-L2 {float(zerr):.3e}, token NLL max {float(err32.max()):.3e} mean "
          f"{float(err32.mean()):.3e}; bf16 path: max {float(err16.max()):.3e} mean {float(err16.mean()):.3e}")
    assert float(zerr) < 1e-4
    assert float(err32.max()) < NLL_BOUND
    assert float(err32.mean()) * 100 <= float(err16.mean())
    assert float((ll.double() - (-(want * mask).sum(-1))).abs().max()) < NLL_BOUND * T


def test_fp32_prefill_decode_follow_forward_and_greedy_follows_fp64():
    from test_gpu_opt_fp32 import _decode_run, _right_padded
    from slamkit_b200.lm import DecodeSession
    c = O.OraclePostLnConfig(n_layers=3, **MID)
    B, T, k = 4, 120, 6
    m, p = _mk(c, 7, B, T + k, fp32=True)
    ids, lens = _right_padded(B, T + k, c.vocab_size, 8, min_len=k + 10)
    full = m.forward(ids.to(DEV)).logits.clone()
    plens = lens - k
    prompt = ids.clone()
    prompt[torch.arange(T + k)[None] >= plens[:, None]] = 0
    sess = DecodeSession(m, B, T + k, k, 0)
    got = [sess.prefill(prompt[:, :T], plens).clone()]
    for i in range(k - 1):
        pos = (plens + i).to(torch.int32)
        got.append(sess.step(ids.gather(1, pos[:, None].long())[:, 0].to(DEV), pos.to(DEV)).clone())
    scale = float(full.abs().max())
    for i, g_ in enumerate(got):
        want = full[torch.arange(B, device=DEV), (plens - 1 + i).to(DEV)]
        assert float((g_ - want).abs().max()) <= 2e-5 * max(1.0, scale), i
    eager = _decode_run(m, ids[:, :70], lens.clamp(max=70), 80, 5, False)
    replay = _decode_run(m, ids[:, :70], lens.clamp(max=70), 80, 5, True)
    for a, b in zip(eager, replay):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32)), "graph replay differs from eager"
    m, p = _mk(c, 11, 2, 64, fp32=True, std=0.05)
    prompt = torch.tensor([[1, 17, 33, 5, 250, 9, 41, 77]])
    seq = m.generate(prompt, max_new_tokens=12, do_sample=False, eos_token_id=[])[0].cpu()
    for t in range(prompt.shape[1], seq.shape[0]):
        z = _fp64_logits(p, c, seq[None, :t])[0, -1]
        top = torch.topk(z, 2).values
        if float(top[0] - top[1]) > 1e-4:
            assert int(seq[t]) == int(z.argmax()), t


# ---- refusals ------------------------------------------------------------------------------------------------------
def test_refusals_name_field_or_mode_before_any_launch():
    import ctypes as C
    from slamkit_b200 import _lib as L
    from slamkit_b200.lm import B200UnitLM
    lib = L.require_cuda()
    c = O.OraclePostLnConfig(vocab_size=502, hidden=128, n_layers=1, n_heads=2, ffn=256, max_positions=64, proj_dim=64)
    n0 = lib.sk_launch_count()
    with pytest.raises(ValueError, match="master_weights"):
        B200UnitLM(_lm_cfg(c), device=DEV, max_batch=1, max_seq=16, master_weights=True)
    assert lib.sk_launch_count() == n0
    m, _ = _mk(c, 1, 1, 16)
    torch.cuda.synchronize()
    n0 = lib.sk_launch_count()
    p32 = torch.zeros(m.n_params, device=DEV)
    assert lib.sk_lm_set_master(m._h, L.ptr(p32), L.ptr(p32)) == -1
    assert b"post_ln" in lib.sk_last_error()
    h = C.c_void_p()
    pre_proj = L.SkOptConfig(502, 128, 1, 2, 256, 64, 1e-5, 1, 0, 64)         # pre-LN with project_in / project_out
    assert lib.sk_lm_create_opt(C.byref(pre_proj), C.byref(h)) == -1
    assert b"proj_dim" in lib.sk_last_error()
    bad = L.SkOptConfig(502, 128, 1, 2, 256, 64, 1e-5, 1, 1, 96)              # not a multiple of 64
    assert lib.sk_lm_create_opt(C.byref(bad), C.byref(h)) == -1
    assert b"proj_dim" in lib.sk_last_error()
    assert lib.sk_launch_count() == n0


# ---- CLIs ----------------------------------------------------------------------------------------------------------
def _tiny_post_ln_dir(path):
    """A tiny random HF post-LN OPTForCausalLM with project_in / project_out, saved as twist_init loads a base."""
    from transformers import OPTConfig, OPTForCausalLM
    cfg = OPTConfig(hidden_size=128, ffn_dim=256, num_hidden_layers=2, num_attention_heads=2, word_embed_proj_dim=64,
                    do_layer_norm_before=False, max_position_embeddings=256, vocab_size=600, dropout=0.0,
                    attention_dropout=0.0, layerdrop=0.0)
    torch.manual_seed(0)
    OPTForCausalLM(cfg).save_pretrained(str(path))
    return str(path)


def test_cli_train_twist_post_ln_trains_saves_resumes_and_loads(tmp_path):
    import shutil
    from safetensors.torch import load_file
    from cli import train
    from test_gpu_round2 import _write_tokens
    from slamkit_b200.lm import B200UnitLM, OptPostLnLMConfig
    base = _tiny_post_ln_dir(tmp_path / "base")
    tok = str(tmp_path / "tok.jsonl")
    _write_tokens(tok, 40, 1)
    common = [f"data.train_path={tok}", f"data.val_path={tok}", "model=twist", "model.tlm_type=b200",
              "model.context_len=64", f"model.config_args.base_model_name={base}",
              "model.config_args.torch_dtype=bfloat16", "training_args.per_device_train_batch_size=4",
              "+training_args.logging_steps=1", "training_args.warmup_steps=2", "training_args.warmup_ratio=0",
              "+training_args.save_steps=4", "+training_args.max_steps=8"]
    log_a = train.main(common + [f"training_args.output_dir={tmp_path}/a"])
    la = [r for r in log_a if "loss" in r]
    assert len(la) == 8 and la[-1]["loss"] < la[0]["loss"]
    c = json.load(open(tmp_path / "a" / "config.json"))
    assert c["base_config"]["do_layer_norm_before"] is False and c["base_config"]["word_embed_proj_dim"] == 64
    os.makedirs(tmp_path / "b")
    shutil.copytree(tmp_path / "a" / "checkpoint-4", tmp_path / "b" / "checkpoint-4")
    log_b = train.main(common + ["cont_training=true", f"training_args.output_dir={tmp_path}/b"])
    lb = [r for r in log_b if "loss" in r]
    assert [r["loss"] for r in la][-4:] == [r["loss"] for r in lb][-4:]
    a, b = load_file(str(tmp_path / "a" / "model.safetensors")), load_file(str(tmp_path / "b" / "model.safetensors"))
    assert set(a) == set(b) and all(torch.equal(a[k], b[k]) for k in a)
    from slamkit_b200.integration import tlm_b200_from_cfg
    from transformers import OPTForCausalLM
    node = {"context_len": 64, "config_args": {"base_model_name": base, "vocab_size": 502, "torch_dtype": "bfloat16"}}
    init = tlm_b200_from_cfg(node, device=DEV, max_batch=1).state_dict_hf()
    hf = OPTForCausalLM.from_pretrained(base, dtype=torch.bfloat16)
    hf.resize_token_embeddings(502)                 # twist_init: the HF weights, the first vocab_size table rows
    for k, v in hf.state_dict().items():
        assert torch.equal(init["lm." + k].cpu(), v), k
    m = B200UnitLM.from_pretrained(str(tmp_path / "a"), device=DEV)
    assert isinstance(m.config, OptPostLnLMConfig) and m.config.proj_dim == 64 and not m.fp32
    sd = m.state_dict_hf()
    assert all(torch.equal(sd[k].cpu(), a[k]) for k in a)


def test_cli_eval_scores_a_float32_post_ln_checkpoint(tmp_path, caplog):
    import logging
    import cli.eval as E
    from cli.extract_features import build_tokeniser
    from slamkit_b200 import metrics as M
    from slamkit_b200.config import load_config
    from slamkit_b200.lm import OptPostLnLMConfig, write_unit_lm_checkpoint
    from slamkit_b200.speech_lm import B200SpeechLM
    from test_gpu_eval import _write_clips
    c = O.OraclePostLnConfig(vocab_size=502, hidden=128, n_layers=2, n_heads=2, ffn=256, max_positions=256, proj_dim=64)
    p = O.init_params(c, seed=4, std=0.05, dtype=torch.float32)
    ck = tmp_path / "ck"
    write_unit_lm_checkpoint(str(ck), {**p, "lm.lm_head.weight": p["lm.model.decoder.embed_tokens.weight"]}, _lm_cfg(c),
                             torch_dtype="float32")
    g = torch.Generator().manual_seed(13)
    sw = tmp_path / "swuggy"
    _write_clips(sw, [f"{d}/{i}_w.wav" for d in ("a", "b") for i in range(4)], g)
    argv = [f"model.pretrained_model={ck}", "+synthetic_weights=true", "batch_size=2", "num_workers=2",
            "metric=swuggy_inter", f"metric.data_path={sw}"]
    with caplog.at_level(logging.INFO):
        res = E.main(argv)
    assert "fp32 inference" in caplog.text
    cfg = load_config("eval", argv)
    model = E.load_model(cfg, DEV)
    assert model.fp32 and isinstance(model.config, OptPostLnLMConfig)
    slm = B200SpeechLM(model, build_tokeniser(cfg, DEV))
    assert res == M.swuggy(slm, str(sw), None, True, 2, 2, True, True)
