"""CPU checks of fp32 OPT inference: which checkpoints select it, what is refused, and that the per-token fp64 bound of
tests/test_gpu_opt_fp32.py discriminates -- a clean fp32 forward passes it, and each defect a split-bf16 forward could
carry (a bf16 rounding of the residual stream, a dropped lo product, an off-by-one causal boundary, scores rounded to
bf16) fails it."""
import json

import pytest
import torch
import torch.nn.functional as F

from oracle import opt_oracle as O
from test_gpu_opt_fp32 import NLL_BOUND, _fp64_token_nll, _right_padded

CFG = O.OracleOptConfig(vocab_size=502, hidden=256, n_layers=3, n_heads=4, ffn=1024, max_positions=512)


def _forward(p, c, ids, *, round_residual=False, drop_lo=False, causal_shift=0):
    """OPTForCausalLM in fp32 (or fp64 when p is), with one optional defect."""
    B, T = ids.shape
    pre = "lm.model.decoder."
    bf = lambda t: t.to(torch.bfloat16).to(t.dtype)
    lin = (lambda x, w, b=None: F.linear(x, bf(w), b)) if drop_lo else F.linear   # hi * hi + hi * lo + lo * hi ~ hi only
    pos = torch.arange(T)[None].expand(B, T)
    x = F.embedding(ids, p[pre + "embed_tokens.weight"]) + F.embedding(pos + 2, p[pre + "embed_positions.weight"])
    d, H, hd = c.hidden, c.n_heads, c.head_dim
    keep = torch.arange(T)[None] <= torch.arange(T)[:, None] + causal_shift
    for l in range(c.n_layers):
        h = f"{pre}layers.{l}."
        y = F.layer_norm(x, (d,), p[h + "self_attn_layer_norm.weight"], p[h + "self_attn_layer_norm.bias"], c.ln_eps)
        q = lin(y, p[h + "self_attn.q_proj.weight"], p[h + "self_attn.q_proj.bias"]) * hd ** -0.5
        k = lin(y, p[h + "self_attn.k_proj.weight"], p[h + "self_attn.k_proj.bias"])
        v = lin(y, p[h + "self_attn.v_proj.weight"], p[h + "self_attn.v_proj.bias"])
        q, k, v = (t.view(B, T, H, hd).transpose(1, 2) for t in (q, k, v))
        a = F.scaled_dot_product_attention(q, k, v, attn_mask=keep, scale=1.0).transpose(1, 2).reshape(B, T, d)
        x = x + lin(a, p[h + "self_attn.out_proj.weight"], p[h + "self_attn.out_proj.bias"])
        if round_residual:
            x = bf(x)
        y = F.layer_norm(x, (d,), p[h + "final_layer_norm.weight"], p[h + "final_layer_norm.bias"], c.ln_eps)
        x = x + lin(F.relu(lin(y, p[h + "fc1.weight"], p[h + "fc1.bias"])), p[h + "fc2.weight"], p[h + "fc2.bias"])
        if round_residual:
            x = bf(x)
    x = F.layer_norm(x, (d,), p[pre + "final_layer_norm.weight"], p[pre + "final_layer_norm.bias"], c.ln_eps)
    return lin(x, p[pre + "embed_tokens.weight"])


@pytest.fixture(scope="module")
def case():
    p = O.init_params(CFG, seed=5, std=0.05, dtype=torch.float32)
    ids, _ = _right_padded(4, 96, CFG.vocab_size, 6, min_len=48)
    p64 = {k: v.double() for k, v in p.items()}
    with torch.no_grad():
        want, mask = _fp64_token_nll(O.forward_logits(p64, CFG, ids), ids)
    return p, ids, want, mask


def _err(p, ids, want, mask, round_scores=False, **defect):
    with torch.no_grad():
        tok, _ = _fp64_token_nll(_forward(p, CFG, ids, **defect).double(), ids)
    if round_scores:
        tok = tok.to(torch.bfloat16).double()
    return float((tok - want).abs()[mask].max())


def test_fp64_restatement_matches_the_oracle(case):
    p, ids, want, mask = case
    p64 = {k: v.double() for k, v in p.items()}
    with torch.no_grad():
        z = _forward(p64, CFG, ids)
        assert float((z - O.forward_logits(p64, CFG, ids)).abs().max()) < 1e-12


def test_clean_fp32_forward_is_within_the_bound(case):
    assert _err(*case) < NLL_BOUND / 4


@pytest.mark.parametrize("defect", [dict(round_residual=True), dict(drop_lo=True), dict(causal_shift=1),
                                    dict(round_scores=True)], ids=["bf16-residual", "dropped-lo", "causal+1", "bf16-scores"])
def test_bound_catches_defects(case, defect):
    assert _err(*case, **defect) > NLL_BOUND


def golden_fp32(golden_dir):
    """tests/golden/opt_fp32_tiny.npz (oracle/make_opt_fp32_golden.py: the reference's UnitLM in fp32) and its model."""
    import os
    import numpy as np
    z = np.load(os.path.join(golden_dir, "opt_fp32_tiny.npz"))
    c = z["cfg"]
    cfg = O.OracleOptConfig(vocab_size=int(c[0]), hidden=int(c[1]), n_layers=int(c[2]), n_heads=int(c[3]), ffn=int(c[4]),
                            max_positions=int(c[5]))
    return z, cfg, O.init_params(cfg, seed=int(c[6]), std=float(z["std"]), dtype=torch.float32)


def calc_nll_ll(logits, tokens, mean_nll, ignore=None, pad=0):
    """UnitLM.log_likelihood's tail (calc_nll) on given logits, in the logits' dtype."""
    logits = logits.clone()
    if ignore is not None:
        logits[:, :, ignore] = float("-inf")
    x = tokens[:, 1:]
    mask = x != pad
    lp = torch.log_softmax(logits[:, :-1], -1).gather(-1, x.clamp(min=0)[..., None])[..., 0] * mask
    s = lp.sum(-1)
    return s / mask.sum(-1) if mean_nll else s


def test_fp32_oracle_reproduces_the_reference_golden(golden_dir):
    z, cfg, p = golden_fp32(golden_dir)
    ids = torch.from_numpy(z["logits/ids"])
    with torch.no_grad():
        got = O.forward_logits(p, cfg, ids)
    want = torch.from_numpy(z["logits/z"])
    assert float((got - want).norm() / want.norm()) < 1e-6
    tokens = torch.from_numpy(z["loglik/tokens"])
    ignore = torch.from_numpy(z["loglik/ignore"]).tolist()
    with torch.no_grad():
        zt = O.forward_logits(p, cfg, tokens)
    for key, mean_nll, ign in (("sum", False, None), ("mean", True, None), ("sum_ign", False, ignore),
                               ("mean_ign", True, ignore)):
        ll = calc_nll_ll(zt, tokens, mean_nll, ign)
        assert float((ll - torch.from_numpy(z["loglik/" + key])).abs().max()) < 1e-5 * (1 if mean_nll else 40), key


def test_checkpoint_dtype_selects_the_mode():
    from slamkit_b200.lm import checkpoint_is_fp32
    assert checkpoint_is_fp32({"torch_dtype": "float32", "base_config": {"torch_dtype": "float32"}})
    assert checkpoint_is_fp32({"base_config": {"torch_dtype": "torch.float32"}})
    assert not checkpoint_is_fp32({"torch_dtype": "bfloat16", "base_config": {"torch_dtype": "float32"}})
    assert not checkpoint_is_fp32({"base_config": {}})
    # transformers >= 4.56 writes `dtype` instead of `torch_dtype`
    assert checkpoint_is_fp32({"dtype": "float32", "base_config": {"dtype": "float32"}})
    assert checkpoint_is_fp32({"base_config": {"dtype": "float32"}})
    assert not checkpoint_is_fp32({"dtype": "bfloat16", "base_config": {"dtype": "float32"}})


def test_written_config_round_trips(tmp_path):
    from slamkit_b200.lm import OptLMConfig, checkpoint_is_fp32, write_unit_lm_checkpoint
    c = OptLMConfig(hidden=128, n_layers=1, n_heads=2, ffn=256)
    for dt, want in (("float32", True), ("bfloat16", False)):
        write_unit_lm_checkpoint(str(tmp_path / dt), {}, c, torch_dtype=dt)
        assert checkpoint_is_fp32(json.load(open(tmp_path / dt / "config.json"))) is want


def test_other_architectures_and_training_are_refused():
    from slamkit_b200.lm import B200UnitLM, LMConfig, NeoxLMConfig, OptLMConfig
    for cfg in (LMConfig(vocab_size=502, hidden=128, n_layers=1, n_heads=2, n_kv_heads=1, head_dim=64, ffn=256),
                NeoxLMConfig(hidden=128, n_layers=1, n_heads=2, ffn=512)):
        with pytest.raises(ValueError, match="fp32_inference"):
            B200UnitLM(cfg, trainable=False, fp32_inference=True)
    with pytest.raises(ValueError, match="trainable=False"):
        B200UnitLM(OptLMConfig(), trainable=True, fp32_inference=True)
    with pytest.raises(ValueError, match="master_weights"):
        B200UnitLM(OptLMConfig(), trainable=False, master_weights=True, fp32_inference=True)
