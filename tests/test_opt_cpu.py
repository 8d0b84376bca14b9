"""OPT decoder, host side (no GPU): oracle/opt_oracle.py against tests/golden/opt_tiny.npz (produced by the reference's own
UnitLM over HF OPTForCausalLM), OptLMConfig.from_hf's accept / refuse matrix, lm_config_from_hf dispatch, the OPT
checkpoint layout and tlm_b200_from_cfg's torch_dtype rule."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import opt_oracle as O
from helpers import rel_err, u16_to_bf16


def _golden(golden_dir):
    z = np.load(os.path.join(golden_dir, "opt_tiny.npz"))
    c = z["cfg"]
    cfg = O.OracleOptConfig(vocab_size=int(c[0]), hidden=int(c[1]), n_layers=int(c[2]), n_heads=int(c[3]), ffn=int(c[4]),
                            max_positions=int(c[5]))
    return z, cfg, O.init_params(cfg, seed=int(c[6]))


def test_oracle_forward_matches_reference(golden_dir):
    z, cfg, p = _golden(golden_dir)
    ids, labels = torch.from_numpy(z["train/ids"]), torch.from_numpy(z["train/labels"])
    logits = O.forward_logits(p, cfg, ids)
    # without an attention_mask and autocast the reference takes the same plain bf16 path: bit-identical logits and loss
    assert torch.equal(logits, u16_to_bf16(z["nomask/logits_u16"]))
    loss = O.compute_loss(logits, labels, float(z["train/num_items"]))
    assert abs(float(loss) - float(z["nomask/loss"])) <= 1e-6 * abs(float(z["nomask/loss"]))
    # the Trainer path (attention_mask, autocast): non-pad rows agree to bf16 rounding; pad rows are not compared (HF moves
    # their positions to table row 1 and masks their keys; they carry no loss)
    ref = O.golden_masked_logits(z)
    valid = ids != 0
    assert rel_err(logits[valid], ref[valid]) < 4e-3
    assert abs(float(loss) - float(z["train/loss"])) <= 2e-3 * abs(float(z["train/loss"]))


def test_oracle_masked_positions_follow_hf():
    ids = torch.tensor([[5, 6, 7, 0, 0]])
    assert O.positions(ids).tolist() == [[0, 1, 2, 3, 4]]
    assert O.positions(ids, (ids != 0).long()).tolist() == [[0, 1, 2, -1, -1]]


def test_oracle_backward_matches_reference(golden_dir):
    z, cfg, p = _golden(golden_dir)
    ids, labels = torch.from_numpy(z["train/ids"]), torch.from_numpy(z["train/labels"])
    _, _, grads = O.forward_backward(p, cfg, ids, labels, float(z["train/num_items"]))
    for k, g in grads.items():
        ref = u16_to_bf16(z["grad/" + k]).view_as(g)
        if k.endswith("embed_positions.weight"):
            # HF's masked positions put the pad rows' (zero) gradient at row 1, not at their in-row positions: compare the rest
            g, ref = g[2:], ref[2:]
        assert rel_err(g, ref) < 2e-2, k


def test_oracle_optimizer_step_matches_reference(golden_dir):
    z, cfg, p = _golden(golden_dir)
    ids, labels = torch.from_numpy(z["train/ids"]), torch.from_numpy(z["train/labels"])
    tr = O.OracleOptTrainer(p, cfg, lr=1e-3, max_grad_norm=0.5)
    tr.train_step(ids, labels)
    assert abs(float(tr.last_total_norm) - float(z["train/total_norm"])) <= 0.01 * float(z["train/total_norm"])
    for k, v in tr.p.items():
        upd = v.float() - p[k].float()
        # a first AdamW step moves every element with a gradient by ~lr: compare the update's direction elementwise and
        # its mean size per tensor
        agree = (torch.sign(upd) == torch.from_numpy(z["upd_sign/" + k]).float().view_as(upd)).float().mean()
        assert agree > 0.97, (k, float(agree))
        ref_size = float(z["upd_absmean/" + k])
        assert abs(float(upd.abs().mean()) - ref_size) <= 0.05 * ref_size + 1e-9, k


def test_oracle_packed_row_matches_reference(golden_dir):
    z, cfg, p = _golden(golden_dir)
    ids, pos, labels = (torch.from_numpy(z["packed/" + k]) for k in ("ids", "position_ids", "labels"))
    logits = O.forward_logits(p, cfg, ids, pos, packed=True)
    assert rel_err(logits, u16_to_bf16(z["packed/logits_u16"])) < 4e-3
    loss = O.compute_loss(logits, labels, float(z["packed/num_items"]))
    assert abs(float(loss) - float(z["packed/loss"])) <= 2e-3 * abs(float(z["packed/loss"]))


# ---- configuration --------------------------------------------------------------------------------------------------
def _opt(**kw):
    from transformers import OPTConfig
    base = dict(hidden_size=768, ffn_dim=3072, num_hidden_layers=12, num_attention_heads=12, word_embed_proj_dim=768,
                dropout=0.0, attention_dropout=0.0, layerdrop=0.0)
    base.update(kw)
    return OPTConfig(**base)


def test_opt_config_from_hf_accepts_opt_125m_geometry():
    from slamkit_b200.lm import OptLMConfig
    c = OptLMConfig.from_hf(_opt(), vocab_size=502)
    assert (c.vocab_size, c.hidden, c.n_layers, c.n_heads, c.ffn, c.max_positions) == (502, 768, 12, 12, 3072, 2048)
    assert c.tie_embeddings and c.ln_eps == 1e-5 and c.head_dim == 64
    c = OptLMConfig.from_hf(_opt(hidden_size=2048, ffn_dim=8192, num_attention_heads=32, word_embed_proj_dim=2048))
    assert c.hidden == 2048 and c.n_heads == 32                                    # opt-1.3b


@pytest.mark.parametrize("kw,field", [
    (dict(do_layer_norm_before=False), "do_layer_norm_before"),
    (dict(word_embed_proj_dim=512), "word_embed_proj_dim"),
    (dict(_remove_final_layer_norm=True), "_remove_final_layer_norm"),
    (dict(enable_bias=False), "enable_bias"),
    (dict(layer_norm_elementwise_affine=False), "layer_norm_elementwise_affine"),
    (dict(activation_function="gelu"), "activation_function"),
    (dict(num_attention_heads=16), "head_dim"),
    (dict(dropout=0.1), "dropout"),
    (dict(attention_dropout=0.1), "attention_dropout"),
    (dict(layerdrop=0.1), "layerdrop"),
])
def test_opt_config_from_hf_refuses_by_field(kw, field):
    from slamkit_b200.lm import OptLMConfig
    with pytest.raises(ValueError, match=field):
        OptLMConfig.from_hf(_opt(**kw))


def test_lm_config_from_hf_dispatches_on_model_type():
    from transformers import LlamaConfig, Qwen2Config
    from slamkit_b200.lm import LMConfig, OptLMConfig, lm_config_from_hf
    assert isinstance(lm_config_from_hf(_opt(), vocab_size=502), OptLMConfig)
    q = lm_config_from_hf(Qwen2Config(hidden_size=896, num_attention_heads=14, num_key_value_heads=2), vocab_size=502)
    assert isinstance(q, LMConfig)
    with pytest.raises(ValueError, match="llama"):
        lm_config_from_hf(LlamaConfig())
    with pytest.raises(ValueError):
        LMConfig.from_hf(_opt())                        # LMConfig.from_hf stays Qwen2-only


# ---- checkpoint layout ---------------------------------------------------------------------------------------------
def test_checkpoint_layout_equals_reference_state_dict(golden_dir, tmp_path):
    """write_unit_lm_checkpoint on an OPT config writes the keys and shapes the reference's UnitLM.from_pretrained gives
    (fixture), and a base_config that round-trips through OptLMConfig.from_hf."""
    from safetensors.torch import load_file
    from transformers import OPTConfig
    from slamkit_b200.lm import OptLMConfig, write_unit_lm_checkpoint
    z, _, _ = _golden(golden_dir)
    cfg = O.OracleOptConfig(vocab_size=502, hidden=128, n_layers=1, n_heads=2, ffn=256, max_positions=64)
    p = O.init_params(cfg, seed=int(z["ckpt/seed_params"]))
    lm_cfg = OptLMConfig(vocab_size=502, hidden=128, n_layers=1, n_heads=2, ffn=256, max_positions=64)
    write_unit_lm_checkpoint(str(tmp_path), {**p, "lm.lm_head.weight": p["lm.model.decoder.embed_tokens.weight"]}, lm_cfg)
    sd = load_file(str(tmp_path / "model.safetensors"))
    keys = [str(k) for k in z["ckpt/keys"]]
    shapes = {k: json.loads(str(s)) for k, s in zip(keys, z["ckpt/shapes"])}
    # tied: the reference's state dict lists lm.lm_head.weight too, the file stores the table once
    assert sorted(sd) == sorted(k for k in keys if k != "lm.lm_head.weight")
    for k, t in sd.items():
        assert list(t.shape) == shapes[k], k
        d = np.array([float(t.double().sum()), float((t.double().flatten() * torch.arange(t.numel(), dtype=torch.float64)).sum())])
        assert np.allclose(d, z["ckpt/digests"][keys.index(k)], rtol=1e-12, atol=1e-9), k
    c = json.load(open(tmp_path / "config.json"))
    assert c["base_model_name"] == "facebook/opt-125m" and c["vocab_size"] == 502
    base = c["base_config"]
    assert base == json.loads(str(z["ckpt/base_config"]))
    back = OptLMConfig.from_hf(OPTConfig(**{k: v for k, v in base.items() if k not in ("model_type", "architectures")}),
                               vocab_size=c["vocab_size"])
    assert back == lm_cfg


def test_tlm_b200_from_cfg_refuses_opt_without_bf16(tmp_path):
    from transformers import OPTConfig
    from slamkit_b200.integration import tlm_b200_from_cfg
    OPTConfig(hidden_size=128, ffn_dim=256, num_hidden_layers=2, num_attention_heads=2, word_embed_proj_dim=128,
              max_position_embeddings=256).save_pretrained(str(tmp_path))
    cfg = {"context_len": 64, "config_args": {"base_model_name": str(tmp_path), "vocab_size": 502, "twist_init": False,
                                              "dropout": 0.0, "attention_dropout": 0.0, "layerdrop": 0.0,
                                              "torch_dtype": None}}
    with pytest.raises(ValueError, match="torch_dtype=bfloat16"):
        tlm_b200_from_cfg(cfg, device="cpu")
    # the base's own dropout (0.1 in OPTConfig) is replaced by config_args' 0.0 before the refusal matrix runs
    cfg["config_args"]["torch_dtype"] = "bfloat16"
    cfg["config_args"]["dropout"] = 0.1
    with pytest.raises(ValueError, match="dropout"):
        tlm_b200_from_cfg(cfg, device="cpu")
