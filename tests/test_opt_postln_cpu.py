"""Post-LayerNorm OPT (the opt-350m layout) without a GPU: config dispatch and refusals, the CPU oracle against the
reference fixture tests/golden/opt_postln_tiny.npz (bf16 forward / backward / AdamW step / packed row, fp32 logits /
log-likelihoods / greedy generate), the checkpoint layout and the integration's precision refusal."""
import json
import os

import numpy as np
import pytest
import torch

from helpers import rel_err, u16_to_bf16
from oracle import opt_postln_oracle as O


def _opt(**kw):
    from transformers import OPTConfig
    base = dict(hidden_size=1024, ffn_dim=4096, num_hidden_layers=24, num_attention_heads=16, word_embed_proj_dim=512,
                do_layer_norm_before=False, dropout=0.0, attention_dropout=0.0, layerdrop=0.0)
    base.update(kw)
    return OPTConfig(**base)


def golden(golden_dir):
    z = np.load(os.path.join(golden_dir, "opt_postln_tiny.npz"))
    c = z["cfg"]
    cfg = O.OraclePostLnConfig(vocab_size=int(c[0]), hidden=int(c[1]), n_layers=int(c[2]), n_heads=int(c[3]),
                               ffn=int(c[4]), max_positions=int(c[5]), proj_dim=int(c[6]))
    return z, cfg, int(c[7])


# ---- config ---------------------------------------------------------------------------------------------------------
def test_opt350m_geometry_becomes_a_post_ln_config():
    from slamkit_b200.lm import OptLMConfig, OptPostLnLMConfig, lm_config_from_hf
    c = lm_config_from_hf(_opt(), vocab_size=502)
    assert isinstance(c, OptPostLnLMConfig) and isinstance(c, OptLMConfig)      # every OPT path takes it
    assert (c.vocab_size, c.hidden, c.n_layers, c.n_heads, c.ffn, c.proj_dim) == (502, 1024, 24, 16, 4096, 512)
    assert c.has_proj and c.tie_embeddings and c.head_dim == 64
    assert OptPostLnLMConfig() == OptPostLnLMConfig(vocab_size=502, hidden=1024, n_layers=24, n_heads=16, ffn=4096,
                                                    proj_dim=512)
    flat = lm_config_from_hf(_opt(word_embed_proj_dim=1024), vocab_size=502)      # post-LN without projections
    assert isinstance(flat, OptPostLnLMConfig) and not flat.has_proj
    assert type(lm_config_from_hf(_opt(do_layer_norm_before=True, word_embed_proj_dim=1024))) is OptLMConfig


@pytest.mark.parametrize("kw,field", [
    (dict(_remove_final_layer_norm=True), "_remove_final_layer_norm"),
    (dict(enable_bias=False), "enable_bias"),
    (dict(layer_norm_elementwise_affine=False), "layer_norm_elementwise_affine"),
    (dict(activation_function="gelu"), "activation_function"),
    (dict(num_attention_heads=8), "head_dim"),
    (dict(dropout=0.1), "dropout"),
    (dict(attention_dropout=0.1), "attention_dropout"),
    (dict(layerdrop=0.1), "layerdrop"),
    (dict(word_embed_proj_dim=500), "word_embed_proj_dim"),
    (dict(do_layer_norm_before=True), "do_layer_norm_before"),
])
def test_post_ln_refusals_name_their_field(kw, field):
    from slamkit_b200.lm import OptPostLnLMConfig
    with pytest.raises(ValueError, match=field):
        OptPostLnLMConfig.from_hf(_opt(**kw))


def test_pre_ln_with_projections_stays_refused():
    from slamkit_b200.lm import OptLMConfig, lm_config_from_hf
    with pytest.raises(ValueError, match="word_embed_proj_dim"):
        lm_config_from_hf(_opt(do_layer_norm_before=True))
    with pytest.raises(ValueError, match="do_layer_norm_before"):
        OptLMConfig.from_hf(_opt(word_embed_proj_dim=1024))


# ---- oracle against the reference fixture ---------------------------------------------------------------------------
def test_oracle_reproduces_bf16_golden(golden_dir):
    z, c, seed = golden(golden_dir)
    p = O.init_params(c, seed=seed)
    ids, labels = torch.from_numpy(z["train/ids"]), torch.from_numpy(z["train/labels"])
    tr = O.OraclePostLnTrainer(p, c, lr=1e-3, max_grad_norm=0.5)
    loss, logits, grads = O.forward_backward(p, c, ids, labels, float(z["train/num_items"]))
    assert abs(float(loss) - float(z["train/loss"])) < 1e-4 * abs(float(z["train/loss"]))
    assert rel_err(logits, u16_to_bf16(z["train/logits_u16"])) < 1e-3
    assert set(grads) == {k[len("grad/"):] for k in z.files if k.startswith("grad/")} - {"lm.lm_head.weight"}
    for k, g in grads.items():
        assert rel_err(g, u16_to_bf16(z["grad/" + k]).view_as(g)) < 1e-2, k
    tr.train_step(ids, labels)
    assert abs(float(tr.last_total_norm) - float(z["train/total_norm"])) < 1e-3 * float(z["train/total_norm"])
    for k in p:
        upd = tr.p[k].float() - p[k].float()
        ref = torch.from_numpy(z["upd_sign/" + k]).float().view_as(upd)
        assert float((torch.sign(upd) == ref).float().mean()) > 0.97, k
        assert abs(float(upd.abs().mean()) - float(z["upd_absmean/" + k])) <= 0.05 * float(z["upd_absmean/" + k]) + 1e-9, k
    ids, pos, labels = (torch.from_numpy(z["packed/" + k]) for k in ("ids", "position_ids", "labels"))
    loss, logits, _ = O.forward_backward(p, c, ids, labels, float(z["packed/num_items"]), position_ids=pos, packed=True)
    assert rel_err(logits, u16_to_bf16(z["packed/logits_u16"])) < 1e-3
    assert abs(float(loss) - float(z["packed/loss"])) < 1e-4 * abs(float(z["packed/loss"]))


def fp32_golden(golden_dir):
    z, c, _ = golden(golden_dir)
    p = O.init_params(c, seed=int(z["f32/seed_params"]), std=float(z["f32/std"]), dtype=torch.float32)
    return z, c, p


def test_oracle_reproduces_fp32_golden(golden_dir):
    z, c, p = fp32_golden(golden_dir)
    with torch.no_grad():
        got = O.forward_logits(p, c, torch.from_numpy(z["f32/ids"]))
        assert rel_err(got, torch.from_numpy(z["f32/logits"])) < 1e-6
        tokens = torch.from_numpy(z["f32/loglik_tokens"])
        ignore = z["f32/loglik_ignore"].tolist()
        lo = O.forward_logits(p, c, tokens)
        for key, mean, ban in (("sum", False, None), ("mean", True, None), ("sum_ign", False, ignore),
                               ("mean_ign", True, ignore)):
            zz = lo.clone()
            if ban:
                zz[..., ban] = float("-inf")
            lp = torch.log_softmax(zz[:, :-1], -1).gather(-1, tokens[:, 1:, None])[..., 0]
            mask = tokens[:, 1:] != 0
            ll = (lp * mask).sum(-1)
            ll = ll / mask.sum(-1) if mean else ll
            assert float((ll - torch.from_numpy(z["f32/loglik_" + key])).abs().max()) < 1e-4, key
        seq = torch.from_numpy(z["f32/gen_prompt"])
        want = torch.from_numpy(z["f32/gen_out"])
        for t in range(seq.shape[1], want.shape[1]):
            nxt = O.forward_logits(p, c, want[:, :t])[0, -1].argmax()
            assert int(nxt) == int(want[0, t]), t


# ---- checkpoint layout and integration ------------------------------------------------------------------------------
def test_checkpoint_layout_equals_reference_state_dict(golden_dir, tmp_path):
    """write_unit_lm_checkpoint on a post-LN config writes the keys and shapes of the reference's UnitLM.state_dict()
    (project_in / project_out, no decoder final_layer_norm) and a base_config that round-trips through
    lm_config_from_hf."""
    from safetensors.torch import load_file
    from transformers import OPTConfig
    from slamkit_b200.lm import OptPostLnLMConfig, lm_config_from_hf, write_unit_lm_checkpoint
    z, c, _ = golden(golden_dir)
    p = O.init_params(c, seed=int(z["ckpt/seed_params"]))
    lm_cfg = OptPostLnLMConfig(vocab_size=502, hidden=128, n_layers=2, n_heads=2, ffn=256, max_positions=64, proj_dim=64)
    write_unit_lm_checkpoint(str(tmp_path), {**p, "lm.lm_head.weight": p["lm.model.decoder.embed_tokens.weight"]}, lm_cfg)
    sd = load_file(str(tmp_path / "model.safetensors"))
    keys = [str(k) for k in z["ckpt/keys"]]
    shapes = {k: json.loads(str(s)) for k, s in zip(keys, z["ckpt/shapes"])}
    assert "lm.model.decoder.project_in.weight" in keys and "lm.model.decoder.project_out.weight" in keys
    assert not any("decoder.final_layer_norm" in k for k in keys)
    assert sorted(sd) == sorted(k for k in keys if k != "lm.lm_head.weight")
    for k, t in sd.items():
        assert list(t.shape) == shapes[k], k
    cfg = json.load(open(tmp_path / "config.json"))
    assert cfg["base_model_name"] == "facebook/opt-350m"
    base = cfg["base_config"]
    written = json.loads(str(z["ckpt/base_config"]))
    assert base["do_layer_norm_before"] is False and base["word_embed_proj_dim"] == 64
    assert {k: v for k, v in base.items()} == {k: v for k, v in written.items()}
    back = lm_config_from_hf(OPTConfig(**{k: v for k, v in base.items() if k not in ("model_type", "architectures")}),
                             vocab_size=cfg["vocab_size"])
    assert back == lm_cfg


def test_integration_refuses_float32_for_post_ln(tmp_path):
    from slamkit_b200.integration import tlm_b200_config
    from slamkit_b200.lm import OptPostLnLMConfig
    _opt(hidden_size=128, ffn_dim=256, num_hidden_layers=2, num_attention_heads=2, word_embed_proj_dim=64,
         max_position_embeddings=256, vocab_size=600).save_pretrained(str(tmp_path))
    node = {"context_len": 64, "config_args": {"base_model_name": str(tmp_path), "vocab_size": 502,
                                               "torch_dtype": "float32"}}
    with pytest.raises(ValueError, match="bfloat16"):
        tlm_b200_config(node)
    node["config_args"]["torch_dtype"] = "bfloat16"
    c, master = tlm_b200_config(node)
    assert isinstance(c, OptPostLnLMConfig) and c.proj_dim == 64 and not master
