"""OPT with fp32 master weights, host side: the autocast oracle (oracle/opt_amp_oracle.py) against the reference's own
run (tests/golden/opt_amp_tiny.npz: UnitLM with fp32 parameters under bf16 autocast), the config rules that select the
mode, and the fp32 checkpoint."""
import hashlib
import json
import os

import numpy as np
import pytest
import torch

from oracle import opt_amp_oracle as A
from oracle.opt_oracle import OracleOptConfig


def _golden(golden_dir):
    z = np.load(os.path.join(golden_dir, "opt_amp_tiny.npz"))
    c = z["cfg"]
    cfg = OracleOptConfig(vocab_size=int(c[0]), hidden=int(c[1]), n_layers=int(c[2]), n_heads=int(c[3]), ffn=int(c[4]),
                          max_positions=int(c[5]))
    return z, cfg, A.init_params_fp32(cfg, seed=int(c[6]))


def test_amp_oracle_reproduces_reference_bit_for_bit(golden_dir):
    """Loss, logits and every fp32 gradient are the reference's exactly (same ops in the same order); the clip norm too."""
    z, cfg, p = _golden(golden_dir)
    ids, labels = torch.from_numpy(z["ids"]), torch.from_numpy(z["labels"])
    loss, logits, g = A.forward_backward_amp(p, cfg, ids, labels, float(z["num_items"]), attention_mask=(ids != 0).long())
    assert float(loss) == float(z["loss"])
    assert logits.dtype == torch.bfloat16
    ref_logits = torch.from_numpy(z["logits_u16"].view(np.int16)).view(torch.bfloat16)
    valid = ids != 0           # pad queries: the reference's mask and the causal mask differ there, neither is scored
    assert torch.equal(logits[valid], ref_logits[valid])
    for k in p:
        flat = g[k].contiguous().view(-1)
        assert g[k].dtype == torch.float32 and torch.equal(flat[A.sample_index(flat.numel())], torch.from_numpy(z["grad/" + k])), k
        assert hashlib.sha256(flat.numpy().astype("<f4").tobytes()).hexdigest() == str(z["grad_sha256/" + k]), k
    tr = A.OracleOptAmpTrainer(p, cfg, lr=1e-3, max_grad_norm=0.5)
    tr.apply(g)
    assert float(tr.last_total_norm) == float(z["total_norm"])


def test_amp_oracle_adamw_step_within_one_ulp_of_reference(golden_dir):
    """After clip + AdamW each fp32 parameter is within 2 ulps of max(|p_old|, |p_new|, lr) of the reference's: torch's
    fused CPU AdamW contracts some multiply-adds that the oracle (like the GPU kernel) rounds one by one, which moves
    the update (about lr on a first step) by an ulp or two of its own and the subtraction p - update by one ulp of p."""
    z, cfg, p = _golden(golden_dir)
    ids, labels = torch.from_numpy(z["ids"]), torch.from_numpy(z["labels"])
    _, _, g = A.forward_backward_amp(p, cfg, ids, labels, float(z["num_items"]), attention_mask=(ids != 0).long())
    tr = A.OracleOptAmpTrainer(p, cfg, lr=1e-3, max_grad_norm=0.5)
    tr.apply(g)
    for k in p:
        idx = A.sample_index(p[k].numel())            # the fixture keeps ~1024 evenly spaced elements per tensor
        ref = torch.from_numpy(z["post/" + k])
        ours, old = tr.p[k].reshape(-1)[idx], p[k].reshape(-1)[idx]
        big = torch.maximum(torch.maximum(ref.abs(), ours.abs()), old.abs()).clamp(min=1e-3)
        ulp = torch.nextafter(big, torch.tensor(float("inf"))) - big
        assert bool(((ours - ref).abs() <= 2 * ulp).all()), k
        assert float((tr.p[k] - p[k]).abs().max()) > 0, k


def _base(tmp_path, model_type="opt"):
    if model_type == "opt":
        from transformers import OPTConfig
        OPTConfig(hidden_size=128, ffn_dim=256, num_hidden_layers=2, num_attention_heads=2, word_embed_proj_dim=128,
                  max_position_embeddings=256).save_pretrained(str(tmp_path))
    else:
        from transformers import GPTNeoXConfig
        GPTNeoXConfig(hidden_size=128, intermediate_size=512, num_hidden_layers=2, num_attention_heads=2,
                      rotary_pct=0.25, max_position_embeddings=256).save_pretrained(str(tmp_path))
    return {"context_len": 64, "config_args": {"base_model_name": str(tmp_path), "vocab_size": 502, "twist_init": False,
                                               "dropout": 0.0, "attention_dropout": 0.0, "layerdrop": 0.0,
                                               "hidden_dropout": 0.0}}


def test_float32_selects_master_weights_and_other_dtypes_are_refused_by_name(tmp_path):
    from slamkit_b200.integration import tlm_b200_config
    from slamkit_b200.lm import OptLMConfig
    cfg = _base(tmp_path)
    for dt, want in (("float32", True), ("torch.float32", True), ("bfloat16", False)):
        cfg["config_args"]["torch_dtype"] = dt
        lm_cfg, master = tlm_b200_config(cfg)
        assert isinstance(lm_cfg, OptLMConfig) and master is want, dt
    assert tlm_b200_config(cfg, autocast_bf16=True)[1] is False
    cfg["config_args"]["torch_dtype"] = "float32"
    assert tlm_b200_config(cfg, autocast_bf16=True)[1] is True
    with pytest.raises(ValueError, match=r"training_args\.bf16"):
        tlm_b200_config(cfg, autocast_bf16=False)
    for dt in (None, "float16"):
        cfg["config_args"]["torch_dtype"] = dt
        with pytest.raises(ValueError, match="torch_dtype=bfloat16") as e:
            tlm_b200_config(cfg)
        assert "torch_dtype=float32" in str(e.value)


def test_neox_float32_stays_refused(tmp_path):
    from slamkit_b200.integration import tlm_b200_config
    cfg = _base(tmp_path, "gpt_neox")
    cfg["config_args"]["torch_dtype"] = "float32"
    with pytest.raises(ValueError, match="torch_dtype"):
        tlm_b200_config(cfg)
    cfg["config_args"]["torch_dtype"] = "bfloat16"
    assert tlm_b200_config(cfg)[1] is False


def test_checkpoint_writer_emits_fp32_tensors_and_dtype(tmp_path):
    from safetensors.torch import load_file
    from slamkit_b200.lm import OptLMConfig, write_unit_lm_checkpoint
    cfg = OracleOptConfig(vocab_size=502, hidden=128, n_layers=1, n_heads=2, ffn=256, max_positions=64)
    p = A.init_params_fp32(cfg, seed=1)
    lm_cfg = OptLMConfig(vocab_size=502, hidden=128, n_layers=1, n_heads=2, ffn=256, max_positions=64)
    write_unit_lm_checkpoint(str(tmp_path), {**p, "lm.lm_head.weight": p["lm.model.decoder.embed_tokens.weight"]}, lm_cfg,
                             base_model_name="facebook/opt-125m", torch_dtype="float32")
    sd = load_file(os.path.join(tmp_path, "model.safetensors"))
    assert set(sd) == set(p) and all(v.dtype == torch.float32 and torch.equal(v, p[k]) for k, v in sd.items())
    c = json.load(open(os.path.join(tmp_path, "config.json")))
    assert c["torch_dtype"] == "float32" and c["base_config"]["torch_dtype"] == "float32"
    from transformers import OPTConfig
    from slamkit_b200.lm import OptLMConfig as OC
    base = {k: v for k, v in c["base_config"].items() if k not in ("model_type", "architectures")}
    assert OC.from_hf(OPTConfig(**base), vocab_size=c["vocab_size"]) == lm_cfg
