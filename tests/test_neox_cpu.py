"""CPU checks of the GPT-NeoX path: the fixture against the oracle, the config refusals, the fused-QKV permutation, the
checkpoint writer and the gradient-sync bucket plan of the NeoX layout.  No GPU needed."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import neox_oracle as O


def _golden(golden_dir):
    z = np.load(os.path.join(golden_dir, "neox_tiny.npz"))
    c = z["cfg"]
    cfg = O.OracleNeoxConfig(vocab_size=int(c[0]), hidden=int(c[1]), n_layers=int(c[2]), n_heads=int(c[3]), ffn=int(c[4]),
                             max_positions=int(c[5]), rot_dims=int(c[6]))
    return z, cfg, int(c[7])


def test_oracle_reproduces_fixture_logits_bitwise(golden_dir):
    z, c, seed = _golden(golden_dir)
    p = O.init_params(c, seed=seed)
    lo = O.forward_logits(p, c, torch.from_numpy(z["train/ids"]))
    ref = torch.from_numpy(z["nomask/logits_u16"].astype(np.uint16)).view(torch.bfloat16)
    assert torch.equal(lo.view(torch.int16), ref.view(torch.int16))
    pk = O.forward_logits(p, c, torch.from_numpy(z["packed/ids"]), torch.from_numpy(z["packed/position_ids"]), packed=True)
    refp = torch.from_numpy(z["packed/logits_u16"].astype(np.uint16)).view(torch.bfloat16)
    assert torch.equal(pk.view(torch.int16), refp.view(torch.int16))


def test_oracle_loss_and_gradients_near_fixture(golden_dir):
    z, c, seed = _golden(golden_dir)
    p = O.init_params(c, seed=seed)
    ids, labels = torch.from_numpy(z["train/ids"]), torch.from_numpy(z["train/labels"])
    loss, _, g = O.forward_backward(p, c, ids, labels, float(z["train/num_items"]))
    assert abs(float(loss) - float(z["nomask/loss"])) < 1e-3 * abs(float(z["nomask/loss"]))
    assert set(g) == {k[9:] for k in z.files if k.startswith("grad_d16/")}
    # the reference's Trainer-path gradients are stored as the difference from this backward: it is zero everywhere, so
    # the oracle reproduces every reference gradient bit for bit
    ref = O.golden_grads(z, p, c)
    assert all(not z["grad_d16/" + k].any() for k in p)
    assert all(torch.equal(ref[k].view(torch.int16), g[k].view(torch.int16)) for k in p)


def _hf_cfg(**kw):
    from transformers import GPTNeoXConfig
    base = dict(vocab_size=502, hidden_size=768, num_hidden_layers=12, num_attention_heads=12, intermediate_size=3072,
                max_position_embeddings=2048, tie_word_embeddings=False,
                rope_parameters={"rope_theta": 10000.0, "partial_rotary_factor": 0.25, "rope_type": "default"})
    base.update(kw)
    return GPTNeoXConfig(**base)


def test_pythia_160m_config_accepted():
    from slamkit_b200.lm import NeoxLMConfig, lm_config_from_hf
    c = lm_config_from_hf(_hf_cfg(), vocab_size=502)
    assert isinstance(c, NeoxLMConfig)
    assert (c.hidden, c.n_layers, c.n_heads, c.ffn, c.rot_dims, c.max_positions) == (768, 12, 12, 3072, 16, 2048)


@pytest.mark.parametrize("kw,field", [
    (dict(use_parallel_residual=False), "use_parallel_residual"),
    (dict(hidden_size=128, num_attention_heads=4, intermediate_size=512), "head_dim"),       # pythia-14m
    (dict(hidden_size=2048, num_attention_heads=8, intermediate_size=8192), "head_dim"),     # pythia-1b
    (dict(rope_parameters={"rope_theta": 10000.0, "partial_rotary_factor": 0.1, "rope_type": "default"}),
     "partial_rotary_factor"),
    (dict(rope_parameters={"rope_theta": 10000.0, "partial_rotary_factor": 0.25, "rope_type": "linear", "factor": 2.0}),
     "rope_type"),
    (dict(hidden_act="gelu_new"), "hidden_act"),
    (dict(attention_bias=False), "attention_bias"),
    (dict(tie_word_embeddings=True), "tie_word_embeddings"),
    (dict(attention_dropout=0.1), "attention_dropout"),
    (dict(hidden_dropout=0.1), "hidden_dropout"),
])
def test_unsupported_variants_refused_by_name(kw, field):
    from slamkit_b200.lm import lm_config_from_hf
    with pytest.raises(ValueError, match=field):
        lm_config_from_hf(_hf_cfg(**kw), vocab_size=502)


def test_qkv_permutation_round_trip():
    from slamkit_b200.lm import neox_qkv_segments
    H, hd = 5, 64
    d = H * hd
    segs = neox_qkv_segments(H, hd)
    hf = torch.randn(3 * d, 7)
    flat = torch.empty_like(hf)
    for f0, h0, n in segs:
        flat[f0:f0 + n] = hf[h0:h0 + n]
    # [Q; K; V]: q rows of head h at h*64, k rows at d + h*64, v rows at 2d + h*64
    view = hf.view(H, 3, hd, 7)
    for j in range(3):
        assert torch.equal(flat[j * d:(j + 1) * d], view[:, j].reshape(d, 7))
    back = torch.cat([flat[f0:f0 + n] for f0, h0, n in segs])   # segments are listed in HF row order
    assert torch.equal(back, hf)
    assert sorted(f0 for f0, _, _ in segs) == list(range(0, 3 * d, hd))


def test_checkpoint_writer_layout(golden_dir, tmp_path):
    """write_unit_lm_checkpoint writes the state dict and the gpt_neox base_config the reference's
    UnitLM.from_pretrained was shown (in the fixture) to load into the same keys and shapes."""
    from safetensors.torch import load_file
    from slamkit_b200.lm import NeoxLMConfig, write_unit_lm_checkpoint
    z, c, _ = _golden(golden_dir)
    p = O.init_params(c, seed=int(z["ckpt/seed_params"]))
    cfg = NeoxLMConfig(vocab_size=502, hidden=128, n_layers=2, n_heads=2, ffn=512, max_positions=64, rot_dims=16,
                       bos_token_id=1, eos_token_id=1)
    write_unit_lm_checkpoint(str(tmp_path), p, cfg, base_model_name="base")
    j = json.load(open(tmp_path / "config.json"))
    assert j["base_config"] == json.loads(str(z["ckpt/base_config"]))
    assert j["tie_word_embeddings"] is False and j["base_config"]["model_type"] == "gpt_neox"
    sd = load_file(str(tmp_path / "model.safetensors"))
    keys = [str(k) for k in z["ckpt/keys"]]
    shapes = [json.loads(str(s)) for s in z["ckpt/shapes"]]
    assert sorted(sd) == sorted(keys)
    for k, s in zip(keys, shapes):
        assert list(sd[k].shape) == s, k
        assert torch.equal(sd[k], p[k]), k
    assert str(z["ckpt/model_type"]) == "gpt_neox"


def test_gradsync_bucket_plan_covers_neox_layout():
    """The data-parallel gradient buckets (layer ranges from each layer's first tensor, `ln1`, plus the tail from
    `final_norm`) tile the NeoX flat layout: every layer tensor lies inside exactly one bucket."""
    from slamkit_b200.trainer import plan_buckets
    per_layer = ("ln1", "ln1_b", "ln2", "ln2_b", "wqkv", "bqkv", "wo", "bo", "w1", "b1", "w2", "b2")
    d, F, nl, V = 128, 512, 5, 512
    shape = {"ln1": d, "ln1_b": d, "ln2": d, "ln2_b": d, "wqkv": 3 * d * d, "bqkv": 3 * d, "wo": d * d, "bo": d,
             "w1": F * d, "b1": F, "w2": d * F, "b2": d}
    off, t = 0, {}
    for l in range(nl):
        for n in per_layer:
            t[f"layers.{l}.{n}"] = off
            off += (shape[n] + 63) // 64 * 64
    for n, size in (("final_norm", d), ("final_norm_b", d), ("embed", V * d), ("lm_head", V * d)):
        t[n] = off
        off += size
    layer_start = [t[f"layers.{l}.ln1"] for l in range(nl)] + [t["final_norm"]]
    buckets, tail = plan_buckets(layer_start, off, 2)
    spans = sorted((a, b) for _, a, b in buckets) + [tail]
    assert spans[0][0] == 0 and spans[-1][1] == off
    assert all(b0 == a1 for (_, b0), (a1, _) in zip(spans, spans[1:]))
    for l in range(nl):
        lo, hi = t[f"layers.{l}.ln1"], t[f"layers.{l}.b2"]
        assert sum(1 for a, b in spans if a <= lo and hi < b) == 1
