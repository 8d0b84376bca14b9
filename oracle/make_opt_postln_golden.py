"""Generate tests/golden/opt_postln_tiny.npz by running the REFERENCE's own `slamkit.model.unit_lm.UnitLM` over a tiny
post-LayerNorm OPT base (the opt-350m layout: do_layer_norm_before=False, word_embed_proj_dim < hidden_size, no decoder
final_layer_norm).

TEST INFRASTRUCTURE ONLY -- run once by hand (`python oracle/make_opt_postln_golden.py`) where the reference is
importable; the fixture is committed and nothing at test or bench time imports the reference.

The base has 2 layers, hidden 128, 2 heads, ffn 256, word_embed_proj_dim 64, vocab 502, written as a config.json in a
temporary directory and loaded the way config/model/twist.yaml does (twist_init=false), with the seeded parameters of
oracle.opt_postln_oracle.init_params.  Recorded, under the keys below:
  train/*     bf16 (torch_dtype bfloat16, no autocast): loss, logits, every gradient, the clip_grad_norm_(0.5) total
              norm and one fused AdamW step (lr 1e-3) kept as the sign of every element's update (upd_sign/*) and each
              tensor's mean |update| (upd_absmean/*), on a right-padded [2, 32] batch whose pad targets are -100
  packed/*    one packed row (4 documents, restarting position_ids) with the explicit block-diagonal causal 4-D mask
  f32/*       float32 (torch_dtype float32): logits of a right-padded batch, log_likelihood summed and mean with and
              without ignore_tokens, and a greedy generate with its per-step top-1 / top-2 margins
  ckpt/*      the state-dict keys and shapes UnitLM.from_pretrained gives on a directory written by
              slamkit_b200.lm.write_unit_lm_checkpoint for a post-LN config, and its base_config
"""
import json
import os
import sys
import tempfile

import numpy as np
import torch

os.environ.setdefault("HF_HUB_OFFLINE", "1")       # everything below is local: never look anything up on the hub
os.environ.setdefault("TRANSFORMERS_OFFLINE", "1")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle.make_goldens import REF, _stub_omegaconf, bf16_to_u16  # noqa: E402
from oracle.opt_postln_oracle import OraclePostLnConfig, init_params, packed_mask  # noqa: E402

CFG = OraclePostLnConfig(vocab_size=502, hidden=128, n_layers=2, n_heads=2, ffn=256, max_positions=64, proj_dim=64)
SEED_PARAMS = 123
SEED_F32 = 321
STD_F32 = 0.1


def base_config(c: OraclePostLnConfig, torch_dtype: str = "bfloat16") -> dict:
    return {"model_type": "opt", "architectures": ["OPTForCausalLM"], "hidden_size": c.hidden, "ffn_dim": c.ffn,
            "num_hidden_layers": c.n_layers, "num_attention_heads": c.n_heads, "vocab_size": c.vocab_size,
            "max_position_embeddings": c.max_positions, "do_layer_norm_before": False, "word_embed_proj_dim": c.proj_dim,
            "activation_function": "relu", "enable_bias": True, "layer_norm_elementwise_affine": True,
            "dropout": 0.0, "attention_dropout": 0.0, "layerdrop": 0.0, "init_std": 0.02, "tie_word_embeddings": True,
            "pad_token_id": 0, "bos_token_id": 1, "eos_token_id": 1, "torch_dtype": torch_dtype}


def reference_model(params, dtype=torch.bfloat16):
    from slamkit.model.unit_lm import UnitLM, UnitLMConfig
    tmp = tempfile.mkdtemp()
    name = "float32" if dtype == torch.float32 else "bfloat16"
    json.dump(base_config(CFG, name), open(os.path.join(tmp, "config.json"), "w"))
    cfg = UnitLMConfig(base_model_name=tmp, vocab_size=CFG.vocab_size, twist_init=False,
                       torch_dtype=None if dtype == torch.float32 else "bfloat16")
    torch.manual_seed(0)
    model = UnitLM(cfg)
    sd = model.state_dict()
    for k, v in params.items():
        assert k in sd and sd[k].shape == v.shape and sd[k].dtype == dtype, k
    missing = [k for k in sd if k not in params and k != "lm.lm_head.weight"]
    assert not missing, missing
    assert not any("decoder.final_layer_norm" in k for k in sd), "post-LN OPT has no decoder final_layer_norm"
    model.load_state_dict({**params, "lm.lm_head.weight": params["lm.model.decoder.embed_tokens.weight"]}, strict=True)
    assert model.lm.lm_head.weight.data_ptr() == model.lm.model.decoder.embed_tokens.weight.data_ptr(), "embeddings not tied"
    return model


def train_blob(blob):
    params = init_params(CFG, seed=SEED_PARAMS)
    model = reference_model(params)
    model.train()
    g = torch.Generator().manual_seed(7)
    B, T = 2, 32
    ids = torch.randint(2, 502, (B, T), generator=g)
    ids[:, 0] = 1
    ids[1, 26:] = 0                      # right padding as DataCollatorForLanguageModeling emits
    labels = ids.clone()
    labels[ids == 0] = -100
    num_items = float((labels != -100).sum())
    out = model(input_ids=ids, labels=labels, num_items_in_batch=num_items)
    out.loss.backward()
    grads = {k: p.grad.detach().clone() for k, p in model.named_parameters()}
    opt = torch.optim.AdamW(model.parameters(), lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0, fused=True)
    total_norm = torch.nn.utils.clip_grad_norm_(model.parameters(), 0.5)
    opt.step()
    blob.update({"train/ids": ids.numpy(), "train/labels": labels.numpy(), "train/num_items": np.float32(num_items),
                 "train/loss": np.float32(out.loss.item()), "train/logits_u16": bf16_to_u16(out.logits.detach()),
                 "train/total_norm": np.float32(float(total_norm)),
                 "cfg": np.array([CFG.vocab_size, CFG.hidden, CFG.n_layers, CFG.n_heads, CFG.ffn, CFG.max_positions,
                                  CFG.proj_dim, SEED_PARAMS], dtype=np.int64)})
    for k, v in grads.items():
        blob["grad/" + k] = bf16_to_u16(v)
    for k, p in model.named_parameters():
        upd = p.detach().float() - params[k].float()
        blob["upd_sign/" + k] = torch.sign(upd).to(torch.int8).numpy()
        blob["upd_absmean/" + k] = np.float32(upd.abs().mean())
    print("post-LN train: loss", out.loss.item(), "total_norm", float(total_norm))


def packed_blob(blob):
    model = reference_model(init_params(CFG, seed=SEED_PARAMS))
    model.eval()
    g = torch.Generator().manual_seed(9)
    lens = [16, 1, 15, 16]
    docs = [torch.randint(2, 502, (n,), generator=g) for n in lens]
    ids = torch.cat(docs)[None]
    pos = torch.cat([torch.arange(n) for n in lens])[None]
    labels = ids.clone()
    for a in np.cumsum([0] + lens[:-1]):
        labels[0, a] = -100
    num_items = float((labels[:, 1:] != -100).sum())
    T = ids.shape[1]
    mask4d = torch.zeros(1, 1, T, T, dtype=torch.bfloat16).masked_fill(~packed_mask(pos), torch.finfo(torch.bfloat16).min)
    with torch.no_grad():
        out = model(input_ids=ids, attention_mask=mask4d, position_ids=pos, labels=labels, num_items_in_batch=num_items)
    blob.update({"packed/ids": ids.numpy(), "packed/position_ids": pos.numpy(), "packed/labels": labels.numpy(),
                 "packed/num_items": np.float32(num_items), "packed/loss": np.float32(out.loss.item()),
                 "packed/logits_u16": bf16_to_u16(out.logits)})
    print("post-LN packed: loss", out.loss.item())


def f32_blob(blob):
    model = reference_model(init_params(CFG, seed=SEED_F32, std=STD_F32, dtype=torch.float32), dtype=torch.float32)
    model.eval()
    g = torch.Generator().manual_seed(7)
    ids = torch.randint(2, 502, (2, 32), generator=g)
    ids[:, 0] = 1
    ids[1, 26:] = 0
    with torch.no_grad():
        z = model(input_ids=ids).logits
    assert z.dtype == torch.float32
    blob.update({"f32/seed_params": np.int64(SEED_F32), "f32/std": np.float32(STD_F32), "f32/ids": ids.numpy(),
                 "f32/logits": z.numpy()})
    g = torch.Generator().manual_seed(11)
    tokens = torch.randint(2, 502, (3, 40), generator=g)
    tokens[:, 0] = 1
    tokens[1, 25:] = 0
    tokens[2, 33:] = 0
    present = set(tokens.flatten().tolist())
    ignore = sorted(i for i in torch.randperm(500, generator=g).add(2).tolist() if i not in present)[:100]
    ll = {"sum": model.log_likelihood(tokens.clone(), mean_nll=False),
          "mean": model.log_likelihood(tokens.clone(), mean_nll=True),
          "sum_ign": model.log_likelihood(tokens.clone(), mean_nll=False, ignore_tokens=ignore),
          "mean_ign": model.log_likelihood(tokens.clone(), mean_nll=True, ignore_tokens=ignore)}
    for k, v in ll.items():
        assert v.dtype == torch.float32, k
        blob["f32/loglik_" + k] = v.numpy()
    blob.update({"f32/loglik_tokens": tokens.numpy(), "f32/loglik_ignore": np.array(ignore, dtype=np.int64)})
    prompt = torch.tensor([[1, 17, 33, 5, 250, 9, 41, 77]])
    out = model.generate(prompt, max_new_tokens=16, do_sample=False, return_dict_in_generate=True, output_scores=True)
    top2 = torch.stack([torch.topk(s[0].float(), 2).values for s in out.scores])
    blob.update({"f32/gen_prompt": prompt.numpy(), "f32/gen_out": out.sequences.numpy(),
                 "f32/gen_margin": (top2[:, 0] - top2[:, 1]).numpy()})
    print("post-LN fp32: loglik", {k: v.tolist() for k, v in ll.items()})
    print("post-LN fp32: generate", out.sequences.tolist(), "min margin", float(blob["f32/gen_margin"].min()))


def checkpoint_blob(blob):
    import slamkit.model.unit_lm as ref_mod
    from slamkit.model.unit_lm import UnitLM
    from slamkit_b200.lm import OptPostLnLMConfig, write_unit_lm_checkpoint
    from transformers import OPTConfig
    real = ref_mod.AutoConfig.from_pretrained
    # the reference's default base model is looked up on the hub (unit_lm.py:37,66-70): stand in for that one lookup
    ref_mod.AutoConfig.from_pretrained = staticmethod(
        lambda name, *a, **k: OPTConfig() if name == "facebook/opt-350M" else real(name, *a, **k))
    p = init_params(CFG, seed=5)
    tmp = tempfile.mkdtemp()
    base, ck = os.path.join(tmp, "base"), os.path.join(tmp, "ck")
    os.makedirs(base)
    cfg = OptPostLnLMConfig(vocab_size=502, hidden=128, n_layers=2, n_heads=2, ffn=256, max_positions=64, proj_dim=64)
    write_unit_lm_checkpoint(ck, {**p, "lm.lm_head.weight": p["lm.model.decoder.embed_tokens.weight"]}, cfg,
                             base_model_name=base)
    written = json.load(open(os.path.join(ck, "config.json")))["base_config"]
    json.dump(written, open(os.path.join(base, "config.json"), "w"))
    model = UnitLM.from_pretrained(ck, torch_dtype=torch.bfloat16)
    sd = model.state_dict()
    keys = sorted(sd)
    for k in keys:
        if k in p:
            assert torch.equal(sd[k], p[k]), k
    blob.update({"ckpt/keys": np.array(keys), "ckpt/shapes": np.array([json.dumps(list(sd[k].shape)) for k in keys]),
                 "ckpt/base_config": np.array(json.dumps(written)), "ckpt/seed_params": np.int64(5)})
    print("post-LN checkpoint:", len(keys), "keys")


if __name__ == "__main__":
    assert os.path.isdir(REF), "the reference must be importable to produce the fixture"
    _stub_omegaconf()
    sys.path.insert(0, REF)
    blob = {}
    train_blob(blob)
    packed_blob(blob)
    f32_blob(blob)
    checkpoint_blob(blob)
    out = os.path.join(ROOT, "tests", "golden", "opt_postln_tiny.npz")
    np.savez_compressed(out, **blob)
    print("->", out, os.path.getsize(out), "bytes")
