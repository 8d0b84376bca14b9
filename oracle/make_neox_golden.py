"""Generate tests/golden/neox_tiny.npz by running the REFERENCE's own `slamkit.model.unit_lm.UnitLM` over a tiny GPT-NeoX
base.

TEST INFRASTRUCTURE ONLY -- run once by hand (`python oracle/make_neox_golden.py`) where the reference is importable; the
fixture is committed and nothing at test or bench time imports the reference.

The base is a parallel-residual GPT-NeoX (2 layers, hidden 128, 2 heads, ffn 512, vocab 502, 64 positions,
partial_rotary_factor 0.25, untied embed_out, bf16) written as a config.json in a temporary directory, loaded the way
config/train_inter_scale.yaml does (torch_dtype bfloat16; twist_init=false), with the seeded parameters of
oracle.neox_oracle.init_params.  Recorded, under the keys below:
  train/*     loss, logits, every gradient, the clip_grad_norm_(0.5) total norm and the parameters after one fused
              AdamW step (lr 1e-3), on a right-padded [2, 32] batch with its attention_mask under bf16 autocast
              (the HF Trainer path); nomask/* the same batch without mask and autocast (pure causal path).  The
              Trainer-path logits are stored as the bit-pattern difference from the unmasked logits
              (oracle.neox_oracle.golden_masked_logits decodes them exactly), every gradient as the bit-pattern difference from
              the CPU oracle's bf16 backward (oracle.neox_oracle.golden_grads); the AdamW step is kept as the sign of every element's update (upd_sign/*, int8) and each
              tensor's mean |update| (upd_absmean/*): a first step moves each element by about lr * sign(grad)
  packed/*    one packed row (4 documents, restarting position_ids) with the explicit block-diagonal causal 4-D mask
  loglik/*    UnitLM.log_likelihood, summed and mean, on a right-padded batch
  ckpt/*      the state-dict keys, shapes and fingerprints UnitLM.from_pretrained gives on a directory written by
              slamkit_b200.lm.write_unit_lm_checkpoint, and its base_config
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

from oracle.make_goldens import REF, _param_digest, _stub_omegaconf, bf16_to_u16  # noqa: E402
from oracle.neox_oracle import OracleNeoxConfig, forward_backward, init_params, packed_mask, u16_delta  # noqa: E402

CFG = OracleNeoxConfig(vocab_size=502, hidden=128, n_layers=2, n_heads=2, ffn=512, max_positions=64, rot_dims=16)
SEED_PARAMS = 123


def base_config(c: OracleNeoxConfig) -> dict:
    return {"model_type": "gpt_neox", "architectures": ["GPTNeoXForCausalLM"], "hidden_size": c.hidden,
            "intermediate_size": c.ffn, "num_hidden_layers": c.n_layers, "num_attention_heads": c.n_heads,
            "vocab_size": c.vocab_size, "max_position_embeddings": c.max_positions, "layer_norm_eps": c.ln_eps,
            "use_parallel_residual": True, "hidden_act": "gelu", "attention_bias": True, "attention_dropout": 0.0,
            "hidden_dropout": 0.0, "initializer_range": 0.02, "tie_word_embeddings": False,
            "rope_parameters": {"rope_theta": c.rope_theta, "partial_rotary_factor": c.rot_dims / c.head_dim,
                                "rope_type": "default"},
            "pad_token_id": 0, "bos_token_id": 1, "eos_token_id": 1, "torch_dtype": "bfloat16"}


def reference_model(params):
    from slamkit.model.unit_lm import UnitLM, UnitLMConfig
    tmp = tempfile.mkdtemp()
    json.dump(base_config(CFG), open(os.path.join(tmp, "config.json"), "w"))
    cfg = UnitLMConfig(base_model_name=tmp, vocab_size=CFG.vocab_size, twist_init=False, torch_dtype="bfloat16")
    torch.manual_seed(0)
    model = UnitLM(cfg)
    sd = model.state_dict()
    for k, v in params.items():
        assert k in sd and sd[k].shape == v.shape and sd[k].dtype == torch.bfloat16, k
    missing = [k for k in sd if k not in params]
    assert not missing, missing
    model.load_state_dict(params, strict=True)
    assert model.lm.embed_out.weight.data_ptr() != model.lm.gpt_neox.embed_in.weight.data_ptr(), "embeddings tied"
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
    attn = (ids != 0).long()
    num_items = float((labels != -100).sum())
    with torch.autocast("cpu", dtype=torch.bfloat16):
        out = model(input_ids=ids, attention_mask=attn, labels=labels, num_items_in_batch=num_items)
    out.loss.backward()
    with torch.no_grad():
        nomask = model(input_ids=ids, labels=labels, num_items_in_batch=num_items)
    grads = {k: p.grad.detach().clone() for k, p in model.named_parameters()}
    opt = torch.optim.AdamW(model.parameters(), lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0, fused=True)
    total_norm = torch.nn.utils.clip_grad_norm_(model.parameters(), 0.5)
    opt.step()
    blob.update({"train/ids": ids.numpy(), "train/labels": labels.numpy(), "train/num_items": np.float32(num_items),
                 "train/loss": np.float32(out.loss.item()),
                 "train/logits_d16": u16_delta(bf16_to_u16(out.logits.detach()), bf16_to_u16(nomask.logits)),
                 "train/total_norm": np.float32(float(total_norm)),
                 "nomask/loss": np.float32(nomask.loss.item()), "nomask/logits_u16": bf16_to_u16(nomask.logits),
                 "cfg": np.array([CFG.vocab_size, CFG.hidden, CFG.n_layers, CFG.n_heads, CFG.ffn, CFG.max_positions,
                                  CFG.rot_dims, SEED_PARAMS], dtype=np.int64)})
    # every gradient as the bit-pattern difference from the CPU oracle's bf16 backward on the same batch (the two agree
    # almost everywhere, so the difference compresses to almost nothing); oracle.neox_oracle.golden_grads decodes it
    _, _, ograds = forward_backward(params, CFG, ids, labels, num_items)
    for k, v in grads.items():
        blob["grad_d16/" + k] = u16_delta(bf16_to_u16(v), bf16_to_u16(ograds[k]))
    for k, p in model.named_parameters():
        upd = p.detach().float() - params[k].float()
        blob["upd_sign/" + k] = torch.sign(upd).to(torch.int8).numpy()
        blob["upd_absmean/" + k] = np.float32(upd.abs().mean())
    print("neox train: loss", out.loss.item(), "total_norm", float(total_norm))


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
        alone = [model(input_ids=d[None]).logits[0] for d in docs]
    off = 0
    for n, a in zip(lens, alone):
        assert float((a.float() - out.logits[0, off:off + n].float()).abs().max()) < 2e-2
        off += n
    blob.update({"packed/ids": ids.numpy(), "packed/position_ids": pos.numpy(), "packed/labels": labels.numpy(),
                 "packed/num_items": np.float32(num_items), "packed/loss": np.float32(out.loss.item()),
                 "packed/logits_u16": bf16_to_u16(out.logits)})
    print("neox packed: loss", out.loss.item())


def loglik_blob(blob):
    model = reference_model(init_params(CFG, seed=3))
    model.eval()
    g = torch.Generator().manual_seed(11)
    tokens = torch.randint(2, 502, (3, 40), generator=g)
    tokens[:, 0] = 1
    tokens[1, 25:] = 0
    tokens[2, 33:] = 0
    ll_sum = model.log_likelihood(tokens.clone(), mean_nll=False)
    ll_mean = model.log_likelihood(tokens.clone(), mean_nll=True)
    blob.update({"loglik/tokens": tokens.numpy(), "loglik/sum": ll_sum.float().numpy(), "loglik/mean": ll_mean.float().numpy(),
                 "loglik/seed_params": np.int64(3)})
    print("neox loglik:", ll_sum.tolist(), ll_mean.tolist())


def checkpoint_blob(blob):
    import slamkit.model.unit_lm as ref_mod
    from slamkit.model.unit_lm import UnitLM
    from slamkit_b200.lm import NeoxLMConfig, write_unit_lm_checkpoint
    from transformers import OPTConfig
    real = ref_mod.AutoConfig.from_pretrained
    # the reference's default base model is looked up on the hub (unit_lm.py:37,66-70): stand in for that one lookup
    ref_mod.AutoConfig.from_pretrained = staticmethod(
        lambda name, *a, **k: OPTConfig() if name == "facebook/opt-350M" else real(name, *a, **k))
    p = init_params(CFG, seed=5)
    tmp = tempfile.mkdtemp()
    base, ck = os.path.join(tmp, "base"), os.path.join(tmp, "ck")
    os.makedirs(base)
    cfg = NeoxLMConfig(vocab_size=502, hidden=128, n_layers=2, n_heads=2, ffn=512, max_positions=64, rot_dims=16,
                       bos_token_id=1, eos_token_id=1)
    write_unit_lm_checkpoint(ck, p, cfg, base_model_name=base)
    written = json.load(open(os.path.join(ck, "config.json")))["base_config"]
    json.dump(written, open(os.path.join(base, "config.json"), "w"))
    model = UnitLM.from_pretrained(ck, torch_dtype=torch.bfloat16)
    sd = model.state_dict()
    keys = sorted(sd)
    for k in keys:
        if k in p:
            assert torch.equal(sd[k], p[k]), k
    blob.update({"ckpt/keys": np.array(keys), "ckpt/digests": np.stack([_param_digest(sd[k]) for k in keys]),
                 "ckpt/shapes": np.array([json.dumps(list(sd[k].shape)) for k in keys]),
                 "ckpt/base_config": np.array(json.dumps(written)), "ckpt/seed_params": np.int64(5),
                 "ckpt/model_type": np.array(model.lm.config.model_type)})
    print("neox checkpoint:", len(keys), "keys")


if __name__ == "__main__":
    assert os.path.isdir(REF), "the reference must be importable to produce the fixture"
    _stub_omegaconf()
    sys.path.insert(0, REF)
    blob = {}
    train_blob(blob)
    packed_blob(blob)
    loglik_blob(blob)
    checkpoint_blob(blob)
    out = os.path.join(ROOT, "tests", "golden", "neox_tiny.npz")
    np.savez_compressed(out, **blob)
    print("->", out, os.path.getsize(out), "bytes")
