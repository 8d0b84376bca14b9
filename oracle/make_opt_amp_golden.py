"""Generate tests/golden/opt_amp_tiny.npz by running the REFERENCE's own `slamkit.model.unit_lm.UnitLM` with fp32
parameters under bf16 autocast: its default TWIST / GSLM training precision (`torch_dtype: null` -> fp32, `bf16: True`).

TEST INFRASTRUCTURE ONLY -- run once by hand (`python oracle/make_opt_amp_golden.py`) where the reference is importable;
the fixture is committed and nothing at test or bench time imports the reference.

The base is the tiny pre-LayerNorm OPT of oracle/make_opt_golden.py (1 layer, hidden 128, 2 heads, ffn 256, vocab 502),
loaded with torch_dtype=float32 and the seeded fp32 parameters of oracle.opt_amp_oracle.init_params_fp32.  On the same
right-padded [2, 32] batch with its attention_mask, under torch.autocast("cpu", bfloat16), recorded:
  loss, logits_u16 (bf16 bit patterns) and total_norm (clip_grad_norm_(0.5));
  grad_sha256/<name>   SHA-256 of the fp32 .grad of every parameter (its little-endian bytes): a bit-exact check of the
                       whole tensor in 64 bytes;
  grad/<name>, post/<name>   the fp32 .grad and the fp32 parameter after one fused AdamW step (lr 1e-3) at the elements
                       sample_index(numel) picks (about 1024 per tensor, evenly spaced), which keeps the fixture small.
"""
import hashlib
import json
import os
import sys
import tempfile

import numpy as np
import torch

os.environ.setdefault("HF_HUB_OFFLINE", "1")
os.environ.setdefault("TRANSFORMERS_OFFLINE", "1")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle.make_goldens import REF, _stub_omegaconf, bf16_to_u16  # noqa: E402
from oracle.make_opt_golden import CFG, SEED_PARAMS, base_config  # noqa: E402
from oracle.opt_amp_oracle import init_params_fp32, sample_index  # noqa: E402


def reference_model(params):
    from slamkit.model.unit_lm import UnitLM, UnitLMConfig
    tmp = tempfile.mkdtemp()
    json.dump({**base_config(CFG), "torch_dtype": "float32"}, open(os.path.join(tmp, "config.json"), "w"))
    cfg = UnitLMConfig(base_model_name=tmp, vocab_size=CFG.vocab_size, twist_init=False, torch_dtype="float32")
    torch.manual_seed(0)
    model = UnitLM(cfg)
    sd = model.state_dict()
    for k, v in params.items():
        assert k in sd and sd[k].shape == v.shape and sd[k].dtype == torch.float32, k
    model.load_state_dict({**params, "lm.lm_head.weight": params["lm.model.decoder.embed_tokens.weight"]}, strict=True)
    assert model.lm.lm_head.weight.data_ptr() == model.lm.model.decoder.embed_tokens.weight.data_ptr(), "embeddings not tied"
    return model


def train_blob(blob):
    params = init_params_fp32(CFG, seed=SEED_PARAMS)
    model = reference_model(params)
    model.train()
    g = torch.Generator().manual_seed(7)
    B, T = 2, 32
    ids = torch.randint(2, 502, (B, T), generator=g)
    ids[:, 0] = 1
    ids[1, 26:] = 0
    labels = ids.clone()
    labels[ids == 0] = -100
    attn = (ids != 0).long()
    num_items = float((labels != -100).sum())
    with torch.autocast("cpu", dtype=torch.bfloat16):
        out = model(input_ids=ids, attention_mask=attn, labels=labels, num_items_in_batch=num_items)
    out.loss.backward()
    grads = {k: p.grad.detach().clone() for k, p in model.named_parameters()}
    assert all(v.dtype == torch.float32 for v in grads.values())
    opt = torch.optim.AdamW(model.parameters(), lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0, fused=True)
    total_norm = torch.nn.utils.clip_grad_norm_(model.parameters(), 0.5)
    opt.step()
    blob.update({"ids": ids.numpy(), "labels": labels.numpy(), "num_items": np.float32(num_items),
                 "loss": np.float32(out.loss.item()), "logits_u16": bf16_to_u16(out.logits.detach()),
                 "total_norm": np.float32(float(total_norm)),
                 "cfg": np.array([CFG.vocab_size, CFG.hidden, CFG.n_layers, CFG.n_heads, CFG.ffn, CFG.max_positions,
                                  SEED_PARAMS], dtype=np.int64)})
    for k, v in grads.items():
        flat = v.contiguous().view(-1)
        blob["grad_sha256/" + k] = np.array(hashlib.sha256(flat.numpy().astype("<f4").tobytes()).hexdigest())
        blob["grad/" + k] = flat[sample_index(flat.numel())].numpy()
    for k, p in model.named_parameters():
        blob["post/" + k] = p.detach().reshape(-1)[sample_index(p.numel())].numpy().copy()
    print("opt amp train: loss", out.loss.item(), "total_norm", float(total_norm), "logits", out.logits.dtype)


if __name__ == "__main__":
    assert os.path.isdir(REF), "the reference must be importable to produce the fixture"
    _stub_omegaconf()
    sys.path.insert(0, REF)
    blob = {}
    train_blob(blob)
    out = os.path.join(ROOT, "tests", "golden", "opt_amp_tiny.npz")
    np.savez_compressed(out, **blob)
    print("->", out, os.path.getsize(out), "bytes")
