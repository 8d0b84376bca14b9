"""Generate tests/golden/opt_fp32_tiny.npz by running the REFERENCE's own `slamkit.model.unit_lm.UnitLM` in fp32: how the
reference scores and generates a float32 TWIST / GSLM checkpoint (`torch_dtype` null loads fp32; cli/eval.py runs no
autocast).

TEST INFRASTRUCTURE ONLY -- run once by hand (`python oracle/make_opt_fp32_golden.py`) where the reference is importable;
the fixture is committed and nothing at test or bench time imports the reference.

The base is the tiny pre-LayerNorm OPT of oracle/make_opt_golden.py (1 layer, hidden 128, 2 heads, ffn 256, vocab 502),
loaded with torch_dtype None (fp32) on the CPU, with fp32 parameters from oracle.opt_oracle.init_params (std 0.1, so that
greedy steps have clear margins).  Recorded:
  logits/ids, logits/z        fp32 logits of a right-padded [2, 32] batch passed without a mask, as log_likelihood does
  loglik/tokens, loglik/ignore, loglik/{sum,mean,sum_ign,mean_ign}
                              UnitLM.log_likelihood summed and mean, without and with ignore_tokens
  gen/prompt, gen/out, gen/margin
                              greedy UnitLM.generate (max_new_tokens 16) and the top-1 / top-2 margin of each step's logits
"""
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

from oracle.make_goldens import REF, _stub_omegaconf  # noqa: E402
from oracle.make_opt_golden import CFG, base_config  # noqa: E402
from oracle.opt_oracle import init_params  # noqa: E402

SEED_PARAMS = 321
STD = 0.1


def reference_model(params):
    from slamkit.model.unit_lm import UnitLM, UnitLMConfig
    tmp = tempfile.mkdtemp()
    json.dump({**base_config(CFG), "torch_dtype": "float32"}, open(os.path.join(tmp, "config.json"), "w"))
    cfg = UnitLMConfig(base_model_name=tmp, vocab_size=CFG.vocab_size, twist_init=False, torch_dtype=None)
    torch.manual_seed(0)
    model = UnitLM(cfg)
    sd = model.state_dict()
    for k, v in params.items():
        assert k in sd and sd[k].shape == v.shape and sd[k].dtype == torch.float32, k
    model.load_state_dict({**params, "lm.lm_head.weight": params["lm.model.decoder.embed_tokens.weight"]}, strict=True)
    assert model.lm.lm_head.weight.data_ptr() == model.lm.model.decoder.embed_tokens.weight.data_ptr(), "embeddings not tied"
    model.eval()
    return model


def main():
    params = init_params(CFG, seed=SEED_PARAMS, std=STD, dtype=torch.float32)
    model = reference_model(params)
    blob = {"cfg": np.array([CFG.vocab_size, CFG.hidden, CFG.n_layers, CFG.n_heads, CFG.ffn, CFG.max_positions,
                             SEED_PARAMS], dtype=np.int64), "std": np.float32(STD)}
    g = torch.Generator().manual_seed(7)
    ids = torch.randint(2, 502, (2, 32), generator=g)
    ids[:, 0] = 1
    ids[1, 26:] = 0
    with torch.no_grad():
        z = model(input_ids=ids).logits
    assert z.dtype == torch.float32
    blob.update({"logits/ids": ids.numpy(), "logits/z": z.numpy()})

    g = torch.Generator().manual_seed(11)
    tokens = torch.randint(2, 502, (3, 40), generator=g)
    tokens[:, 0] = 1
    tokens[1, 25:] = 0
    tokens[2, 33:] = 0
    present = set(tokens.flatten().tolist())      # ignore_tokens are never targets (the other modality's ids)
    ignore = sorted(i for i in torch.randperm(500, generator=g).add(2).tolist() if i not in present)[:100]
    ll = {"sum": model.log_likelihood(tokens.clone(), mean_nll=False),
          "mean": model.log_likelihood(tokens.clone(), mean_nll=True),
          "sum_ign": model.log_likelihood(tokens.clone(), mean_nll=False, ignore_tokens=ignore),
          "mean_ign": model.log_likelihood(tokens.clone(), mean_nll=True, ignore_tokens=ignore)}
    for k, v in ll.items():
        assert v.dtype == torch.float32, k
        blob["loglik/" + k] = v.numpy()
    blob.update({"loglik/tokens": tokens.numpy(), "loglik/ignore": np.array(ignore, dtype=np.int64)})

    prompt = torch.tensor([[1, 17, 33, 5, 250, 9, 41, 77]])
    out = model.generate(prompt, max_new_tokens=16, do_sample=False, return_dict_in_generate=True, output_scores=True)
    seq = out.sequences
    top2 = torch.stack([torch.topk(s[0].float(), 2).values for s in out.scores])
    blob.update({"gen/prompt": prompt.numpy(), "gen/out": seq.numpy(), "gen/margin": (top2[:, 0] - top2[:, 1]).numpy()})
    print("logits", tuple(z.shape), "loglik", {k: v.tolist() for k, v in ll.items()})
    print("generate", seq.tolist(), "margins", blob["gen/margin"].tolist())
    dst = os.path.join(ROOT, "tests", "golden", "opt_fp32_tiny.npz")
    np.savez_compressed(dst, **blob)
    print("->", dst, os.path.getsize(dst), "bytes")


if __name__ == "__main__":
    assert os.path.isdir(REF), "the reference must be importable to produce the fixture"
    _stub_omegaconf()
    sys.path.insert(0, REF)
    main()
