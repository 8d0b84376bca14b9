"""CPU oracle for the OPT decoder on hot path (ii): forward, `compute_loss`, autograd backward and the HF-Trainer
optimiser step.

TEST INFRASTRUCTURE ONLY.  Nothing under slamkit_b200/ may import this module; only tests/, __graft_entry__.smoke()
and tools/opt_bench.py use it, as the checker.

A plain-PyTorch (CPU) restatement of the pre-LayerNorm OPT decoder as HF `OPTForCausalLM` runs it under bf16
(transformers 5.5.0, `transformers/models/opt/modeling_opt.py`; "HF:" below): the reference's default `model: twist` /
`gslm` base (config/model/default.yaml: facebook/opt-125m) behind `slamkit.model.unit_lm.UnitLM`.  The restatement is
pinned by tests/golden/opt_tiny.npz, which oracle/make_opt_golden.py produced with the reference's own `UnitLM`.
The loss, clipping and AdamW parts are the model-independent ones of oracle/lm_oracle.py.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, List, Optional

import numpy as np
import torch
import torch.nn.functional as F

from oracle.lm_oracle import adamw_step_, clip_grad_norm_, compute_loss, packed_mask  # noqa: F401  (re-exported)


@dataclass
class OracleOptConfig:
    vocab_size: int = 502
    hidden: int = 768
    n_layers: int = 12
    n_heads: int = 12
    ffn: int = 3072
    max_positions: int = 2048
    ln_eps: float = 1e-5
    tie_embeddings: bool = True
    pad_token_id: int = 0

    @property
    def head_dim(self) -> int:
        return self.hidden // self.n_heads


def init_params(cfg: OracleOptConfig, seed: int = 0, std: float = 0.02, dtype=torch.bfloat16) -> Dict[str, torch.Tensor]:
    """Seeded random parameters with the names of `UnitLM.state_dict()` over OPTForCausalLM (prefix `lm.`).  Biases and
    LayerNorm parameters are random too (HF initialises them to 0 / 1), so that every one of them is exercised."""
    g = torch.Generator().manual_seed(seed)

    def rn(*shape, s=std):
        return (torch.randn(shape, generator=g) * s).to(dtype)

    d = cfg.hidden
    p: Dict[str, torch.Tensor] = {}
    p["lm.model.decoder.embed_tokens.weight"] = rn(cfg.vocab_size, d)
    p["lm.model.decoder.embed_positions.weight"] = rn(cfg.max_positions + 2, d)
    for l in range(cfg.n_layers):
        h = f"lm.model.decoder.layers.{l}."
        for n in ("k", "v", "q", "out"):
            p[h + f"self_attn.{n}_proj.weight"] = rn(d, d)
            p[h + f"self_attn.{n}_proj.bias"] = rn(d)
        p[h + "self_attn_layer_norm.weight"] = (1.0 + 0.1 * torch.randn(d, generator=g)).to(dtype)
        p[h + "self_attn_layer_norm.bias"] = rn(d, s=0.1)
        p[h + "fc1.weight"] = rn(cfg.ffn, d)
        p[h + "fc1.bias"] = rn(cfg.ffn)
        p[h + "fc2.weight"] = rn(d, cfg.ffn)
        p[h + "fc2.bias"] = rn(d)
        p[h + "final_layer_norm.weight"] = (1.0 + 0.1 * torch.randn(d, generator=g)).to(dtype)
        p[h + "final_layer_norm.bias"] = rn(d, s=0.1)
    p["lm.model.decoder.final_layer_norm.weight"] = (1.0 + 0.1 * torch.randn(d, generator=g)).to(dtype)
    p["lm.model.decoder.final_layer_norm.bias"] = rn(d, s=0.1)
    if not cfg.tie_embeddings:
        p["lm.lm_head.weight"] = rn(cfg.vocab_size, d)
    return p


def positions(input_ids: torch.Tensor, attention_mask: Optional[torch.Tensor] = None,
              position_ids: Optional[torch.Tensor] = None) -> torch.Tensor:
    """OPTDecoder.forward (HF:modeling_opt.py:500-515): the given position_ids, else cumsum(mask) * mask - 1 (pad
    positions -> -1, i.e. table row 1), with an all-ones mask when none is given."""
    if position_ids is not None:
        return position_ids
    if attention_mask is None:
        attention_mask = torch.ones_like(input_ids)
    return (torch.cumsum(attention_mask, dim=1) * attention_mask - 1).long()


def forward_logits(p: Dict[str, torch.Tensor], cfg: OracleOptConfig, input_ids: torch.Tensor,
                   position_ids: Optional[torch.Tensor] = None, attention_mask: Optional[torch.Tensor] = None,
                   packed: bool = False) -> torch.Tensor:
    """OPTForCausalLM.forward without cache: embed_tokens + embed_positions(pos + 2) (HF:modeling_opt.py:45-70) ->
    L x [LayerNorm, q/k/v (+bias), q * head_dim^-0.5, causal MHA, out_proj (+bias), residual, LayerNorm, fc1 (+bias), ReLU,
    fc2 (+bias), residual] (HF:modeling_opt.py:135-182, 202-260) -> final LayerNorm -> tied lm_head.  Tensors carry the
    parameters' dtype (bf16); nn.LayerNorm on bf16 computes in fp32 and rounds once, which is also what its autocast
    form (fp32 output, cast to bf16 by the next linear) gives.  packed=True: block-diagonal causal attention over the
    documents that position_ids == 0 starts (the reference's varlen path)."""
    B, T = input_ids.shape
    pre = "lm.model.decoder."
    pos = positions(input_ids, attention_mask, position_ids)
    x = F.embedding(input_ids, p[pre + "embed_tokens.weight"]) + F.embedding(pos + 2, p[pre + "embed_positions.weight"])
    d, H, hd = cfg.hidden, cfg.n_heads, cfg.head_dim
    mask = packed_mask(pos) if packed else None
    for l in range(cfg.n_layers):
        h = f"{pre}layers.{l}."
        res = x
        y = F.layer_norm(x, (d,), p[h + "self_attn_layer_norm.weight"], p[h + "self_attn_layer_norm.bias"], cfg.ln_eps)
        q = F.linear(y, p[h + "self_attn.q_proj.weight"], p[h + "self_attn.q_proj.bias"]) * hd ** -0.5
        k = F.linear(y, p[h + "self_attn.k_proj.weight"], p[h + "self_attn.k_proj.bias"])
        v = F.linear(y, p[h + "self_attn.v_proj.weight"], p[h + "self_attn.v_proj.bias"])
        q, k, v = (t.view(B, T, H, hd).transpose(1, 2) for t in (q, k, v))
        if mask is not None:
            a = F.scaled_dot_product_attention(q, k, v, attn_mask=mask, scale=1.0)
        else:
            a = F.scaled_dot_product_attention(q, k, v, is_causal=True, scale=1.0)
        a = a.transpose(1, 2).reshape(B, T, d)
        x = res + F.linear(a, p[h + "self_attn.out_proj.weight"], p[h + "self_attn.out_proj.bias"])
        res = x
        y = F.layer_norm(x, (d,), p[h + "final_layer_norm.weight"], p[h + "final_layer_norm.bias"], cfg.ln_eps)
        y = F.relu(F.linear(y, p[h + "fc1.weight"], p[h + "fc1.bias"]))
        x = res + F.linear(y, p[h + "fc2.weight"], p[h + "fc2.bias"])
    x = F.layer_norm(x, (d,), p[pre + "final_layer_norm.weight"], p[pre + "final_layer_norm.bias"], cfg.ln_eps)
    head = p[pre + "embed_tokens.weight"] if cfg.tie_embeddings else p["lm.lm_head.weight"]
    return F.linear(x, head)


def forward_backward(p: Dict[str, torch.Tensor], cfg: OracleOptConfig, input_ids, labels,
                     num_items_in_batch: Optional[float] = None, position_ids=None, packed: bool = False,
                     row_weight: Optional[torch.Tensor] = None):
    """Loss, logits and parameter gradients via autograd (Trainer.training_step for one micro-batch).  row_weight [B]:
    the loss is instead sum_b row_weight[b] * (summed NLL of row b) -- the per-sequence weighting of the DPO path."""
    leaves = {k: v.detach().clone().requires_grad_(True) for k, v in p.items()}
    logits = forward_logits(leaves, cfg, input_ids, position_ids, packed=packed)
    if row_weight is None:
        loss = compute_loss(logits, labels, num_items_in_batch)
    else:
        nll = F.cross_entropy(logits.float()[:, :-1].reshape(-1, logits.shape[-1]), labels[:, 1:].reshape(-1),
                              reduction="none", ignore_index=-100).view(labels.shape[0], -1)
        loss = (nll.sum(-1) * row_weight).sum()
    loss.backward()
    return loss.detach(), logits.detach(), {k: v.grad for k, v in leaves.items()}


class OracleOptTrainer:
    """One HF-Trainer-equivalent optimiser step on CPU: forward / backward with num_items_in_batch, clip_grad_norm_ over
    every parameter, AdamW (oracle/lm_oracle.py restatements)."""

    def __init__(self, params: Dict[str, torch.Tensor], cfg: OracleOptConfig, lr=1e-3, betas=(0.9, 0.999), eps=1e-8,
                 weight_decay=0.0, max_grad_norm=0.5):
        self.p = {k: v.clone() for k, v in params.items()}
        self.cfg = cfg
        self.lr, self.betas, self.eps, self.wd, self.max_grad_norm = lr, betas, eps, weight_decay, max_grad_norm
        self.m = {k: torch.zeros_like(v) for k, v in self.p.items()}
        self.v = {k: torch.zeros_like(v) for k, v in self.p.items()}
        self.step_count = 0
        self.last_total_norm = None

    def train_step(self, input_ids, labels, lr: Optional[float] = None, position_ids=None, packed: bool = False) -> float:
        num_items = float((labels != -100).sum().item())
        loss, _, grads = forward_backward(self.p, self.cfg, input_ids, labels, num_items, position_ids, packed)
        names: List[str] = list(self.p.keys())
        if self.max_grad_norm and self.max_grad_norm > 0:
            self.last_total_norm = clip_grad_norm_([grads[k] for k in names], self.max_grad_norm)
        self.step_count += 1
        for k in names:
            adamw_step_(self.p[k], grads[k], self.m[k], self.v[k], lr=self.lr if lr is None else lr, beta1=self.betas[0],
                        beta2=self.betas[1], eps=self.eps, weight_decay=self.wd, step=self.step_count)
        return float(loss)


def flops_per_token(cfg: OracleOptConfig, T: int) -> float:
    """Model FLOPs of one trained token (forward + backward = 3 x forward): 2 x the matmul parameters (q/k/v, out, fc1,
    fc2, lm_head) plus causal attention's 2 x 2 x T/2 x hidden per layer."""
    d, Fd, V = cfg.hidden, cfg.ffn, cfg.vocab_size
    per_layer = 2 * (4 * d * d + 2 * d * Fd) + 2 * 2 * (T / 2) * d
    return 3.0 * (cfg.n_layers * per_layer + 2 * d * V)



# ---- tests/golden/opt_tiny.npz stores the Trainer-path (masked, autocast) logits as the bit-pattern difference from the
# unmasked ones, which compresses to a fraction of the raw values and decodes exactly.
def u16_delta(new_u16: np.ndarray, base_u16: np.ndarray) -> np.ndarray:
    """(new - base) mod 2^16 of two uint16 bf16 bit patterns"""
    return ((new_u16.astype(np.int64) - base_u16.astype(np.int64)) % 65536).astype(np.uint16)


def golden_masked_logits(z) -> torch.Tensor:
    """the fixture's Trainer-path (attention_mask, autocast) logits"""
    bits = (z["nomask/logits_u16"].astype(np.int64) + z["train/logits_d16"].astype(np.int64)) % 65536
    return torch.from_numpy(bits.astype(np.uint16)).view(torch.bfloat16)
