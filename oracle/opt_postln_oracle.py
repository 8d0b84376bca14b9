"""CPU oracle for the post-LayerNorm OPT decoder (facebook/opt-350m layout): forward, `compute_loss`, autograd backward and
the HF-Trainer optimiser step.

TEST INFRASTRUCTURE ONLY.  Nothing under slamkit_b200/ may import this module; only tests/ and tools/ use it, as the
checker.

A plain-PyTorch (CPU) restatement of HF `OPTForCausalLM` with `do_layer_norm_before=False` and, when `proj_dim` is
neither 0 nor `hidden`, the bias-free `project_in` / `project_out` pair (transformers 5.5.0,
`transformers/models/opt/modeling_opt.py`: OPTDecoderLayer, OPTDecoder).  The tensors carry the parameters' dtype: bf16
parameters give the bf16 path (every linear and every residual add rounded to bf16, LayerNorm in fp32 rounded once), fp32
parameters the fp32 path.  The restatement is pinned by tests/golden/opt_postln_tiny.npz, which
oracle/make_opt_postln_golden.py produced with the reference's own `UnitLM`.  The pre-LayerNorm decoder, the loss,
clipping and AdamW are those of oracle/opt_oracle.py and oracle/lm_oracle.py.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, List, Optional

import torch
import torch.nn.functional as F

from oracle.lm_oracle import adamw_step_, clip_grad_norm_, compute_loss, packed_mask  # noqa: F401  (re-exported)
from oracle.opt_oracle import OracleOptConfig, positions


@dataclass
class OraclePostLnConfig(OracleOptConfig):
    proj_dim: int = 0            # word_embed_proj_dim; 0 or hidden: no projections

    @property
    def has_proj(self) -> bool:
        return self.proj_dim not in (0, self.hidden)

    @property
    def embed_dim(self) -> int:
        return self.proj_dim if self.has_proj else self.hidden


def init_params(cfg: OraclePostLnConfig, seed: int = 0, std: float = 0.02, dtype=torch.bfloat16) -> Dict[str, torch.Tensor]:
    """Seeded random parameters with the names of `UnitLM.state_dict()` over a post-LN OPTForCausalLM (prefix `lm.`):
    no decoder `final_layer_norm`, and `project_in` / `project_out` when projecting.  Biases and LayerNorm parameters are
    random too, so that every one of them is exercised."""
    g = torch.Generator().manual_seed(seed)

    def rn(*shape, s=std):
        return (torch.randn(shape, generator=g) * s).to(dtype)

    d, e = cfg.hidden, cfg.embed_dim
    p: Dict[str, torch.Tensor] = {}
    p["lm.model.decoder.embed_tokens.weight"] = rn(cfg.vocab_size, e)
    p["lm.model.decoder.embed_positions.weight"] = rn(cfg.max_positions + 2, d)
    if cfg.has_proj:
        p["lm.model.decoder.project_out.weight"] = rn(e, d, s=d ** -0.5)
        p["lm.model.decoder.project_in.weight"] = rn(d, e, s=e ** -0.5)
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
    if not cfg.tie_embeddings:
        p["lm.lm_head.weight"] = rn(cfg.vocab_size, e)
    return p


def forward_logits(p: Dict[str, torch.Tensor], cfg: OraclePostLnConfig, input_ids: torch.Tensor,
                   position_ids: Optional[torch.Tensor] = None, attention_mask: Optional[torch.Tensor] = None,
                   packed: bool = False) -> torch.Tensor:
    """OPTForCausalLM.forward without cache, post-LN:
        e = embed_tokens[id];  x = project_in(e) + embed_positions(pos + 2)
        per layer: x = LN1(x + out_proj(attn(x)));  x = LN2(x + fc2(relu(fc1(x))))
        h = project_out(x);  logits = h @ embed_tokens^T
    packed=True: block-diagonal causal attention over the documents that position_ids == 0 starts."""
    B, T = input_ids.shape
    pre = "lm.model.decoder."
    pos = positions(input_ids, attention_mask, position_ids)
    x = F.embedding(input_ids, p[pre + "embed_tokens.weight"])
    if cfg.has_proj:
        x = F.linear(x, p[pre + "project_in.weight"])
    x = x + F.embedding(pos + 2, p[pre + "embed_positions.weight"])
    d, H, hd = cfg.hidden, cfg.n_heads, cfg.head_dim
    mask = packed_mask(pos) if packed else None
    for l in range(cfg.n_layers):
        h = f"{pre}layers.{l}."
        q = F.linear(x, p[h + "self_attn.q_proj.weight"], p[h + "self_attn.q_proj.bias"]) * hd ** -0.5
        k = F.linear(x, p[h + "self_attn.k_proj.weight"], p[h + "self_attn.k_proj.bias"])
        v = F.linear(x, p[h + "self_attn.v_proj.weight"], p[h + "self_attn.v_proj.bias"])
        q, k, v = (t.view(B, T, H, hd).transpose(1, 2) for t in (q, k, v))
        if mask is not None:
            a = F.scaled_dot_product_attention(q, k, v, attn_mask=mask, scale=1.0)
        else:
            a = F.scaled_dot_product_attention(q, k, v, is_causal=True, scale=1.0)
        a = a.transpose(1, 2).reshape(B, T, d)
        x = x + F.linear(a, p[h + "self_attn.out_proj.weight"], p[h + "self_attn.out_proj.bias"])
        x = F.layer_norm(x, (d,), p[h + "self_attn_layer_norm.weight"], p[h + "self_attn_layer_norm.bias"], cfg.ln_eps)
        y = F.relu(F.linear(x, p[h + "fc1.weight"], p[h + "fc1.bias"]))
        x = x + F.linear(y, p[h + "fc2.weight"], p[h + "fc2.bias"])
        x = F.layer_norm(x, (d,), p[h + "final_layer_norm.weight"], p[h + "final_layer_norm.bias"], cfg.ln_eps)
    if cfg.has_proj:
        x = F.linear(x, p[pre + "project_out.weight"])
    head = p[pre + "embed_tokens.weight"] if cfg.tie_embeddings else p["lm.lm_head.weight"]
    return F.linear(x, head)


def forward_backward(p: Dict[str, torch.Tensor], cfg: OraclePostLnConfig, input_ids, labels,
                     num_items_in_batch: Optional[float] = None, position_ids=None, packed: bool = False,
                     row_weight: Optional[torch.Tensor] = None):
    """Loss, logits and parameter gradients via autograd (one micro-batch).  row_weight [B]: the loss is instead
    sum_b row_weight[b] * (summed NLL of row b), the per-sequence weighting of the DPO path."""
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


class OraclePostLnTrainer:
    """One HF-Trainer-equivalent optimiser step on CPU: forward / backward with num_items_in_batch, clip_grad_norm_ over
    every parameter, AdamW."""

    def __init__(self, params: Dict[str, torch.Tensor], cfg: OraclePostLnConfig, lr=1e-3, betas=(0.9, 0.999), eps=1e-8,
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


def flops_per_token(cfg: OraclePostLnConfig, T: int) -> float:
    """Model FLOPs of one trained token (forward + backward = 3 x forward): 2 x the matmul parameters (q/k/v, out, fc1,
    fc2, project_in / project_out, lm_head) plus causal attention's 2 x 2 x T/2 x hidden per layer."""
    d, Fd, V, e = cfg.hidden, cfg.ffn, cfg.vocab_size, cfg.embed_dim
    per_layer = 2 * (4 * d * d + 2 * d * Fd) + 2 * 2 * (T / 2) * d
    proj = 2 * 2 * d * e if cfg.has_proj else 0
    return 3.0 * (cfg.n_layers * per_layer + proj + 2 * e * V)
