"""CPU oracle for the GPT-NeoX decoder on hot path (ii): forward, `compute_loss`, autograd backward and the HF-Trainer
optimiser step.

TEST INFRASTRUCTURE ONLY.  Nothing under slamkit_b200/ may import this module; only tests/, __graft_entry__.smoke()
and tools/neox_bench.py use it, as the checker.

A plain-PyTorch (CPU) restatement of the parallel-residual GPT-NeoX decoder as HF `GPTNeoXForCausalLM` runs it under
bf16 (transformers 5.5.0, `transformers/models/gpt_neox/modeling_gpt_neox.py`; "HF:" below): the Pythia bases of the
reference's config/train_inter_scale.yaml behind `slamkit.model.unit_lm.UnitLM`.  The restatement is pinned by
tests/golden/neox_tiny.npz, which oracle/make_neox_golden.py produced with the reference's own `UnitLM`.  The loss,
clipping and AdamW parts are the model-independent ones of oracle/lm_oracle.py.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, List, Optional

import numpy as np
import torch
import torch.nn.functional as F

from oracle.lm_oracle import adamw_step_, clip_grad_norm_, compute_loss, packed_mask  # noqa: F401  (re-exported)
from oracle.opt_oracle import golden_masked_logits, u16_delta  # noqa: F401  (the same fixture encodings)


@dataclass
class OracleNeoxConfig:
    vocab_size: int = 502
    hidden: int = 768
    n_layers: int = 12
    n_heads: int = 12
    ffn: int = 3072
    max_positions: int = 2048
    rot_dims: int = 16
    rope_theta: float = 10000.0
    ln_eps: float = 1e-5

    @property
    def head_dim(self) -> int:
        return self.hidden // self.n_heads


def init_params(cfg: OracleNeoxConfig, seed: int = 0, std: float = 0.02, dtype=torch.bfloat16) -> Dict[str, torch.Tensor]:
    """Seeded random parameters with the names of `UnitLM.state_dict()` over GPTNeoXForCausalLM (prefix `lm.`).  Biases
    and LayerNorm parameters are random too (HF initialises them to 0 / 1), so that every one of them is exercised."""
    g = torch.Generator().manual_seed(seed)

    def rn(*shape, s=std):
        return (torch.randn(shape, generator=g) * s).to(dtype)

    def ln_w(n):
        return (1.0 + 0.1 * torch.randn(n, generator=g)).to(dtype)

    d = cfg.hidden
    p: Dict[str, torch.Tensor] = {}
    p["lm.gpt_neox.embed_in.weight"] = rn(cfg.vocab_size, d)
    for l in range(cfg.n_layers):
        h = f"lm.gpt_neox.layers.{l}."
        p[h + "input_layernorm.weight"] = ln_w(d)
        p[h + "input_layernorm.bias"] = rn(d, s=0.1)
        p[h + "post_attention_layernorm.weight"] = ln_w(d)
        p[h + "post_attention_layernorm.bias"] = rn(d, s=0.1)
        p[h + "attention.query_key_value.weight"] = rn(3 * d, d)
        p[h + "attention.query_key_value.bias"] = rn(3 * d)
        p[h + "attention.dense.weight"] = rn(d, d)
        p[h + "attention.dense.bias"] = rn(d)
        p[h + "mlp.dense_h_to_4h.weight"] = rn(cfg.ffn, d)
        p[h + "mlp.dense_h_to_4h.bias"] = rn(cfg.ffn)
        p[h + "mlp.dense_4h_to_h.weight"] = rn(d, cfg.ffn)
        p[h + "mlp.dense_4h_to_h.bias"] = rn(d)
    p["lm.gpt_neox.final_layer_norm.weight"] = ln_w(d)
    p["lm.gpt_neox.final_layer_norm.bias"] = rn(d, s=0.1)
    p["lm.embed_out.weight"] = rn(cfg.vocab_size, d)
    return p


def rope_cos_sin(cfg: OracleNeoxConfig, pos: torch.Tensor, dtype=torch.bfloat16):
    """GPTNeoXRotaryEmbedding (HF:modeling_gpt_neox.py:53-116): inv_freq over the rotary_ndims columns, fp32 outer
    product, cat(freqs, freqs), cos / sin cast to the activation dtype.  [B, T, rot]."""
    rot = cfg.rot_dims
    inv_freq = 1.0 / (cfg.rope_theta ** (torch.arange(0, rot, 2, dtype=torch.int64).to(dtype=torch.float) / rot))
    freqs = pos[..., None].float() * inv_freq[None, None, :].float()
    emb = torch.cat((freqs, freqs), dim=-1)
    return emb.cos().to(dtype), emb.sin().to(dtype)


def rotate_half(x: torch.Tensor) -> torch.Tensor:
    h = x.shape[-1] // 2
    return torch.cat((-x[..., h:], x[..., :h]), dim=-1)


def forward_logits(p: Dict[str, torch.Tensor], cfg: OracleNeoxConfig, input_ids: torch.Tensor,
                   position_ids: Optional[torch.Tensor] = None, packed: bool = False) -> torch.Tensor:
    """GPTNeoXForCausalLM.forward without cache: embed_in -> L x [h1 = LN1(x), h2 = LN2(x); query_key_value (+bias)
    viewed as per-head [q | k | v]; RoPE on the first rot_dims columns of q and k (HF:modeling_gpt_neox.py:126-159);
    causal attention with scale head_dim^-0.5; dense (+bias); mlp = dense_4h_to_h(gelu(dense_h_to_4h(h2)));
    x = mlp + attn + x (HF:modeling_gpt_neox.py:280-282)] -> final LayerNorm -> embed_out.  Tensors carry the
    parameters' dtype (bf16).  packed=True: block-diagonal causal attention over the documents that position_ids == 0
    starts (the reference's varlen path)."""
    B, T = input_ids.shape
    pre = "lm.gpt_neox."
    pos = position_ids if position_ids is not None else torch.arange(T)[None].expand(B, T)
    d, H, hd, rot = cfg.hidden, cfg.n_heads, cfg.head_dim, cfg.rot_dims
    x = F.embedding(input_ids, p[pre + "embed_in.weight"])
    cos, sin = rope_cos_sin(cfg, pos, x.dtype)
    cos, sin = cos[:, None], sin[:, None]
    mask = packed_mask(pos) if packed else None
    for l in range(cfg.n_layers):
        h = f"{pre}layers.{l}."
        h1 = F.layer_norm(x, (d,), p[h + "input_layernorm.weight"], p[h + "input_layernorm.bias"], cfg.ln_eps)
        qkv = F.linear(h1, p[h + "attention.query_key_value.weight"], p[h + "attention.query_key_value.bias"])
        q, k, v = qkv.view(B, T, H, 3 * hd).transpose(1, 2).chunk(3, dim=-1)
        q = torch.cat([q[..., :rot] * cos + rotate_half(q[..., :rot]) * sin, q[..., rot:]], dim=-1)
        k = torch.cat([k[..., :rot] * cos + rotate_half(k[..., :rot]) * sin, k[..., rot:]], dim=-1)
        if mask is not None:
            a = F.scaled_dot_product_attention(q, k, v, attn_mask=mask, scale=hd ** -0.5)
        else:
            a = F.scaled_dot_product_attention(q, k, v, is_causal=True, scale=hd ** -0.5)
        a = a.transpose(1, 2).reshape(B, T, d)
        attn = F.linear(a, p[h + "attention.dense.weight"], p[h + "attention.dense.bias"])
        h2 = F.layer_norm(x, (d,), p[h + "post_attention_layernorm.weight"], p[h + "post_attention_layernorm.bias"],
                          cfg.ln_eps)
        m = F.gelu(F.linear(h2, p[h + "mlp.dense_h_to_4h.weight"], p[h + "mlp.dense_h_to_4h.bias"]))
        m = F.linear(m, p[h + "mlp.dense_4h_to_h.weight"], p[h + "mlp.dense_4h_to_h.bias"])
        x = m + attn + x
    x = F.layer_norm(x, (d,), p[pre + "final_layer_norm.weight"], p[pre + "final_layer_norm.bias"], cfg.ln_eps)
    return F.linear(x, p["lm.embed_out.weight"])


def forward_backward(p: Dict[str, torch.Tensor], cfg: OracleNeoxConfig, input_ids, labels,
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


class OracleNeoxTrainer:
    """One HF-Trainer-equivalent optimiser step on CPU: forward / backward with num_items_in_batch, clip_grad_norm_ over
    every parameter, AdamW (oracle/lm_oracle.py restatements)."""

    def __init__(self, params: Dict[str, torch.Tensor], cfg: OracleNeoxConfig, lr=1e-3, betas=(0.9, 0.999), eps=1e-8,
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


def flops_per_token(cfg: OracleNeoxConfig, T: int) -> float:
    """Model FLOPs of one trained token (forward + backward = 3 x forward): 2 x the matmul parameters (query_key_value,
    dense, dense_h_to_4h, dense_4h_to_h, embed_out) plus causal attention's 2 x 2 x T/2 x hidden per layer."""
    d, Fd, V = cfg.hidden, cfg.ffn, cfg.vocab_size
    per_layer = 2 * (4 * d * d + 2 * d * Fd) + 2 * 2 * (T / 2) * d
    return 3.0 * (cfg.n_layers * per_layer + 2 * d * V)


def golden_grads(z, p: Dict[str, torch.Tensor], cfg: OracleNeoxConfig) -> Dict[str, torch.Tensor]:
    """tests/golden/neox_tiny.npz's reference gradients: stored as the bf16 bit-pattern difference from this oracle's
    bf16 backward on the fixture's training batch (parameters `p` = init_params(cfg, seed of the fixture))."""
    ids, labels = torch.from_numpy(z["train/ids"]), torch.from_numpy(z["train/labels"])
    _, _, g = forward_backward(p, cfg, ids, labels, float(z["train/num_items"]))
    out = {}
    for k, v in g.items():
        base = v.contiguous().view(torch.int16).numpy().view(np.uint16).astype(np.int64)
        bits = (base + z["grad_d16/" + k].astype(np.int64).reshape(base.shape)) % 65536
        out[k] = torch.from_numpy(bits.astype(np.uint16)).view(torch.bfloat16)
    return out
