"""CPU oracle for OPT trained with fp32 master weights under bf16 autocast: the reference's default recipe
(config/model/default.yaml `torch_dtype: null` loads OPTForCausalLM in fp32, config/training_args/default.yaml
`bf16: True` makes HF Trainer run forward and backward under torch.autocast(bfloat16)).

TEST INFRASTRUCTURE ONLY.  Nothing under slamkit_b200/ may import this module; only tests/ and tools/ use it, as the
checker.  Pinned by tests/golden/opt_amp_tiny.npz, which oracle/make_opt_amp_golden.py produced with the reference's
own `UnitLM`.

The restatement is oracle/opt_oracle.py's forward with fp32 leaves, run under CPU autocast, and autograd for the
backward.  What autocast does to each op of that forward (the numerics slamkit_b200's master-weight path implements):
  embed_tokens + embed_positions       fp32 tables, fp32 sum: the residual stream starts fp32
  layer_norm (both per layer, final)   fp32 input and parameters, fp32 output; the next linear rounds it once to bf16
  q/k/v/out_proj, fc1, fc2, lm_head    weight, bias and input cast to bf16, bf16 output
  attention, ReLU, q scaling           bf16
  residual + branch                    fp32 + bf16 -> fp32, the residual is never rounded
  loss                                 compute_loss upcasts the bf16 logits
Backward: autocast's casts make every linear's dW / db a bf16 tensor that is widened into the fp32 .grad; LayerNorm and
embedding gradients and the residual gradient are fp32.  clip_grad_norm_ and AdamW then run on fp32 tensors with fp32
moments (oracle/lm_oracle.py's restatements are dtype-generic).
"""
from __future__ import annotations

from typing import Dict, List, Optional

import torch

from oracle.lm_oracle import adamw_step_, clip_grad_norm_, compute_loss
from oracle.opt_oracle import OracleOptConfig, forward_logits, init_params


def sample_index(n: int, target: int = 1024) -> torch.Tensor:
    """Evenly spaced element indices (about `target`, always including 0) of a flattened tensor of n elements: the
    elements tests/golden/opt_amp_tiny.npz stores values of."""
    return torch.arange(0, n, max(1, n // target))


def init_params_fp32(cfg: OracleOptConfig, seed: int = 0, std: float = 0.02) -> Dict[str, torch.Tensor]:
    """opt_oracle.init_params drawn in fp32 (the same normal draws, not rounded to bf16)."""
    return init_params(cfg, seed=seed, std=std, dtype=torch.float32)


def forward_backward_amp(p: Dict[str, torch.Tensor], cfg: OracleOptConfig, input_ids, labels,
                         num_items_in_batch: Optional[float] = None, position_ids=None, attention_mask=None,
                         packed: bool = False):
    """Loss, bf16 logits and fp32 parameter gradients of one micro-batch: fp32 leaves, forward under
    torch.autocast("cpu", bfloat16), autograd backward outside it (Trainer.training_step with bf16=True)."""
    leaves = {k: v.detach().float().clone().requires_grad_(True) for k, v in p.items()}
    with torch.autocast("cpu", dtype=torch.bfloat16):
        logits = forward_logits(leaves, cfg, input_ids, position_ids, attention_mask=attention_mask, packed=packed)
        loss = compute_loss(logits, labels, num_items_in_batch)
    loss.backward()
    return loss.detach(), logits.detach(), {k: v.grad for k, v in leaves.items()}


class OracleOptAmpTrainer:
    """HF-Trainer-equivalent optimiser steps on fp32 master weights: gradients accumulated in fp32 over micro-batches,
    clip_grad_norm_ over the fp32 gradients, AdamW with fp32 moments."""

    def __init__(self, params: Dict[str, torch.Tensor], cfg: OracleOptConfig, lr=1e-3, betas=(0.9, 0.999), eps=1e-8,
                 weight_decay=0.0, max_grad_norm=0.5):
        self.p = {k: v.detach().float().clone() for k, v in params.items()}
        self.cfg = cfg
        self.lr, self.betas, self.eps, self.wd, self.max_grad_norm = lr, betas, eps, weight_decay, max_grad_norm
        self.m = {k: torch.zeros_like(v) for k, v in self.p.items()}
        self.v = {k: torch.zeros_like(v) for k, v in self.p.items()}
        self.step_count = 0
        self.last_total_norm = None

    def accumulate(self, micro_batches, num_items: float) -> Dict[str, torch.Tensor]:
        """fp32 .grad after the micro-batches (each: (input_ids, labels[, position_ids, packed]))."""
        acc: Dict[str, torch.Tensor] = {}
        self.losses: List[float] = []
        for mb in micro_batches:
            ids, labels = mb[0], mb[1]
            pos = mb[2] if len(mb) > 2 else None
            packed = bool(mb[3]) if len(mb) > 3 else False
            loss, _, g = forward_backward_amp(self.p, self.cfg, ids, labels, num_items, position_ids=pos, packed=packed)
            self.losses.append(float(loss))
            for k, v in g.items():
                acc[k] = v if k not in acc else acc[k] + v
        return acc

    def apply(self, grads: Dict[str, torch.Tensor], lr: Optional[float] = None) -> None:
        names = list(self.p.keys())
        if self.max_grad_norm and self.max_grad_norm > 0:
            self.last_total_norm = clip_grad_norm_([grads[k] for k in names], self.max_grad_norm)
        self.step_count += 1
        for k in names:
            adamw_step_(self.p[k], grads[k], self.m[k], self.v[k], lr=self.lr if lr is None else lr, beta1=self.betas[0],
                        beta2=self.betas[1], eps=self.eps, weight_decay=self.wd, step=self.step_count)

    def train_step(self, input_ids, labels, lr: Optional[float] = None) -> float:
        num_items = float((labels != -100).sum().item())
        self.apply(self.accumulate([(input_ids, labels)], num_items), lr)
        return self.losses[0]
