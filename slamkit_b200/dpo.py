"""DPO step on the GPU train path (SURVEY.md §8 f-2): mirror of `SLAMDPOTrainer` (slamkit/trainer/slam_dpo_trainer.py:4-64,
a `trl.DPOTrainer` whose `tokenize_row` prepends BOS to the prompt and appends EOS to both completions) with trl's default
sigmoid loss, beta 0.1 (config/training_args/dpo_training_args.yaml:5-6), frozen reference model.

    loss = -log sigmoid(beta * [(pi_c - pi_r) - (ref_c - ref_r)]),   pi_x = sum_{completion tokens} log p(token)

The loss is not a CE, but d loss / d logits is a per-sequence-weighted CE gradient, so the step is
reference forward -> policy forward (per-position NLL) -> per-sequence weights (tiny device ops) -> weighted backward
(`sk_lm_forward_rows` / `sk_lm_backward_weighted`), i.e. the same kernels as pre-training."""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence

import torch

from . import _lib as L
from .lm import B200AdamW, B200UnitLM


def tokenize_row(features: Dict[str, str], tokeniser, max_prompt_length: Optional[int], max_completion_length: Optional[int],
                 add_special_tokens: bool = False) -> Dict[str, List[int]]:
    """SLAMDPOTrainer.tokenize_row (slam_dpo_trainer.py:40-64): BOS + prompt (left-truncated), completion + EOS
    (right-truncated); unit strings tokenised WITHOUT the `<S> $0 <S>` template."""
    def raw(s: str) -> List[int]:
        return tokeniser.string_tokenise(s)["input_ids"][1:-1]
    prompt = [tokeniser.bos_token_id] + raw(features["prompt"])
    if add_special_tokens and tokeniser.eos_token_id is not None:
        prompt = prompt + [tokeniser.eos_token_id]
    chosen = raw(features["chosen"]) + [tokeniser.eos_token_id]
    rejected = raw(features["rejected"]) + [tokeniser.eos_token_id]
    if max_prompt_length is not None:
        prompt = prompt[-max_prompt_length:]
    if max_completion_length is not None:
        chosen, rejected = chosen[:max_completion_length], rejected[:max_completion_length]
    return {"prompt_input_ids": prompt, "chosen_input_ids": chosen, "rejected_input_ids": rejected}


def collate_pairs(rows: Sequence[Dict[str, List[int]]], pad_id: int = 0):
    """trl concatenated batch: first all prompt+chosen, then all prompt+rejected, right-padded; labels cover the
    completion tokens only (prompt and padding -> -100)."""
    seqs, labs = [], []
    for key in ("chosen_input_ids", "rejected_input_ids"):
        for r in rows:
            p, c = r["prompt_input_ids"], r[key]
            seqs.append(p + c)
            labs.append([-100] * len(p) + c)
    n = max(len(s) for s in seqs)
    ids = torch.full((len(seqs), n), pad_id, dtype=torch.int64)
    labels = torch.full((len(seqs), n), -100, dtype=torch.int64)
    for i, (s, l) in enumerate(zip(seqs, labs)):
        ids[i, :len(s)] = torch.tensor(s)
        labels[i, :len(l)] = torch.tensor(l)
    return ids, labels


class B200DPOTrainer:
    """One optimiser step = `gradient_accumulation_steps` micro-batches of concatenated [chosen ; rejected] rows.  Under
    torchrun every rank holds its own micro-batches; trl runs DDP, i.e. the MEAN over ranks of each rank's mean loss, so
    the per-sequence weights carry 1 / (pairs_per_micro_batch * grad_accum * world) and the flat gradient buffer is
    SUM-all-reduced (`trainer.GradSync`, overlapped with the backward pass) before the clip + AdamW step."""

    def __init__(self, policy: B200UnitLM, reference: B200UnitLM, beta: float = 0.1, lr: float = 5e-5,
                 max_grad_norm: float = 0.5, weight_decay: float = 0.0, grad_accum: int = 1, overlap_comm: bool = True):
        from .trainer import GradSync
        if getattr(policy, "master", False) or getattr(reference, "master", False):
            raise NotImplementedError("B200DPOTrainer does not take models with fp32 master weights")
        self.policy, self.reference, self.beta = policy, reference, beta
        self.opt = B200AdamW(policy, lr=lr, max_grad_norm=max_grad_norm, weight_decay=weight_decay)
        self.sync = GradSync(policy, overlap=overlap_comm)
        self.grad_accum = grad_accum

    @staticmethod
    def _seq_logps(model: B200UnitLM, ids: torch.Tensor, labels: torch.Tensor) -> torch.Tensor:
        B, T = ids.shape
        model._ensure(B, T)
        row_nll = torch.empty(B * T, device=model.device, dtype=torch.float32)
        L.check(model.lib.sk_lm_forward_rows(model._h, L.ptr(ids), L.ptr(labels), None, B, T, L.ptr(row_nll),
                                             L.ptr(model.stats), L.stream_ptr()))
        return -row_nll.view(B, T).sum(dim=1)

    def micro_step(self, ids: torch.Tensor, labels: torch.Tensor, accumulate: bool) -> Dict[str, torch.Tensor]:
        """Forward of reference + policy and the weighted backward of one concatenated [2N, T] batch of `collate_pairs`;
        gradients are written (accumulate=False) or added (True) to the policy's flat gradient buffer."""
        pol, ref = self.policy, self.reference
        ids, labels = ids.to(pol.device).contiguous(), labels.to(pol.device).contiguous()
        n = ids.shape[0] // 2
        B, T = ids.shape
        ref_lp = self._seq_logps(ref, ids, labels)
        pol_lp = self._seq_logps(pol, ids, labels)
        z = self.beta * ((pol_lp[:n] - pol_lp[n:]) - (ref_lp[:n] - ref_lp[n:]))
        loss = -torch.nn.functional.logsigmoid(z).mean()
        # d loss / d pi_c = -beta*sigmoid(-z)/n ; d loss / d pi_r = +beta*sigmoid(-z)/n ; pi = -sum nll, and the kernel
        # applies w * (softmax - onehot) = w * d nll / d logits  ->  w_c = +beta*sigmoid(-z)/n, w_r = -beta*sigmoid(-z)/n
        g = self.beta * torch.sigmoid(-z) / (n * self.grad_accum * self.sync.world)
        w_seq = torch.cat([g, -g])
        row_w = w_seq[:, None].expand(B, T).contiguous().view(-1).float()
        L.check(pol.lib.sk_lm_backward_weighted(pol._h, L.ptr(ids), L.ptr(labels), None, B, T, L.ptr(row_w), int(accumulate),
                                                L.ptr(pol.stats), L.stream_ptr()))
        return {"loss": loss, "rewards_chosen": self.beta * (pol_lp[:n] - ref_lp[:n]),
                "rewards_rejected": self.beta * (pol_lp[n:] - ref_lp[n:]), "logits_z": z}

    def step(self, ids, labels, lr: Optional[float] = None) -> Dict[str, torch.Tensor]:
        """One optimiser step.  ids / labels: one concatenated batch (grad_accum == 1) or lists of `grad_accum` batches.
        Returns device tensors of the LAST micro-batch plus `loss` = mean over the accumulation window (this rank)."""
        if torch.is_tensor(ids):
            ids, labels = [ids], [labels]
        assert len(ids) == self.grad_accum == len(labels), "one [2N, T] batch per accumulation step"
        out, loss = None, 0.0
        for i, (a, b) in enumerate(zip(ids, labels)):
            out = self.micro_step(a, b, accumulate=i > 0)
            loss = loss + out["loss"] / self.grad_accum
        self.sync.reduce()
        self.opt.step(lr=lr)
        out["loss"] = loss
        return out
