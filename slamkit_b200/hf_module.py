"""HF-Trainer-compatible face of the GPU train step (SURVEY.md §8 b-2): an `nn.Module` whose `forward(input_ids,
attention_mask, position_ids, labels, num_items_in_batch)` returns `CausalLMOutputWithPast(loss, logits)` under autograd,
as `slamkit.model.unit_lm.UnitLM.forward` does (slamkit/model/unit_lm.py:135-182), so that `SLAMTrainer` / HF `Trainer`,
the reference collators and callbacks can drive it unchanged:

    model = B200UnitLMModule(B200UnitLM(LMConfig(...)))
    loss = model(input_ids=ids, labels=labels, num_items_in_batch=n).loss
    loss.backward()                     # model.flat.grad is the flat bf16 gradient buffer
    torch.optim.AdamW(model.parameters()).step()

The module has ONE parameter, `flat`: the flat bf16 buffer the sm_90a kernels read (same storage as `core.params`), so
optimisers and `clip_grad_norm_` see every weight; `state_dict()` / `load_state_dict()` speak the reference's names
(`lm.model.layers.N...`).  Forward + backward run in one C-ABI call (`sk_lm_forward_backward`) inside the
`autograd.Function`'s forward -- the gradient of a scalar loss with respect to the flat buffer is known as soon as the
loss is -- and `backward` hands it to autograd scaled by the incoming gradient.  The fast path for training remains
`trainer.B200Trainer` (fused clip + AdamW, overlapped all-reduce); this class is the drop-in boundary."""
from __future__ import annotations

from typing import Dict, Optional

import torch

from .lm import B200UnitLM, check_right_padded


class _LMStep(torch.autograd.Function):
    @staticmethod
    def forward(ctx, flat, core, input_ids, labels, position_ids, num_items):
        out = core.forward_backward(input_ids, labels, position_ids, num_items_in_batch=num_items)
        ctx.core = core
        return out.stats[0].clone()

    @staticmethod
    def backward(ctx, grad_out):
        g = ctx.core.grads
        return g * grad_out.to(g.dtype), None, None, None, None, None


class B200UnitLMModule(torch.nn.Module):
    def __init__(self, core: B200UnitLM):
        super().__init__()
        if core.grads is None:
            raise ValueError("B200UnitLMModule needs a trainable B200UnitLM (trainable=True)")
        if getattr(core, "master", False):
            raise NotImplementedError("B200UnitLMModule does not take a model with fp32 master weights (train it with "
                                      "slamkit_b200.trainer.B200Trainer / cli/train.py)")
        self.core = core
        self.flat = torch.nn.Parameter(core.params, requires_grad=True)      # shares storage with the bound buffer
        self.config = core.config

    @property
    def device(self) -> torch.device:
        return self.core.device

    def forward(self, input_ids: torch.Tensor = None, attention_mask: Optional[torch.Tensor] = None,
                position_ids: Optional[torch.Tensor] = None, labels: Optional[torch.Tensor] = None,
                num_items_in_batch=None, **unused):
        from transformers.modeling_outputs import CausalLMOutputWithPast
        check_right_padded(attention_mask)
        ni = None if num_items_in_batch is None else float(num_items_in_batch)
        if labels is not None and torch.is_grad_enabled() and self.flat.requires_grad:
            loss = _LMStep.apply(self.flat, self.core, input_ids, labels, position_ids, ni)
            return CausalLMOutputWithPast(loss=loss, logits=None)
        out = self.core.forward(input_ids, None, position_ids, labels, ni)
        loss = out.loss.clone() if out.loss is not None else None
        return CausalLMOutputWithPast(loss=loss, logits=out.logits)

    # ---- the reference's parameter names (UnitLM.state_dict(): prefix `lm.`) -----------------------------------------
    def state_dict(self, *args, **kwargs) -> Dict[str, torch.Tensor]:
        return self.core.state_dict_hf()

    def load_state_dict(self, state_dict: Dict[str, torch.Tensor], strict: bool = True, **kwargs):
        self.core.load_hf_state_dict(state_dict)
        return torch.nn.modules.module._IncompatibleKeys([], [])

    def save_pretrained(self, save_directory: str, **kwargs) -> None:
        self.core.save_pretrained(save_directory, **{k: v for k, v in kwargs.items() if k == "base_model_name"})

    @torch.inference_mode()
    def log_likelihood(self, tokens: torch.Tensor, mean_nll: bool, ignore_tokens=None) -> torch.Tensor:
        return self.core.log_likelihood(tokens, mean_nll, ignore_tokens)

    def generate(self, *a, **k):
        return self.core.generate(*a, **k)
