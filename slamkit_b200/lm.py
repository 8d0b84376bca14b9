"""B200UnitLM -- host-side mirror of the reference's TokenLM plugin for hot path (ii).

Mirrors `slamkit.model.unit_lm.UnitLM` (slamkit/model/unit_lm.py:82-212) and the `TokenLM` ABC
(slamkit/model/token_lm.py:7-27): same `forward(input_ids, attention_mask, position_ids, labels,
num_items_in_batch)` contract, `log_likelihood`, HF-compatible state-dict names (`lm.model.layers.N...`), but the
compute is the hand-written sm_90a train step behind the C ABI (`sk_lm_*` in include/slamkit_b200.h).  PyTorch only
owns the flat bf16 parameter / gradient / workspace buffers.
"""
from __future__ import annotations

import ctypes as C
import math
from dataclasses import dataclass
from typing import Dict, Iterator, List, Optional, Tuple

import torch

from . import _lib as L


@dataclass
class LMConfig:
    """Shape of the decoder (defaults = Qwen2.5-0.5B body with the 502-entry unit vocab, config/model/slam.yaml)."""
    vocab_size: int = 502
    hidden: int = 896
    n_layers: int = 24
    n_heads: int = 14
    n_kv_heads: int = 2
    head_dim: int = 64
    ffn: int = 4864
    max_positions: int = 2048
    rms_eps: float = 1e-6
    rope_theta: float = 10000.0          # config/model/slam.yaml:8 (see SURVEY.md §3.2 RoPE-theta hazard)
    tie_embeddings: bool = True
    qkv_bias: bool = True
    pad_token_id: int = 0

    @staticmethod
    def from_hf(cfg, vocab_size: Optional[int] = None, max_positions: int = 2048) -> "LMConfig":
        """From an HF config of the base model.  Only the Qwen2 decoder architecture (RMSNorm, rotary GQA attention with
        q/k/v bias, SwiGLU, no o/MLP bias) has sm_90a kernels behind it: anything else (e.g. the OPT-125M of
        config/model/twist.yaml) is refused instead of being silently trained as a different model."""
        mt = getattr(cfg, "model_type", None)
        if mt != "qwen2":
            raise ValueError(f"unsupported base architecture '{mt}': the GPU train path implements the Qwen2 decoder "
                             "(use model=slam, config/model/slam.yaml)")
        if getattr(cfg, "head_dim", None) not in (None, 64) or cfg.hidden_size // cfg.num_attention_heads != 64:
            raise ValueError("unsupported attention geometry: the sm_90a attention kernels need head_dim 64")
        rp = getattr(cfg, "rope_parameters", None) or {}
        theta = rp.get("rope_theta", getattr(cfg, "rope_theta", 10000.0))
        return LMConfig(
            vocab_size=vocab_size or cfg.vocab_size, hidden=cfg.hidden_size, n_layers=cfg.num_hidden_layers,
            n_heads=cfg.num_attention_heads, n_kv_heads=cfg.num_key_value_heads,
            head_dim=getattr(cfg, "head_dim", None) or cfg.hidden_size // cfg.num_attention_heads,
            ffn=cfg.intermediate_size, max_positions=max_positions, rms_eps=cfg.rms_norm_eps, rope_theta=float(theta),
            tie_embeddings=bool(cfg.tie_word_embeddings), qkv_bias=bool(getattr(cfg, "attention_bias", True)),
            pad_token_id=cfg.pad_token_id or 0)


def rope_tables(theta: float, head_dim: int, max_positions: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """cos/sin tables exactly as HF computes them (HF:models/qwen2/modeling_qwen2.py Qwen2RotaryEmbedding.forward):
    fp32 inv_freq, fp32 outer product, cos()/sin(), then cast to the activation dtype (bf16). Shape [P, head_dim/2]."""
    inv_freq = 1.0 / (theta ** (torch.arange(0, head_dim, 2, dtype=torch.int64).to(dtype=torch.float) / head_dim))
    pos = torch.arange(max_positions, dtype=torch.float32)
    freqs = (inv_freq[:, None].float() @ pos[None, :].float()).transpose(0, 1)  # [P, hd/2]
    return freqs.cos().to(torch.bfloat16).contiguous(), freqs.sin().to(torch.bfloat16).contiguous()


@dataclass
class LMOutput:
    loss: Optional[torch.Tensor]
    logits: Optional[torch.Tensor]
    stats: Optional[torch.Tensor] = None   # device fp32[3]: loss, n_valid_targets, nll_sum


def write_unit_lm_checkpoint(save_directory: str, state_dict_hf: Dict[str, torch.Tensor], config: "LMConfig",
                             base_model_name: str = "Qwen/Qwen2.5-0.5B") -> None:
    """Writes `model.safetensors` with the `lm.`-prefixed names of `UnitLM.state_dict()` (base_model_prefix = "lm",
    slamkit/model/unit_lm.py:87) and a `config.json` in the `UnitLMConfig` layout (unit_lm.py:32-79), so that the
    reference's `UnitLM.from_pretrained(dir)` / cli/eval.py consume a model trained with this package.  Pure host code (no CUDA):
    tests/test_host_cpu.py loads such a directory with the reference's own class."""
    import json
    import os
    from safetensors.torch import save_file
    os.makedirs(save_directory, exist_ok=True)
    c = config
    sd = {k: v.detach().contiguous().cpu() for k, v in state_dict_hf.items()
          if k != "lm.lm_head.weight" or not c.tie_embeddings}
    save_file(sd, os.path.join(save_directory, "model.safetensors"), metadata={"format": "pt"})
    base = {"model_type": "qwen2", "architectures": ["Qwen2ForCausalLM"], "hidden_size": c.hidden,
            "intermediate_size": c.ffn, "num_hidden_layers": c.n_layers, "num_attention_heads": c.n_heads,
            "num_key_value_heads": c.n_kv_heads, "vocab_size": c.vocab_size, "rms_norm_eps": c.rms_eps,
            "max_position_embeddings": c.max_positions, "tie_word_embeddings": c.tie_embeddings, "hidden_act": "silu",
            "rope_parameters": {"rope_theta": c.rope_theta, "rope_type": "default"}, "rope_theta": c.rope_theta,
            "pad_token_id": c.pad_token_id, "bos_token_id": 1, "eos_token_id": 1, "torch_dtype": "bfloat16"}
    cfg = {"model_type": "speech_language_model", "architectures": ["UnitLM"], "base_model_name": base_model_name,
           "base_config": base, "vocab_size": c.vocab_size, "twist_init": False, "use_cache": False,
           "tie_word_embeddings": c.tie_embeddings, "torch_dtype": "bfloat16",
           "max_position_embeddings": c.max_positions}
    with open(os.path.join(save_directory, "config.json"), "w") as f:
        json.dump(cfg, f, indent=2)


def check_right_padded(attention_mask: Optional[torch.Tensor]) -> None:
    """The kernels apply the causal mask only (plus document boundaries from position_ids).  That is exact for the
    reference's batches -- right-padded by DataCollatorForLanguageModeling / `padding_side = "right"`
    (slamkit/data/hf_dataset.py:61-64, unit_tokeniser.py:45) -- because a non-pad query never looks at a later pad key.
    Any other mask (left padding, holes) would silently change the result, so it is refused."""
    if attention_mask is None:
        return
    m = attention_mask
    if m.dim() != 2:
        raise ValueError("attention_mask must be [batch, seq] (explicit 4-D masks are not supported on the GPU path)")
    ok = bool(((m[:, 1:] != 0) <= (m[:, :-1] != 0)).all()) if m.shape[1] > 1 else True
    if not ok:
        raise ValueError("attention_mask is not right-padding (ones then zeros per row): the GPU attention kernels "
                         "implement causal masking only")


class B200UnitLM:
    """Causal unit LM whose forward/backward/optimiser run in libslamkit_b200.so."""

    def __init__(self, config: LMConfig, device: str = "cuda:0", max_batch: int = 8, max_seq: int = 1024,
                 trainable: bool = True, seed: Optional[int] = None):
        self.lib = L.require_cuda()
        self.config = config
        self.device = torch.device(device)
        torch.cuda.set_device(self.device)
        c = L.SkLmConfig(config.vocab_size, config.hidden, config.n_layers, config.n_heads, config.n_kv_heads,
                         config.head_dim, config.ffn, config.max_positions, config.rms_eps,
                         int(config.tie_embeddings), int(config.qkv_bias))
        self._h = C.c_void_p()
        L.check(self.lib.sk_lm_create(C.byref(c), C.byref(self._h)))
        self.n_params = int(self.lib.sk_lm_param_count(self._h))
        self.tensors: Dict[str, Tuple[int, int, int]] = {}
        n = self.lib.sk_lm_tensor_info(self._h, -1, None, 0, None, None, None)
        buf = C.create_string_buffer(64)
        for i in range(n):
            off, r, cc = C.c_int64(), C.c_int32(), C.c_int32()
            L.check(self.lib.sk_lm_tensor_info(self._h, i, buf, 64, C.byref(off), C.byref(r), C.byref(cc)))
            self.tensors[buf.value.decode()] = (off.value, r.value, cc.value)
        self.vocab_padded = self.tensors["embed"][1]
        self.params = torch.zeros(self.n_params, device=self.device, dtype=torch.bfloat16)
        self.grads = torch.zeros(self.n_params, device=self.device, dtype=torch.bfloat16) if trainable else None
        cos, sin = rope_tables(config.rope_theta, config.head_dim, config.max_positions)
        self.rope_cos, self.rope_sin = cos.to(self.device), sin.to(self.device)
        self.max_batch, self.max_seq = max_batch, max_seq
        self.workspace = None
        self._bind(max_batch, max_seq)
        self.stats = torch.zeros(3, device=self.device, dtype=torch.float32)
        if seed is not None:
            self.init_weights(seed)

    # ---- memory ------------------------------------------------------------------------------------------------
    def _bind(self, B: int, T: int) -> None:
        need = int(self.lib.sk_lm_workspace_bytes(self._h, B, T))
        if self.workspace is None or self.workspace.numel() < need:
            self.workspace = torch.empty(need, device=self.device, dtype=torch.uint8)
        L.check(self.lib.sk_lm_bind(self._h, L.ptr(self.params), L.ptr(self.grads), L.ptr(self.rope_cos),
                                    L.ptr(self.rope_sin), L.ptr(self.workspace), C.c_int64(self.workspace.numel())))

    def _ensure(self, B: int, T: int) -> None:
        need = int(self.lib.sk_lm_workspace_bytes(self._h, B, T))
        if need > self.workspace.numel():
            self._bind(B, T)

    def tensor(self, name: str, grad: bool = False) -> torch.Tensor:
        off, r, c = self.tensors[name]
        flat = self.grads if grad else self.params
        return flat[off:off + r * c].view(r, c)

    def __del__(self):
        try:
            if getattr(self, "_h", None):
                self.lib.sk_lm_destroy(self._h)
                self._h = None
        except Exception:
            pass

    # ---- weights -----------------------------------------------------------------------------------------------
    def init_weights(self, seed: int = 0, std: float = 0.02) -> None:
        """HF `_init_weights` equivalent: normal(0, std) for linear/embedding weights, zeros for biases, ones for
        norms (HF:modeling_utils.py PreTrainedModel._init_weights)."""
        g = torch.Generator(device="cpu").manual_seed(seed)
        V = self.config.vocab_size
        for name, (off, r, c) in self.tensors.items():
            t = self.params[off:off + r * c].view(r, c)
            base = name.split(".")[-1]
            if base in ("ln1", "ln2", "final_norm"):
                t.fill_(1.0)
            elif base == "bqkv":
                t.zero_()
            elif base in ("embed", "lm_head"):
                t.zero_()
                t[:V].copy_((torch.randn((V, c), generator=g) * std).to(torch.bfloat16))
            else:
                t.copy_((torch.randn((r, c), generator=g) * std).to(torch.bfloat16))

    def _hf_map(self) -> Iterator[Tuple[str, str, List[Tuple[int, int, int]]]]:
        """(flat tensor name, HF parameter name, [(row in the flat tensor, row in the HF tensor, n rows), ...]).

        q/k/v are row ranges of the fused `wqkv` / `bqkv`.  gate_proj and up_proj share `wgu` in 128-row blocks --
        flat rows [256b, 256b+128) = gate rows [128b, 128b+128), flat rows [256b+128, 256b+256) = the same up rows -- so
        that one 256-column GEMM tile holds gate AND up of the same hidden units and SwiGLU runs in the GEMM epilogue."""
        cfg = self.config
        q, kv = cfg.n_heads * cfg.head_dim, cfg.n_kv_heads * cfg.head_dim
        nb = cfg.ffn // 128
        for l in range(cfg.n_layers):
            p, h = f"layers.{l}.", f"lm.model.layers.{l}."
            yield p + "ln1", h + "input_layernorm.weight", [(0, 0, 1)]
            yield p + "wqkv", h + "self_attn.q_proj.weight", [(0, 0, q)]
            yield p + "wqkv", h + "self_attn.k_proj.weight", [(q, 0, kv)]
            yield p + "wqkv", h + "self_attn.v_proj.weight", [(q + kv, 0, kv)]
            if cfg.qkv_bias:
                yield p + "bqkv", h + "self_attn.q_proj.bias", [(0, 0, q)]
                yield p + "bqkv", h + "self_attn.k_proj.bias", [(q, 0, kv)]
                yield p + "bqkv", h + "self_attn.v_proj.bias", [(q + kv, 0, kv)]
            yield p + "wo", h + "self_attn.o_proj.weight", [(0, 0, cfg.hidden)]
            yield p + "ln2", h + "post_attention_layernorm.weight", [(0, 0, 1)]
            yield p + "wgu", h + "mlp.gate_proj.weight", [(256 * b, 128 * b, 128) for b in range(nb)]
            yield p + "wgu", h + "mlp.up_proj.weight", [(256 * b + 128, 128 * b, 128) for b in range(nb)]
            yield p + "wd", h + "mlp.down_proj.weight", [(0, 0, cfg.hidden)]
        yield "final_norm", "lm.model.norm.weight", [(0, 0, 1)]
        yield "embed", "lm.model.embed_tokens.weight", [(0, 0, cfg.vocab_size)]
        if not cfg.tie_embeddings:
            yield "lm_head", "lm.lm_head.weight", [(0, 0, cfg.vocab_size)]

    def _flat_rows(self, flat: str, grad: bool) -> torch.Tensor:
        """The flat tensor as a [rows, cols] matrix; 1-row tensors (norm weights, the fused bias) as a column so that
        the segment rows of `_hf_map` index elements."""
        t = self.tensor(flat, grad=grad)
        return t.view(-1, 1) if t.shape[0] == 1 else t

    def load_hf_state_dict(self, sd: Dict[str, torch.Tensor], grads: bool = False) -> None:
        """Load parameters named as in `UnitLM.state_dict()` (prefix `lm.`, slamkit/model/unit_lm.py:87)."""
        for flat, hf, segs in self._hf_map():
            src = sd[hf].to(torch.bfloat16)
            dst = self._flat_rows(flat, grads)
            if src.dim() == 1:
                src = src.view(-1, 1)
            if segs == [(0, 0, 1)]:                       # whole norm weight
                dst.view(-1).copy_(src.view(-1))
                continue
            for f0, h0, n in segs:
                dst[f0:f0 + n].copy_(src[h0:h0 + n])

    def state_dict_hf(self, grads: bool = False) -> Dict[str, torch.Tensor]:
        out = {}
        for flat, hf, segs in self._hf_map():
            t = self._flat_rows(flat, grads)
            if segs == [(0, 0, 1)]:
                out[hf] = t.view(-1).clone()
                continue
            parts = [t[f0:f0 + n] for f0, h0, n in segs]    # segments are listed in HF row order
            v = torch.cat(parts, dim=0) if len(parts) > 1 else parts[0].clone()
            out[hf] = v.view(-1) if flat.endswith("bqkv") else v
        if self.config.tie_embeddings:
            out["lm.lm_head.weight"] = out["lm.model.embed_tokens.weight"]
        return out

    # ---- checkpoints (HF layout, SURVEY.md §5 / §8 f-4) ------------------------------------------------------------
    def save_pretrained(self, save_directory: str, base_model_name: str = "Qwen/Qwen2.5-0.5B") -> None:
        write_unit_lm_checkpoint(save_directory, self.state_dict_hf(), self.config, base_model_name)

    @classmethod
    def from_pretrained(cls, directory: str, device: str = "cuda:0", max_batch: int = 8, max_seq: int = 1024,
                        trainable: bool = True) -> "B200UnitLM":
        import json
        import os
        from safetensors.torch import load_file
        cfg = json.load(open(os.path.join(directory, "config.json")))
        b = cfg["base_config"]
        theta = (b.get("rope_parameters") or {}).get("rope_theta", b.get("rope_theta", 10000.0))
        lm_cfg = LMConfig(vocab_size=cfg["vocab_size"], hidden=b["hidden_size"], n_layers=b["num_hidden_layers"],
                          n_heads=b["num_attention_heads"], n_kv_heads=b["num_key_value_heads"],
                          head_dim=b["hidden_size"] // b["num_attention_heads"], ffn=b["intermediate_size"],
                          max_positions=max(max_seq, 2048), rms_eps=b["rms_norm_eps"], rope_theta=float(theta),
                          tie_embeddings=bool(b.get("tie_word_embeddings", True)), pad_token_id=b.get("pad_token_id", 0))
        m = cls(lm_cfg, device=device, max_batch=max_batch, max_seq=max_seq, trainable=trainable)
        m.load_hf_state_dict(load_file(os.path.join(directory, "model.safetensors")))
        return m

    # ---- compute -----------------------------------------------------------------------------------------------

    def _prep(self, input_ids: torch.Tensor, position_ids: Optional[torch.Tensor]):
        assert input_ids.dim() == 2 and input_ids.dtype == torch.int64
        B, T = input_ids.shape
        self._ensure(B, T)
        ids = input_ids.to(self.device, non_blocking=True).contiguous()
        pos = None
        if position_ids is not None:
            pos = position_ids.to(self.device, non_blocking=True).to(torch.int32).contiguous().view(-1)
        return B, T, ids, pos

    def logits_view(self, B: int, T: int) -> torch.Tensor:
        """Zero-copy view of the bf16 logits of the last forward: [B, T, vocab_size]."""
        p = self.lib.sk_lm_logits(self._h)
        ld = self.lib.sk_lm_logits_ld(self._h)
        off = p - self.workspace.data_ptr()
        flat = self.workspace[off:off + B * T * ld * 2].view(torch.bfloat16).view(B, T, ld)
        return flat[:, :, :self.config.vocab_size]

    def forward(self, input_ids: torch.Tensor, attention_mask: Optional[torch.Tensor] = None,
                position_ids: Optional[torch.Tensor] = None, labels: Optional[torch.Tensor] = None,
                num_items_in_batch: Optional[float] = None, **_) -> LMOutput:
        """Forward only (eval / scoring). Padding is right-padding as produced by the reference collators
        (slamkit/data/hf_dataset.py:61-64), so the causal mask alone is exact for the non-pad positions."""
        check_right_padded(attention_mask)
        B, T, ids, pos = self._prep(input_ids, position_ids)
        lab = labels.to(self.device).contiguous() if labels is not None else None
        ni = float(num_items_in_batch) if num_items_in_batch is not None else 0.0
        L.check(self.lib.sk_lm_forward(self._h, L.ptr(ids), L.ptr(lab), L.ptr(pos), B, T, L.f32(ni), L.ptr(self.stats),
                                       L.stream_ptr()))
        return LMOutput(loss=self.stats[0] if labels is not None else None, logits=self.logits_view(B, T),
                        stats=self.stats)

    __call__ = forward

    def forward_backward(self, input_ids: torch.Tensor, labels: torch.Tensor, position_ids: Optional[torch.Tensor] = None,
                         num_items_in_batch: Optional[float] = None, loss_scale: float = 1.0,
                         accumulate: bool = False) -> LMOutput:
        """One micro-batch of training: loss (slamkit/model/unit_lm.py:13-29 semantics) and gradients into self.grads."""
        B, T, ids, pos = self._prep(input_ids, position_ids)
        lab = labels.to(self.device, non_blocking=True).contiguous()
        ni = float(num_items_in_batch) if num_items_in_batch is not None else 0.0
        L.check(self.lib.sk_lm_forward_backward(self._h, L.ptr(ids), L.ptr(lab), L.ptr(pos), B, T, L.f32(ni),
                                                L.f32(loss_scale), int(accumulate), L.ptr(self.stats), L.stream_ptr()))
        return LMOutput(loss=self.stats[0], logits=None, stats=self.stats)

    @torch.inference_mode()
    def log_likelihood(self, tokens: torch.Tensor, mean_nll: bool, ignore_tokens=None) -> torch.Tensor:
        """TokenLM.log_likelihood (slamkit/model/unit_lm.py:184-194): per-sample (mean or summed) log-likelihood."""
        out = self.forward(tokens)
        logits = out.logits.float()
        if ignore_tokens is not None:
            logits[:, :, ignore_tokens] = float("-inf")
        x = tokens.to(self.device)[..., 1:].clone()
        x[x == self.config.pad_token_id] = -100
        lp = torch.log_softmax(logits[..., :-1, :], dim=-1)
        mask = x.ne(-100)
        tok = lp.gather(-1, x.clamp(min=0).unsqueeze(-1)).squeeze(-1) * mask
        ll = tok.sum(-1)
        return ll / mask.sum(-1) if mean_nll else ll

    @torch.inference_mode()
    def generate(self, inputs: Optional[torch.Tensor] = None, generation_config=None, **kwargs) -> torch.Tensor:
        """TokenLM.generate (slamkit/model/token_lm.py:19-27; UnitLM.generate -> HF GenerationMixin, unit_lm.py:196-198):
        greedy or sampled continuation of left-padded prompts with HF's logits processing (generation.py).  No KV cache --
        decoding is not a hot path here -- so every new token re-runs the forward kernels on one sequence's prefix."""
        from .generation import generate_tokens
        if inputs is None:
            inputs = kwargs.pop("input_ids", None)
        if inputs is None:
            raise ValueError("generate: no prompt (inputs / input_ids)")
        keys = ("max_new_tokens", "max_length", "do_sample", "temperature", "top_k", "top_p", "eos_token_id", "pad_token_id",
                "bad_words_ids")
        opts = {}
        if generation_config is not None:
            for k in keys:
                v = getattr(generation_config, k, None)
                if v is not None:
                    opts[k] = v
            if "max_new_tokens" in opts:
                opts.pop("max_length", None)
        for k in keys:
            if kwargs.get(k) is not None:
                opts[k] = kwargs[k]
                if k == "max_new_tokens":
                    opts.pop("max_length", None)
        attention_mask = kwargs.get("attention_mask")
        ignored = {"attention_mask", "token_type_ids", "use_cache", "return_dict_in_generate", "output_scores", "synced_gpus"}
        unknown = sorted(k for k in kwargs if k not in keys and k not in ignored and kwargs[k] is not None)
        if unknown:
            raise NotImplementedError(f"generate: unsupported arguments {unknown} (greedy / sampling with temperature, top_k, "
                                      "top_p, bad_words_ids, eos / pad ids and length limits are implemented)")
        opts.setdefault("eos_token_id", getattr(self.config, "eos_token_id", 1))      # UnitTokeniser: bos = eos = 1
        opts.setdefault("pad_token_id", self.config.pad_token_id)
        if opts.get("do_sample") and "top_k" not in opts:
            opts["top_k"] = 50                                    # transformers' GenerationConfig default
        V = self.config.vocab_size

        def next_logits(ids: torch.Tensor) -> torch.Tensor:
            if ids.shape[1] > self.max_seq:
                raise L.SkError(f"generate: sequence of {ids.shape[1]} tokens exceeds the bound workspace (max_seq = {self.max_seq})")
            return self.forward(ids).logits[0, -1, :V].float().cpu()

        return generate_tokens(next_logits, inputs, attention_mask=attention_mask, max_positions=self.config.max_positions, **opts)


class B200AdamW:
    """Gradient clipping + AdamW exactly as HF Trainer applies them (HF:trainer.py clip_grad_norm_ -> optimizer.step):
    one `sk_lm_optimizer_step` call = grad-norm reduction + fused clip-scale/AdamW pass over the flat buffers."""

    def __init__(self, model: B200UnitLM, lr: float = 1e-3, betas=(0.9, 0.999), eps: float = 1e-8,
                 weight_decay: float = 0.0, max_grad_norm: float = 0.5, emulate_bf16_norm: bool = True):
        self.model = model
        self.lr, self.betas, self.eps, self.wd = lr, betas, eps, weight_decay
        self.max_grad_norm = max_grad_norm
        self.emulate = emulate_bf16_norm
        self.exp_avg = torch.zeros_like(model.params)
        self.exp_avg_sq = torch.zeros_like(model.params)
        self.step_count = 0
        self.stats = torch.zeros(3, device=model.device, dtype=torch.float32)  # total_norm, clip_coef, exact norm

    def step(self, lr: Optional[float] = None) -> None:
        self.step_count += 1
        m = self.model
        L.check(m.lib.sk_lm_optimizer_step(m._h, L.ptr(self.exp_avg), L.ptr(self.exp_avg_sq),
                                           L.f32(self.lr if lr is None else lr), L.f32(self.betas[0]),
                                           L.f32(self.betas[1]), L.f32(self.eps), L.f32(self.wd), self.step_count,
                                           L.f32(self.max_grad_norm or 0.0), int(self.emulate), L.ptr(self.stats),
                                           L.stream_ptr()))


def cosine_with_min_lr(step: int, *, base_lr: float, min_lr: float, warmup_steps: int, total_steps: int,
                       num_cycles: float = 0.5) -> float:
    """HF `get_cosine_with_min_lr_schedule_with_warmup` (HF:optimization.py:326-385) evaluated at `step`."""
    min_lr_rate = min_lr / base_lr
    if step < warmup_steps:
        return base_lr * float(step) / float(max(1, warmup_steps))
    progress = float(step - warmup_steps) / float(max(1, total_steps - warmup_steps))
    factor = 0.5 * (1.0 + math.cos(math.pi * float(num_cycles) * 2.0 * progress))
    factor = factor * (1 - min_lr_rate) + min_lr_rate
    return base_lr * max(0, factor)
