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


@dataclass
class OptLMConfig:
    """Shape of a pre-LayerNorm OPT decoder (defaults = facebook/opt-125m with the 502-entry unit vocabulary, the base of
    config/model/twist.yaml and gslm.yaml).  `max_positions` is the checkpoint's `max_position_embeddings`: the learned
    position table has max_positions + 2 rows (HF OPTLearnedPositionalEmbedding, offset 2)."""
    vocab_size: int = 502
    hidden: int = 768
    n_layers: int = 12
    n_heads: int = 12
    ffn: int = 3072
    max_positions: int = 2048
    ln_eps: float = 1e-5
    tie_embeddings: bool = True
    pad_token_id: int = 0
    bos_token_id: int = 1
    eos_token_id: int = 1
    init_std: float = 0.02
    head_dim: int = 64

    @staticmethod
    def from_hf(cfg, vocab_size: Optional[int] = None) -> "OptLMConfig":
        """From an HF `OPTConfig`.  Only what the sm_90a kernels implement is accepted; every other variant is refused by
        name: post-LayerNorm OPT and the project_in / project_out pair (opt-350m), the legacy `_remove_final_layer_norm`,
        bias-free linears, non-affine LayerNorms, activations other than ReLU, head_dim other than 64, and any dropout or
        layerdrop (there are no dropout kernels: set them to 0.0 as config/model/default.yaml does)."""
        if getattr(cfg, "model_type", None) != "opt":
            raise ValueError(f"OptLMConfig.from_hf: model_type is '{getattr(cfg, 'model_type', None)}', not 'opt'")
        if not getattr(cfg, "do_layer_norm_before", True):
            raise ValueError("unsupported OPT variant: do_layer_norm_before=False (post-LayerNorm OPT, e.g. opt-350m)")
        if getattr(cfg, "word_embed_proj_dim", cfg.hidden_size) != cfg.hidden_size:
            raise ValueError(f"unsupported OPT variant: word_embed_proj_dim={cfg.word_embed_proj_dim} != hidden_size="
                             f"{cfg.hidden_size} (project_in / project_out, e.g. opt-350m)")
        OptLMConfig._check_common(cfg)
        return OptLMConfig(**OptLMConfig._fields_from_hf(cfg, vocab_size))

    @staticmethod
    def _check_common(cfg) -> None:
        """The refusals that pre- and post-LayerNorm OPT share, each naming its field."""
        if getattr(cfg, "_remove_final_layer_norm", False):
            raise ValueError("unsupported OPT variant: _remove_final_layer_norm=True")
        if not getattr(cfg, "enable_bias", True):
            raise ValueError("unsupported OPT variant: enable_bias=False")
        if not getattr(cfg, "layer_norm_elementwise_affine", True):
            raise ValueError("unsupported OPT variant: layer_norm_elementwise_affine=False")
        if getattr(cfg, "activation_function", "relu") != "relu":
            raise ValueError(f"unsupported OPT variant: activation_function='{cfg.activation_function}' (only relu)")
        if cfg.hidden_size % cfg.num_attention_heads or cfg.hidden_size // cfg.num_attention_heads != 64:
            raise ValueError(f"unsupported attention geometry: hidden_size / num_attention_heads = "
                             f"{cfg.hidden_size / cfg.num_attention_heads:g}; the sm_90a attention kernels need head_dim 64")
        for k in ("dropout", "attention_dropout", "layerdrop"):
            if float(getattr(cfg, k, 0.0) or 0.0) != 0.0:
                raise ValueError(f"unsupported OPT setting: {k}={getattr(cfg, k)} (there are no dropout kernels; set it to 0.0)")

    @staticmethod
    def _fields_from_hf(cfg, vocab_size: Optional[int]) -> dict:
        return dict(
            vocab_size=vocab_size or cfg.vocab_size, hidden=cfg.hidden_size, n_layers=cfg.num_hidden_layers,
            n_heads=cfg.num_attention_heads, ffn=cfg.ffn_dim, max_positions=cfg.max_position_embeddings,
            tie_embeddings=bool(getattr(cfg, "tie_word_embeddings", True)),
            pad_token_id=cfg.pad_token_id if cfg.pad_token_id is not None else 0,
            bos_token_id=cfg.bos_token_id if cfg.bos_token_id is not None else 1,
            eos_token_id=cfg.eos_token_id if cfg.eos_token_id is not None else 1,
            init_std=float(getattr(cfg, "init_std", 0.02)))


@dataclass
class OptPostLnLMConfig(OptLMConfig):
    """Shape of a post-LayerNorm OPT decoder (HF `do_layer_norm_before=False`; defaults = facebook/opt-350m with the
    502-entry unit vocabulary, TWIST-350M's base).  Each layer normalises after its residual add and there is no final
    LayerNorm.  `proj_dim` is `word_embed_proj_dim`: when it is neither 0 nor `hidden`, the token table and the tied head
    are `proj_dim` wide and the bias-free project_in / project_out map them to and from the residual stream.  It is an
    `OptLMConfig`, so every OPT path (learned positions, checkpoints, generate, scoring) takes it."""
    hidden: int = 1024
    n_layers: int = 24
    n_heads: int = 16
    ffn: int = 4096
    proj_dim: int = 512

    @property
    def has_proj(self) -> bool:
        return self.proj_dim not in (0, self.hidden)

    @staticmethod
    def from_hf(cfg, vocab_size: Optional[int] = None) -> "OptPostLnLMConfig":
        """From an HF `OPTConfig` with `do_layer_norm_before=False`, with or without `word_embed_proj_dim != hidden_size`.
        Every other variant that `OptLMConfig.from_hf` refuses is refused here too, by the same field names."""
        if getattr(cfg, "model_type", None) != "opt":
            raise ValueError(f"OptPostLnLMConfig.from_hf: model_type is '{getattr(cfg, 'model_type', None)}', not 'opt'")
        if getattr(cfg, "do_layer_norm_before", True):
            raise ValueError("OptPostLnLMConfig.from_hf: do_layer_norm_before=True is the pre-LayerNorm OPT (OptLMConfig)")
        OptLMConfig._check_common(cfg)
        pd = int(getattr(cfg, "word_embed_proj_dim", None) or cfg.hidden_size)
        if pd != cfg.hidden_size and (pd % 64 or pd > cfg.hidden_size):
            raise ValueError(f"unsupported OPT variant: word_embed_proj_dim={pd} (project_in / project_out need a multiple "
                             f"of 64 below hidden_size={cfg.hidden_size})")
        return OptPostLnLMConfig(**OptLMConfig._fields_from_hf(cfg, vocab_size), proj_dim=pd)


@dataclass
class NeoxLMConfig:
    """Shape of a GPT-NeoX decoder with the parallel residual (defaults = EleutherAI/pythia-160m with the 502-entry unit
    vocabulary; the base family of config/train_inter_scale.yaml).  `rot_dims` = head_dim * partial_rotary_factor
    columns of each q / k head are rotated; `max_positions` is the number of RoPE table rows."""
    vocab_size: int = 502
    hidden: int = 768
    n_layers: int = 12
    n_heads: int = 12
    ffn: int = 3072
    max_positions: int = 2048
    rot_dims: int = 16
    rope_theta: float = 10000.0
    ln_eps: float = 1e-5
    init_std: float = 0.02
    pad_token_id: int = 0
    bos_token_id: int = 0
    eos_token_id: int = 0
    head_dim: int = 64
    tie_embeddings: bool = False          # embed_out is always a separate matrix here (tied heads are refused)

    @staticmethod
    def from_hf(cfg, vocab_size: Optional[int] = None, max_positions: Optional[int] = None) -> "NeoxLMConfig":
        """From an HF `GPTNeoXConfig`.  Only what the sm_90a kernels implement is accepted; every other variant is refused
        by name: the sequential residual (use_parallel_residual=False), head_dim other than 64 (pythia-14m / -31m have 32,
        pythia-1b and up 128 or 256), a rotary width other than 16, 32 or 64 columns, rope types other than default,
        activations other than exact gelu, bias-free attention, tied input / output embeddings and any dropout."""
        if getattr(cfg, "model_type", None) != "gpt_neox":
            raise ValueError(f"NeoxLMConfig.from_hf: model_type is '{getattr(cfg, 'model_type', None)}', not 'gpt_neox'")
        if not getattr(cfg, "use_parallel_residual", True):
            raise ValueError("unsupported GPT-NeoX variant: use_parallel_residual=False (sequential residual)")
        hd = getattr(cfg, "head_dim", None) or cfg.hidden_size // cfg.num_attention_heads
        if cfg.hidden_size % cfg.num_attention_heads or hd != 64:
            raise ValueError(f"unsupported attention geometry: head_dim = hidden_size / num_attention_heads = "
                             f"{cfg.hidden_size / cfg.num_attention_heads:g}; the sm_90a attention kernels need head_dim 64")
        rp = dict(getattr(cfg, "rope_parameters", None) or {})
        rope_type = rp.get("rope_type", rp.get("type", "default"))
        if rope_type != "default":
            raise ValueError(f"unsupported GPT-NeoX setting: rope_type='{rope_type}' (only default RoPE)")
        factor = rp.get("partial_rotary_factor", getattr(cfg, "partial_rotary_factor", getattr(cfg, "rotary_pct", 1.0)))
        rot = int(hd * float(factor))
        if rot not in (16, 32, 64):
            raise ValueError(f"unsupported GPT-NeoX setting: partial_rotary_factor={factor} gives rotary_ndims={rot}; "
                             "the RoPE epilogue rotates 16, 32 or 64 columns per head")
        theta = rp.get("rope_theta", getattr(cfg, "rope_theta", getattr(cfg, "rotary_emb_base", 10000.0)))
        act = getattr(cfg, "hidden_act", "gelu")
        if act != "gelu":
            raise ValueError(f"unsupported GPT-NeoX setting: hidden_act='{act}' (only the exact erf gelu)")
        if not getattr(cfg, "attention_bias", True):
            raise ValueError("unsupported GPT-NeoX setting: attention_bias=False")
        if getattr(cfg, "tie_word_embeddings", False):
            raise ValueError("unsupported GPT-NeoX setting: tie_word_embeddings=True (embed_out must be untied)")
        for k in ("attention_dropout", "hidden_dropout"):
            if float(getattr(cfg, k, 0.0) or 0.0) != 0.0:
                raise ValueError(f"unsupported GPT-NeoX setting: {k}={getattr(cfg, k)} (there are no dropout kernels; "
                                 "set it to 0.0)")
        bos = getattr(cfg, "bos_token_id", None)
        eos = getattr(cfg, "eos_token_id", None)
        return NeoxLMConfig(
            vocab_size=vocab_size or cfg.vocab_size, hidden=cfg.hidden_size, n_layers=cfg.num_hidden_layers,
            n_heads=cfg.num_attention_heads, ffn=cfg.intermediate_size,
            max_positions=max_positions or cfg.max_position_embeddings, rot_dims=rot, rope_theta=float(theta),
            ln_eps=float(cfg.layer_norm_eps), init_std=float(getattr(cfg, "initializer_range", 0.02)),
            pad_token_id=getattr(cfg, "pad_token_id", None) or 0, bos_token_id=bos if bos is not None else 0,
            eos_token_id=eos if isinstance(eos, int) else 0)


def lm_config_from_hf(base, vocab_size: Optional[int] = None, max_positions: int = 2048):
    """The decoder config for an HF base config, by `model_type`: `LMConfig` for qwen2 (RoPE tables of `max_positions`
    rows), `OptLMConfig` for opt (`OptPostLnLMConfig` when `do_layer_norm_before` is False; both have their own learned
    position table and ignore `max_positions`), `NeoxLMConfig` for
    gpt_neox (RoPE tables of max(max_positions, max_position_embeddings) rows).  Anything else is refused."""
    mt = getattr(base, "model_type", None)
    if mt == "opt":
        if not getattr(base, "do_layer_norm_before", True):   # post-LayerNorm OPT (opt-350m)
            return OptPostLnLMConfig.from_hf(base, vocab_size=vocab_size)
        return OptLMConfig.from_hf(base, vocab_size=vocab_size)
    if mt == "qwen2":
        return LMConfig.from_hf(base, vocab_size=vocab_size, max_positions=max_positions)
    if mt == "gpt_neox":
        return NeoxLMConfig.from_hf(base, vocab_size=vocab_size,
                                    max_positions=max(max_positions, int(getattr(base, "max_position_embeddings", 0) or 0)))
    raise ValueError(f"unsupported base architecture '{mt}': the GPU path implements the Qwen2, OPT (pre- and "
                     "post-LayerNorm) and GPT-NeoX (parallel residual) decoders")


def neox_qkv_segments(n_heads: int, head_dim: int = 64) -> List[Tuple[int, int, int]]:
    """(row in the kernels' [Q; K; V] layout, row in HF's per-head [q | k | v] query_key_value, n rows) for every head's
    q, k and v block, in HF row order: the permutation applied to the fused weight and bias on load and undone on save."""
    d = n_heads * head_dim
    return [(j * d + h * head_dim, h * 3 * head_dim + j * head_dim, head_dim) for h in range(n_heads) for j in range(3)]


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


def _opt_base_config(c: "OptLMConfig", torch_dtype: str = "bfloat16") -> dict:
    """The HF `OPTConfig` fields of an OPT decoder of this shape: the opt-125m layout, or for `OptPostLnLMConfig` the
    opt-350m one (post-LayerNorm, `word_embed_proj_dim`)."""
    post = isinstance(c, OptPostLnLMConfig)
    return {"model_type": "opt", "architectures": ["OPTForCausalLM"], "hidden_size": c.hidden, "ffn_dim": c.ffn,
            "num_hidden_layers": c.n_layers, "num_attention_heads": c.n_heads, "vocab_size": c.vocab_size,
            "max_position_embeddings": c.max_positions, "do_layer_norm_before": not post,
            "word_embed_proj_dim": c.proj_dim if post and c.has_proj else c.hidden,
            "activation_function": "relu", "enable_bias": True, "layer_norm_elementwise_affine": True,
            "_remove_final_layer_norm": False, "dropout": 0.0, "attention_dropout": 0.0, "layerdrop": 0.0,
            "init_std": c.init_std, "tie_word_embeddings": c.tie_embeddings, "pad_token_id": c.pad_token_id,
            "bos_token_id": c.bos_token_id, "eos_token_id": c.eos_token_id, "torch_dtype": torch_dtype}


def _neox_base_config(c: "NeoxLMConfig") -> dict:
    """The HF `GPTNeoXConfig` fields of a parallel-residual GPT-NeoX decoder of this shape (Pythia layout)."""
    return {"model_type": "gpt_neox", "architectures": ["GPTNeoXForCausalLM"], "hidden_size": c.hidden,
            "intermediate_size": c.ffn, "num_hidden_layers": c.n_layers, "num_attention_heads": c.n_heads,
            "vocab_size": c.vocab_size, "max_position_embeddings": c.max_positions, "layer_norm_eps": c.ln_eps,
            "use_parallel_residual": True, "hidden_act": "gelu", "attention_bias": True, "attention_dropout": 0.0,
            "hidden_dropout": 0.0, "initializer_range": c.init_std, "tie_word_embeddings": False,
            "rope_parameters": {"rope_theta": c.rope_theta, "partial_rotary_factor": c.rot_dims / c.head_dim,
                                "rope_type": "default"},
            "pad_token_id": c.pad_token_id, "bos_token_id": c.bos_token_id, "eos_token_id": c.eos_token_id,
            "torch_dtype": "bfloat16"}


def write_unit_lm_checkpoint(save_directory: str, state_dict_hf: Dict[str, torch.Tensor], config,
                             base_model_name: Optional[str] = None, torch_dtype: str = "bfloat16") -> None:
    """Writes `model.safetensors` with the `lm.`-prefixed names of `UnitLM.state_dict()` (base_model_prefix = "lm",
    slamkit/model/unit_lm.py:87) and a `config.json` in the `UnitLMConfig` layout (unit_lm.py:32-79), so that the
    reference's `UnitLM.from_pretrained(dir)` / cli/eval.py consume a model trained with this package.  Pure host code (no CUDA):
    tests/test_host_cpu.py loads such a directory with the reference's own class.  `torch_dtype` names the tensors' dtype
    ("float32" for an OPT model trained with fp32 master weights, as the reference's own run saves it)."""
    import json
    import os
    from safetensors.torch import save_file
    os.makedirs(save_directory, exist_ok=True)
    c = config
    is_opt = isinstance(c, OptLMConfig)
    is_neox = isinstance(c, NeoxLMConfig)
    if base_model_name is None:
        base_model_name = (("facebook/opt-350m" if isinstance(c, OptPostLnLMConfig) else "facebook/opt-125m") if is_opt
                           else ("EleutherAI/pythia-160m" if is_neox else "Qwen/Qwen2.5-0.5B"))
    sd = {k: v.detach().contiguous().cpu() for k, v in state_dict_hf.items()
          if k != "lm.lm_head.weight" or not c.tie_embeddings}
    save_file(sd, os.path.join(save_directory, "model.safetensors"), metadata={"format": "pt"})
    base = _opt_base_config(c, torch_dtype) if is_opt else _neox_base_config(c) if is_neox else {"model_type": "qwen2", "architectures": ["Qwen2ForCausalLM"], "hidden_size": c.hidden,
            "intermediate_size": c.ffn, "num_hidden_layers": c.n_layers, "num_attention_heads": c.n_heads,
            "num_key_value_heads": c.n_kv_heads, "vocab_size": c.vocab_size, "rms_norm_eps": c.rms_eps,
            "max_position_embeddings": c.max_positions, "tie_word_embeddings": c.tie_embeddings, "hidden_act": "silu",
            "rope_parameters": {"rope_theta": c.rope_theta, "rope_type": "default"}, "rope_theta": c.rope_theta,
            "pad_token_id": c.pad_token_id, "bos_token_id": 1, "eos_token_id": 1, "torch_dtype": "bfloat16"}
    cfg = {"model_type": "speech_language_model", "architectures": ["UnitLM"], "base_model_name": base_model_name,
           "base_config": base, "vocab_size": c.vocab_size, "twist_init": False, "use_cache": False,
           "tie_word_embeddings": c.tie_embeddings, "torch_dtype": torch_dtype,
           "max_position_embeddings": c.max_positions}
    with open(os.path.join(save_directory, "config.json"), "w") as f:
        json.dump(cfg, f, indent=2)


def checkpoint_is_fp32(config: dict) -> bool:
    """Whether a `save_pretrained` config.json (top level, else its base_config) names float32 as its dtype, under
    `torch_dtype` or under `dtype` (the key transformers writes since 4.56)."""
    def dtype_of(c: dict):
        return c.get("dtype", c.get("torch_dtype"))
    dt = dtype_of(config)
    if dt is None:
        dt = dtype_of(config.get("base_config") or {})
    return str(dt).replace("torch.", "") == "float32"


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

    def __init__(self, config, device: str = "cuda:0", max_batch: int = 8, max_seq: int = 1024,
                 trainable: bool = True, seed: Optional[int] = None, master_weights: bool = False,
                 fp32_inference: bool = False):
        """`config`: `LMConfig` (Qwen2 decoder), `OptLMConfig` (pre-LayerNorm OPT decoder), `OptPostLnLMConfig`
        (post-LayerNorm OPT, opt-350m; bf16 training and both inference modes, no master weights) or `NeoxLMConfig`
        (GPT-NeoX).

        `master_weights` (OPT only): train fp32 parameters, fp32 gradients and fp32 AdamW moments under bf16 autocast
        numerics -- the reference's default recipe (`torch_dtype: null`, `bf16: true`).  `params32` / `grads32` then hold
        the model; `params` is their bf16 shadow that the GEMMs read and `grads` the per-micro-batch bf16 scratch of the
        linear gradients.  Such a model trains and scores; `generate` refuses it (generate from its saved checkpoint).

        `fp32_inference` (OPT, `trainable=False`): score and generate in fp32, as the reference runs a float32 checkpoint
        (`from_pretrained` picks it for one).  `params32` holds the model; the linears run as split-bf16 three-product
        GEMMs on its (hi, lo) copy, and logits, log-likelihoods and the sampled distribution are fp32-grade."""
        self.fp32 = bool(fp32_inference)
        if self.fp32 and (not isinstance(config, OptLMConfig) or trainable or master_weights):
            raise ValueError("fp32_inference=True is a forward-only mode of the OPT decoder: it needs an OPT config and "
                             "trainable=False, without master_weights (the Qwen2 and GPT-NeoX recipes are bf16)")
        self.lib = L.require_cuda()
        self.config = config
        self.is_opt = isinstance(config, OptLMConfig)
        self.is_neox = isinstance(config, NeoxLMConfig)
        self.master = bool(master_weights)
        self.post_ln = isinstance(config, OptPostLnLMConfig)
        if self.master and not self.is_opt:
            raise ValueError("master_weights=True is implemented for the OPT decoder only (the Qwen2 and GPT-NeoX recipes "
                             "train bf16 parameters)")
        if self.master and self.post_ln:
            raise ValueError("master_weights=True is implemented for the pre-LayerNorm OPT decoder only; a post-LayerNorm "
                             "OPT (OptPostLnLMConfig, e.g. opt-350m) trains bf16 parameters (torch_dtype bfloat16)")
        self.device = torch.device(device)
        torch.cuda.set_device(self.device)
        self._h = C.c_void_p()
        if self.is_neox:
            c = L.SkNeoxConfig(config.vocab_size, config.hidden, config.n_layers, config.n_heads, config.ffn,
                               config.max_positions, config.rot_dims, config.ln_eps)
            L.check(self.lib.sk_lm_create_neox(C.byref(c), C.byref(self._h)))
        elif self.is_opt:
            c = L.SkOptConfig(config.vocab_size, config.hidden, config.n_layers, config.n_heads, config.ffn,
                              config.max_positions, config.ln_eps, int(config.tie_embeddings))
            if self.post_ln:
                c.post_ln, c.proj_dim = 1, config.proj_dim
            L.check(self.lib.sk_lm_create_opt(C.byref(c), C.byref(self._h)))
        else:
            c = L.SkLmConfig(config.vocab_size, config.hidden, config.n_layers, config.n_heads, config.n_kv_heads,
                             config.head_dim, config.ffn, config.max_positions, config.rms_eps,
                             int(config.tie_embeddings), int(config.qkv_bias))
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
        # fp32 inference reads params32 and its split copy only: the bf16 buffer that sk_lm_bind requires is a placeholder
        self.params = torch.zeros(64 if self.fp32 else self.n_params, device=self.device, dtype=torch.bfloat16)
        self.grads = torch.zeros(self.n_params, device=self.device, dtype=torch.bfloat16) if trainable else None
        self.rope_cos = self.rope_sin = None          # OPT: learned positions, no RoPE tables
        if not self.is_opt:          # GPT-NeoX: tables over the rotated columns only (partial rotary)
            cos, sin = rope_tables(config.rope_theta, config.rot_dims if self.is_neox else config.head_dim,
                                   config.max_positions)
            self.rope_cos, self.rope_sin = cos.to(self.device), sin.to(self.device)
        self.max_batch, self.max_seq = max_batch, max_seq
        self.workspace = None
        self.params32 = self.grads32 = None
        self._bind(max_batch, max_seq)
        if self.master:
            self.params32 = torch.zeros(self.n_params, device=self.device, dtype=torch.float32)
            self.grads32 = torch.zeros(self.n_params, device=self.device, dtype=torch.float32) if trainable else None
            L.check(self.lib.sk_lm_set_master(self._h, L.ptr(self.params32), L.ptr(self.grads32)))
            self._bind(max_batch, max_seq)                # the fp32 residual stream needs the larger workspace
        if self.fp32:
            self.params32 = torch.zeros(self.n_params, device=self.device, dtype=torch.float32)
            self.prepared = torch.empty(int(self.lib.sk_lm_fp32_prepared_bytes(self._h)), device=self.device,
                                        dtype=torch.uint8)
            self.refresh_shadow()
            self._bind(max_batch, max_seq)                # (hi, lo) activations and fp32 logits: a larger workspace
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
        """A parameter (or its gradient) as a [rows, cols] view of the flat buffers: the fp32 ones with master weights
        or fp32 inference, else the bf16 ones."""
        off, r, c = self.tensors[name]
        if self.master or self.fp32:
            flat = self.grads32 if grad else self.params32
        else:
            flat = self.grads if grad else self.params
        return flat[off:off + r * c].view(r, c)

    def refresh_shadow(self) -> None:
        """Master weights: rewrite the bf16 shadow from the fp32 masters; fp32 inference: rewrite the split (hi, lo) copy
        of params32 (after they are loaded or changed by hand)."""
        if self.master:
            self.params.copy_(self.params32)
        if self.fp32:
            L.check(self.lib.sk_lm_set_fp32(self._h, L.ptr(self.params32), L.ptr(self.prepared),
                                            C.c_int64(self.prepared.numel()), L.stream_ptr()))

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
        if self.is_opt or self.is_neox:
            return self._init_weights_opt(seed)
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

    def _init_weights_opt(self, seed: int) -> None:
        """HF OPT init (PreTrainedModel._init_weights with config.init_std): normal(0, init_std) for the linear weights
        and both embedding tables, zero for the token table's pad_token_id row (nn.Embedding(padding_idx)), LayerNorm
        weights 1 and biases 0, linear biases 0.  GPT-NeoX's init is the same with initializer_range as the std and no
        padding row (embed_in has no padding_idx)."""
        g = torch.Generator(device="cpu").manual_seed(seed)
        cfg = self.config
        std = cfg.init_std
        dt = torch.float32 if self.master or self.fp32 else torch.bfloat16
        for name, (off, r, c) in self.tensors.items():
            t = self.tensor(name)
            base = name.split(".")[-1]
            if base in ("ln1", "ln2", "final_norm"):
                t.fill_(1.0)
            elif r == 1:                                   # LayerNorm and linear biases
                t.zero_()
            elif base in ("embed", "lm_head"):
                t.zero_()
                t[:cfg.vocab_size].copy_((torch.randn((cfg.vocab_size, c), generator=g) * std).to(dt))
                if base == "embed" and self.is_opt and 0 <= cfg.pad_token_id < cfg.vocab_size:
                    t[cfg.pad_token_id].zero_()
            else:
                t.copy_((torch.randn((r, c), generator=g) * std).to(dt))
        self.refresh_shadow()

    def _hf_map_opt(self) -> Iterator[Tuple[str, str, List[Tuple[int, int, int]]]]:
        """OPT names of `UnitLM.state_dict()` over OPTForCausalLM: q/k/v are row ranges of the fused `wqkv` / `bqkv`."""
        cfg = self.config
        d = cfg.hidden
        for l in range(cfg.n_layers):
            p, h = f"layers.{l}.", f"lm.model.decoder.layers.{l}."
            yield p + "ln1", h + "self_attn_layer_norm.weight", [(0, 0, 1)]
            yield p + "ln1_b", h + "self_attn_layer_norm.bias", [(0, 0, 1)]
            for j, n in enumerate("qkv"):
                yield p + "wqkv", h + f"self_attn.{n}_proj.weight", [(j * d, 0, d)]
                yield p + "bqkv", h + f"self_attn.{n}_proj.bias", [(j * d, 0, d)]
            yield p + "wo", h + "self_attn.out_proj.weight", [(0, 0, d)]
            yield p + "bo", h + "self_attn.out_proj.bias", [(0, 0, 1)]
            yield p + "ln2", h + "final_layer_norm.weight", [(0, 0, 1)]
            yield p + "ln2_b", h + "final_layer_norm.bias", [(0, 0, 1)]
            yield p + "w1", h + "fc1.weight", [(0, 0, cfg.ffn)]
            yield p + "b1", h + "fc1.bias", [(0, 0, 1)]
            yield p + "w2", h + "fc2.weight", [(0, 0, d)]
            yield p + "b2", h + "fc2.bias", [(0, 0, 1)]
        if not self.post_ln:                              # post-LN OPT has no decoder-level final LayerNorm
            yield "final_norm", "lm.model.decoder.final_layer_norm.weight", [(0, 0, 1)]
            yield "final_norm_b", "lm.model.decoder.final_layer_norm.bias", [(0, 0, 1)]
        yield "embed", "lm.model.decoder.embed_tokens.weight", [(0, 0, cfg.vocab_size)]
        yield "pos_embed", "lm.model.decoder.embed_positions.weight", [(0, 0, cfg.max_positions + 2)]
        if self.post_ln and cfg.has_proj:
            yield "proj_in", "lm.model.decoder.project_in.weight", [(0, 0, d)]
            yield "proj_out", "lm.model.decoder.project_out.weight", [(0, 0, cfg.proj_dim)]
        if not cfg.tie_embeddings:
            yield "lm_head", "lm.lm_head.weight", [(0, 0, cfg.vocab_size)]

    def _hf_map_neox(self) -> Iterator[Tuple[str, str, List[Tuple[int, int, int]]]]:
        """GPT-NeoX names of `UnitLM.state_dict()` over GPTNeoXForCausalLM.  HF's fused query_key_value holds per-head
        [q | k | v] blocks of 3 x 64 rows; the flat `wqkv` / `bqkv` hold [Q; K; V] (what the attention kernels read), so
        each head's three 64-row blocks are segments, listed in HF row order."""
        cfg = self.config
        d = cfg.hidden
        qkv = neox_qkv_segments(cfg.n_heads, cfg.head_dim)
        for l in range(cfg.n_layers):
            p, h = f"layers.{l}.", f"lm.gpt_neox.layers.{l}."
            yield p + "ln1", h + "input_layernorm.weight", [(0, 0, 1)]
            yield p + "ln1_b", h + "input_layernorm.bias", [(0, 0, 1)]
            yield p + "ln2", h + "post_attention_layernorm.weight", [(0, 0, 1)]
            yield p + "ln2_b", h + "post_attention_layernorm.bias", [(0, 0, 1)]
            yield p + "wqkv", h + "attention.query_key_value.weight", qkv
            yield p + "bqkv", h + "attention.query_key_value.bias", qkv
            yield p + "wo", h + "attention.dense.weight", [(0, 0, d)]
            yield p + "bo", h + "attention.dense.bias", [(0, 0, 1)]
            yield p + "w1", h + "mlp.dense_h_to_4h.weight", [(0, 0, cfg.ffn)]
            yield p + "b1", h + "mlp.dense_h_to_4h.bias", [(0, 0, 1)]
            yield p + "w2", h + "mlp.dense_4h_to_h.weight", [(0, 0, d)]
            yield p + "b2", h + "mlp.dense_4h_to_h.bias", [(0, 0, 1)]
        yield "final_norm", "lm.gpt_neox.final_layer_norm.weight", [(0, 0, 1)]
        yield "final_norm_b", "lm.gpt_neox.final_layer_norm.bias", [(0, 0, 1)]
        yield "embed", "lm.gpt_neox.embed_in.weight", [(0, 0, cfg.vocab_size)]
        yield "lm_head", "lm.embed_out.weight", [(0, 0, cfg.vocab_size)]

    def _hf_map(self) -> Iterator[Tuple[str, str, List[Tuple[int, int, int]]]]:
        """(flat tensor name, HF parameter name, [(row in the flat tensor, row in the HF tensor, n rows), ...]).

        q/k/v are row ranges of the fused `wqkv` / `bqkv`.  gate_proj and up_proj share `wgu` in 128-row blocks --
        flat rows [256b, 256b+128) = gate rows [128b, 128b+128), flat rows [256b+128, 256b+256) = the same up rows -- so
        that one 256-column GEMM tile holds gate AND up of the same hidden units and SwiGLU runs in the GEMM epilogue."""
        if self.is_opt:
            yield from self._hf_map_opt()
            return
        if self.is_neox:
            yield from self._hf_map_neox()
            return
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
        """Load parameters named as in `UnitLM.state_dict()` (prefix `lm.`, slamkit/model/unit_lm.py:87).  With master
        weights or fp32 inference the fp32 buffer takes the values exactly (fp16 / bf16 checkpoints are widened) and the
        bf16 shadow or the split copy is refreshed from them."""
        for flat, hf, segs in self._hf_map():
            src = sd[hf].to(torch.float32 if self.master or self.fp32 else torch.bfloat16)
            dst = self._flat_rows(flat, grads)
            if src.dim() == 1:
                src = src.view(-1, 1)
            if segs == [(0, 0, 1)]:                       # whole norm weight
                dst.view(-1).copy_(src.view(-1))
                continue
            for f0, h0, n in segs:
                dst[f0:f0 + n].copy_(src[h0:h0 + n])
        if not grads:
            self.refresh_shadow()

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
            out["lm.lm_head.weight"] = out["lm.model.decoder.embed_tokens.weight" if self.is_opt else
                                           "lm.model.embed_tokens.weight"]
        return out

    # ---- checkpoints (HF layout, SURVEY.md §5 / §8 f-4) ------------------------------------------------------------
    def save_pretrained(self, save_directory: str, base_model_name: Optional[str] = None) -> None:
        """With master weights or fp32 inference the checkpoint holds the fp32 values and says `torch_dtype: float32`."""
        write_unit_lm_checkpoint(save_directory, self.state_dict_hf(), self.config, base_model_name,
                                 torch_dtype="float32" if self.master or self.fp32 else "bfloat16")

    @classmethod
    def from_pretrained(cls, directory: str, device: str = "cuda:0", max_batch: int = 8, max_seq: int = 1024,
                        trainable: bool = True, master_weights: bool = False) -> "B200UnitLM":
        """An OPT checkpoint whose config says `torch_dtype: float32`, loaded for inference (`trainable=False`, no
        `master_weights`), runs in fp32 (`fp32_inference`): the checkpoint's dtype decides the precision, as for the
        reference's `UnitLM`.  Every other checkpoint runs in bf16."""
        import json
        import os
        from safetensors.torch import load_file
        cfg = json.load(open(os.path.join(directory, "config.json")))
        b = cfg["base_config"]
        if b.get("model_type") == "gpt_neox":
            from transformers import GPTNeoXConfig
            b = {k: v for k, v in b.items() if k not in ("model_type", "architectures")}
            lm_cfg = NeoxLMConfig.from_hf(GPTNeoXConfig(**b), vocab_size=cfg["vocab_size"],
                                          max_positions=max(max_seq, int(b.get("max_position_embeddings", 2048))))
            m = cls(lm_cfg, device=device, max_batch=max_batch, max_seq=max_seq, trainable=trainable)
            m.load_hf_state_dict(load_file(os.path.join(directory, "model.safetensors")))
            return m
        if b.get("model_type") == "opt":
            from transformers import OPTConfig
            b = {k: v for k, v in b.items() if k not in ("model_type", "architectures")}
            if not trainable:                              # dropout is inactive in eval mode
                b.update(dropout=0.0, attention_dropout=0.0, layerdrop=0.0)
            lm_cfg = lm_config_from_hf(OPTConfig(**b), vocab_size=cfg["vocab_size"])
            m = cls(lm_cfg, device=device, max_batch=max_batch, max_seq=max_seq, trainable=trainable,
                    master_weights=master_weights,
                    fp32_inference=checkpoint_is_fp32(cfg) and not trainable and not master_weights)
            m.load_hf_state_dict(load_file(os.path.join(directory, "model.safetensors")))
            return m
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

    def _logits_ptr(self) -> int:
        return self.lib.sk_lm_logits_f32(self._h) if self.fp32 else self.lib.sk_lm_logits(self._h)

    def logits_view(self, B: int, T: int) -> torch.Tensor:
        """Zero-copy view of the logits of the last forward: [B, T, vocab_size], bf16 (fp32 with fp32 inference)."""
        p = self._logits_ptr()
        ld = self.lib.sk_lm_logits_ld(self._h)
        off = p - self.workspace.data_ptr()
        dt = torch.float32 if self.fp32 else torch.bfloat16
        es = 4 if self.fp32 else 2
        flat = self.workspace[off:off + B * T * ld * es].view(dt).view(B, T, ld)
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

    def _ban_bits(self, ignore_tokens) -> Optional[torch.Tensor]:
        """Device bitmask (`generation.ban_bitmask` layout) of an ignore list, built once per distinct list."""
        if ignore_tokens is None:
            return None
        key = tuple(int(i) for i in ignore_tokens)
        cache = self.__dict__.setdefault("_ban_cache", {})
        bits = cache.get(key)
        if bits is None:
            V = self.config.vocab_size
            ids = torch.as_tensor(key, dtype=torch.long).to(self.device)
            if ids.numel() and bool(((ids < 0) | (ids >= V)).any()):
                raise ValueError(f"ignore_tokens: ids must be in [0, {V})")
            flags = torch.zeros((V + 31) // 32 * 32, dtype=torch.int64, device=self.device)
            flags[ids] = 1
            words = (flags.view(-1, 32) << torch.arange(32, device=self.device)).sum(1)
            bits = torch.where(words >= 2 ** 31, words - 2 ** 32, words).to(torch.int32)
            if len(cache) >= 4:
                cache.pop(next(iter(cache)))
            cache[key] = bits
        return bits

    @torch.inference_mode()
    def sequence_log_likelihood(self, tokens: torch.Tensor, mean_nll: bool, ignore_tokens=None,
                                attention_mask: Optional[torch.Tensor] = None,
                                return_token_nll: bool = False):
        """`UnitLM.log_likelihood` of the reference model (slamkit/model/unit_lm.py:184-194): [B] per-sequence (mean or
        summed) log-likelihood on the device.  A bf16 model gives bf16 scores with the reference's bf16 rounding of each
        token's log-prob, of the sum and of the mean (the metric's 0.5 tie rule sees those roundings); an fp32 inference
        model gives fp32 scores with no rounding, as calc_nll on fp32 logits.  One forward pass, then `sk_seq_loglik` /
        `sk_seq_loglik_f32` reads the logits once.  Targets equal to the model's pad id are masked; `ignore_tokens` are
        -inf columns.  With `return_token_nll`, also returns the fp32 [B, T-1] per-token values."""
        check_right_padded(attention_mask)
        if tokens.dim() != 2:
            raise ValueError("tokens must be [batch, seq]")
        B, T = tokens.shape
        if T > self.config.max_positions:
            raise ValueError(f"sequence_log_likelihood: a row of {T} tokens is longer than max_positions = "
                             f"{self.config.max_positions} (rows are not truncated)")
        if B == 0:
            ll = torch.empty((0,), device=self.device, dtype=torch.float32 if self.fp32 else torch.bfloat16)
            return (ll, torch.empty((0, max(T - 1, 0)), device=self.device)) if return_token_nll else ll
        ids = tokens.to(self.device, dtype=torch.int64).contiguous()
        self.forward(ids)
        return self.score_last_forward(ids, mean_nll, ignore_tokens, return_token_nll)

    def score_last_forward(self, ids: torch.Tensor, mean_nll: bool, ignore_tokens=None, return_token_nll: bool = False):
        """The scoring half of `sequence_log_likelihood`: `sk_seq_loglik` (`sk_seq_loglik_f32` with fp32 inference) on the
        logits of the last `forward(ids)` (ids: device int64 [B, T], B >= 1)."""
        B, T = ids.shape
        ll = torch.empty((B,), device=self.device, dtype=torch.float32 if self.fp32 else torch.bfloat16)
        token_nll = torch.empty((B * max(T - 1, 1),), device=self.device, dtype=torch.float32)
        ban = self._ban_bits(ignore_tokens)
        fn = self.lib.sk_seq_loglik_f32 if self.fp32 else self.lib.sk_seq_loglik
        L.check(fn(C.c_void_p(self._logits_ptr()), self.lib.sk_lm_logits_ld(self._h), self.config.vocab_size, L.ptr(ids), B,
                   T, int(self.config.pad_token_id), L.ptr(ban), int(bool(mean_nll)), L.ptr(token_nll), L.ptr(ll),
                   L.stream_ptr()))
        return (ll, token_nll[:B * (T - 1)].view(B, T - 1)) if return_token_nll else ll

    @torch.inference_mode()
    def generate(self, inputs: Optional[torch.Tensor] = None, generation_config=None, **kwargs) -> torch.Tensor:
        """TokenLM.generate (slamkit/model/token_lm.py:19-27; UnitLM.generate -> HF GenerationMixin, unit_lm.py:196-198):
        greedy or sampled continuation of left-padded prompts with HF's logits processing (rules: generation.py).

        All rows decode together on the device: one prefill pass writes the prompts' K/V into a cache, then every new
        token is one batched decode step plus on-device token selection, captured once as a CUDA graph and replayed.
        The host looks at the rows' `finished` flags every 16 steps only.  Sampling draws from a Philox stream whose seed
        comes from `generator` (or torch's default CPU generator), so `torch.manual_seed` makes runs reproducible.
        Prompt plus continuation is bounded by `max_positions`.  `repetition_penalty`, `no_repeat_ngram_size` and
        `min_length` / `min_new_tokens` run inside the selection kernel on a device copy of each row's history;
        `num_return_sequences = k` prefills each prompt once and copies its KV cache to k rows (output [B*k, ...],
        rows of one prompt adjacent, as HF orders them).

        `allowed_token_ids = A` restricts every step to the ids in A: the result is that of
        `bad_words_ids=[[i] for i not in A]`.  The decode steps then run the head GEMM on the rows of A only and select
        over those columns (`sk_lm_decode_step_sub`, `sk_select_next_sub`); with history rules (repetition_penalty,
        no_repeat_ngram_size, min_length / min_new_tokens) or on an fp32 inference handle they ban the complement on the
        full vocabulary instead."""
        if self.master:
            raise NotImplementedError("generate: this model trains fp32 master weights; generate from its saved checkpoint "
                                      "(B200UnitLM.from_pretrained without master_weights)")
        generator = kwargs.pop("generator", None)
        if inputs is None:
            inputs = kwargs.pop("input_ids", None)
        if inputs is None:
            raise ValueError("generate: no prompt (inputs / input_ids)")
        keys = ("max_new_tokens", "max_length", "do_sample", "temperature", "top_k", "top_p", "eos_token_id", "pad_token_id",
                "bad_words_ids", "repetition_penalty", "no_repeat_ngram_size", "min_length", "min_new_tokens",
                "num_return_sequences", "allowed_token_ids")
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
                                      "top_p, bad_words_ids, repetition_penalty, no_repeat_ngram_size, min_length, "
                                      "min_new_tokens, num_return_sequences, allowed_token_ids, eos / pad ids and "
                                      "length limits are implemented)")
        opts.setdefault("eos_token_id", getattr(self.config, "eos_token_id", 1))      # UnitTokeniser: bos = eos = 1
        opts.setdefault("pad_token_id", self.config.pad_token_id)
        if opts.get("do_sample") and "top_k" not in opts:
            opts["top_k"] = 50                                    # transformers' GenerationConfig default
        return self._generate_cached(inputs, attention_mask, generator=generator, **opts)

    def _allowed_ids(self, allowed_token_ids, with_bans: bool) -> Optional[torch.Tensor]:
        """allowed_token_ids as ascending int64 ids, after the checks generate makes (None when not given)."""
        if allowed_token_ids is None:
            return None
        if with_bans:
            raise ValueError("generate: pass allowed_token_ids or bad_words_ids, not both")
        ids = torch.as_tensor(allowed_token_ids).reshape(-1)
        if ids.numel() == 0:
            raise ValueError("generate: allowed_token_ids is empty")
        if ids.is_floating_point() or ids.dtype == torch.bool:
            raise ValueError("generate: allowed_token_ids must be integer token ids")
        ids = ids.to("cpu", torch.long)
        V = self.config.vocab_size
        if bool(((ids < 0) | (ids >= V)).any()):
            raise ValueError(f"generate: allowed_token_ids must be in [0, {V})")
        ids = ids.sort().values
        if bool((ids[1:] == ids[:-1]).any()):
            raise ValueError("generate: allowed_token_ids has duplicate ids")
        return ids

    def _generate_cached(self, inputs: torch.Tensor, attention_mask: Optional[torch.Tensor], max_new_tokens=None,
                         max_length=None, do_sample=False, temperature=None, top_k=None, top_p=None, eos_token_id=None,
                         pad_token_id=None, bad_words_ids=None, generator=None, repetition_penalty=None,
                         no_repeat_ngram_size=None, min_length=None, min_new_tokens=None,
                         num_return_sequences=None, allowed_token_ids=None) -> torch.Tensor:
        from .generation import _single_token_bans, ban_bitmask, min_step
        if inputs.dim() != 2:
            raise ValueError("generate: inputs must be [batch, time]")
        B, T = inputs.shape
        k = int(num_return_sequences or 1)
        if k < 1:
            raise ValueError("num_return_sequences must be >= 1")
        if k > 1 and not do_sample:
            raise ValueError("Greedy methods (do_sample != True) without beam search do not support `num_return_sequences` "
                             f"different than 1 (got {k}).")
        penalty = float(repetition_penalty) if repetition_penalty is not None else 1.0
        if penalty <= 0:
            raise ValueError(f"repetition_penalty has to be a strictly positive float, but is {repetition_penalty}")
        ngram = int(no_repeat_ngram_size or 0)
        if max_new_tokens is None:
            max_new_tokens = (max_length if max_length is not None else 20) - T      # HF's default: max_length = 20 in total
        if max_new_tokens < 0:
            raise ValueError(f"generate: the prompt ({T} tokens) is already longer than max_length={max_length}")
        eos = [] if eos_token_id is None else ([int(eos_token_id)] if isinstance(eos_token_id, int) else
                                               [int(e) for e in eos_token_id])
        eos = sorted(set(eos))
        if len(eos) > 8:
            raise NotImplementedError("generate: at most 8 eos_token_id values are supported")
        if eos and pad_token_id is None:
            pad_token_id = min(eos)                                   # HF: "Setting pad_token_id to eos_token_id"
        fill = int(pad_token_id) if pad_token_id is not None else 0
        banned = _single_token_bans(bad_words_ids)
        allowed = self._allowed_ids(allowed_token_ids, bool(banned))
        lens = torch.full((B,), T, dtype=torch.long)
        if attention_mask is not None:
            m = attention_mask.to("cpu").bool()
            lens = m.sum(1)
            left = torch.arange(T)[None, :] >= (T - lens)[:, None]
            if B and (bool((lens == 0).any()) or not torch.equal(m, left)):
                raise ValueError("generate: attention_mask must be left-padding (zeros first, then ones) for every row")
        bound = min_step(T, min_length, min_new_tokens) if eos else 0
        rules = penalty != 1.0 or ngram > 0 or bound > 0
        V = self.config.vocab_size
        if allowed is not None and (rules or self.fp32):
            keep = set(allowed.tolist())                 # the same result through the full-vocabulary ban bitmask
            banned, allowed = [i for i in range(V) if i not in keep], None
        if rules and B and bool(((inputs < 0) | (inputs >= V)).any()):
            raise ValueError(f"generate: repetition_penalty / no_repeat_ngram_size read every prompt id, pads included; "
                             f"all must be in [0, {V})")
        if B == 0 or max_new_tokens == 0:
            return inputs.repeat_interleave(k, dim=0) if k > 1 else inputs.clone()
        P = self.config.max_positions
        Lmax = int(lens.max())
        if Lmax > P:
            raise L.SkError(f"generate: a prompt of {Lmax} tokens is longer than max_positions = {P}")
        if self.is_opt and Lmax + max_new_tokens > P:
            raise ValueError(f"generate: prompt ({Lmax}) + max_new_tokens ({max_new_tokens}) exceeds the {P} learned positions "
                             "of the OPT position table")
        T_cache = min(Lmax + max_new_tokens, P)
        # left-padded [B, T] -> right-padded [B, Lmax]: row b's real tokens at positions 0..lens[b]-1
        cols = torch.arange(Lmax)[None, :]
        src = ((T - lens)[:, None] + cols).clamp(max=T - 1)
        ids = torch.where(cols < lens[:, None], inputs.to("cpu").gather(1, src), torch.zeros((), dtype=torch.long))
        seed = 0
        if do_sample:
            gen = generator if generator is not None else torch.default_generator
            seed = int(torch.randint(0, 2 ** 62, (1,), generator=gen))
        cfg = L.SkSampling(seed=seed, top_p=float(top_p) if top_p is not None else 1.0,
                           temperature=float(temperature) if temperature is not None else 1.0, do_sample=int(bool(do_sample)),
                           top_k=int(top_k) if top_k else 0, n_eos=len(eos), pad_token_id=fill, max_length=T_cache)
        for i, e in enumerate(eos):
            cfg.eos[i] = e
        if do_sample and cfg.temperature <= 0:
            raise ValueError("temperature must be > 0")
        sess = DecodeSession(self, B * k, T_cache, max_new_tokens, fill, allowed)
        if rules:
            sess.set_rules(inputs.repeat_interleave(k, dim=0), penalty, ngram, bound)
        ban = ban_bitmask(banned, V).to(self.device) if banned else None
        sess.prefill(ids, lens, k)
        sess.select(cfg, ban)
        n_steps = max_new_tokens - 1
        if n_steps > 0:
            def step():
                sess.step()
                sess.select(cfg, ban)
            step()                        # eager: sets every one-time kernel attribute before the capture
            done = 1
            if done < n_steps and not bool(sess.finished.all()):
                # captured on a side stream without torch.cuda.graph's gc.collect / empty_cache, which cost more than a
                # short generation
                g, cur, side = torch.cuda.CUDAGraph(), torch.cuda.current_stream(), torch.cuda.Stream()
                side.wait_stream(cur)
                with torch.cuda.stream(side):
                    g.capture_begin()
                    try:
                        step()
                    finally:
                        g.capture_end()
                cur.wait_stream(side)
                while done < n_steps:
                    if done % 16 == 0 and bool(sess.finished.all()):
                        break
                    g.replay()
                    done += 1
        n_new = int(sess.n_gen.max())
        prompts = inputs.repeat_interleave(k, dim=0) if k > 1 else inputs
        out = torch.cat([prompts.to(self.device), sess.out[:, :n_new]], dim=1)
        return out.to(inputs.device)


class DecodeSession:
    """Device buffers of one batched incremental decode of a `B200UnitLM`: the KV cache of all layers, the decode
    workspace, the [B, vocab] logits of the current step and the selection state (`SkDecodeState`).  PyTorch owns the
    memory; `prefill`, `step` and `select` enqueue `sk_lm_prefill`, `sk_lm_decode_step` and `sk_select_next` on the
    current stream.  `step` and `select` take the same arguments every call, so they can be captured in a CUDA graph.
    After `set_rules`, `select` runs `sk_select_next_ex` over the rows' device history instead."""

    def __init__(self, model: B200UnitLM, B: int, T_cache: int, max_new: int, pad_token_id: int = 0,
                 allowed: Optional[torch.Tensor] = None):
        self.m, self.B, self.T_cache = model, B, T_cache
        lib, h, dev = model.lib, model._h, model.device
        self.ldl = model.vocab_padded
        # allowed ids (ascending): the head is gathered once into `head` [n_pad, width] and the logits are [B, n_pad]
        self.sub_ids, self.head = None, None
        if allowed is not None:
            n = int(allowed.numel())
            self.ldl = (n + 63) // 64 * 64
            self.sub_ids = allowed.to(dev, torch.int32)
            width = model.tensors.get("lm_head", model.tensors["embed"])[2]
            self.head = torch.empty(self.ldl, width, device=dev, dtype=torch.bfloat16)
            L.check(lib.sk_lm_gather_head(h, L.ptr(self.sub_ids), n, self.ldl, L.ptr(self.head), L.stream_ptr()))
        self.kv = torch.empty(int(lib.sk_lm_kv_cache_bytes(h, B, T_cache)), device=dev, dtype=torch.uint8)
        self.ws = torch.empty(int(lib.sk_lm_decode_workspace_bytes(h, B, T_cache)), device=dev, dtype=torch.uint8)
        self.logits_buf = torch.empty(B, self.ldl, device=dev, dtype=torch.float32 if model.fp32 else torch.bfloat16)
        self.tokens = torch.zeros(B, device=dev, dtype=torch.long)
        self.pos = torch.zeros(B, device=dev, dtype=torch.int32)
        self.finished = torch.zeros(B, device=dev, dtype=torch.int32)
        self.n_gen = torch.zeros(B, device=dev, dtype=torch.int32)
        self.out = torch.full((B, max(max_new, 1)), pad_token_id, device=dev, dtype=torch.long)
        self.step_ctr = torch.zeros(2, device=dev, dtype=torch.int32)
        self.state = L.SkDecodeState(self.tokens.data_ptr(), self.pos.data_ptr(), self.finished.data_ptr(),
                                     self.n_gen.data_ptr(), self.out.data_ptr(), self.step_ctr.data_ptr(), self.out.shape[1], 0)
        self.rules = None

    def set_rules(self, prompts: torch.Tensor, penalty: float = 1.0, ngram: int = 0, min_step: int = 0) -> None:
        """Turns on the history processors (SkLogitRules): prompts are the [B, T] padded prompts exactly as passed to
        generate.  Allocates the history [B, T + max_new] and, as the rules need them, the presence and ban bitmaps;
        call before `prefill`, which builds the presence bitmap."""
        B, T = prompts.shape
        if B != self.B:
            raise ValueError(f"set_rules: {B} prompts for a session of {self.B} rows")
        dev, W = self.m.device, (self.m.config.vocab_size + 31) // 32
        self.history = torch.zeros(B, T + self.out.shape[1], device=dev, dtype=torch.long)
        self.history[:, :T] = prompts.to(dev)
        self.presence = torch.empty(B, W, device=dev, dtype=torch.int32) if penalty != 1.0 else None
        self.scratch = torch.empty(B, W, device=dev, dtype=torch.int32) if ngram > 0 or min_step > 0 else None
        self.rules = L.SkLogitRules(self.history.data_ptr(), L.ptr(self.presence).value, L.ptr(self.scratch).value,
                                    float(penalty), int(ngram), int(min_step), T, self.history.shape[1], 0)

    @property
    def logits(self) -> torch.Tensor:
        """[B, vocab_size] logits of the last prefill / decode step (bf16; fp32 with fp32 inference); with allowed ids,
        [B, n]: column c is the logit of sub_ids[c]."""
        if self.sub_ids is not None:
            return self.logits_buf[:, :self.sub_ids.numel()]
        return self.logits_buf[:, :self.m.config.vocab_size]

    def prefill(self, ids: torch.Tensor, lens: torch.Tensor, k: int = 1) -> torch.Tensor:
        """ids: right-padded [B, T] prompts, lens: real tokens per row.  Fills the cache; the next token of row b goes
        to position lens[b] (its last prompt token, at lens[b] - 1, is the state's current token).  k > 1
        (num_return_sequences): the session has B*k rows; each prompt is prefilled once at [B, T] and its cache rows,
        logits, token and position are copied to rows b*k .. b*k + k - 1 (`sk_lm_kv_fanout`)."""
        m = self.m
        B, T = ids.shape
        if B * k != self.B:
            raise ValueError(f"prefill: {B} prompts x {k} for a session of {self.B} rows")
        m._ensure(B, T)
        ids_d = ids.to(m.device, dtype=torch.long).contiguous()
        lens_d = lens.to(m.device, dtype=torch.int32).contiguous()
        tok = ids_d.gather(1, (lens_d.long() - 1).clamp(min=0)[:, None])[:, 0]
        kv = self.kv if k == 1 else torch.empty(int(m.lib.sk_lm_kv_cache_bytes(m._h, B, self.T_cache)), device=m.device,
                                                dtype=torch.uint8)
        if self.head is None:
            L.check(m.lib.sk_lm_prefill(m._h, L.ptr(ids_d), L.ptr(lens_d), B, T, L.ptr(kv), self.T_cache,
                                        L.ptr(self.logits_buf), self.ldl, L.ptr(self.ws), C.c_int64(self.ws.numel()),
                                        L.stream_ptr()))
        else:
            L.check(m.lib.sk_lm_prefill_sub(m._h, L.ptr(ids_d), L.ptr(lens_d), B, T, L.ptr(kv), self.T_cache,
                                            L.ptr(self.head), self.ldl, L.ptr(self.logits_buf), self.ldl, L.ptr(self.ws),
                                            C.c_int64(self.ws.numel()), L.stream_ptr()))
        if k > 1:
            L.check(m.lib.sk_lm_kv_fanout(m._h, L.ptr(kv), B, k, L.ptr(self.kv), self.T_cache, L.ptr(lens_d),
                                          L.stream_ptr()))
            self.logits_buf.copy_(self.logits_buf[:B].repeat_interleave(k, dim=0))
            tok, lens_d = tok.repeat_interleave(k), lens_d.repeat_interleave(k)
        self.tokens.copy_(tok)
        self.pos.copy_(lens_d - 1)
        if self.rules is not None and self.presence is not None:
            L.check(m.lib.sk_presence_init(L.ptr(self.history), self.history.shape[1], self.rules.prompt_len, self.B,
                                           m.config.vocab_size, L.ptr(self.presence), L.stream_ptr()))
        return self.logits

    def step(self, tokens: Optional[torch.Tensor] = None, pos: Optional[torch.Tensor] = None) -> torch.Tensor:
        """One decode step: tokens int64 [B] at positions pos int32 [B] (default: the selection state's)."""
        m = self.m
        t = self.tokens if tokens is None else tokens
        p = self.pos if pos is None else pos
        if self.head is None:
            L.check(m.lib.sk_lm_decode_step(m._h, L.ptr(t), L.ptr(p), self.B, L.ptr(self.kv), self.T_cache,
                                            L.ptr(self.logits_buf), self.ldl, L.ptr(self.ws), C.c_int64(self.ws.numel()),
                                            L.stream_ptr()))
        else:
            L.check(m.lib.sk_lm_decode_step_sub(m._h, L.ptr(t), L.ptr(p), self.B, L.ptr(self.kv), self.T_cache,
                                                L.ptr(self.head), self.ldl, L.ptr(self.logits_buf), self.ldl,
                                                L.ptr(self.ws), C.c_int64(self.ws.numel()), L.stream_ptr()))
        return self.logits

    def select(self, cfg: "L.SkSampling", ban: Optional[torch.Tensor] = None, uniforms: Optional[torch.Tensor] = None) -> None:
        m = self.m
        if self.sub_ids is not None:
            if ban is not None or self.rules is not None:
                raise ValueError("select: a session with allowed ids takes no ban bitmask or rules")
            L.check(m.lib.sk_select_next_sub(L.ptr(self.logits_buf), self.ldl, L.ptr(self.sub_ids), self.sub_ids.numel(),
                                             m.config.vocab_size, self.B, C.byref(cfg), L.ptr(uniforms),
                                             C.byref(self.state), L.stream_ptr()))
            return
        args = (L.ptr(self.logits_buf), self.ldl, m.config.vocab_size, self.B, L.ptr(ban), C.byref(cfg), L.ptr(uniforms),
                C.byref(self.state))
        if self.rules is None:
            fn = m.lib.sk_select_next_f32 if m.fp32 else m.lib.sk_select_next
            L.check(fn(*args, L.stream_ptr()))
        else:
            fn = m.lib.sk_select_next_ex_f32 if m.fp32 else m.lib.sk_select_next_ex
            L.check(fn(*args, C.byref(self.rules), L.stream_ptr()))


class B200AdamW:
    """Gradient clipping + AdamW exactly as HF Trainer applies them (HF:trainer.py clip_grad_norm_ -> optimizer.step):
    one `sk_lm_optimizer_step` call = grad-norm reduction + fused clip-scale/AdamW pass over the flat buffers."""

    def __init__(self, model: B200UnitLM, lr: float = 1e-3, betas=(0.9, 0.999), eps: float = 1e-8,
                 weight_decay: float = 0.0, max_grad_norm: float = 0.5, emulate_bf16_norm: bool = True):
        self.model = model
        self.lr, self.betas, self.eps, self.wd = lr, betas, eps, weight_decay
        self.max_grad_norm = max_grad_norm
        self.emulate = emulate_bf16_norm
        # fp32 moments with master weights (torch.optim.AdamW keeps its state in the parameters' dtype)
        self.exp_avg = torch.zeros_like(model.params32 if model.master else model.params)
        self.exp_avg_sq = torch.zeros_like(self.exp_avg)
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
