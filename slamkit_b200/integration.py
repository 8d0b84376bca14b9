"""Factory hooks for the reference's two string-keyed factories (INTEGRATION.md):
`feature_extractor_type: hubert_b200` (slamkit/tokeniser/audio_tokeniser.py:99-104) and `tlm_type: b200`
(slamkit/model/token_lm.py:30-43).  Constructor keys and defaults are the reference's own."""
from __future__ import annotations

import os
import warnings
from typing import Optional, Tuple


def hubert_b200_from_cfg(pretrained_model: str = "facebook/hubert-base-ls960",
                         kmeans_path: str = "https://dl.fbaipublicfiles.com/hubert/hubert_base_ls960_L9_km500.bin",
                         layer: int = 9, num_units: int = 500, compile: bool = False, cache_path: Optional[str] = None,
                         load_config_only: bool = False, device: str = "cuda:0", max_batch: int = 64,
                         max_samples: int = 480000):
    """Same keys as HubertFeatureExtractor.__init__ (hubert_feature_extractor.py:17-37); `compile` is accepted and
    ignored (there is no tracing compiler on this path)."""
    from transformers import HubertConfig, HubertModel
    from .feature_extractor import HubertB200Config, HubertB200FeatureExtractor, from_hf_state_dict

    hf_cfg = HubertConfig.from_pretrained(pretrained_model)
    cfg = HubertB200Config.from_hf(hf_cfg, layer=layer, n_units=num_units)
    if load_config_only:
        return HubertB200FeatureExtractor(cfg, load_config_only=True)
    if cache_path is None:
        cache_path = os.environ.get("SLAMKIT_CACHE", os.path.expanduser("~/.cache/slamkit"))
    os.makedirs(cache_path, exist_ok=True)
    km_file = f"{cache_path}/kmeans_model.bin"
    if not os.path.exists(km_file):
        from torch.hub import download_url_to_file
        download_url_to_file(kmeans_path, km_file)
    import joblib
    with open(km_file, "rb") as fd, warnings.catch_warnings():
        warnings.simplefilter("ignore")
        km = joblib.load(fd)
    model = HubertModel.from_pretrained(pretrained_model)
    params = from_hf_state_dict(model.state_dict(), km.cluster_centers_, cfg)
    return HubertB200FeatureExtractor(cfg, params, device=device, max_batch=max_batch, max_samples=max_samples)


def tlm_b200_config(cfg, autocast_bf16: Optional[bool] = None):
    """The decoder config and precision for the reference's model config node (config/model/*.yaml): context_len,
    config_args{base_model_name, vocab_size, twist_init, rope_theta, torch_dtype, dropout, ...}.  Host code only (reads the
    base config, builds nothing on the GPU).  Returns (lm_cfg, master_weights).

    The base config decides the decoder: Qwen2 (`LMConfig`), pre-LayerNorm OPT (`OptLMConfig`, the default TWIST / GSLM
    base), post-LayerNorm OPT (`OptPostLnLMConfig`, opt-350m, bfloat16 only) or parallel-residual GPT-NeoX (`NeoxLMConfig`, the Pythia bases of config/train_inter_scale.yaml).  For OPT the
    reference's `config_args` overrides are applied to the base config as `UnitLMConfig` does (pad / bos / eos ids,
    dropout, attention_dropout, layerdrop), `rope_theta` is ignored, and `torch_dtype` picks the precision:
      - bfloat16: bf16 parameters with bf16 AdamW moments;
      - float32: fp32 master weights, fp32 gradients and fp32 AdamW moments with bf16 autocast numerics -- the
        reference's default recipe, whose `torch_dtype: null` loads the model in fp32 and whose `bf16: true` trains under
        autocast.  `autocast_bf16` is `training_args.bf16` where the caller has it: False asks for pure fp32 training,
        which is refused.
    `torch_dtype: null` is refused by name (pass bfloat16 or float32 explicitly).  GPT-NeoX takes the same overrides and
    requires bfloat16.  Raises OSError when the base model cannot be reached (offline box) and ValueError when its
    architecture or settings have no kernels here."""
    from transformers import AutoConfig
    from .lm import OptLMConfig, lm_config_from_hf

    args = cfg["config_args"] if isinstance(cfg, dict) else cfg.config_args
    get = args.get if hasattr(args, "get") else (lambda k, d=None: getattr(args, k, d))
    base = AutoConfig.from_pretrained(get("base_model_name"))
    ctx = int(cfg["context_len"] if isinstance(cfg, dict) else cfg.context_len)
    master = False
    if getattr(base, "model_type", None) == "opt":
        # slamkit/model/unit_lm.py:59-63 passes these to AutoConfig.from_pretrained; the yaml's dropout keys arrive as
        # the same keyword arguments
        for k in ("pad_token_id", "bos_token_id", "eos_token_id", "dropout", "attention_dropout", "layerdrop"):
            if get(k) is not None:
                setattr(base, k, get(k))
        dt = str(get("torch_dtype")).replace("torch.", "")
        if dt == "float32" and not getattr(base, "do_layer_norm_before", True):
            raise ValueError("a post-LayerNorm OPT base (do_layer_norm_before=False, e.g. opt-350m) trains bf16 parameters "
                             "with bf16 AdamW moments on the GPU path; fp32 master weights (torch_dtype=float32) are "
                             "implemented for the pre-LayerNorm OPT only (pass model.config_args.torch_dtype=bfloat16)")
        if dt == "float32":
            if autocast_bf16 is False:
                raise ValueError("OPT with model.config_args.torch_dtype=float32 trains fp32 master weights under bf16 autocast; "
                                 "training_args.bf16=false asks for pure fp32 training, which the GPU path does not implement "
                                 "(set training_args.bf16=true)")
            master = True
        elif dt != "bfloat16":
            raise ValueError(f"OPT on the GPU path trains bf16 parameters with bf16 AdamW moments (torch_dtype=bfloat16) or "
                             f"fp32 master weights under bf16 autocast (torch_dtype=float32); torch_dtype={get('torch_dtype')} "
                             "names neither (pass model.config_args.torch_dtype=bfloat16 or model.config_args.torch_dtype=float32)")
    elif getattr(base, "model_type", None) == "gpt_neox":
        # UnitLMConfig (slamkit/model/unit_lm.py:59-63) hands pad / bos / eos (defaults 0 / 1 / 1) and the yaml's
        # remaining config_args to AutoConfig.from_pretrained
        for k, dflt in (("pad_token_id", 0), ("bos_token_id", 1), ("eos_token_id", 1)):
            setattr(base, k, get(k) if get(k) is not None else dflt)
        for k in ("attention_dropout", "hidden_dropout", "use_parallel_residual", "hidden_act", "tie_word_embeddings"):
            if get(k) is not None:
                setattr(base, k, get(k))
        dt = get("torch_dtype")
        if str(dt).replace("torch.", "") != "bfloat16":
            raise ValueError(f"GPT-NeoX on the GPU path trains bf16 parameters with bf16 AdamW moments; torch_dtype={dt} asks "
                             "for fp32 master weights, which it does not implement (pass model.config_args.torch_dtype=bfloat16)")
    lm_cfg = lm_config_from_hf(base, vocab_size=get("vocab_size", 502), max_positions=max(2048, ctx))
    if get("rope_theta") is not None and not isinstance(lm_cfg, OptLMConfig):
        lm_cfg.rope_theta = float(get("rope_theta"))
    return lm_cfg, master


def tlm_b200_from_cfg(cfg, device: str = "cuda:0", max_batch: int = 8, max_seq: Optional[int] = None,
                      autocast_bf16: Optional[bool] = None):
    """The `B200UnitLM` of the reference's model config node, with the decoder and precision `tlm_b200_config` picks
    (OPT with `torch_dtype: float32` trains fp32 master weights, `master_weights=True`).  `twist_init` loads the base
    model's HF weights (opt-125m ships fp16: with master weights they are widened to fp32, as the reference loads them;
    the Pythia weights come from a local directory or cache), else the HF init is seeded."""
    from .lm import B200UnitLM

    args = cfg["config_args"] if isinstance(cfg, dict) else cfg.config_args
    get = args.get if hasattr(args, "get") else (lambda k, d=None: getattr(args, k, d))
    lm_cfg, master = tlm_b200_config(cfg, autocast_bf16)
    ctx = int(cfg["context_len"] if isinstance(cfg, dict) else cfg.context_len)
    model = B200UnitLM(lm_cfg, device=device, max_batch=max_batch, max_seq=int(max_seq or ctx), master_weights=master)
    if get("twist_init", True):
        from transformers import AutoModelForCausalLM
        import torch
        hf = AutoModelForCausalLM.from_pretrained(get("base_model_name"), dtype=torch.float32 if master else torch.bfloat16)
        hf.resize_token_embeddings(lm_cfg.vocab_size)
        model.load_hf_state_dict({"lm." + k: v for k, v in hf.state_dict().items()})
    else:
        model.init_weights(seed=0)
    return model


# textlesslib checkpoint names (`<dense>-<quantizer>-<vocab>-hifigan[-<suffix>]`) -> file names under its disk root
TEXTLESS_VOCODER_FILES = {
    "mhubert-base-25hz-kmeans-500-hifigan": "hifigan_lj_mhubert_base_25hz.pt",
    "mhubert-base-25hz-kmeans-500-hifigan-config": "hifigan_lj_mhubert_base_25hz_config.json",
    "hubert-base-ls960-layer-9-kmeans-500-hifigan": "hifigan_expresso_lj_vctk_hubert_base_ls960_L9_km500_generator.pt",
    "hubert-base-ls960-layer-9-kmeans-500-hifigan-config": "hifigan_expresso_lj_vctk_hubert_base_ls960_L9_km500_config.json",
    "hubert-base-ls960-layer-9-kmeans-expresso-2000-hifigan":
        "hifigan_expresso_lj_vctk_hubert_base_ls960_L9_km2000_expresso_generator.pt",
    "hubert-base-ls960-layer-9-kmeans-expresso-2000-hifigan-config":
        "hifigan_expresso_lj_vctk_hubert_base_ls960_L9_km2000_expresso_config.json",
    "mhubert-base-vp_mls_cv_8lang-kmeans-2000-hifigan":
        "hifigan_expresso_lj_vctk_mhubert_base_vp_mls_cv_8lang_it3_L12_km2000_generator.pt",
    "mhubert-base-vp_mls_cv_8lang-kmeans-2000-hifigan-config":
        "hifigan_expresso_lj_vctk_mhubert_base_vp_mls_cv_8lang_it3_L12_km2000_config.json",
    "mhubert-base-vp_mls_cv_8lang-kmeans-expresso-2000-hifigan":
        "hifigan_expresso_lj_vctk_mhubert_base_vp_mls_cv_8lang_it3_L12_km2000_expresso_generator.pt",
    "mhubert-base-vp_mls_cv_8lang-kmeans-expresso-2000-hifigan-config":
        "hifigan_expresso_lj_vctk_mhubert_base_vp_mls_cv_8lang_it3_L12_km2000_expresso_config.json",
}


def vocoder_checkpoint_paths(dense_model_name: str, quantizer_model_name: str, vocab_size: int,
                             vocoder_suffix: Optional[str] = None) -> Tuple[str, str]:
    """(generator, config) paths where textlesslib's checkpoint manager keeps them: $TEXTLESS_CHECKPOINT_ROOT, default
    ~/.textless/ (CodeHiFiGANVocoder.by_name, slamkit/vocoder/hifigan/vocoder.py:98-140)."""
    name = f"{dense_model_name}-{quantizer_model_name}-{vocab_size}-hifigan"
    if vocoder_suffix is not None:
        name += "-" + vocoder_suffix
    root = os.path.expanduser(os.environ.get("TEXTLESS_CHECKPOINT_ROOT", "~/.textless/"))
    if name not in TEXTLESS_VOCODER_FILES:
        raise FileNotFoundError(f"unknown textless vocoder checkpoint '{name}': pass model_path= and config_path=")
    return (os.path.join(root, TEXTLESS_VOCODER_FILES[name]), os.path.join(root, TEXTLESS_VOCODER_FILES[name + "-config"]))


def vocoder_b200_from_cfg(cfg, device: str = "cuda:0", max_rows: int = 64, max_frames: int = 16384):
    """`vocoder_factory` (slamkit/vocoder/audio_vocoder.py:13-25) for `vocoder_type: hifigan` / `hifigan_b200`, with the
    reference's keys (dense_model_name, quantizer_model_name, vocab_size, vocoder_suffix, speaker_meta, style_meta) or
    explicit `model_path` / `config_path`.  Nothing is downloaded: a missing file raises FileNotFoundError naming the
    path it was expected at.  `vocoder_type: null` gives None."""
    get = cfg.get if hasattr(cfg, "get") else (lambda k, d=None: getattr(cfg, k, d))
    vt = get("vocoder_type")
    if vt is None:
        return None
    if vt not in ("hifigan", "hifigan_b200"):
        raise ValueError(f"Unknown vocoder type: {vt}")
    model_path, config_path = get("model_path"), get("config_path")
    if not (model_path and config_path):
        mp, cp = vocoder_checkpoint_paths(get("dense_model_name"), get("quantizer_model_name"), get("vocab_size"),
                                          get("vocoder_suffix"))
        model_path, config_path = model_path or mp, config_path or cp
    for p in (model_path, config_path):
        if not os.path.exists(p):
            raise FileNotFoundError(f"vocoder file not found: {p} (this package never downloads; place the textlesslib "
                                    "checkpoint there or pass vocoder.model_path / vocoder.config_path)")
    from .vocoder import HifiGanB200Vocoder
    return HifiGanB200Vocoder.from_checkpoint(model_path, config_path, device=device, max_rows=max_rows,
                                              max_frames=max_frames)
