"""Factory hooks for the reference's two string-keyed factories (INTEGRATION.md):
`feature_extractor_type: hubert_b200` (slamkit/tokeniser/audio_tokeniser.py:99-104) and `tlm_type: b200`
(slamkit/model/token_lm.py:30-43).  Constructor keys and defaults are the reference's own."""
from __future__ import annotations

import os
import warnings
from typing import Optional


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


def tlm_b200_from_cfg(cfg, device: str = "cuda:0", max_batch: int = 8, max_seq: Optional[int] = None):
    """`cfg` is the reference's model config node (config/model/*.yaml): context_len, config_args{base_model_name,
    vocab_size, twist_init, rope_theta, ...}.  Raises OSError when the base model cannot be reached (offline box) and
    ValueError when its architecture has no kernels here (anything but Qwen2)."""
    from transformers import AutoConfig
    from .lm import B200UnitLM, LMConfig

    args = cfg["config_args"] if isinstance(cfg, dict) else cfg.config_args
    get = args.get if hasattr(args, "get") else (lambda k, d=None: getattr(args, k, d))
    base = AutoConfig.from_pretrained(get("base_model_name"))
    ctx = int(cfg["context_len"] if isinstance(cfg, dict) else cfg.context_len)
    lm_cfg = LMConfig.from_hf(base, vocab_size=get("vocab_size", 502), max_positions=max(2048, ctx))
    if get("rope_theta") is not None:
        lm_cfg.rope_theta = float(get("rope_theta"))
    model = B200UnitLM(lm_cfg, device=device, max_batch=max_batch, max_seq=int(max_seq or ctx))
    if get("twist_init", True):
        from transformers import AutoModelForCausalLM
        import torch
        hf = AutoModelForCausalLM.from_pretrained(get("base_model_name"), dtype=torch.bfloat16)
        hf.resize_token_embeddings(lm_cfg.vocab_size)
        model.load_hf_state_dict({"lm." + k: v for k, v in hf.state_dict().items()})
    else:
        model.init_weights(seed=0)
    return model
