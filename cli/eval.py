"""cli/eval.py -- drop-in for the reference entry point (cli/eval.py): the modelling metrics of a trained checkpoint on
the GPU, with the reference's argument grammar and output.

    python cli/eval.py model.pretrained_model=<dir written by cli/train.py> metric=swuggy_inter \
        metric.data_path=<dir> tokeniser=unit_hubert_25 tokeniser.feature_extractor_type=hubert_b200 batch_size=8

Metrics: swuggy, sblimp, storycloze (sStoryCloze / tStoryCloze) and salmon, with `metric.mean_nll`,
`metric.used_token_modality`, `metric.subfolder` and `metric.parts`.  Prints one `key: value` line per result and
`main(argv)` returns the result dict.  The generative metrics (generate, asr_perplexity, llm_as_judge) and cross-modal
metrics need a vocoder, Whisper or an external LLM, which this package does not provide; they raise
NotImplementedError.  `+synthetic_weights=true` builds a seeded random mHuBERT-geometry extractor (no checkpoint
reachable offline)."""
import json
import logging
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

from slamkit_b200.config import load_config  # noqa: E402

logger = logging.getLogger(__name__)

MODELLING = ("swuggy", "sblimp", "storycloze", "salmon")
GENERATIVE = ("generate", "asr_perplexity", "llm_as_judge")


def check_metric(cfg) -> str:
    """The metric type this CLI runs; raises for the ones it cannot."""
    mt = cfg.metric.metric_type
    if cfg.metric.get("cross_modal", False):
        raise NotImplementedError(f"cross-modal metric '{mt}': it needs a vocoder, Whisper or an external LLM, which this "
                                  "package does not provide")
    if mt in GENERATIVE:
        raise NotImplementedError(f"metric '{mt}' needs a vocoder, Whisper or an external LLM, which this package does "
                                  "not provide; the modelling metrics are swuggy, sblimp, storycloze and salmon")
    if mt not in MODELLING:
        raise ValueError(f"Unknown metric type: {mt}")
    return mt


def load_model(cfg, device: str):
    """`model.pretrained_model` (a directory written by `save_pretrained` / cli/train.py) as a `B200UnitLM`."""
    from slamkit_b200.lm import B200UnitLM
    path = cfg.model.get("pretrained_model")
    if not path:
        raise ValueError("no pretrained model: pass model.pretrained_model=<dir>")
    base = json.load(open(os.path.join(path, "config.json"))).get("base_config", {})
    if base.get("model_type") != "qwen2":
        raise ValueError(f"unsupported base architecture '{base.get('model_type')}' in {path}: the GPU scoring path "
                         "implements the Qwen2 decoder")
    return B200UnitLM.from_pretrained(path, device=device, max_batch=cfg.batch_size, max_seq=256, trainable=False)


def build_tokeniser(cfg, device: str):
    """The unit tokeniser as cli/extract_features builds it; the interleaved tokeniser wraps the same extractor."""
    from cli.extract_features import build_tokeniser as build_unit
    t = cfg.tokeniser
    if t.tokeniser_type == "unit":
        return build_unit(cfg, device)
    if t.tokeniser_type == "interleave":
        from slamkit_b200.config import Cfg
        from slamkit_b200.tokeniser import B200InterleavingTokeniser
        unit_cfg = Cfg({**cfg, "tokeniser": Cfg({**t, "tokeniser_type": "unit"})})
        fe = build_unit(unit_cfg, device).model
        p = t.params
        return B200InterleavingTokeniser(fe, dedup=p.dedup, pad_token_id=p.pad_token_id,
                                         num_units=p.get("num_units") or t.feature_extractor["num_units"],
                                         text_tokeniser_path=p.get("text_tokeniser_path", "facebook/opt-125m"))
    raise ValueError(f"Unknown tokeniser type: {t.tokeniser_type}")


def main(argv=None):
    from slamkit_b200 import metrics as M
    from slamkit_b200.speech_lm import B200SpeechLM
    cfg = load_config("eval", argv if argv is not None else sys.argv[1:])
    mt = check_metric(cfg)
    if cfg.vocoder.get("vocoder_type") is not None:
        logger.warning("the modelling metrics do not use a vocoder; vocoder=%s is ignored", cfg.vocoder.vocoder_type)
    if cfg.logger.get("report_to") not in (None, "none"):
        logger.warning("results are printed only; logger.report_to=%s is ignored", cfg.logger.report_to)
    device = cfg.device if str(cfg.device).startswith("cuda:") else "cuda:0"
    torch.cuda.set_device(device)
    tokeniser = build_tokeniser(cfg, device)
    model = B200SpeechLM(load_model(cfg, device), tokeniser)
    if len(tokeniser) > model.model.config.vocab_size:
        raise ValueError(f"the tokeniser has {len(tokeniser)} ids but the model's vocabulary is "
                         f"{model.model.config.vocab_size}")
    path = M.resolve_reference_path(cfg.metric.data_path, cfg.get("reference_path"))
    m = cfg.metric
    used, mean_nll = m.get("used_token_modality", None), m.get("mean_nll", True)
    args = (cfg.batch_size, cfg.num_workers, cfg.pin_memory)
    with torch.inference_mode():
        if mt == "salmon":
            res = M.salmon(model, path, used, mean_nll, m.parts, *args)
        else:
            res = getattr(M, mt)(model, path, used, mean_nll, *args, m.get("subfolder", False))
    for key, val in res.items():
        if isinstance(val, list):
            print(f"{key}:")
            for i, v in enumerate(val):
                print(f"\t{i}: {v}")
        else:
            print(f"{key}: {val}")
    return res


if __name__ == "__main__":
    main()
