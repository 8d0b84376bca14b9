"""cli/eval.py -- drop-in for the reference entry point (cli/eval.py): the modelling metrics of a trained checkpoint on
the GPU, with the reference's argument grammar and output.

    python cli/eval.py model.pretrained_model=<dir written by cli/train.py> metric=swuggy_inter \
        metric.data_path=<dir> tokeniser=unit_hubert_25 tokeniser.feature_extractor_type=hubert_b200 batch_size=8

Metrics: swuggy, sblimp, storycloze (sStoryCloze / tStoryCloze) and salmon, with `metric.mean_nll`,
`metric.used_token_modality`, `metric.subfolder` and `metric.parts`.  Prints one `key: value` line per result and
`main(argv)` returns the result dict.  `metric=generate` with a vocoder (`vocoder=vocoder_hubert_25`, vocoder_type
hifigan / hifigan_b200) continues the first `prompt_length` seconds of each file and writes
`<out_path>/generate_<i>.wav`; without a vocoder it raises NotImplementedError.  asr_perplexity, llm_as_judge and the
cross-modal metrics need Whisper or an external LLM, which this package does not provide; they raise
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
VOCODERS = ("hifigan", "hifigan_b200")


def check_metric(cfg) -> str:
    """The metric type this CLI runs; raises for the ones it cannot."""
    mt = cfg.metric.metric_type
    if cfg.metric.get("cross_modal", False):
        raise NotImplementedError(f"cross-modal metric '{mt}': it needs a vocoder, Whisper or an external LLM, which this "
                                  "package does not provide")
    if mt == "generate" and cfg.vocoder.get("vocoder_type") in VOCODERS:
        return mt
    if mt in GENERATIVE:
        raise NotImplementedError(f"metric '{mt}' needs a vocoder, Whisper or an external LLM, which this package does "
                                  "not provide; the modelling metrics are swuggy, sblimp, storycloze and salmon")
    if mt not in MODELLING:
        raise ValueError(f"Unknown metric type: {mt}")
    return mt


def load_model(cfg, device: str, max_seq: int = 256):
    """`model.pretrained_model` (a directory written by `save_pretrained` / cli/train.py) as a `B200UnitLM`."""
    from slamkit_b200.lm import B200UnitLM
    path = cfg.model.get("pretrained_model")
    if not path:
        raise ValueError("no pretrained model: pass model.pretrained_model=<dir>")
    base = json.load(open(os.path.join(path, "config.json"))).get("base_config", {})
    if base.get("model_type") not in ("qwen2", "opt", "gpt_neox"):
        raise ValueError(f"unsupported base architecture '{base.get('model_type')}' in {path}: the GPU scoring path "
                         "implements the Qwen2, OPT and GPT-NeoX decoders")
    m = B200UnitLM.from_pretrained(path, device=device, max_batch=cfg.batch_size, max_seq=max_seq, trainable=False)
    logger.info("%s: %s", path, "float32 checkpoint, fp32 inference (split-bf16 GEMMs, fp32 logits and scores)" if m.fp32
                else "bf16 inference")
    return m


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
    if mt != "generate" and cfg.vocoder.get("vocoder_type") is not None:
        logger.warning("the modelling metrics do not use a vocoder; vocoder=%s is ignored", cfg.vocoder.vocoder_type)
    if cfg.logger.get("report_to") not in (None, "none"):
        logger.warning("results are printed only; logger.report_to=%s is ignored", cfg.logger.report_to)
    device = cfg.device if str(cfg.device).startswith("cuda:") else "cuda:0"
    torch.cuda.set_device(device)
    tokeniser = build_tokeniser(cfg, device)
    if mt == "generate":
        return run_generate(cfg, tokeniser, device)
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


def generate_max_seq(cfg, tokeniser, dataset) -> int:
    """LM rows needed by `metric=generate`: the units of the longest prompt (at most one per HuBERT frame), what the
    tokeniser puts around them (the unit tokeniser's BOS; the interleaved tokeniser's prefix and `<speech>` marker) and
    max_new_tokens."""
    from slamkit_b200.audio_io import audio_info
    sr = tokeniser.fe_sample_rate
    longest = 0
    for i, path in enumerate(dataset.data):
        n, file_sr = audio_info(path)
        n = -(-n * sr // file_sr)
        cut = dataset.crop(i)
        longest = max(longest, n if cut is None else min(n, cut))
    new = int(cfg.metric.get("generate_kwargs", {}).get("max_new_tokens", 20))
    extra = len(tokeniser.prompt_layout()["prefix"]) + 1 if hasattr(tokeniser, "prompt_layout") else 1
    return tokeniser.model.frames(max(longest, 1)) + extra + new


def run_generate(cfg, tokeniser, device: str) -> dict:
    """cli/eval.py's `metric=generate` branch: continue the prompts and write `<out_path>/generate_<i>.wav` (32-bit
    float at the tokeniser's sample rate) for the first `num_log` non-empty continuations, numbered in the result list's
    order (with `num_return_sequences = k`, the k continuations of a prompt are adjacent).  Prints no metric lines."""
    from slamkit_b200 import metrics as M
    from slamkit_b200.audio_io import write_wav_float
    from slamkit_b200.integration import vocoder_b200_from_cfg
    from slamkit_b200.speech_lm import B200SpeechLM
    m = cfg.metric
    path = M.resolve_reference_path(m.data_path, cfg.get("reference_path"))
    ds = M.PromptDataset(path, prompt_length=m.prompt_length, sample_rate=tokeniser.fe_sample_rate,
                         num_files=m.num_files, min_file_length=m.get("min_file_length", None),
                         use_alignment=m.get("use_alignment", False), alignment_folder=m.get("alignment_folder", None))
    assert len(ds) > 0, f"no samples found for {path}"
    # every prompt yields num_return_sequences continuations, vocoded in one batch
    n_ret = int(m.get("generate_kwargs", {}).get("num_return_sequences", None) or 1)
    vocoder = vocoder_b200_from_cfg(cfg.vocoder, device=device, max_rows=cfg.batch_size * n_ret)
    model = B200SpeechLM(load_model(cfg, device, max_seq=generate_max_seq(cfg, tokeniser, ds)), tokeniser, vocoder=vocoder)
    if len(tokeniser) > model.model.config.vocab_size:
        raise ValueError(f"the tokeniser has {len(tokeniser)} ids but the model's vocabulary is "
                         f"{model.model.config.vocab_size}")
    res = M.generate(model, path, cfg.batch_size, m.get("used_token_modality", None), m.prompt_length,
                     m.get("min_file_length", None), m.get("alignment_folder", None), m.get("use_alignment", False),
                     tokeniser.fe_sample_rate, m.num_files, cfg.num_workers, cfg.pin_memory, **m.get("generate_kwargs", {}))
    if m.get("out_path", False):
        os.makedirs(m.out_path, exist_ok=True)
        for i, gen in enumerate(res["generate"]):
            if i == m.get("num_log", -1):
                print(f"Only saving first {i} samples")
                break
            if gen.shape[-1] == 0:
                continue
            write_wav_float(os.path.join(m.out_path, f"{m.metric_type}_{i}.{m.get('ext', 'wav')}"), gen,
                            tokeniser.fe_sample_rate)
    return res


if __name__ == "__main__":
    main()
