"""Modelling metrics of cli/eval.py (slamkit/metric/modelling_metric.py): sWUGGY, sBLIMP, sStoryCloze / tStoryCloze and
SALMon.  Each metric is a list of (positive, negative) clip pairs; a pair scores 1 when the model gives the positive clip
the higher log-likelihood, 0.5 on a tie and 0 otherwise (also when a score is NaN), and the metric is the mean.

Scores are the values of `B200SpeechLM.log_likelihood` in the model's own precision, as the reference model returns them:
bf16 for a bf16 checkpoint, fp32 for a float32 OPT checkpoint (fp32 inference), so ties happen where the reference has
them.  Batching follows the reference exactly: `batch_size` positives form one batch and the
same pairs' negatives another, each zero-padded to its own longest clip, in dataset order.  HuBERT sees the padding
(no attention mask, GroupNorm over time), so the batch composition is part of what decides a clip's units."""
from __future__ import annotations

import logging
import os
from pathlib import Path
from typing import List, Optional, Sequence, Tuple

import torch

logger = logging.getLogger(__name__)

SALMON_PARTS = ["bg_alignment/", "bg_all_consistency/", "bg_domain_consistency/", "gender_consistency/",
                "rir_consistency/", "sentiment_alignment/", "sentiment_consistency/", "speaker_consistency/"]


def resolve_reference_path(path: str, default_path: Optional[str]) -> str:
    """A `//reference` prefix becomes $SLAM_REFERENCE_PATH, or `default_path` (cfg.reference_path) when that is unset."""
    if path.startswith("//reference"):
        ref = os.environ.get("SLAM_REFERENCE_PATH", default_path)
        if ref is None:
            raise ValueError("data_path starts with //reference but neither SLAM_REFERENCE_PATH nor reference_path is set")
        path = path.replace("//reference", ref)
    return path


class ModellingMetricDataset:
    """Pairs of consecutive files: for each sub-directory in `Path.iterdir()` order (or `path` itself without
    `subfolder`), the `*.wav` files stably sorted by the integer before the first `sep`; pair i = files 2i (positive)
    and 2i + 1 (negative)."""

    def __init__(self, path: str, sep: str = "_", subfolder: bool = True):
        self.data: List[Path] = []
        key = lambda x: int(x.name.split(sep)[0])  # noqa: E731
        if subfolder:
            for f in Path(path).iterdir():
                if f.is_dir():
                    self.data += sorted(list(f.glob("*.wav")), key=key)
        else:
            self.data += sorted(list(Path(path).glob("*.wav")), key=key)

    def __len__(self) -> int:
        return len(self.data) // 2

    def pair(self, idx: int) -> Tuple[str, str]:
        return str(self.data[2 * idx]), str(self.data[2 * idx + 1])


class SalmonDataset:
    """One SALMon part: files grouped by the integer after the first `_` of the stem, each group sorted; [0] is the
    positive, [1] the negative.  Empty groups are dropped."""

    def __init__(self, path: str, part: str):
        paths = list((Path(path) / part).glob("*.wav"))
        idx = [int(p.stem.split("_")[1]) for p in paths]
        groups: List[List[str]] = [[] for _ in range(max(idx, default=-1) + 1)]
        for p, i in zip(paths, idx):
            groups[i].append(str(p))
        for g in groups:
            g.sort()
        self.data = [g for g in groups if g]

    def __len__(self) -> int:
        return len(self.data)

    def pair(self, idx: int) -> Tuple[str, str]:
        return self.data[idx][0], self.data[idx][1]


def score_pairs(pos: torch.Tensor, neg: torch.Tensor) -> torch.Tensor:
    """modelling_metric.py tie rule: 1 if pos > neg, 0.5 if equal, else 0 (a NaN on either side compares false: 0)."""
    res = torch.zeros_like(pos)
    res[pos > neg] = 1
    res[pos == neg] = 0.5
    res[pos < neg] = 0
    return res


def pair_scores(model, dataset, used_token_modality: Optional[str], mean_nll: bool = True, batch_size: int = 1,
                num_workers: int = 8, pin_memory: bool = True) -> torch.Tensor:
    """Per-pair results (the dtype of the scores: bf16, or fp32 for an fp32 inference model) in dataset order.  Audio
    is decoded by `num_workers` threads ahead of the GPU into pinned buffers (cli/extract_features.BatchPrefetcher; it
    always pins, so `pin_memory` is accepted for the reference's signature only)."""
    from cli.extract_features import BatchPrefetcher
    n = len(dataset)
    batches = []
    for i in range(0, n, batch_size):
        pairs = [dataset.pair(j) for j in range(i, min(i + batch_size, n))]
        batches.append([(p, None) for p, _ in pairs])       # positives, padded to their own longest clip
        batches.append([(q, None) for _, q in pairs])       # negatives, separately
    sr = model.tokeniser.fe_sample_rate
    out, pos = [], None
    for k, (_, wav, lens) in enumerate(BatchPrefetcher(batches, sr, str(model.device), num_workers=max(1, num_workers))):
        ll = model.log_likelihood(wav, lens, mean_nll=mean_nll, used_token_modality=used_token_modality)
        if k % 2 == 0:
            pos = ll
        else:
            out.append(score_pairs(pos, ll))
    return torch.cat(out) if out else torch.zeros(0)


def modelling_metric(model, dataset, used_token_modality: Optional[str], mean_nll: bool = True, batch_size: int = 1,
                     num_workers: int = 8, pin_memory: bool = True) -> float:
    res = pair_scores(model, dataset, used_token_modality, mean_nll, batch_size, num_workers, pin_memory)
    return res.float().mean().cpu().item()


def salmon(model, salmon_path: str, used_token_modality, mean_nll, parts: Sequence[str], batch_size: int,
           num_workers: int = 8, pin_memory: bool = True) -> dict:
    if parts[0] == "all":
        parts = SALMON_PARTS
    out = {}
    for part in parts:
        dataset = SalmonDataset(salmon_path, part)
        assert len(dataset) > 0, f"no samples found for {part}"
        out[part] = modelling_metric(model, dataset, used_token_modality, mean_nll, batch_size, num_workers, pin_memory)
        logger.info(f"SALMon - {part}: {out[part]:.4f}")
    return out


def _paired(name: str, sep: str):
    def metric(model, data_path: str, used_token_modality, mean_nll: bool = True, batch_size: int = 1,
               num_workers: int = 8, pin_memory: bool = True, subfolder: bool = False) -> dict:
        dataset = ModellingMetricDataset(data_path, sep=sep, subfolder=subfolder)
        assert len(dataset) > 0, f"no samples found for {data_path}"
        res = modelling_metric(model, dataset, used_token_modality, mean_nll, batch_size, num_workers, pin_memory)
        logger.info(f"{name}: {res:.4f}")
        return {name: res}
    metric.__name__ = name
    return metric


swuggy = _paired("sWUGGY", "_")
sblimp = _paired("sBLIMP", "+")
storycloze = _paired("StoryCloze", "_")


# ---- generative metric (slamkit/metric/generative_metric.py) ----------------------------------------------------------
def get_cut_location(alignment, prompt_length: float) -> float:
    """generative_metric.py:18-26: the end time of the aligned word whose end is nearest to `prompt_length` (first on
    ties)."""
    endtimes = torch.tensor([word[2] for word in alignment])
    return endtimes[torch.abs(endtimes - prompt_length).argmin()].item()


def _is_shorter(path: str, min_file_length: float) -> bool:
    from .audio_io import audio_info
    n, sr = audio_info(path)
    return n < min_file_length * sr


class PromptDataset:
    """generative_metric.py:34-81: files matched by `glob_path` (recursive), the first `num_files` of `iglob` when it is
    set, skipping files shorter than `min_file_length` seconds; each prompt is the resampled, channel-averaged clip cut
    to `int(prompt_length * sample_rate)` samples, or with `use_alignment` to the aligned word end nearest to
    `prompt_length` (alignments: `<file>.json` next to a `.wav`, or `<alignment_folder>/<stem>.json`)."""

    def __init__(self, glob_path: str, prompt_length: Optional[float] = None, sample_rate: int = 16000,
                 num_files: Optional[int] = None, min_file_length: Optional[float] = None, use_alignment: bool = False,
                 alignment_folder: Optional[str] = None):
        from glob import glob, iglob
        self.prompt_length, self.sample_rate = prompt_length, sample_rate
        if num_files is None:
            self.data = glob(glob_path, recursive=True)
            if min_file_length is not None:
                self.data = [p for p in self.data if not _is_shorter(p, min_file_length)]
        else:
            self.data = []
            for path in iglob(glob_path, recursive=True):
                if len(self.data) >= num_files:
                    break
                if min_file_length is not None and _is_shorter(path, min_file_length):
                    continue
                self.data.append(path)
        self.use_alignment, self.alignment_folder = use_alignment, alignment_folder

    def __len__(self) -> int:
        return len(self.data)

    def crop(self, idx: int) -> Optional[int]:
        """Samples kept of file `idx` (None: all)."""
        if self.prompt_length is None:
            return None
        if not self.use_alignment:
            return int(self.prompt_length * self.sample_rate)
        import json
        with open(self.get_alignment_path(self.data[idx])) as f:
            alignment = json.load(f)["aligned_text"]
        return int(get_cut_location(alignment, self.prompt_length) * self.sample_rate)

    def __getitem__(self, idx: int):
        from .audio_io import load_audio
        audio = load_audio(self.data[idx], self.sample_rate)
        n = self.crop(idx)
        if n is not None:
            audio = audio[:n]
        return audio, audio.shape[-1]

    def get_alignment_path(self, file: str) -> str:
        if self.alignment_folder is None:
            return file.replace(".wav", ".json")
        base = os.path.basename(file)
        return os.path.join(self.alignment_folder, base[:base.find(".")] + ".json")


def generate(model, data_path: str, batch_size: int, used_tokens_modality: Optional[str] = None,
             prompt_length: Optional[float] = None, min_file_length: Optional[float] = None,
             alignment_folder: Optional[str] = None, use_alignment: bool = False, sample_rate: int = 16000,
             num_files: Optional[int] = None, num_workers: int = 8, pin_memory: bool = True, **generate_kwargs) -> dict:
    """generative_metric.py:89-106: `batch_size` prompts at a time, in dataset order, zero-padded to the batch's longest
    prompt, each batch continued by `model.generate`.  Audio is decoded ahead of the GPU by `num_workers` threads
    (cli/extract_features.BatchPrefetcher); the prefetcher decodes whole files, and the crop is applied on the device."""
    from cli.extract_features import BatchPrefetcher
    dataset = PromptDataset(data_path, prompt_length=prompt_length, sample_rate=sample_rate, num_files=num_files,
                            min_file_length=min_file_length, alignment_folder=alignment_folder, use_alignment=use_alignment)
    assert len(dataset) > 0, f"no samples found for {data_path}"
    idx = list(range(len(dataset)))
    batches = [[(dataset.data[i], i) for i in idx[s:s + batch_size]] for s in range(0, len(idx), batch_size)]
    res, prompts = [], []
    with torch.inference_mode():
        for batch, wav, lens in BatchPrefetcher(batches, sample_rate, str(model.device), num_workers=max(1, num_workers)):
            cut = [dataset.crop(i) for _, i in batch]
            lens = torch.stack([lens[r].clamp(max=c) if c is not None else lens[r] for r, c in enumerate(cut)])
            S = int(lens.max())
            wav = wav[:, :S] * (torch.arange(S, device=wav.device)[None, :] < lens[:, None])
            res.extend(model.generate(wav, lens, used_tokens_modality or "SPEECH", **generate_kwargs))
            prompts.extend(wav[r, :int(lens[r])] for r in range(wav.shape[0]))
    return {"generate": res, "prompts": prompts}
