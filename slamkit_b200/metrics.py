"""Modelling metrics of cli/eval.py (slamkit/metric/modelling_metric.py): sWUGGY, sBLIMP, sStoryCloze / tStoryCloze and
SALMon.  Each metric is a list of (positive, negative) clip pairs; a pair scores 1 when the model gives the positive clip
the higher log-likelihood, 0.5 on a tie and 0 otherwise (also when a score is NaN), and the metric is the mean.

Scores are the bf16 values of `B200SpeechLM.log_likelihood`, as the bf16 reference model returns them, so ties happen
where the reference has them.  Batching follows the reference exactly: `batch_size` positives form one batch and the
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
    """Per-pair results (the dtype of the scores, bf16) in dataset order.  Audio is decoded by `num_workers` threads
    ahead of the GPU into pinned buffers (cli/extract_features.BatchPrefetcher; it always pins, so `pin_memory` is
    accepted for the reference's signature only)."""
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
