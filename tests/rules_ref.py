"""Reference for the history-dependent logits processors of slamkit_b200.generation (`apply_rules`) and of the selection
kernel's `sk_select_next_ex`: transformers' own RepetitionPenalty, NoRepeatNGram, NoBadWords, MinLength and
MinNewTokensLength processors, applied in HF's order on fp32 scores of padded rows, and the rows to compare on.

`hf_rules` restates how `generate` builds them: a set `min_new_tokens` replaces `min_length` by `min_new_tokens + T`,
and both processors count the padded prompt width T.  `rule_cases` are constructed rows (pads in the history, repeated
ids, n = 1..4, eos lists on either side of the length bound) and random ones.  `mismatches(impl)` names the cases where
an implementation with `apply_rules`' signature differs from HF's processors in any element, -inf pattern included.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Callable, List, Optional

import torch

PAD = 0


@dataclass
class RuleCase:
    name: str
    scores: torch.Tensor                  # fp32 [V]
    history: List[int]                    # padded prompt (prompt_len ids) + generated tokens
    prompt_len: int
    repetition_penalty: Optional[float] = None
    no_repeat_ngram_size: int = 0
    banned: List[int] = field(default_factory=list)
    eos: List[int] = field(default_factory=list)
    min_length: Optional[int] = None
    min_new_tokens: Optional[int] = None

    def kwargs(self) -> dict:
        return dict(history=self.history, prompt_len=self.prompt_len, repetition_penalty=self.repetition_penalty,
                    no_repeat_ngram_size=self.no_repeat_ngram_size, banned=self.banned, eos=self.eos,
                    min_length=self.min_length, min_new_tokens=self.min_new_tokens)


def hf_rules(c: RuleCase) -> torch.Tensor:
    from transformers.generation.logits_process import (MinLengthLogitsProcessor, MinNewTokensLengthLogitsProcessor,
                                                       NoBadWordsLogitsProcessor, NoRepeatNGramLogitsProcessor,
                                                       RepetitionPenaltyLogitsProcessor)
    ids = torch.tensor([c.history], dtype=torch.long)
    s = c.scores.float().clone()[None]
    eos = torch.tensor(c.eos, dtype=torch.long) if c.eos else None
    min_length = c.min_length
    if c.min_new_tokens is not None:
        min_length = c.min_new_tokens + c.prompt_len
    procs = []
    if c.repetition_penalty is not None and c.repetition_penalty != 1.0:
        procs.append(RepetitionPenaltyLogitsProcessor(c.repetition_penalty))
    if c.no_repeat_ngram_size and c.no_repeat_ngram_size > 0:
        procs.append(NoRepeatNGramLogitsProcessor(c.no_repeat_ngram_size))
    if c.banned:
        procs.append(NoBadWordsLogitsProcessor([[b] for b in c.banned], eos_token_id=eos))
    if eos is not None and min_length is not None and min_length > 0:
        procs.append(MinLengthLogitsProcessor(min_length, eos))
    if eos is not None and c.min_new_tokens is not None and c.min_new_tokens > 0:
        procs.append(MinNewTokensLengthLogitsProcessor(c.prompt_len, c.min_new_tokens, eos))
    for p in procs:
        s = p(ids, s)
    return s[0]


def rule_cases(V: int = 64, seed: int = 0) -> List[RuleCase]:
    g = torch.Generator().manual_seed(seed)
    rnd = lambda: torch.randn(V, generator=g) * 3.0
    out: List[RuleCase] = []
    # pads in the history: a left-padded prompt of 3 pads, repeated ids, the pad id with the largest (positive) and a
    # negative score
    hist = [PAD, PAD, PAD, 5, 9, 5, 9, 5, 12, 9]
    for p in (1.5, 0.5, 2.0):
        s = rnd()
        s[PAD], s[9] = 7.0, -2.0
        out.append(RuleCase(f"penalty{p}-pads-repeats", s, hist, 8, repetition_penalty=p))
    # n-grams 1..4 over a history whose tail recurs (pads included in the recurring n-grams)
    hist2 = [PAD, PAD, 7, PAD, PAD, 7, 3, PAD, PAD, 7, 3, 4, PAD, PAD, 7]
    for n in (1, 2, 3, 4):
        out.append(RuleCase(f"ngram{n}-pads", rnd(), hist2, 6, no_repeat_ngram_size=n))
    out.append(RuleCase("ngram5-too-short", rnd(), [1, 2, 1], 3, no_repeat_ngram_size=5))
    out.append(RuleCase("ngram4-at-length", rnd(), [1, 2, 1], 3, no_repeat_ngram_size=4))   # cur_len + 1 == n
    # eos lists on either side of the length bound (padded prompt width 6)
    for gen in (0, 1, 2, 3):
        h = [PAD, PAD, 4, 5, 6, 7] + [8] * gen
        out.append(RuleCase(f"min_new3-step{gen}", rnd(), h, 6, eos=[1, 33], min_new_tokens=3))
        out.append(RuleCase(f"min_length8-step{gen}", rnd(), h, 6, eos=[2], min_length=8))
        out.append(RuleCase(f"min_new2-overrides-min_length-step{gen}", rnd(), h, 6, eos=[1, 2, 3], min_new_tokens=2,
                            min_length=20))
    # everything at once, and random rows
    out.append(RuleCase("all", rnd(), hist2, 6, repetition_penalty=1.3, no_repeat_ngram_size=2, banned=[3, 11],
                        eos=[7], min_new_tokens=20))
    for r in range(8):
        T = int(torch.randint(1, 12, (), generator=g))
        h = torch.randint(0, 8, (T + int(torch.randint(0, 10, (), generator=g)),), generator=g).tolist()
        out.append(RuleCase(f"random{r}", rnd(), h, T, repetition_penalty=[None, 1.2, 0.7, 1.0][r % 4],
                            no_repeat_ngram_size=r % 5, eos=[int(h[-1])] if r % 2 else [],
                            min_new_tokens=(r % 3) * 2 if r % 2 else None, min_length=T + 3 if r % 4 == 3 else None))
    return out


def mismatches(impl: Callable[..., torch.Tensor], V: int = 64, seed: int = 0) -> List[str]:
    bad = []
    for c in rule_cases(V, seed):
        want = hf_rules(c)
        got = impl(c.scores.float().clone(), **c.kwargs())
        if not torch.equal(got, want):
            bad.append(c.name)
    return bad
