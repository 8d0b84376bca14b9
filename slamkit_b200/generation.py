"""`TokenLM.generate` rules for the GPU unit LM (slamkit/model/token_lm.py:19-27; `UnitLM.generate` hands the call to HF's
`GenerationMixin.generate`, slamkit/model/unit_lm.py:196-198; callers: `SpeechLM.generate`, slamkit/model/speech_lm.py:38-55,
with `config/metric/generate.yaml`'s `temperature / top_k / max_new_tokens / do_sample` and `bad_words_ids`).

`B200UnitLM.generate` decodes on the device: a prefill pass fills a KV cache, then one batched decode step per token
(`sk_lm_decode_step`) and on-device token selection (`sk_select_next`), replayed as a CUDA graph.  This module is the
CPU statement of the rules that path implements, so that a model trained here can be sampled through the reference's
`SpeechLM` with HF's semantics:
  * decoder-only conventions: prompts arrive LEFT-padded with an `attention_mask` (speech_lm.py:44-45); each row is decoded
    without the pads (positions start at 0 at the first real token, as HF derives them from the mask) and the result is
    the padded prompt followed by the continuation, right-padded with `pad_token_id` after `eos_token_id`;
  * logits processing in HF's order: `bad_words_ids` (single-token entries) -> temperature -> top-k -> top-p -> softmax ->
    multinomial (`do_sample=True`) or argmax.
`select_next` and `generate_tokens` are pure torch functions of a `next_logits(ids[1,t]) -> [vocab]` callable (one row at
a time, no cache), which is how the CPU tests check them against `transformers`' own `generate` and logits warpers and
how the GPU tests check the device sampler.
"""
from __future__ import annotations

from typing import Callable, List, Optional, Sequence

import torch


def process_logits(logits: torch.Tensor, temperature: float = 1.0, top_k: Optional[int] = None, top_p: Optional[float] = None,
                   banned: Optional[Sequence[int]] = None) -> torch.Tensor:
    """fp32 scores after HF's NoBadWords -> Temperature -> TopK -> TopP processors (filtered entries = -inf)."""
    s = logits.float().clone()
    if banned is not None and len(banned):
        s[..., list(banned)] = float("-inf")
    if temperature is not None and temperature != 1.0:
        if temperature <= 0:
            raise ValueError("temperature must be > 0")
        s = s / temperature
    if top_k is not None and top_k > 0:
        k = min(int(top_k), s.shape[-1])
        kth = torch.topk(s, k, dim=-1).values[..., -1, None]
        s = s.masked_fill(s < kth, float("-inf"))
    if top_p is not None and top_p < 1.0:
        # HF TopPLogitsWarper: sort ascending, drop the tokens whose cumulative probability stays <= 1 - top_p, always keep
        # the most probable one
        sorted_s, idx = torch.sort(s, descending=False, dim=-1)
        cum = sorted_s.softmax(dim=-1).cumsum(dim=-1)
        remove = cum <= (1.0 - top_p)
        remove[..., -1:] = False
        s = s.masked_fill(remove.scatter(-1, idx, remove), float("-inf"))
    return s


def select_next(logits: torch.Tensor, do_sample: bool, temperature: float = 1.0, top_k: Optional[int] = None,
                top_p: Optional[float] = None, banned: Optional[Sequence[int]] = None,
                generator: Optional[torch.Generator] = None) -> int:
    if not do_sample:          # greedy: the warpers are not applied (HF only builds them when sampling)
        s = logits.float().clone()
        if banned is not None and len(banned):
            s[..., list(banned)] = float("-inf")
        return int(torch.argmax(s, dim=-1))
    s = process_logits(logits, temperature, top_k, top_p, banned)
    return int(torch.multinomial(torch.softmax(s, dim=-1), 1, generator=generator))


def _single_token_bans(bad_words_ids) -> List[int]:
    if not bad_words_ids:
        return []
    out = []
    for w in bad_words_ids:
        w = list(w)
        if len(w) != 1:
            raise NotImplementedError("bad_words_ids: only single-token entries are supported (what SpeechLM passes, "
                                      "slamkit/model/speech_lm.py:46-48)")
        out.append(int(w[0]))
    return out


def ban_bitmask(banned: Sequence[int], vocab_size: int) -> torch.Tensor:
    """int32 [ceil(V/32)] bitmask of banned ids (bit i % 32 of word i // 32), the form `sk_select_next` takes: one bit per
    id, so banning every text id of an interleaved 152 k vocabulary costs 19 KB."""
    n_words = (vocab_size + 31) // 32
    bits = torch.zeros(n_words * 32, dtype=torch.bool)
    if len(banned):
        ids = torch.as_tensor(list(banned), dtype=torch.long)
        if bool(((ids < 0) | (ids >= vocab_size)).any()):
            raise ValueError(f"bad_words_ids: ids must be in [0, {vocab_size})")
        bits[ids] = True
    words = (bits.view(n_words, 32).long() << torch.arange(32)).sum(1)
    return torch.where(words >= 2 ** 31, words - 2 ** 32, words).to(torch.int32)


def generate_tokens(next_logits: Callable[[torch.Tensor], torch.Tensor], inputs: torch.Tensor,
                    attention_mask: Optional[torch.Tensor] = None, max_new_tokens: Optional[int] = None,
                    max_length: Optional[int] = None, do_sample: bool = False, temperature: float = 1.0,
                    top_k: Optional[int] = None, top_p: Optional[float] = None, eos_token_id=None,
                    pad_token_id: Optional[int] = None, bad_words_ids=None, max_positions: Optional[int] = None,
                    generator: Optional[torch.Generator] = None) -> torch.Tensor:
    """inputs [B, T] (left-padded when attention_mask has leading zeros) -> [B, T + n_new] int64 on inputs' device."""
    if inputs.dim() != 2:
        raise ValueError("generate: inputs must be [batch, time]")
    B, T = inputs.shape
    if max_new_tokens is None:
        max_new_tokens = (max_length if max_length is not None else 20) - T          # HF's default: max_length = 20 in total
    if max_new_tokens < 0:
        raise ValueError(f"generate: the prompt ({T} tokens) is already longer than max_length={max_length}")
    eos = set([] if eos_token_id is None else ([int(eos_token_id)] if isinstance(eos_token_id, int) else [int(e) for e in eos_token_id]))
    if eos and pad_token_id is None:
        pad_token_id = min(eos)                                  # HF: "Setting pad_token_id to eos_token_id"
    banned = _single_token_bans(bad_words_ids)
    rows: List[List[int]] = []
    for b in range(B):
        row = inputs[b]
        if attention_mask is not None:
            m = attention_mask[b].bool()
            n_real = int(m.sum())
            if n_real == 0 or not bool(m[T - n_real:].all()):
                raise ValueError("generate: attention_mask must be left-padding (zeros first, then ones) for every row")
            row = row[T - n_real:]
        seq = row.tolist()
        new: List[int] = []
        for _ in range(max_new_tokens):
            if max_positions is not None and len(seq) + len(new) >= max_positions:
                break
            ids = torch.tensor([seq + new], dtype=torch.long)
            tok = select_next(next_logits(ids), do_sample, temperature, top_k, top_p, banned, generator)
            new.append(tok)
            if tok in eos:
                break
        rows.append(new)
    n_new = max((len(r) for r in rows), default=0)
    fill = pad_token_id if pad_token_id is not None else 0
    out = torch.full((B, T + n_new), fill, dtype=torch.long)
    out[:, :T] = inputs.to("cpu")
    for b, r in enumerate(rows):
        if r:
            out[b, T:T + len(r)] = torch.tensor(r, dtype=torch.long)
    return out.to(inputs.device)
