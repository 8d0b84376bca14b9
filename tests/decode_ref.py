"""Reference for the token selection of decode.cu (`sk_select_next`, `sk_select_next_f32`): HF's selection rules, the
Philox4x32-10 draws, and constructed rows whose expected token needs no tolerance.

Selection rule (`expected_token`): slamkit_b200.generation.process_logits (bans -> temperature -> top-k -> top-p) with
top-p ties broken by id (a stable ascending sort), then the inverse CDF in token-id order at u: the first id whose
cumulative probability exceeds u.  -0.0 and +0.0 are one value, as in torch.argmax and HF's warpers.

Draws: with uniforms = NULL the kernel draws u = (r.x >> 8) * 2^-24 from Philox4x32-10 (Salmon et al., SC'11) with
counter (step, row, 0, 0) and key (seed & 0xffffffff, seed >> 32); `philox_uniform` restates it in numpy.

Constructed rows (`constructed_cases`).  Every kept score is equal, or is so far below the kept maximum that its exp
underflows to exactly 0 in fp32 (FILL), so the kept probabilities are exactly 1/n.  With n a power of two the CDF
steps are dyadic, and u placed on a step is exact in the kernel's fp32 draw (target = u * n, running sums of 1.0).
Where n is not a power of two, u is 0 or the largest float below 1, which no rounding can move across a step.  Scores
are bf16 values, so the bf16 and fp32 entry points see the same row; temperatures are powers of two, so the scaled
scores are exact too.  Each case spreads its ids over the vocabulary (`spread`), so at V = 152,167 they fall in
different thread chunks of the kernel.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import List, Sequence

import numpy as np
import torch

FILL = -16384.0                    # a bf16 value whose exp(FILL - 0) is exactly 0 in fp32: probability 0, not banned
ONE_MINUS = float(np.float32(1.0) - np.float32(2.0 ** -24))   # the largest float below 1


# ----------------------------------------------------------------------------------------------------- Philox4x32-10
_M0, _M1 = 0xD2511F53, 0xCD9E8D57
_W0, _W1 = 0x9E3779B9, 0xBB67AE85
_U32 = np.uint64(0xFFFFFFFF)


def philox4x32_10(ctr, key):
    """Philox4x32-10 of counters ctr (4 uint32 arrays, broadcast) under key (2 uint32 arrays) -> 4 uint32 arrays."""
    c = [np.asarray(x, dtype=np.uint64) & _U32 for x in ctr]
    k0, k1 = (np.asarray(x, dtype=np.uint64) & _U32 for x in key)
    for _ in range(10):
        p0 = np.uint64(_M0) * c[0]
        p1 = np.uint64(_M1) * c[2]
        hi0, lo0 = p0 >> np.uint64(32), p0 & _U32
        hi1, lo1 = p1 >> np.uint64(32), p1 & _U32
        c = [hi1 ^ c[1] ^ k0, lo1, hi0 ^ c[3] ^ k1, lo0]
        k0 = (k0 + np.uint64(_W0)) & _U32
        k1 = (k1 + np.uint64(_W1)) & _U32
    return [x.astype(np.uint32) for x in c]


def philox_uniform(seed: int, step: int, rows) -> np.ndarray:
    """float32 [len(rows)]: the kernel's draw of `rows` at `step` under `seed` (counter (step, row, 0, 0))."""
    rows = np.asarray(rows, dtype=np.uint64)
    z = np.zeros_like(rows)
    r = philox4x32_10((np.full_like(rows, step), rows, z, z), (seed & 0xFFFFFFFF, seed >> 32))
    return (r[0] >> np.uint32(8)).astype(np.float32) * np.float32(2.0 ** -24)


# ----------------------------------------------------------------------------------------------------- selection rule
def _canonical(s: torch.Tensor) -> torch.Tensor:
    return s + 0.0                                       # -0.0 + 0.0 = +0.0: one value for both zeros


def expected_token(logits, do_sample, temperature, top_k, top_p, banned, u):
    """generation.process_logits (top-p restated with a stable sort), softmax, inverse CDF at u in token-id order.
    Returns (token, distance of u to the nearest CDF boundary)."""
    from slamkit_b200.generation import process_logits
    logits = _canonical(logits.float())
    if not do_sample:
        s = logits.clone()
        if banned:
            s[list(banned)] = float("-inf")
        return int(torch.nonzero(s == s.max())[0]), 1.0
    s = _canonical(process_logits(logits, temperature, top_k, None, banned))
    if top_p is not None and top_p < 1.0:
        ss, idx = torch.sort(s, descending=False, stable=True)
        cum = ss.softmax(-1).cumsum(-1)
        remove = cum <= (1.0 - top_p)
        remove[-1] = False
        s = s.masked_fill(remove.scatter(0, idx, remove), float("-inf"))
    cdf = torch.softmax(s.double(), -1).cumsum(-1)
    tok = int(torch.searchsorted(cdf, torch.tensor([u], dtype=torch.float64), right=True)[0])
    tok = min(tok, int(torch.nonzero(s > float("-inf"))[-1]))
    return tok, float((cdf - u).abs().min())


def kept_ids(logits, temperature, top_k, top_p, banned) -> List[int]:
    """Ids with a non-zero probability after the sampling processors (stable top-p)."""
    s = _canonical(logits.float())
    from slamkit_b200.generation import process_logits
    s = process_logits(s, temperature, top_k, None, banned)
    if top_p is not None and top_p < 1.0:
        ss, idx = torch.sort(s, descending=False, stable=True)
        remove = ss.softmax(-1).cumsum(-1) <= (1.0 - top_p)
        remove[-1] = False
        s = s.masked_fill(remove.scatter(0, idx, remove), float("-inf"))
    p = torch.softmax(s.double(), -1)
    return torch.nonzero(p > 0)[:, 0].tolist()


# ----------------------------------------------------------------------------------------------------- constructed rows
@dataclass
class SelCase:
    name: str
    logits: torch.Tensor                               # fp32 [V] holding bf16 values
    do_sample: bool
    temperature: float = 1.0
    top_k: int = 0
    top_p: float = 1.0
    u: float = 0.5
    banned: List[int] = field(default_factory=list)
    n_kept: int = 0                                    # the kept set's size the case is built for (0: greedy)

    @property
    def want(self) -> int:
        return expected_token(self.logits, self.do_sample, self.temperature, self.top_k or None,
                              self.top_p if self.top_p < 1.0 else None, self.banned, self.u)[0]


def spread(V: int, n: int) -> List[int]:
    """n distinct ids spread over [0, V): the first and the last id included (n <= V)."""
    assert 1 <= n <= V
    if n == 1:
        return [V // 2]
    return sorted(set(round(i * (V - 1) / (n - 1)) for i in range(n)))


def _row(V: int, ids: Sequence[int], vals: Sequence[float], fill: float = FILL) -> torch.Tensor:
    x = torch.full((V,), fill)
    for i, v in zip(ids, vals):
        x[i] = v
    return x


def signed_zero_cases(V: int) -> List[SelCase]:
    """Rows whose answer depends on -0.0 == +0.0: greedy over a -0.0 at a lower id than a +0.0; top-k and top-p over a
    group of alternating zeros (a key order that puts -0.0 below +0.0 keeps only the +0.0 ids in top-k and drops the
    -0.0 ids first in top-p)."""
    out = []
    if V >= 2:
        a, b = spread(V, 2)
        out.append(SelCase("greedy-signed-zero", _row(V, [a, b], [-0.0, 0.0], -5.0), False))
    if V >= 4:
        z = spread(V, 4)
        vals = [0.0, -0.0, 0.0, -0.0]
        out.append(SelCase("top_k-signed-zero", _row(V, z, vals), True, top_k=2, u=0.8, n_kept=4))
        out.append(SelCase("top_p-signed-zero", _row(V, z, vals), True, top_p=0.5, u=0.0, n_kept=2))
    return out


def constructed_cases(V: int) -> List[SelCase]:
    """The constructed rows that fit a vocabulary of V ids (see the module docstring)."""
    cases: List[SelCase] = []
    # greedy: tied maxima far apart (ids 3 and 150000 at the 152 k vocabulary: thread chunks 0 and 503)
    a, b = (3, 150000) if V == 152167 else spread(V, 2) if V >= 2 else (0, 0)
    if V >= 2:
        cases.append(SelCase("greedy-tie", _row(V, [a, b], [3.0, 3.0]), False))
        cases.append(SelCase("greedy-banned-max", _row(V, [a, b], [7.0, 3.0]), False, banned=[a]))
        keep = spread(V, 1)[0]
        rest = [i for i in range(V) if i != keep]
        x = _row(V, [keep], [-100.0], 50.0)
        cases.append(SelCase("greedy-all-but-one-banned", x, False, banned=rest))
        cases.append(SelCase("sample-all-but-one-banned", x, True, top_k=1, u=ONE_MINUS, banned=rest, n_kept=1))
    # top_k = 1 over distinct scores: the argmax whatever u is
    if V >= 3:
        g = torch.Generator().manual_seed(V)
        x = (torch.randn(V, generator=g) * 3.0).to(torch.bfloat16).float()
        m = spread(V, 3)[1]
        x[m] = float(x.max()) + 1.0
        cases.append(SelCase("top_k1", x, True, top_k=1, u=ONE_MINUS, n_kept=1))
    if V >= 8:
        s8 = spread(V, 8)
        # top-k at a tie: the k-th score is shared by four ids, all kept; u on the dyadic step 1/2
        x = _row(V, s8, [1.0 if i % 2 == 0 else 0.5 for i in range(8)])
        cases.append(SelCase("top_k-tie-at-k", x, True, top_k=2, u=0.5, n_kept=4))
        # top-k at least the number of finite scores (all but four ids banned): the k-th score is -inf, every finite
        # score is kept; u on the step 1/4
        four = s8[1::2]
        ban = [i for i in range(V) if i not in four]
        x = _row(V, four, [2.0] * 4)
        cases.append(SelCase("top_k>=finite-with-bans", x, True, top_k=6, u=0.25, banned=ban, n_kept=4))
        # no top-k, no top-p: eight equal scores, u on the step 3/8, u = 0 and u just below 1
        x = _row(V, s8, [1.5] * 8)
        for u, tag in ((0.375, "step3/8"), (0.0, "u=0"), (ONE_MINUS, "u<1")):
            cases.append(SelCase(f"equal8-{tag}", x, True, u=u, n_kept=8))
        # top-p on the exact cumulative steps of eight equal scores: 1 - top_p = 1/4, 1/2, 3/4 drops 2, 4, 6 of them in
        # id order (the cut lies inside the tie group)
        for p, n, u in ((0.75, 6, 0.0), (0.5, 4, 0.5), (0.25, 2, 0.5)):
            cases.append(SelCase(f"top_p{p}-cut-in-tie", x, True, top_p=p, u=u, n_kept=n))
        cases.append(SelCase("top_p0.75-cut-in-tie-u<1", x, True, top_p=0.75, u=ONE_MINUS, n_kept=6))
        # a power-of-two temperature decides the top-p cut: at 1/8 the four low ids carry ~3e-4 of the mass and go, at
        # temperature 1 they would carry 0.27 and three of them would stay
        x = _row(V, s8, [1.0 if i % 2 else 0.0 for i in range(8)])
        cases.append(SelCase("temp1/8-top_p0.9", x, True, temperature=0.125, top_p=0.9, u=0.5, n_kept=4))
        cases.append(SelCase("temp2-top_k-tie", _row(V, s8, [1.0] * 4 + [0.5] * 4), True, temperature=2.0, top_k=3,
                             u=0.75, n_kept=4))
    return cases


def check_case(c: SelCase) -> None:
    """The arithmetic claims of a constructed row: bf16 scores, the kept set of the size it was built for, and equal
    probabilities on it (so every CDF step is k / n exactly)."""
    assert torch.equal(c.logits.to(torch.bfloat16).float(), c.logits), c.name
    if not c.do_sample:
        return
    kept = kept_ids(c.logits, c.temperature, c.top_k or None, c.top_p if c.top_p < 1.0 else None, c.banned)
    assert len(kept) == c.n_kept, (c.name, kept)
    s = _canonical(c.logits.float())
    if c.temperature != 1.0:
        s = s / c.temperature
    assert len(set(s[kept].tolist())) == 1, c.name
    if c.n_kept & (c.n_kept - 1) and c.u not in (0.0, ONE_MINUS):
        raise AssertionError(f"{c.name}: u must be 0 or just below 1 when the kept count is not a power of two")
