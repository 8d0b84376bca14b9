"""CPU checks of tests/decode_ref.py and of the fp32-cache decode references in tests/attn_ref.py: Philox4x32-10 against
the Random123 known-answer vectors, the selection rule against transformers' own warpers on every constructed row, and
the arithmetic claims behind the exact decode expectations."""
import numpy as np
import pytest
import torch

import attn_ref as A
import decode_ref as D

V_SHAPES = [2, 3, 31, 33, 511, 513, 152167]


# ----------------------------------------------------------------------------------------------------- Philox
@pytest.mark.parametrize("ctr,key,want", [
    ((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
    ((0xFFFFFFFF,) * 4, (0xFFFFFFFF,) * 2, (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
    ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0),
     (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1)),
])
def test_philox_known_answers(ctr, key, want):
    got = D.philox4x32_10(tuple(np.uint32(c) for c in ctr), tuple(np.uint32(k) for k in key))
    assert tuple(int(x) for x in got) == want


def test_philox_uniform_layout():
    """u = (x >> 8) 2^-24 of counter (step, row, 0, 0) under key (seed lo, seed hi): in [0, 1) on the 2^-24 grid, the
    seed's high word and the counter words each change the draw, and step and row are not interchangeable."""
    seed = 0x9E3779B97F4A7C15
    u = D.philox_uniform(seed, 3, range(300))
    assert u.dtype == np.float32 and bool(((u >= 0) & (u < 1)).all())
    assert bool((u * 2 ** 24 == np.round(u * 2 ** 24)).all())
    r = D.philox4x32_10((3, 5, 0, 0), (seed & 0xFFFFFFFF, seed >> 32))
    assert float(D.philox_uniform(seed, 3, [5])[0]) == float(np.uint32(r[0]) >> np.uint32(8)) * 2.0 ** -24
    assert not np.array_equal(u, D.philox_uniform(seed & 0xFFFFFFFF, 3, range(300)))
    assert D.philox_uniform(seed, 3, [5])[0] != D.philox_uniform(seed, 5, [3])[0]
    assert len(set(u.tolist())) > 290


# ----------------------------------------------------------------------------------------------------- selection rule
def _hf(c: D.SelCase) -> torch.Tensor:
    """transformers' processors on the row: bans as -inf, then Temperature / TopK / TopP warpers (sampling only)."""
    from transformers.generation.logits_process import TemperatureLogitsWarper, TopKLogitsWarper, TopPLogitsWarper
    s = c.logits.float().clone()[None]
    if c.banned:
        s[0, c.banned] = float("-inf")
    ids = torch.zeros(1, 1, dtype=torch.long)
    if c.temperature != 1.0:
        s = TemperatureLogitsWarper(c.temperature)(ids, s)
    if c.top_k:
        s = TopKLogitsWarper(c.top_k)(ids, s)
    if c.top_p < 1.0:
        s = TopPLogitsWarper(c.top_p)(ids, s)
    return s[0]


def _cases():
    out = []
    for V in V_SHAPES:
        for c in D.constructed_cases(V) + D.signed_zero_cases(V):
            out.append(pytest.param(V, c.name, id=f"V{V}-{c.name}"))
    return out


def _case(V, name):
    return next(c for c in D.constructed_cases(V) + D.signed_zero_cases(V) if c.name == name)


@pytest.mark.parametrize("V,name", _cases())
def test_constructed_rows_follow_transformers(V, name):
    """The reference's token equals the one the transformers warpers give (argmax with the lowest id for greedy, the
    first id whose cumulative probability exceeds u for sampling), and the case's exactness claims hold."""
    c = _case(V, name)
    D.check_case(c)
    s = _hf(c)
    if not c.do_sample:
        assert c.want == int(torch.argmax(s))
        return
    p = torch.softmax(s.double(), -1)
    kept = torch.nonzero(p > 0)[:, 0].tolist()
    ours = D.kept_ids(c.logits, c.temperature, c.top_k or None, c.top_p if c.top_p < 1.0 else None, c.banned)
    if c.top_p < 1.0 and kept != ours:
        # a cut inside a tie group: HF's unstable sort drops some members of the group, the kernel (and the
        # reference) drop them in id order; the same number of the same scores goes either way
        assert len(kept) == len(ours) and sorted(c.logits[kept].tolist()) == sorted(c.logits[ours].tolist())
        p = torch.zeros_like(p)
        p[ours] = 1.0 / len(ours)
        kept = ours
    assert bool((p[kept] == 1.0 / len(kept)).all()) or len(kept) & (len(kept) - 1)
    cdf = p.cumsum(-1)
    want = int(torch.nonzero(cdf > c.u)[0]) if bool((cdf > c.u).any()) else kept[-1]
    assert c.want == want, (c.want, want)


def test_signed_zero_rows_match_hf_examples():
    """The two cases of the issue against torch.argmax / TopKLogitsWarper, and -0.0 kept like +0.0 by top-p."""
    from transformers.generation.logits_process import TopKLogitsWarper, TopPLogitsWarper
    x = torch.tensor([-5.0, -0.0, 0.0, -3.0])
    assert int(torch.argmax(x)) == 1 and D.expected_token(x, False, 1.0, None, None, [], 0.5)[0] == 1
    y = torch.tensor([[5.0, 0.0, -0.0, -3.0]])
    kept = torch.isfinite(TopKLogitsWarper(2)(None, y.clone()))[0].tolist()
    assert kept == [True, True, True, False]
    assert D.kept_ids(y[0], 1.0, 2, None, []) == [0, 1, 2]
    z = torch.tensor([[0.0, -0.0, 0.0, -0.0]])
    assert torch.isfinite(TopPLogitsWarper(0.5)(None, z.clone()))[0].tolist() == [False, False, True, True]
    for c in D.signed_zero_cases(8):
        D.check_case(c)
    assert [c.want for c in D.signed_zero_cases(8)] == [0, 7, 5]


# ----------------------------------------------------------------------------------------------------- fp32 decode
def test_decode_split_onehot_margin_and_pairs():
    B, H, Tc = 5, 4, 130
    lens = torch.tensor([1, 63, 64, 65, 130])
    (q_hi, q_lo, k, v), (o_hi, o_lo) = A.decode_split_onehot(B, H, Tc, lens, A.modes_for(H), seed=3)
    assert A.is_bf16(q_hi) and A.is_bf16(q_lo) and A.is_bf16(o_hi) and A.is_bf16(o_lo)
    assert float((q_lo != 0).float().sum()) > 0
    # the expected output is V[target] exactly as a pair, and V / K are not bf16 values (an fp32 cache is needed)
    tgt = torch.stack([lens - 1 if m == "latest" else torch.zeros_like(lens) for m in A.modes_for(H)], 1)
    o = v[torch.arange(B)[:, None], torch.arange(H)[None, :], tgt]
    assert torch.equal(o_hi + o_lo, o)
    assert float((A.bf16(v) != v).float().mean()) > 0.2 and float((A.bf16(k[..., 8:16]) != k[..., 8:16]).float().mean()) > 0.5


def test_decode_split_uniform_exact():
    B, H, Tc = 3, 2, 2048
    lens = torch.tensor([1, 1000, 2048])
    (k, v), (o_hi, o_lo) = A.decode_split_uniform(B, H, Tc, lens, seed=4)
    for b in range(B):
        n = int(lens[b])
        s = v[b, :, :n].double().sum(1)
        want = (s.float() * (torch.ones(()) / torch.tensor(float(n)))).double()
        assert torch.equal((o_hi[b] + o_lo[b]).double(), A.bf16(want) + A.bf16(want - A.bf16(want)))
        assert float(((o_hi[b].double() + o_lo[b].double()) - s / n).abs().max()) <= 2.0 ** -16 * float(s.abs().max() / n + 1)


def test_decode_f32_bound_separates_a_dropped_q_lo():
    """The random-mode bound admits fp32 arithmetic in another order and rejects the result of dropping q_lo."""
    g = torch.Generator().manual_seed(5)
    B, H, Tc = 2, 3, 200
    lens = torch.tensor([130, 200])
    x = torch.randn(B, H, 64, generator=g) * 2
    q_hi = A.bf16(x)
    q_lo = A.bf16(x - q_hi)
    k = torch.randn(B, H, Tc, 64, generator=g)
    v = torch.randn(B, H, Tc, 64, generator=g)
    q = q_hi + q_lo
    O, bo = A.decode_f32_reference(q, k, v, lens, 0.125)
    for b in range(B):
        n = int(lens[b])
        p = torch.softmax(torch.einsum("hd,hjd->hj", q[b], k[b, :, :n]) * 0.125, -1)
        o32 = torch.einsum("hj,hjd->hd", p, v[b, :, :n])
        hi = A.bf16(o32)
        assert bool(((hi.double() + A.bf16(o32 - hi).double() - O[b]).abs() <= bo[b]).all())
        p_hi = torch.softmax(torch.einsum("hd,hjd->hj", q_hi[b], k[b, :, :n]) * 0.125, -1)
        o_hi = torch.einsum("hj,hjd->hd", p_hi, v[b, :, :n]).double()
        assert bool(((o_hi - O[b]).abs() > bo[b]).any())
