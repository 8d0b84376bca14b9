"""The attention reference of tests/attn_ref.py, checked without a GPU: the exact-mode generators' arithmetic claims
hold in fp32 with the FMA emulated, a CPU model of a correct flash kernel passes every check, and each kind of kernel
defect the GPU suite is meant to catch is flagged at its location (exact modes) or breaks the random-mode bound."""
import math

import pytest
import torch

import attn_ref as A

SHAPES = [(2, 1, 2, 1), (2, 63, 4, 2), (2, 65, 2, 2), (2, 129, 4, 1), (2, 200, 6, 2)]


def _onehot(B, T, H, KVH, causal=True, seg=None, seed=0):
    lo, hi = A.bounds(B, T, causal, seg)
    modes = A.modes_for(H)
    tg = A.onehot_targets(lo, hi, modes)
    q, k = A.onehot_q(tg, modes), A.onehot_k(B, T, KVH)
    v = A.int_values((B, T, KVH, 64), 8, seed)
    return q, k, v, tg, lo, hi


PACKED = [[70, 1, 57, 1, 63, 9], [64, 64, 1, 61, 11]]       # length-1 documents, boundaries at 64, 65, 128, 129, ...


# --------------------------------------------------------------------------------------------------- generator claims
@pytest.mark.parametrize("B,T,H,KVH", SHAPES)
@pytest.mark.parametrize("causal", [True, False])
def test_onehot_claims(B, T, H, KVH, causal):
    q, k, v, tg, lo, hi = _onehot(B, T, H, KVH, causal)
    A.check_onehot_claims(q, k, tg, lo, hi, H // KVH)


def test_onehot_claims_packed_and_long_rows():
    seg = A.doc_starts(2, 201, PACKED)
    q, k, v, tg, lo, hi = _onehot(2, 201, 4, 2, True, seg)
    A.check_onehot_claims(q, k, tg, lo, hi, 2)
    # T = 8192: the partial sums stay below 2^27 and the margin holds for the rows that see the most keys
    T = 8192
    lo, hi = A.bounds(1, T, True)
    modes = A.modes_for(2)
    tg = A.onehot_targets(lo, hi, modes)
    rows = torch.tensor([0, 1, 4095, 4096, 8190, 8191])
    A.check_onehot_claims(A.onehot_q(tg, modes), A.onehot_k(1, T, 1), tg, lo, hi, 2, rows=rows)


@pytest.mark.parametrize("B,T,H,KVH", SHAPES)
def test_backward_expectations_match_fp64(B, T, H, KVH):
    """The constructive dQ / dK / dV equal the fp64 chain rule on the same inputs (o = 0, lse = 0), and are bf16 values
    (expect_onehot_bwd asserts the latter)."""
    q, k, _, tg, lo, hi = _onehot(B, T, H, KVH)
    v, do = A.onehot_bwd_inputs(tg, KVH, T, seed=3)
    dq, dk, dv = A.expect_onehot_bwd(q, k, v, do, tg, H // KVH)
    z = torch.zeros(B, T, H, 64)
    rq, rk, rv, *_ = A.bwd_reference(q, k, v, z, do, torch.zeros(B, T, H), lo, hi, 0.125, True)
    assert torch.equal(rq.float(), dq) and torch.equal(rk.float(), dk) and torch.equal(rv.float(), dv)
    dq0, dk0, dv0 = A.expect_onehot_bwd(q, k, v, do, tg, H // KVH, true_o=True)
    assert float(dq0.abs().max()) == 0 and float(dk0.abs().max()) == 0 and torch.equal(dv0, dv)


def test_split_and_decode_claims():
    modes = A.modes_for(4)
    (qh, ql, kh, kl, vh, vl), (oh, ol) = A.split_onehot(2, 130, 4, modes, seed=1)
    s = (torch.einsum("bthd,bjhd->bhtj", qh.double(), kh.double()) + torch.einsum("bthd,bjhd->bhtj", qh.double(), kl.double())
         + torch.einsum("bthd,bjhd->bhtj", ql.double(), kh.double()))
    full = torch.einsum("bthd,bjhd->bhtj", (qh + ql).double(), (kh + kl).double())
    assert torch.equal(s, full)                                          # the kernel's three products are the whole score
    assert torch.equal((oh + ol).double(), (A.expect_onehot_fwd(vh + vl, A.onehot_targets(*A.bounds(2, 130, False), modes), 1)[0]).double())
    lens = torch.tensor([1, 63, 64, 65, 128, 129, 8192, 0])
    A.decode_onehot(8, 16, 1, 8192, lens, A.modes_for(16), seed=2)     # asserts the margin on emulated fp32 scores


# --------------------------------------------------------------------------------------------------- clean model passes
@pytest.mark.parametrize("layout", ["causal", "bidirectional", "packed"])
def test_clean_model_is_exact(layout):
    B, T, H, KVH = 2, 201, 4, 2
    seg = A.doc_starts(B, T, PACKED) if layout == "packed" else None
    causal = layout != "bidirectional"
    q, k, v, tg, lo, hi = _onehot(B, T, H, KVH, causal, seg)
    o, lse = A.flash_emulate(q, k, v, lo, hi, 0.125)
    want_o, want_l = A.expect_onehot_fwd(v, tg, H // KVH)
    assert A.mismatch_exact(o, want_o) is None and A.mismatch_lse_exact(lse, want_l) is None
    vu = A.int_values((B, T, KVH, 64), 64, 5)
    o, lse = A.flash_emulate(torch.zeros_like(q), k, vu, lo, hi, 0.125)
    want_o, want_l = A.expect_uniform_fwd(vu, lo, hi, H // KVH)
    assert A.mismatch_exact(o, want_o) is None
    assert A.mismatch_lse_exact(lse, want_l) is None


@pytest.mark.parametrize("kind", ["rising", "wide", "scale0.1", "midtile"])
def test_clean_model_meets_random_bounds(kind):
    B, T, H, KVH = 2, 300, 4, 2
    scale, seg = 0.125, None
    q, k, v = (A.rising_inputs if kind == "rising" else A.wide_inputs)(B, T, H, KVH, seed=7)
    if kind == "scale0.1":
        scale = 0.1
    if kind == "midtile":
        seg = A.doc_starts(B, T, [[37, 100, 163], [129, 171]])
    lo, hi = A.bounds(B, T, True, seg)
    o, lse = A.flash_emulate(q, k, v, lo, hi, scale)
    O, L, bo, bl = A.fwd_reference(q, k, v, lo, hi, scale, True)
    assert A.mismatch_bound(o, O, bo) is None
    assert A.mismatch_bound(lse, L, bl, "lse") is None
    # backward: an fp32 model with bf16 P and dS, from the model's own o and lse
    do = A.bf16(torch.randn(B, T, H, 64, generator=torch.Generator().manual_seed(8)))
    dq, dk, dv = _bwd_model(q, k, v, o, do, lse, lo, hi, scale)
    rq, rk, rv, bq, bk, bv = A.bwd_reference(q, k, v, o, do, lse, lo, hi, scale, True)
    for name, got, want, bd in (("dq", dq, rq, bq), ("dk", dk, rk, bk), ("dv", dv, rv, bv)):
        assert A.mismatch_bound(got, want, bd, name) is None
    # ... and the bounds are far from vacuous: a 1 % scale error in the backward breaks them
    dq1, dk1, _ = _bwd_model(q, k, v, o, do, lse, lo, hi, scale * 1.01)
    assert A.mismatch_bound(dq1, rq, bq, "dq") is not None and A.mismatch_bound(dk1, rk, bk, "dk") is not None


def _bwd_model(q, k, v, o, do, lse, lo, hi, scale):
    """fp32 backward with P = bf16(exp(s scale - lse)) and dS = bf16(P (dP - delta) scale): what a flash backward does."""
    B, T, H, _ = q.shape
    G = H // k.shape[2]
    kk, vv = k.repeat_interleave(G, 2), v.repeat_interleave(G, 2)
    s = torch.einsum("bthd,bjhd->bhtj", q, kk)
    j = torch.arange(T)
    ok = (j >= lo[:, None, :, None]) & (j <= hi[:, None, :, None])
    p = torch.exp(s * scale - lse.float().permute(0, 2, 1)[..., None]).masked_fill(~ok, 0)
    dp = torch.einsum("bthd,bjhd->bhtj", do, vv)
    delta = (do * o).sum(-1).permute(0, 2, 1)[..., None]
    ds = A.bf16(p * (dp - delta) * scale)
    dq = A.bf16(torch.einsum("bhtj,bjhd->bthd", ds, kk))
    dk = A.bf16(torch.einsum("bhtj,bthd->bjhd", ds, q).reshape(B, T, H // G, G, 64).sum(3))
    dv = A.bf16(torch.einsum("bhtj,bthd->bjhd", A.bf16(p), do).reshape(B, T, H // G, G, 64).sum(3))
    return dq, dk, dv


# --------------------------------------------------------------------------------------------------- defects flagged
def _flag(defect, **kw):
    """Run the model with one defect on the exact modes; -> (mismatch of O, mismatch of lse, the expectations)."""
    B, T, H, KVH = 2, 201, 4, 2
    seg = A.doc_starts(B, T, PACKED)
    q, k, v, tg, lo, hi = _onehot(B, T, H, KVH, True, seg)
    o, lse = A.flash_emulate(q, k, v, lo, hi, 0.125, **kw)
    want_o, want_l = A.expect_onehot_fwd(v, tg, H // KVH)
    mo, ml = A.mismatch_exact(o, want_o, defect), A.mismatch_lse_exact(lse, want_l, defect)
    vu = A.int_values((B, T, KVH, 64), 64, 5)
    ou, lu = A.flash_emulate(torch.zeros_like(q), k, vu, lo, hi, 0.125, **kw)
    wu_o, wu_l = A.expect_uniform_fwd(vu, lo, hi, H // KVH)
    return mo, ml, A.mismatch_exact(ou, wu_o, defect), A.mismatch_lse_exact(lu, wu_l, defect), seg


def test_causal_mask_includes_next_key():
    mo, ml, mu, mlu, _ = _flag("key > row -> key > row + 1", causal_shift=1)
    assert mo is not None and 0 in mo.rows and 0 in mo.heads and 2 in mo.heads and 1 not in mo.heads, mo
    assert mlu is not None and mlu.count >= 2 * 4 * 190, mlu                 # every row but the last of each row


def test_causal_mask_drops_diagonal():
    mo, _, mu, mlu, _ = _flag("key > row -> key >= row", causal_shift=-1)
    assert mo is not None and mo.locs[0][:3] == (0, 0, 0) and {0, 2} <= set(mo.heads), mo   # the latest heads first
    assert mlu is not None and mlu.locs[0][:2] == (0, 0), mlu                # uniform lse: row 0 sees no key at all


def test_document_start_off_by_one():
    mo, _, _, mlu, seg = _flag("document start - 1", lo_shift=-1)
    second = min(s for row in seg.tolist() for s in row if s > 0)         # the earliest start of a second document
    assert mo is not None and set(mo.heads) == {1, 3}, mo                    # the earliest heads
    assert min(mo.rows) == second, (mo, second)
    mo, _, _, mlu, _ = _flag("document start + 1", lo_shift=1)
    assert mo is not None and {1, 3} <= set(mo.heads) and min(mo.rows) == 0, mo   # (latest heads: length-1 documents)
    assert mlu is not None and min(mlu.rows) == 0, mlu


def test_ragged_last_tile_dropped():
    mo, ml, mu, mlu, _ = _flag("last key tile skipped", drop_last_tile=True)
    assert mo is not None and min(mo.rows) == 192 and {r // 64 for r in mo.rows} == {3}, mo
    assert mlu is not None and min(mlu.rows) == 192


def test_wrong_kv_head_for_one_q_head():
    mo, _, mu, _, _ = _flag("q head 1 reads kv head 1", wrong_kv_head=1)
    assert mo is not None and mo.heads == [1], mo
    assert mu is not None and mu.heads == [1], mu


def test_missing_rescale_on_one_tile():
    B, T, H, KVH = 2, 200, 4, 2
    q, k, v, tg, lo, hi = _onehot(B, T, H, KVH)
    o, _ = A.flash_emulate(q, k, v, lo, hi, 0.125, no_corr_tile=1)
    mo = A.mismatch_exact(o, A.expect_onehot_fwd(v, tg, 2)[0], "tile 1 not rescaled")
    assert mo is not None and min(mo.rows) >= 64 and set(mo.heads) == {0, 2}, mo   # latest rows past key tile 1


def test_scale_off_by_one_percent():
    B, T, H, KVH = 2, 200, 4, 2
    q, k, v, tg, lo, hi = _onehot(B, T, H, KVH)
    vu = A.int_values((B, T, KVH, 64), 64, 5)
    # the exact modes are insensitive to the scale by design (p is 1 or 0); the uniform mode is too. Random data is not:
    qr, kr, vr = A.wide_inputs(B, T, H, KVH, seed=4)
    O, L, bo, bl = A.fwd_reference(qr, kr, vr, lo, hi, 0.125, True)
    o, lse = A.flash_emulate(qr, kr, vr, lo, hi, 0.125, scale_mult=1.01)
    mo, ml = A.mismatch_bound(o, O, bo), A.mismatch_bound(lse, L, bl, "lse")
    assert mo is not None and ml is not None and ml.count > B * T * H // 2, (mo, ml)
    del q, k, v, tg, vu


def test_warp_rows_shifted():
    mo, _, mu, _, _ = _flag("rows of warp slice 1 shifted", shift_warp=1)
    assert mo is not None and min(mo.rows) == 17 and max(mo.rows) <= 31, mo
    assert all((r % 64) // 16 == 1 for r in mo.rows)


def test_one_ulp_on_one_element():
    B, T, H, KVH = 2, 200, 4, 2
    q, k, v, tg, lo, hi = _onehot(B, T, H, KVH)
    want = A.expect_onehot_fwd(v, tg, 2)[0]
    got = want.clone()
    x = got[1, 150, 3, 17]
    got[1, 150, 3, 17] = x + (A.ulp_bf16(x.reshape(1)).float()[0] if x != 0 else 2.0 ** -133)
    mo = A.mismatch_exact(got, want, "one ulp")
    assert mo is not None and mo.count == 1 and mo.locs == [(1, 150, 3, 17)], mo
    assert "(1, 3, 150, 17, 2, 1)" in str(mo), mo                          # batch, head, row, col, tile64, warp16


def test_lse_off_by_1e_4():
    B, T, H = 2, 200, 4
    lo, hi = A.bounds(B, T, True)
    want = torch.log((hi - lo + 1).double())[..., None].expand(B, T, H)
    got = want.float().clone()
    got[0, 99, 2] += 1e-4
    ml = A.mismatch_lse_exact(got, want)
    assert ml is not None and ml.count == 1 and ml.locs == [(0, 99, 2)], ml


@pytest.mark.parametrize("kind", ["rising", "wide"])
def test_random_bounds_catch_online_softmax_defects(kind):
    """On adversarial data, a missing rescale on one tile or a 1 % scale error breaks the random-mode contract."""
    B, T, H, KVH = 2, 300, 4, 2
    q, k, v = (A.rising_inputs if kind == "rising" else A.wide_inputs)(B, T, H, KVH, seed=11)
    lo, hi = A.bounds(B, T, True)
    O, L, bo, bl = A.fwd_reference(q, k, v, lo, hi, 0.125, True)
    for kw in (dict(no_corr_tile=2), dict(scale_mult=1.01)):
        o, lse = A.flash_emulate(q, k, v, lo, hi, 0.125, **kw)
        m = A.mismatch_bound(o, O, bo, str(kw))
        assert m is not None and min(m.rows) >= (128 if "no_corr_tile" in kw else 0), (kw, m)
    # and the bound is tight enough to matter: well below the typical size of O
    assert float(bo.median()) < 0.02 * float(O.abs().median())
