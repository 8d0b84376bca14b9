"""Conformance of the 192- and 224-column tiles of the wgmma GEMM, with the exact references of tests/gemm_ref.py.

A 224-wide tile is 3.5 chunks of 64 columns; its last 32 columns leave through a 32-column TMA box.  Covered: every
operand major x every plain epilogue at both widths and with the default column-unit stream-K, RoPE at 192 (three
whole heads per tile), and guard bands that show no tile writes outside [:M, :N] or into its neighbour.
"""
import pytest
import torch

import gemm_ref as R
from test_gpu_gemm_conformance import (DEV, EPILOGUES, MAJOR_IDS, MAJORS, SENT16, AMAX, _data, _layout, _pitched,
                                       run_case)

pytestmark = pytest.mark.gpu

# kind -> ((M, N, K, force_bn, scratch), schedule kinds accepted).  N is not a multiple of the width, so the last
# tile column is partial and the full ones sit next to each other.
WIDTHS = {
    "plain224": ((328, 3 * 224 + 40, 200, 224, False), ("plain224",)),
    "plain192": ((328, 3 * 192 + 40, 200, 192, False), ("plain192",)),
    # 7 x 19 tiles of 256 chosen by the planner: column units, the last wave and the leftover unit end to end
    "colunits": ((896, 4864, 2056, 0, True), ("streamk1",)),
}


@pytest.mark.parametrize("epi", EPILOGUES)
@pytest.mark.parametrize("major", MAJORS, ids=MAJOR_IDS)
@pytest.mark.parametrize("kind", list(WIDTHS))
def test_width_matrix(kind, major, epi):
    shape, expect = WIDTHS[kind]
    plan = run_case(kind, major, epi, shape=shape, expect=expect)
    if kind == "colunits":
        assert plan["sk_colunits"] == 1 and plan["bn"] == 256, plan
    else:
        assert plan["bn"] == shape[3], plan


def test_rope_192():
    """QKV projection + bias + RoPE at a size where the planner takes 192-wide tiles (N = 1152 = 6 x 192)."""
    from slamkit_b200 import ops
    from slamkit_b200.lm import rope_tables
    M, N, K, maxpos, rope_cols = 2000, 1152, 896, 2048, 1024
    x, w = R.int_operand(M, K, AMAX, 1, DEV), R.int_operand(N, K, AMAX, 2, DEV)
    bias = R.real_operand((N,), R.acc_scale(K, AMAX), 3, DEV)
    assert ops.gemm_plan(x, w, bias=bias)["bn"] == 192        # the RoPE launch plans the same width (whole heads)
    cos, sin = (t.to(DEV) for t in rope_tables(10000.0, 64, maxpos))
    pos = torch.randint(0, maxpos + 40, (M,), generator=torch.Generator().manual_seed(0)).to(torch.int32).to(DEV)
    out = ops.linear_rope(x, w, bias, cos, sin, 1, rope_cols, pos_ids=pos)
    rep = R.mismatch_exact(out, R.rope_epilogue(R.exact_acc(x, w), bias, cos, sin, pos, rope_cols), 192, "qkv+rope 192")
    assert rep is None, rep


@pytest.mark.parametrize("out_f32", [False, True], ids=["bf16", "f32"])
@pytest.mark.parametrize("major", MAJORS, ids=MAJOR_IDS)
@pytest.mark.parametrize("kind", ["plain224", "plain192", "colunits"])
def test_guard_bands_and_pitches(kind, major, out_f32):
    """A, B and the residual at pitches wider than their rows with NaN padding; C inside a sentinel-filled buffer:
    exact result, and no element outside [:M, :N] changes (the tail chunk's 32-column box included)."""
    from slamkit_b200 import ops
    (M, N, K, bn, ws), expect = WIDTHS[kind]
    a, b, bias, res, acc = _data(M, N, K)
    a_mn, b_mn = major
    ad = _pitched(_layout(a, a_mn), 24, 64)
    bd = _pitched(_layout(b, b_mn), 40, 64)
    odt = torch.float32 if out_f32 else torch.bfloat16
    sent = float("nan") if out_f32 else torch.tensor([SENT16], dtype=torch.int16).view(torch.bfloat16).item()
    big = torch.full((M + 24, N + 64), sent, dtype=odt, device=DEV)
    before = big.clone()
    out = big[16:16 + M, 8:8 + N]
    rp = _pitched(res, 8, 8)
    kw = dict(a_mn=a_mn, b_mn=b_mn, force_bn=bn, streamk=ws, out=out, out_f32=out_f32, bias=bias, residual=rp,
              round_before_res=True)
    plan = ops.gemm_plan(ad, bd, **kw)
    assert R.schedule_kind(plan, K) in expect and plan["tma_store"] == (0 if out_f32 else 1), plan
    ops.gemm(ad, bd, **kw)
    rep = R.mismatch_exact(out, R.epilogue(acc, bias, res, round_before_res=True, out_f32=out_f32), plan["bn"],
                           f"{kind} pitched")
    assert rep is None, rep
    bits = (lambda t: t.view(torch.int32)) if out_f32 else (lambda t: t.view(torch.int16))
    changed = bits(big) != bits(before)
    changed[16:16 + M, 8:8 + N] = False
    assert not bool(changed.any()), f"{int(changed.sum())} elements outside [:M, :N] were written"


@pytest.mark.parametrize("N,fit", [(896, 224), (1152, 192)])
def test_batch_invariance_across_widths(N, fit):
    """Rows of gemm(A[:m], B) equal the rows of gemm(A, B) bit for bit while the planner moves between 128 and the
    fitted width (the forward GEMMs take no scratch and keep their K order at every width)."""
    from slamkit_b200 import ops
    g = torch.Generator(device=DEV).manual_seed(N)
    A = torch.randn(8192, 896, generator=g, device=DEV).to(torch.bfloat16)
    B = torch.randn(N, 896, generator=g, device=DEV).to(torch.bfloat16)
    full = ops.gemm(A, B)
    assert ops.gemm_plan(A, B)["bn"] == fit
    bns = set()
    for m in (1, 65, 129, 1000, 2048, 3000, 4224, 6000, 8191):
        bns.add(ops.gemm_plan(A[:m], B)["bn"])
        rep = R.mismatch_exact(ops.gemm(A[:m], B), full[:m], fit, f"rows of a batch of {m} vs 8192")
        assert rep is None, rep
    assert {128, fit} <= bns, bns


@pytest.mark.parametrize("M,N,K", [(896, 4864, 2056), (896, 4864, 8192)])
@pytest.mark.parametrize("major", MAJORS, ids=MAJOR_IDS)
def test_colunits_bit_identical_to_whole_tiles(M, N, K, major):
    """Column-unit stream-K carries the first range's fp32 accumulator into the second range, so on real-valued data
    (where any re-association would show) the output equals the whole-tile launch bit for bit."""
    from slamkit_b200 import ops
    g = torch.Generator(device=DEV).manual_seed(K)
    a = torch.randn(M, K, generator=g, device=DEV).to(torch.bfloat16)
    b = torch.randn(N, K, generator=g, device=DEV).to(torch.bfloat16)
    ad, bd = _layout(a, major[0]), _layout(b, major[1])
    kw = dict(a_mn=major[0], b_mn=major[1])
    plan = ops.gemm_plan(ad, bd, streamk=True, **kw)
    assert plan["sk_colunits"] == 1 and plan["sk_units"] > 0, plan
    assert ops.gemm_plan(ad, bd, **kw)["bn"] == plan["bn"]
    whole = ops.gemm(ad, bd, **kw)
    for _ in range(2):
        assert torch.equal(ops.gemm(ad, bd, streamk=True, **kw), whole)
    assert int(ops.gemm_workspace(DEV)[-4096:].max()) == 0, "stream-K flag words not re-armed"
