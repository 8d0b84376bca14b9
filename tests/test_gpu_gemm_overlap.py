"""The register epilogue of the one-pass TMA-store schedule (plain convert and SwiGLU forward) with several tiles per CTA.

On that schedule the producer loads the next tile's k-blocks while the consumer warps still convert and store the
previous tile from their registers, and a staging box is rewritten while older stores may still be in flight.  The
exact one-pass cases of test_gpu_gemm_conformance.py run about one tile per CTA; here every case runs at least three,
with integer operands (exact fp32 accumulator, bit-for-bit comparison) and ragged M / N.
"""
import pytest
import torch

import gemm_ref as R

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
MAJORS = [(False, False), (False, True), (True, False), (True, True)]
MAJOR_IDS = ["KK", "KM", "MK", "MM"]
WIDTHS = [64, 128, 192, 224, 256]
M, K = 8264, 200       # 65 tile rows; ragged M and K
SENT16 = 0x7F81        # a NaN pattern no GEMM output takes


def _ints(rows, cols, seed, amax=8):
    return R.int_operand(rows, cols, amax, seed, DEV)


def _layout(t, mn):
    return t.t().contiguous() if mn else t


def _one_pass(plan, bn):
    assert plan["bn"] == bn and plan["splits"] == 1 and plan["sk_units"] == 0 and plan["tma_store"] == 1, plan


@pytest.mark.parametrize("major", MAJORS, ids=MAJOR_IDS)
@pytest.mark.parametrize("bn", WIDTHS)
def test_plain_convert_many_tiles(bn, major):
    from slamkit_b200 import ops
    N = 1544                                   # ragged: a partial last tile column at every width
    a, b = _ints(M, K, 1), _ints(N, K, 2)
    a_mn, b_mn = major
    ad, bd = _layout(a, a_mn), _layout(b, b_mn)
    kw = dict(a_mn=a_mn, b_mn=b_mn, force_bn=bn)
    plan = ops.gemm_plan(ad, bd, **kw)
    _one_pass(plan, bn)
    tiles = -(-M // 128) * -(-N // bn)
    assert tiles >= 3 * plan["grid"], (tiles, plan)
    out = ops.gemm(ad, bd, **kw)
    rep = R.mismatch_exact(out, R.epilogue(R.exact_acc(a, b)), bn, f"plain bn={bn} a_mn={a_mn} b_mn={b_mn}")
    assert rep is None, rep


@pytest.mark.parametrize("bn", [128, 224, 256])
def test_output_inside_sentinel_buffer(bn):
    """C is a window of a larger sentinel-filled buffer: exact inside, no byte changed outside (the 16-row store boxes
    and the 224-wide tile's 32-column tail box stay inside [:M, :N])."""
    from slamkit_b200 import ops
    N = 1544
    a, b = _ints(M, K, 3), _ints(N, K, 4)
    sent = torch.tensor([SENT16], dtype=torch.int16).view(torch.bfloat16).item()
    big = torch.full((M + 40, N + 72), sent, dtype=torch.bfloat16, device=DEV)
    before = big.clone()
    out = big[24:24 + M, 8:8 + N]
    plan = ops.gemm_plan(a, b, force_bn=bn, out=out)
    _one_pass(plan, bn)
    ops.gemm(a, b, force_bn=bn, out=out)
    rep = R.mismatch_exact(out, R.epilogue(R.exact_acc(a, b)), bn, f"windowed bn={bn}")
    assert rep is None, rep
    changed = big.view(torch.int16) != before.view(torch.int16)
    changed[24:24 + M, 8:8 + N] = False
    assert not bool(changed.any()), f"{int(changed.sum())} elements outside the output were written"


@pytest.mark.parametrize("Mr", [8192, 8264])
def test_swiglu_forward_many_tiles(Mr):
    """gate/up projection with SwiGLU in the epilogue at the LM shape (F = 4864: 19 tile columns, >= 9 tiles per CTA):
    gu exact, act bit-equal to the unfused kernel."""
    from slamkit_b200 import ops
    F, Kx = 4864, 896
    h, wg, wu = _ints(Mr, Kx, 7), _ints(F, Kx, 8), _ints(F, Kx, 9)
    gu_b, act = ops.linear_swiglu_fwd(h, ops.block_gate_up(wg, wu))
    gu_want = R.epilogue(R.exact_acc(h, torch.cat([wg, wu], 0)))
    gu = torch.cat([v.reshape(Mr, F) for v in gu_b.view(Mr, F // 128, 2, 128).unbind(2)], 1)   # [gate | up]
    rep = R.mismatch_exact(gu, gu_want, 256, f"gate/up M={Mr}")
    assert rep is None, rep
    assert torch.equal(act, ops.swiglu_fwd(gu))


def test_back_to_back_dependent():
    """y1 = x W1^T and y2 = y1 W2^T launched back to back (the second reads what the first's last stores wrote);
    small integers keep both products exact."""
    from slamkit_b200 import ops
    x, w1 = _ints(M, 128, 10, 2), _ints(1536, 128, 11, 2)
    w2 = _ints(768, 1536, 12, 1)
    _one_pass(ops.gemm_plan(x, w1), 256)
    y1 = ops.gemm(x, w1)
    y2 = ops.gemm(y1, w2)
    want1 = R.epilogue(R.exact_acc(x, w1))
    rep = R.mismatch_exact(y1, want1, 256, "y1")
    assert rep is None, rep
    rep = R.mismatch_exact(y2, R.epilogue(R.exact_acc(want1.to(torch.bfloat16).to(DEV), w2)), 256, "y2")
    assert rep is None, rep
