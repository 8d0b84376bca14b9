"""The GEMM checker of tests/gemm_ref.py on the CPU: a "kernel output" computed here is passed clean and with the
defects a broken schedule produces (one element off by one ulp, a stale quadrant, a missing k-block, a rounding point
moved); the checker must pass the clean output and flag every defect at the right place."""
import torch

import gemm_ref as R

M, N, K, BN = 256, 512, 320, 256
BIAS_SCALE = R.acc_scale(K, 8)


def _case(seed=0):
    a, b = R.int_operand(M, K, 8, seed), R.int_operand(N, K, 8, seed + 1)
    bias = R.real_operand((N,), BIAS_SCALE, seed + 2)
    res = R.real_operand((M, N), BIAS_SCALE, seed + 3)
    return a, b, bias, res


def _out(a, b, bias, res, round_before_res=True):
    return R.epilogue(R.exact_acc(a, b), bias, res, round_before_res).to(torch.bfloat16)


def test_operands_exercise_bf16_rounding():
    a, b, bias, res = _case()
    acc = R.exact_acc(a, b)
    assert float((acc.abs() > 256).double().mean()) > 0.5          # outputs are not all exact in bf16
    v = R.epilogue(acc, bias, res, round_before_res=True, out_f32=True)
    w = R.epilogue(acc, bias, res, round_before_res=False, out_f32=True)
    assert float((R.bf16_round(v) != R.bf16_round(w)).double().mean()) > 0.05   # the rounding point matters


def test_clean_output_passes():
    a, b, bias, res = _case()
    want = R.epilogue(R.exact_acc(a, b), bias, res, round_before_res=True)
    assert R.mismatch_exact(_out(a, b, bias, res), want, BN) is None


def test_one_ulp_off_is_flagged():
    a, b, bias, res = _case()
    want = R.epilogue(R.exact_acc(a, b), bias, res, round_before_res=True)
    out = _out(a, b, bias, res)
    out.view(torch.int16)[200, 300] += 1
    rep = R.mismatch_exact(out, want, BN)
    assert rep is not None and "1 of" in rep and "(200, 300, 1, 1, 0, 2)" in rep, rep


def test_stale_quadrant_is_flagged():
    a, b, bias, res = _case()
    want = R.epilogue(R.exact_acc(a, b), bias, res, round_before_res=True)
    out = _out(a, b, bias, res)
    a2, b2, _, _ = _case(seed=10)                    # a previous launch's different inputs
    stale = _out(a2, b2, bias, res)
    r0, c0 = 1 * 128 + 3 * 32, 0 * BN + 2 * 64      # tile (1, 0), quadrant 3, chunk 2
    out[r0:r0 + 32, c0:c0 + 64] = stale[r0:r0 + 32, c0:c0 + 64]
    rep = R.mismatch_exact(out, want, BN)
    assert rep is not None, "stale quadrant not flagged"
    assert f"flagged rows [{r0}, {r0 + 31}]" in rep and f"columns [{c0}, {c0 + 63}]" in rep, rep


def test_missing_last_kblock_is_flagged():
    a, b, bias, res = _case()
    want = R.epilogue(R.exact_acc(a, b), bias, res, round_before_res=True)
    out = _out(a, b, bias, res)
    last = (K - 1) // R.BK * R.BK
    r0, c0 = 128, 256                                 # tile (1, 1)
    part = R.exact_acc(a[r0:r0 + 128, :last], b[c0:c0 + BN, :last])
    out[r0:r0 + 128, c0:c0 + BN] = R.epilogue(part, bias[c0:c0 + BN], res[r0:r0 + 128, c0:c0 + BN], True).to(torch.bfloat16)
    rep = R.mismatch_exact(out, want, BN)
    assert rep is not None and "flagged rows [128, 255], columns [256, 511]" in rep, rep


def test_rounding_point_is_flagged():
    a, b, bias, res = _case()
    want = R.epilogue(R.exact_acc(a, b), bias, res, round_before_res=True)
    assert R.mismatch_exact(_out(a, b, bias, res, round_before_res=False), want, BN) is not None
    # and rounding the accumulator before the bias add (a misplaced rounding point in the other direction)
    acc = R.exact_acc(a, b)
    early = R.epilogue(R.bf16_round(acc.float()), bias, res, round_before_res=True).to(torch.bfloat16)
    assert R.mismatch_exact(early, want, BN) is not None


def test_fp32_output_is_checked_bitwise():
    a, b, bias, res = _case()
    want = R.epilogue(R.exact_acc(a, b), bias, res, round_before_res=False, out_f32=True)
    out = want.clone()
    assert R.mismatch_exact(out, want, BN) is None
    out[5, 7] = torch.nextafter(out[5, 7], torch.tensor(float("inf")))
    assert R.mismatch_exact(out, want, BN) is not None


def test_nan_is_never_equal():
    a, b, bias, res = _case()
    want = R.epilogue(R.exact_acc(a, b), bias, res, round_before_res=True)
    out = want.to(torch.bfloat16)
    out[0, 0] = float("nan")
    assert R.mismatch_exact(out, want, BN) is not None
    assert R.mismatch_bound(out, want, torch.full(want.shape, 1e30, dtype=torch.float64), BN) is not None


def test_random_mode_bound():
    g = torch.Generator().manual_seed(3)
    a = torch.randn(256, 896, generator=g).to(torch.bfloat16)
    b = torch.randn(320, 896, generator=g).to(torch.bfloat16)
    out = (a.float() @ b.float().t()).to(torch.bfloat16)            # an fp32-accumulated, bf16-rounded result
    assert R.mismatch_random(out, a, b, BN) is None
    for dr, dc, d in ((17, 33, 2), (255, 319, -2)):                # two bf16 ulps off is outside the bound
        bad = out.clone()
        bad.view(torch.int16)[dr, dc] += d
        rep = R.mismatch_random(bad, a, b, BN)
        assert rep is not None and f"({dr}, {dc}," in rep, rep


def test_gelu_bound():
    v = torch.linspace(-12, 12, 4801, dtype=torch.float32).reshape(1, -1)
    g = R.gelu_exact(v)
    assert R.mismatch_gelu(g.float().to(torch.bfloat16), v) is None
    tanh_gelu = torch.nn.functional.gelu(v, approximate="tanh").to(torch.bfloat16)   # a different GELU is flagged
    assert R.mismatch_gelu(tanh_gelu, v) is not None


def test_ulp_and_rounding_helpers():
    x = torch.tensor([1.0, 1.5, 256.0, 300.0, -1000.0, 0.0])
    assert R.ulp_bf16(x).tolist()[:5] == [2.0 ** -7, 2.0 ** -7, 2.0, 2.0, 4.0]
    assert float(R.ulp_bf16(x)[5]) == 2.0 ** -133
    assert R.bf16_round(torch.tensor([257.0, 259.0, 261.0])).tolist() == [256.0, 260.0, 260.0]   # ties to even


def test_rope_emulation_matches_rotation():
    """At exactly representable values the RoPE emulation is the plain rotate_half formula."""
    M_, cols = 4, 128
    acc = torch.arange(M_ * cols, dtype=torch.float64).reshape(M_, cols) % 7 - 3
    cos = torch.tensor([[1.0] * 32, [0.0] * 32, [0.5] * 32]).to(torch.bfloat16)
    sin = torch.tensor([[0.0] * 32, [1.0] * 32, [0.5] * 32]).to(torch.bfloat16)
    pos = torch.tensor([0, 1, 2, 99])                                # 99 is clamped to the last row
    out = R.rope_epilogue(acc, None, cos, sin, pos, rope_cols=64)
    x1, x2 = acc[:, :32].float(), acc[:, 32:64].float()
    c, s = cos.float()[pos.clamp(max=2)], sin.float()[pos.clamp(max=2)]
    assert torch.equal(out[:, :32], x1 * c - x2 * s) and torch.equal(out[:, 32:64], x2 * c + x1 * s)
    assert torch.equal(out[:, 64:], acc[:, 64:].float())


def test_streamk_contributor_count():
    plan = {"sk_units": 7, "sk_groups": 28, "splits": 1, "bn": 256}
    assert R.streamk_contributors(plan, 2056) == [3] * 7 and R.schedule_kind(plan, 2056) == "streamk2"
    plan = {"sk_units": 11, "sk_groups": 22, "splits": 1, "bn": 256}
    assert R.schedule_kind(plan, 2056) == "streamk1"
    assert R.schedule_kind({"sk_units": 0, "sk_groups": 0, "splits": 7, "bn": 128}, 2112) == "splitk"
    assert R.schedule_kind({"sk_units": 0, "sk_groups": 0, "splits": 1, "bn": 64}, 200) == "plain64"
