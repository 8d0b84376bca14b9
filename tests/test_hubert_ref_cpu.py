"""The HuBERT references of tests/hubert_ref.py on the CPU: a clean emulation of each kernel passes its check, and the
defects a broken kernel or schedule produces (an extra or missing split product, a dropped lo output or lo residual, a
shifted or mis-batched conv window, a row or column written to the wrong place, staging garbage, the wrong variance,
statistics or rounding) are flagged."""
import math

import pytest
import torch

import gemm_ref as G
import hubert_ref as R

torch.set_num_threads(min(8, torch.get_num_threads()))


# ----------------------------------------------------------------------------------------------------- split GEMM
M, N, K = 300, 256, 512        # 3 tile rows (the last one ragged), 4 column groups of 64
LMAX = 64


def _split_case(seed=0, K_=K):
    a = R.split_amax(K_, LMAX)
    ah, al = R.split_int_operand(M, K_, a, LMAX, seed)
    bh, bl = R.split_int_operand(N, K_, a, LMAX, seed + 1)
    scale = G.acc_scale(K_, a)
    g = torch.Generator().manual_seed(seed + 2)
    bias = torch.randn(N, generator=g) * scale
    rh, rl = R.real_split((M, N), scale, seed + 3)
    return ah, al, bh, bl, bias, rh, rl


def _want(c):
    ah, al, bh, bl, bias, rh, rl = c
    return R.split_epilogue(R.split_exact_acc(ah, al, bh, bl), bias, rh, rl)


def _check(out, want, what="split"):
    return [R.mismatch_exact(o, w, M, 64, f"{what} {n}") for o, w, n in zip(out, want, ("hi", "lo"))]


def test_split_amplitudes_are_exact_and_exercise_rounding():
    for K_, a in ((512, 11), (768, 8), (3072, 4), (8192, 2)):
        assert R.split_amax(K_, LMAX) == a
    c = _split_case()
    acc = R.split_exact_acc(*c[:4])
    assert float((acc.abs() > 256).double().mean()) > 0.3               # hi alone does not hold the value
    hi, lo = _want(c)
    assert float((lo != 0).double().mean()) > 0.9                        # the lo output carries information
    with pytest.raises(AssertionError):
        ah, al, bh, bl = R.split_int_operand(4, 8192, 3, LMAX, 0) + R.split_int_operand(4, 8192, 3, LMAX, 1)
        R.split_exact_acc(ah, al, bh, bl)


def test_clean_split_emulation_passes():
    c = _split_case()
    ah, al, bh, bl, bias, rh, rl = c
    acc32 = torch.zeros(M, N, dtype=torch.float32)
    for k0 in range(0, K, R.BK):                     # k-block by k-block in fp32, as the kernel does
        s = slice(k0, k0 + R.BK)
        acc32 += (ah[:, s].double() @ bh[:, s].double().t() + ah[:, s].double() @ bl[:, s].double().t()
                  + al[:, s].double() @ bh[:, s].double().t()).float()
    out = R.split_epilogue(acc32.double(), bias, rh, rl)
    assert _check(out, _want(c)) == [None, None]
    f32 = R.split_epilogue(acc32.double(), bias, rh, rl, out_f32=True)
    assert R.mismatch_exact(f32, R.split_epilogue(R.split_exact_acc(ah, al, bh, bl), bias, rh, rl, out_f32=True), M) is None


def test_added_lo_lo_product_is_flagged():
    c = _split_case()
    ah, al, bh, bl, bias, rh, rl = c
    acc = R.split_exact_acc(ah, al, bh, bl) + al.double() @ bl.double().t()
    rep = _check(R.split_epilogue(acc, bias, rh, rl), _want(c))
    assert rep[0] is not None or rep[1] is not None
    f32 = R.split_epilogue(acc, bias, out_f32=True)
    assert R.mismatch_exact(f32, R.split_epilogue(R.split_exact_acc(ah, al, bh, bl), bias, out_f32=True), M) is not None


def test_missing_hi_lo_on_one_kblock_is_flagged():
    c = _split_case()
    ah, al, bh, bl, bias, rh, rl = c
    acc = R.split_exact_acc(ah, al, bh, bl)
    r0, c0, kb = 128, 64, 5                          # tile row 1, column group 1, k-block 5
    s = slice(kb * R.BK, (kb + 1) * R.BK)
    acc[r0:r0 + 128, c0:c0 + 64] -= ah[r0:r0 + 128, s].double() @ bl[c0:c0 + 64, s].double().t()
    rep = _check(R.split_epilogue(acc, bias, rh, rl), _want(c))
    msg = rep[0] or rep[1]
    assert msg is not None and "rows [128, 255]" in msg and "columns [64, 127]" in msg and "tile 1, group 1" in msg, msg


def test_lo_output_left_at_zero_is_flagged():
    c = _split_case()
    hi, lo = _want(c)
    rep = _check((hi, torch.zeros_like(lo)), (hi, lo))
    assert rep[0] is None and rep[1] is not None


def test_dropped_lo_residual_is_flagged():
    c = _split_case()
    ah, al, bh, bl, bias, rh, rl = c
    out = R.split_epilogue(R.split_exact_acc(ah, al, bh, bl), bias, rh, None)
    rep = _check(out, _want(c))
    assert rep[1] is not None


def test_split_random_bound():
    g = torch.Generator().manual_seed(4)
    x, w = torch.randn(200, 768, generator=g), torch.randn(320, 768, generator=g) / 28
    xh, xl = R.split_f32(x)
    wh, wl = R.split_f32(w)
    ref = R.hilo(xh, xl) @ R.hilo(wh, wl).t() - xl.double() @ wl.double().t()
    out = (xh.float() @ wh.float().t() + xh.float() @ wl.float().t() + xl.float() @ wh.float().t())
    hi, lo = R.split_f32(out)
    bound = R.split_random_bound(xh, xl, wh, wl, ref)
    assert R.mismatch_bound(R.hilo(hi, lo), ref, bound, 200) is None
    bad = R.hilo(hi, lo).clone()
    bad[17, 33] += 0.05                              # above the fp32 accumulation bound (about 5e-3 here)
    assert "(clip 0, frame 17" in (R.mismatch_bound(bad, ref, bound, 200) or "")
    assert R.mismatch_bound(hi.double(), ref, bound, 200) is not None   # the lo half is needed


# ----------------------------------------------------------------------------------------------------- conv layouts
def _conv_case(B=3, Mc=130, k=3, st=2, C=64, seed=0):
    T_in = (Mc - 1) * st + k
    a = R.split_amax(k * C, LMAX)
    ah, al = R.split_int_operand(B * T_in, C, a, LMAX, seed)
    wh, wl = R.split_int_operand(C, k * C, a, LMAX, seed + 1)
    return ah, al, wh, wl, B, Mc, k, st, C


def _conv_out(ah, al, wh, wl, B, Mc, k, st, C):
    A = R.window_rows(ah, B, Mc, k, st, C), R.window_rows(al, B, Mc, k, st, C)
    return R.split_epilogue(R.split_exact_acc(A[0], A[1], wh, wl))


def test_window_rows_is_the_strided_conv():
    ah, al, wh, wl, B, Mc, k, st, C = _conv_case(B=2, Mc=5, C=8)
    x = ah.double().reshape(B, -1, C).transpose(1, 2)                    # [B, C, T_in]
    w = wh.double().reshape(C, k, C).permute(0, 2, 1)                    # [co, ci, j]
    conv = torch.nn.functional.conv1d(x, w, stride=st).transpose(1, 2).reshape(B * Mc, C)
    assert torch.equal(R.window_rows(ah, B, Mc, k, st, C).double() @ wh.double().t(), conv)


def test_conv_window_defects_are_flagged():
    case = _conv_case()
    ah, al, wh, wl, B, Mc, k, st, C = case
    want = _conv_out(*case)
    # shifted by one frame: every window starts C elements late (and the last reads past the clip: zero)
    sh = lambda t: torch.cat([t.reshape(B, -1)[:, C:], torch.zeros(B, C, dtype=t.dtype)], 1)
    got = _conv_out(sh(ah), sh(al), wh, wl, B, Mc, k, st, C)
    assert R.mismatch_exact(got[0], want[0], Mc, 64) is not None
    # clip b reads clip b - 1 (batch stride off by one clip)
    prev = lambda t: torch.cat([t.reshape(B, -1)[:1], t.reshape(B, -1)[:-1]], 0)
    got = _conv_out(prev(ah), prev(al), wh, wl, B, Mc, k, st, C)
    rep = R.mismatch_exact(got[0], want[0], Mc, 64)
    assert rep is not None and "flagged clips [1, 2]" in rep, rep
    # a row of clip 1 written into clip 2 (the last row of a ragged tile)
    bad = want[0].clone()
    bad[2 * Mc + 129] = want[0][Mc + 129]
    rep = R.mismatch_exact(bad, want[0], Mc, 64)
    assert rep is not None and "(clip 2, frame 129, tile 1" in rep, rep


# ----------------------------------------------------------------------------------------------------- positional conv
def _pos_case(B=2, Tf=70, Kpos=16, groups=4, cg=48, seed=0):
    halo = Kpos // 2
    Kd = Kpos * R.GROUP_PAD
    a = R.split_amax(Kd, LMAX)
    xh, xl = R.split_int_operand(B * (Tf + 2 * halo), groups * R.GROUP_PAD, a, LMAX, seed)
    wh, wl = R.split_int_operand(groups * R.GROUP_PAD, Kd, a, LMAX, seed + 1)
    bias = torch.randn(groups * R.GROUP_PAD, generator=torch.Generator().manual_seed(seed + 2)) * 50
    sh = (B, Tf + 2 * halo, groups * R.GROUP_PAD)
    return xh.reshape(sh), xl.reshape(sh), wh, wl, bias, Tf, Kpos, groups, cg


def test_posconv_windows_are_the_grouped_conv():
    xh, xl, wh, wl, bias, Tf, Kpos, groups, cg = _pos_case(Tf=9, Kpos=4, groups=2, cg=64)
    x = xh.double().transpose(1, 2)                                       # [B, G*64, Tp]
    w = wh.double().reshape(groups * 64, Kpos, 64).permute(0, 2, 1)       # [co, ci, j]
    conv = torch.nn.functional.conv1d(x, w, groups=groups)[:, :, :Tf].transpose(1, 2).reshape(-1, groups * 64)
    acc = R.posconv_split_acc(xh, torch.zeros_like(xl), wh, torch.zeros_like(wl), Tf, Kpos, groups)
    assert torch.equal(acc, conv)


def test_posconv_compaction_defects_are_flagged():
    xh, xl, wh, wl, bias, Tf, Kpos, groups, cg = _pos_case()
    acc = R.posconv_split_acc(xh, xl, wh, wl, Tf, Kpos, groups)
    want = R.split_epilogue(acc, bias, col_gin=64, col_gout=cg)
    assert want[0].shape == (2 * Tf, groups * cg)
    # a compacted column in the neighbouring group: group 1's column 5 lands where group 2's column 5 goes
    bad = want[0].clone()
    bad[:, 2 * cg + 5] = want[0][:, 1 * cg + 5]
    rep = R.mismatch_exact(bad, want[0], Tf, cg)
    assert rep is not None and "group 2 | col 101" in rep, rep
    # bias read at the compacted column instead of the padded one
    comp_bias = torch.cat([bias, torch.zeros(64)])[:groups * 64]
    idx = torch.arange(groups * 64)
    gi, ci = idx // 64, idx % 64
    shifted = torch.where(ci < cg, comp_bias[(gi * cg + ci).clamp(max=groups * 64 - 1)], torch.zeros(()))
    got = R.split_epilogue(acc, shifted, col_gin=64, col_gout=cg)
    rep = R.mismatch_exact(got[0], want[0], Tf, cg)
    assert rep is not None and "group 0" not in rep.splitlines()[1], rep   # group 0's columns coincide; the rest differ


def test_staging_defects_are_flagged():
    """regroup_pad output fed to the grouped conv: a halo row that is not zero, or a pad channel holding a NaN (its
    weights are zero, so only a NaN shows), changes the positional-conv output."""
    B, Tf, Kpos, groups, cg = 2, 40, 16, 4, 48
    halo = Kpos // 2
    g = torch.Generator().manual_seed(7)
    x = torch.randn(B * Tf, groups * cg, generator=g)
    w = torch.zeros(groups * 64, Kpos * 64)
    w.view(groups, 64, Kpos, 64)[:, :cg, :, :cg] = torch.randn(groups, cg, Kpos, cg, generator=g) / 30
    xh, xl = R.split_f32(x)
    wh, wl = R.split_f32(w)
    sh, sl = R.regroup_pad(xh, B, Tf, halo, groups, cg), R.regroup_pad(xl, B, Tf, halo, groups, cg)
    assert torch.equal(sh[:, :halo], torch.zeros_like(sh[:, :halo])) and torch.equal(sh.view(B, -1, groups, 64)[..., cg:],
                                                                                      torch.zeros(B, Tf + 2 * halo, groups, 64 - cg))
    ref = R.posconv_split_acc(sh, sl, wh, wl, Tf, Kpos, groups, exact=False)
    bad_h = sh.clone()
    bad_h[1, halo + Tf + 2] = 1.0                       # a trailing halo row of clip 1
    got = R.posconv_split_acc(bad_h, sl, wh, wl, Tf, Kpos, groups, exact=False)
    bound = torch.full_like(ref, 1e-6)
    rep = R.mismatch_bound(got, ref, bound, Tf)
    assert rep is not None and "flagged clips [1]" in rep, rep
    bad_p = sh.clone()
    bad_p.view(B, -1, groups, 64)[0, halo + 3, 2, cg + 1] = float("nan")   # pad channel of group 2
    got = R.posconv_split_acc(bad_p, sl, wh, wl, Tf, Kpos, groups, exact=False)
    rep = R.mismatch_bound(got, ref, bound, Tf)
    assert rep is not None and "group 2" in rep, rep


# ----------------------------------------------------------------------------------------------------- LayerNorm
def _ln_emulation(xh, xl, g, b, eps, unbiased=False):
    v = xh.float() + xl.float()
    D = v.shape[-1]
    mean = v.sum(-1, keepdim=True) / D
    d = v - mean
    var = (d * d).sum(-1, keepdim=True) / (D - 1 if unbiased else D)
    o = d * torch.rsqrt(var + eps) * g.float() + b.float()
    return R.split_f32(o)


def test_layernorm_bound():
    gen = torch.Generator().manual_seed(2)
    x = torch.randn(64, 768, generator=gen) * 3 + 5 * torch.randn(64, 1, generator=gen)
    gamma, beta = 1 + 0.1 * torch.randn(768, generator=gen), 0.1 * torch.randn(768, generator=gen)
    xh, xl = R.split_f32(x)
    ref, mean, rstd = R.layernorm_reference(R.hilo(xh, xl), gamma, beta, 1e-5)
    bound = R.layernorm_bound(R.hilo(xh, xl), gamma, ref, mean, rstd)
    oh, ol = _ln_emulation(xh, xl, gamma, beta, 1e-5)
    assert R.mismatch_bound(R.hilo(oh, ol), ref, bound, 64, 768) is None
    oh, ol = _ln_emulation(xh, xl, gamma, beta, 1e-5, unbiased=True)
    assert R.mismatch_bound(R.hilo(oh, ol), ref, bound, 64, 768) is not None


# ----------------------------------------------------------------------------------------------------- conv0 front
def _gelu_as(z):
    """GELU with the Abramowitz-Stegun 7.1.26 erf the kernels use (float64)."""
    x = z.abs() / math.sqrt(2.0)
    t = 1.0 / (1.0 + 0.3275911 * x)
    p = t * (0.254829592 + t * (-0.284496736 + t * (1.421413741 + t * (-1.453152027 + t * 1.061405429))))
    erf = 1.0 - p * torch.exp(-x * x)
    return 0.5 * z * (1.0 + torch.sign(z) * erf)


def _conv0_emulation(wav, w, gamma, beta, pad, KW, ST, n_stat=None):
    """conv0 as the kernel computes it: fp64 statistics, fp32 scale / shift, fp32 taps pre-multiplied by the scale and
    an fp32 FMA chain seeded with the shift (fp64 product + add, rounded to fp32 per step), A-S GELU, hi/lo split."""
    x = torch.nn.functional.pad(wav.double(), (pad, pad)).unfold(1, KW, ST)
    wd = w.double().reshape(-1, KW)
    y = x @ wd.t()
    ys = y[:, :(n_stat or y.shape[1])]
    mean, var = ys.mean(1, keepdim=True), ys.var(1, unbiased=False, keepdim=True)
    sc = (gamma.double() / torch.sqrt(var + 1e-5)).float()
    sh = (beta.double() - mean * sc.double()).float()
    taps = (w.float().reshape(-1, KW)[None] * sc.transpose(1, 2)).double()   # [B, C, KW]
    acc = sh.double().expand(y.shape).clone()
    for j in range(KW):
        acc = (acc + taps[:, None, :, j] * x[:, :, None, j].float().double()).float().double()
    hi, lo = R.split_f32(_gelu_as(acc).float())
    return R.hilo(hi, lo)


@pytest.mark.parametrize("clip", ["noise", "dc", "silence"])
def test_conv0_bound(clip):
    C, KW, ST, pad, S = 64, 10, 5, 40, 715
    g = torch.Generator().manual_seed(3)
    w = torch.randn(C, KW, generator=g) * math.sqrt(0.2)
    gamma, beta = 1 + 0.1 * torch.randn(C, generator=g), 0.1 * torch.randn(C, generator=g)
    wav = {"noise": 0.1 * torch.randn(2, S, generator=g),
           "dc": 0.5 + 1e-3 * torch.randn(2, S, generator=g),
           "silence": torch.zeros(2, S)}[clip]
    want, z, mag = R.conv0_reference(wav, w, gamma, beta, pad, KW, ST)
    bound = R.conv0_bound(z, want, mag, KW)
    got = _conv0_emulation(wav, w, gamma, beta, pad, KW, ST)
    T0 = want.shape[1]
    assert R.mismatch_bound(got.reshape(-1, C), want.reshape(-1, C), bound.reshape(-1, C), T0, 64) is None
    if clip != "silence":
        bad = _conv0_emulation(wav, w, gamma, beta, pad, KW, ST, n_stat=T0 - 1)
        assert R.mismatch_bound(bad.reshape(-1, C), want.reshape(-1, C), bound.reshape(-1, C), T0, 64) is not None


# ----------------------------------------------------------------------------------------------------- rel_len, plans
def test_rel_len_float32_differs_from_float64():
    S, T = 160000, 500
    lens = torch.arange(0, S + 1)
    want = R.rel_len(lens, S, T)
    f64 = torch.ceil(lens.double() / S * T).clamp(0, T).to(torch.int32)
    diff = (want != f64).nonzero().flatten()
    assert diff.numel() > 0, "no length separates float32 from float64 rel_len at this S"
    assert int(want[0]) == 0 and int(want[-1]) == T and int(R.rel_len(torch.tensor([S + 5]), S, T)[0]) == T


def test_pick_bn_mirror():
    assert R.pick_bn(3000, 768) == 256 and R.pick_bn(1, 768) == 128 and R.pick_bn(1, 3072) == 128
    assert R.pick_bn(3000, 768, force_bn=64) == 64 and R.pick_bn(3000, 3072, a_mode=1) == 64
    assert R.pick_bn(128 * 132, 512) == 256


def test_boundary_rows_cover_edges():
    rows = set(R.boundary_rows(300, 2, frac=0.0).tolist())
    for r in (0, 1, 126, 127, 128, 129, 254, 255, 256, 257, 298, 299, 300, 301, 599):
        assert r in rows


# ----------------------------------------------------------------------------------------------------- encoder layer
def _layer_case(B=2, T=40, H=128, F=256, seed=0):
    g = torch.Generator().manual_seed(seed)
    rn = lambda *s, std=1.0: torch.randn(*s, generator=g) * std
    w = {"wqkv": rn(3 * H, H, std=H ** -0.5), "bqkv": 0.02 * rn(3 * H), "wo": rn(H, H, std=H ** -0.5), "bo": 0.02 * rn(H),
         "ln1.g": 1 + 0.1 * rn(H), "ln1.b": 0.1 * rn(H), "ff1.w": rn(F, H, std=H ** -0.5), "ff1.b": 0.02 * rn(F),
         "ff2.w": rn(H, F, std=F ** -0.5), "ff2.b": 0.02 * rn(H), "ln2.g": 1 + 0.1 * rn(H), "ln2.b": 0.1 * rn(H)}
    return rn(B * T, H), w, B, T, H


def _layer_steps(x, w, B, T, H, drop_residual=False, swap_heads=False):
    """The device's layer step by step in fp32 (split three-product linears, fp32 attention, torch's LayerNorm), every
    intermediate stored as a hi/lo pair -> {step: (emulated output, reference, bound)}, each reference and bound computed
    from the emulation's own input to that step, as the device test does with the device's taps."""
    pair = lambda v: R.hilo(*R.split_f32(v)).float()

    def lin(v, wn, bn, act=0, res=None):
        vh, vl = R.split_f32(v)
        wh, wl = R.split_f32(w[wn])
        y = vh.float() @ wh.float().t() + vh.float() @ wl.float().t() + vl.float() @ wh.float().t() + w[bn]
        if act:
            y = torch.nn.functional.gelu(y)
        if res is not None:
            y = y + res
        return pair(y)

    ln = lambda v, n: torch.nn.functional.layer_norm(v, (H,), w[n + ".g"], w[n + ".b"], 1e-5)
    steps = {}
    x0 = pair(x)
    qkv = lin(x0, "wqkv", "bqkv")
    steps["qkv"] = (qkv, *R.linear_with_bound(x0.double(), None, w["wqkv"], w["bqkv"]))
    q, k, v = (qkv.reshape(B, T, 3, H // 64, 64)[:, :, i].transpose(1, 2) for i in range(3))
    a = torch.softmax(q @ k.transpose(-1, -2) * 0.125, -1) @ v                    # [B, heads, T, 64]
    if swap_heads:
        a = a.flip(1)
    a = pair(a.transpose(1, 2).reshape(B * T, H))
    steps["attention"] = (a, *R.attention_with_bound(qkv.double(), None, B, T, H // 64, 0.125))
    t1 = lin(a, "wo", "bo", res=None if drop_residual else x0)
    steps["oproj"] = (t1, *R.linear_with_bound(a.double(), None, w["wo"], w["bo"], res=x0.double()))
    h1 = pair(ln(t1, "ln1"))
    steps["ln1"] = (h1, *R.layernorm_with_bound(t1.double(), None, w["ln1.g"], w["ln1.b"], 1e-5))
    f = lin(h1, "ff1.w", "ff1.b", act=1)
    steps["ff1"] = (f, *R.linear_with_bound(h1.double(), None, w["ff1.w"], w["ff1.b"], act=1))
    t2 = lin(f, "ff2.w", "ff2.b", res=h1)
    steps["ff2"] = (t2, *R.linear_with_bound(f.double(), None, w["ff2.w"], w["ff2.b"], res=h1.double()))
    out = ln(t2, "ln2")
    steps["ln2"] = (out, *R.layernorm_with_bound(t2.double(), None, w["ln2.g"], w["ln2.b"], 1e-5, hilo_out=False))
    return steps


def test_encoder_layer_step_bounds():
    x, w, B, T, H = _layer_case()
    for name, (got, want, bound) in _layer_steps(x, w, B, T, H).items():
        assert float((bound / want.abs().clamp(min=1e-2)).median()) < 1e-2, name   # bounds that still mean something
        assert R.mismatch_bound(got, want, bound, T, 64, name) is None
    bad = _layer_steps(x, w, B, T, H, drop_residual=True)["oproj"]
    assert R.mismatch_bound(*bad, T, 64, "oproj") is not None
    bad = _layer_steps(x, w, B, T, H, swap_heads=True)["attention"]
    rep = R.mismatch_bound(*bad, T, 64, "attention")
    assert rep is not None and "group 0" in rep and "columns [0, 127]" in rep, rep
