"""CPU checks of tests/qwen_ref.py: each checker accepts a faithful fp32 model of its kernel, agrees with HF (the oracle's
rms_norm and apply_rope, torch autograd, F.silu on bf16), and flags an injected defect: one bf16 ulp, a missing
rounding of x * rstd, eps added after the rsqrt, rstd two bound-widths off, a tail vector not written, accumulate_dw
ignored, dres dropped, a RoPE position off by one, no clamp, partial rotary paired with i + head_dim / 2, the inverse
with +sin, a sigmoid flushed to zero below 2^-126, and d_gate rounded at a different point."""
import numpy as np
import pytest
import torch

import qwen_ref as Q
from grad_ref import bf16, check_bf16_interval


def _ulp(a, idx, k=1):
    """a with the element at idx moved by k bf16 ulps."""
    b = np.array(a, dtype=np.float32, copy=True)
    t = torch.from_numpy(b[idx].reshape(1).copy()).to(torch.bfloat16)
    b[idx] = (t.view(torch.int16) + k).view(torch.bfloat16).float().numpy()[0]
    return b


# ----------------------------------------------------------------------------------------------------- RMSNorm
def _rms_inputs(M=64, D=896, seed=0):
    r = np.random.default_rng(seed)
    scale = np.exp(r.uniform(-6, 3, size=(M, 1)))             # rows from 2.5e-3 to 20: eps matters on the small ones
    x = bf16(r.normal(size=(M, D)) * scale)
    w = bf16(1 + 0.3 * r.normal(size=D))
    return x, w, 1e-6


def _rms_model(x, w, eps, round_xr=True, eps_after=False, rstd_scale=1.0):
    """fp32 model of rmsnorm_fwd_kernel (the sum in fp32, rsqrt correctly rounded)."""
    x32 = x.astype(np.float32)
    ss = (x32 * x32).sum(axis=1, dtype=np.float32)
    ms = (ss / np.float32(x.shape[1])).astype(np.float32)
    if eps_after:
        rstd = (np.float32(1) / np.sqrt(ms) + np.float32(eps)).astype(np.float32)
    else:
        rstd = (np.float32(1) / np.sqrt((ms + np.float32(eps)).astype(np.float32))).astype(np.float32)
    rstd = (rstd * np.float32(rstd_scale)).astype(np.float32)
    t = (x32 * rstd[:, None]).astype(np.float32)
    if round_xr:
        t = bf16(t)
    return bf16(w[None, :] * t), rstd


def test_rmsnorm_fwd_checker():
    from oracle.lm_oracle import rms_norm
    x, w, eps = _rms_inputs()
    y, rstd = _rms_model(x, w, eps)
    assert Q.check_rmsnorm_fwd(y, rstd, x, w, eps) == []
    hf = rms_norm(torch.from_numpy(x).to(torch.bfloat16), torch.from_numpy(w).to(torch.bfloat16), eps).float().numpy()
    assert Q.check_rmsnorm_fwd(hf, None, x, w, eps) == [], "HF's RMSNorm is not inside the reference"
    two = Q.rmsnorm_two_candidates(x, w, eps)
    print(f"rmsnorm: {two} of {x.size} outputs have two candidates")
    assert two < 0.01 * x.size
    ylo, yhi, _, _ = Q.rmsnorm_fwd_ref(x, w, eps)
    i = tuple(np.argwhere((ylo == yhi) & (y != 0))[7])
    assert Q.check_rmsnorm_fwd(_ulp(y, i), rstd, x, w, eps), "one ulp"
    assert Q.check_rmsnorm_fwd(_rms_model(x, w, eps, round_xr=False)[0], rstd, x, w, eps), "x * rstd not rounded"
    y2, r2 = _rms_model(x, w, eps, eps_after=True)
    assert Q.check_rmsnorm_fwd(y2, r2, x, w, eps), "eps after the rsqrt"
    e = Q.rstd_bound(x.shape[1])
    y3, r3 = _rms_model(x, w, eps, rstd_scale=1 + 2 * e)
    assert Q.check_rmsnorm_fwd(y, r3, x, w, eps), "rstd two bound-widths off"
    y4 = y.copy()
    y4[5, -8:] = 0.0
    assert Q.check_rmsnorm_fwd(y4, rstd, x, w, eps), "tail vector not written"


def _bwd_model(dy, x, w, rstd, dres, dw_old, accumulate=True, drop_dres=False):
    """float64 evaluation of the kernel's formula (exact on exact operands), one rounding of each output."""
    dx, dw, _, _ = Q.rmsnorm_bwd_ref(dy, x, w, rstd, None if drop_dres else dres)
    if accumulate and dw_old is not None:
        dw = dw + dw_old
    from grad_ref import bf16_from64
    return bf16_from64(dx), bf16_from64(dw)


@pytest.mark.parametrize("D", [8, 120, 1000])
def test_rmsnorm_bwd_exact_and_defects(D):
    dy, x, w, rstd, dres = Q.exact_rmsnorm_bwd_operands(9, D, seed=D)
    old = bf16(np.random.default_rng(1).integers(-64, 65, size=D).astype(np.float32))
    for d_res in (None, dres):
        for o in (None, old):
            dx, dw = Q.rmsnorm_bwd_exact(dy, x, w, rstd, d_res, o)
            mdx, mdw = _bwd_model(dy, x, w, rstd, d_res, o)
            assert np.array_equal(dx, mdx) and np.array_equal(dw, mdw)
            assert Q.check_rmsnorm_bwd(dx, dw, dy, x, w, rstd, d_res, o) == []
    dx, dw = Q.rmsnorm_bwd_exact(dy, x, w, rstd, dres, old)
    i = (3, D - 1)
    assert Q.check_rmsnorm_bwd(_ulp(dx, i), dw, dy, x, w, rstd, dres, old), "one ulp in dx"
    assert Q.check_rmsnorm_bwd(dx, _ulp(dw, D - 1), dy, x, w, rstd, dres, old), "one ulp in dw"
    _, dw_noacc = _bwd_model(dy, x, w, rstd, dres, old, accumulate=False)
    assert Q.check_rmsnorm_bwd(dx, dw_noacc, dy, x, w, rstd, dres, old), "accumulate_dw ignored"
    dx_nores, _ = _bwd_model(dy, x, w, rstd, dres, old, drop_dres=True)
    assert Q.check_rmsnorm_bwd(dx_nores, dw, dy, x, w, rstd, dres, old), "dres dropped"
    tail = dx.copy()
    tail[4, -8:] = 0.0
    assert Q.check_rmsnorm_bwd(tail, dw, dy, x, w, rstd, dres, old), "tail vector not written"


def test_rmsnorm_bwd_random_bound():
    x, w, eps = _rms_inputs(M=40, D=896, seed=3)
    r = np.random.default_rng(4)
    dy, dres = bf16(r.normal(size=x.shape)), bf16(r.normal(size=x.shape))
    _, rstd = _rms_model(x, w, eps)
    dx64, dw64, _, _ = Q.rmsnorm_bwd_ref(dy, x, w, rstd, dres)
    from grad_ref import bf16_from64
    dx, dw = bf16_from64(dx64), bf16_from64(dw64)
    assert Q.check_rmsnorm_bwd(dx, dw, dy, x, w, rstd, dres) == []
    # torch autograd of HF's module (the oracle's rms_norm on bf16 tensors) is inside the dx bound (its dw rounds each
    # dy * bf16(xhat) to bf16 before the sum, the kernel sums in fp32)
    from oracle.lm_oracle import rms_norm
    xt = torch.from_numpy(x).to(torch.bfloat16).requires_grad_(True)
    wt = torch.from_numpy(w).to(torch.bfloat16).requires_grad_(True)
    rms_norm(xt, wt, eps).backward(torch.from_numpy(dy).to(torch.bfloat16))
    r32 = torch.rsqrt(torch.from_numpy(x).pow(2).mean(-1) + eps).numpy()
    ref, _, _, _ = Q.rmsnorm_bwd_ref(dy, x, w, r32)
    assert check_bf16_interval(xt.grad.float().numpy(), ref, Q.rmsnorm_dx_bound(dy, x, w, r32), "autograd dx") == []
    assert Q.check_rmsnorm_bwd(_ulp(dx, (2, 5), 2), dw, dy, x, w, rstd, dres), "two ulps in dx"
    assert Q.check_rmsnorm_bwd(dx, dw, dy, x, w, rstd, None), "dres dropped"


# ----------------------------------------------------------------------------------------------------- RoPE
def _rope_case(M=96, T=32, hd=64, H=3, KVH=1, maxpos=40, seed=0, rot=None):
    from slamkit_b200.lm import rope_tables
    g = torch.Generator().manual_seed(seed)
    qkv = torch.randn(M, (H + 2 * KVH) * hd + 16, generator=g).to(torch.bfloat16)
    cos, sin = rope_tables(10000.0, rot or hd, maxpos)
    return qkv, cos, sin, H + KVH


def test_rope_matches_hf_apply_rope():
    from oracle.lm_oracle import OracleLMConfig, apply_rope, rope_cos_sin
    B, T, H, hd = 2, 32, 3, 64
    qkv, cos, sin, nr = _rope_case(M=B * T, T=T, H=H, KVH=1)
    pos = Q.rope_positions(B * T, T, cos.shape[0])
    out = Q.rope_ref(qkv, cos, sin, pos, nr, hd)
    c, s = rope_cos_sin(OracleLMConfig(head_dim=hd), torch.arange(T)[None].expand(B, -1), torch.bfloat16)
    q = qkv[:, :H * hd].reshape(B, T, H, hd).transpose(1, 2)
    k = qkv[:, H * hd:(H + 1) * hd].reshape(B, T, 1, hd).transpose(1, 2)
    qr, kr = apply_rope(q, k, c, s)
    assert torch.equal(out[:, :H * hd].reshape(B, T, H, hd).transpose(1, 2), qr)
    assert torch.equal(out[:, H * hd:(H + 1) * hd].reshape(B, T, 1, hd).transpose(1, 2), kr)
    assert torch.equal(out[:, nr * hd:], qkv[:, nr * hd:])


@pytest.mark.parametrize("rot", [64, 32, 16])
def test_rope_inverse_is_autograd(rot):
    qkv, cos, sin, nr = _rope_case(rot=rot)
    g = torch.Generator().manual_seed(9)
    grad = torch.randn(qkv.shape, generator=g).to(torch.bfloat16)
    pos = Q.rope_positions(qkv.shape[0], 32, cos.shape[0])
    inv = Q.rope_ref(grad, cos, sin, pos, nr, 64, rot, inverse=True)
    auto = Q.rope_autograd(qkv, cos, sin, pos, nr, 64, grad, rot)
    assert torch.equal(inv[:, :nr * 64].reshape(-1, nr, 64)[..., :rot], auto)


def _rope_kernel_model(qkv, cos, sin, pos, nr, hd, rot, inverse=False, pair=None):
    """Element-wise model of rope_kernel in fp32 with its rounding points; pair = the distance of the partner column."""
    x = qkv.float().clone()
    half = rot // 2
    pair = pair or half
    c, s = cos.float()[pos], sin.float()[pos]
    if inverse:
        s = -s
    r = lambda t: t.to(torch.bfloat16).float()
    for h in range(nr):
        b = h * hd
        x1, x2 = x[:, b:b + half].clone(), x[:, b + pair:b + pair + half].clone()
        x[:, b:b + half] = r(r(x1 * c) + r(-x2 * s))
        x[:, b + pair:b + pair + half] = r(r(x2 * c) + r(x1 * s))
    return x.to(torch.bfloat16)


@pytest.mark.parametrize("rot", [64, 32, 16])
def test_rope_checker_flags_defects(rot):
    M, T, maxpos = 96, 32, 40
    qkv, cos, sin, nr = _rope_case(M=M, T=T, maxpos=maxpos, rot=rot)
    pos_ids = torch.arange(M) % 50 - 3                          # below 0 and at or above maxpos: clamped
    pos = Q.rope_positions(M, T, maxpos, pos_ids)
    for inverse in (False, True):
        want = Q.rope_ref(qkv, cos, sin, pos, nr, 64, rot, inverse)
        good = _rope_kernel_model(qkv, cos, sin, pos, nr, 64, rot, inverse)
        assert Q.check_rope(good, want) == []
        bad = good.clone()
        bad.view(torch.int16)[3, 1] += 1
        assert Q.check_rope(bad, want), "one ulp"
        assert Q.check_rope(_rope_kernel_model(qkv, cos, sin, (pos + 1).clamp(0, maxpos - 1), nr, 64, rot, inverse),
                            want), "position off by one"
        raw = (torch.arange(M) % 50 - 3)
        assert Q.check_rope(_rope_kernel_model(qkv, cos, sin, raw.clamp(min=0) % maxpos, nr, 64, rot, inverse), want), \
            "no clamp (the table read wraps)"
        assert Q.check_rope(_rope_kernel_model(qkv, cos, sin, pos, nr, 64, rot, not inverse), want), "sign of sin"
        if rot < 64:
            assert Q.check_rope(_rope_kernel_model(qkv, cos, sin, pos, nr, 64, rot, inverse, pair=32), want), \
                "partial rotary paired with i + head_dim / 2"


# ----------------------------------------------------------------------------------------------------- SwiGLU
def _silu_model(g, flush=False):
    """fp32 x / (1 + exp(-x)) (torch's formula); flush: the sigmoid flushed to 0 below 2^-126 (rcp.approx.ftz)."""
    x = np.asarray(g, np.float32)
    with np.errstate(all="ignore"):
        s = (np.float32(1) / (np.float32(1) + np.exp(-x))).astype(np.float32)
        if flush:
            s = np.where(np.abs(s) < np.float32(2.0 ** -126), np.float32(0), s)
        return (x * s).astype(np.float32), s


def _swiglu_model(g, u, d, flush=False, dgate_mode=0):
    with np.errstate(all="ignore"):
        sil, s = _silu_model(g, flush)
        sb = bf16(sil)
        act = bf16(sb * u)
        ds = (s * (np.float32(1) + g * (np.float32(1) - s))).astype(np.float32)
        if dgate_mode == 0:
            dgate = bf16(bf16(d * u) * ds)
        else:                                                    # rounded after the product with u instead
            dgate = bf16(d * bf16(u * ds))
        dup = bf16(d * sb)
    return act, dgate, dup


def _sweep():
    g = Q.all_bf16()
    us = bf16(np.array([1.0, -1.5, 0.0078125, 3.0e3, 0.0], np.float32))
    ds = bf16(np.array([1.0, 0.375, -2.0, 1.0e-3, 5.0], np.float32))
    G = np.tile(g, (len(us), 1))
    return G, np.broadcast_to(us[:, None], G.shape).copy(), np.broadcast_to(ds[:, None], G.shape).copy()


def test_swiglu_checkers_accept_torch_and_the_fp32_model():
    G, U_, D_ = _sweep()
    act, dg, du = _swiglu_model(G, U_, D_)
    assert Q.check_swiglu_fwd(act, G, U_) == []
    assert Q.check_swiglu_bwd(dg, du, G, U_, D_) == []
    tact, tdg, tdu = Q.torch_swiglu(G, U_, D_)
    assert Q.check_swiglu_fwd(tact, G, U_) == [], "F.silu on bf16 is not inside the bound"
    assert Q.check_swiglu_bwd(tdg, tdu, G, U_, D_) == [], "autograd of F.silu is not inside the bound"
    # NaN exactly where torch's is
    assert np.array_equal(np.isnan(Q.swiglu_fwd_candidates(G, U_)[0]), np.isnan(tact))


def test_swiglu_checkers_flag_defects():
    G, U_, D_ = _sweep()
    act, dg, du = _swiglu_model(G, U_, D_)
    i = (0, int(np.argwhere(Q.all_bf16() == np.float32(0.5))[0][0]))
    assert Q.check_swiglu_fwd(_ulp(act, i), G, U_), "one ulp in act"
    assert Q.check_swiglu_bwd(_ulp(dg, i), du, G, U_, D_), "one ulp in d_gate"
    assert Q.check_swiglu_bwd(dg, _ulp(du, i), G, U_, D_), "one ulp in d_up"
    fact, fdg, fdu = _swiglu_model(G, U_, D_, flush=True)
    rep = Q.check_swiglu_fwd(fact, G, U_)
    assert rep, "sigmoid flushed to zero"
    diff = (fact != act) & ~(np.isnan(fact) & np.isnan(act))
    bad = sorted(set(float(v) for v in G[diff]))
    print(f"flushed sigmoid: act differs at gates {bad}")
    assert bad == [-88.5, -88.0, -87.5]
    rep = Q.check_swiglu_bwd(fdg, fdu, G, U_, D_)
    assert any("d_gate" in r for r in rep) and any("d_up" in r for r in rep)
    _, dg2, _ = _swiglu_model(G, U_, D_, dgate_mode=1)
    assert Q.check_swiglu_bwd(dg2, du, G, U_, D_), "d_gate rounded at a different point"
