"""GPU parity of the individual sm_90a kernels (through the C ABI) against fp32 torch restatements of the same op.
Integer / index outputs are compared exactly; floating-point outputs norm-wise at bf16-rounding tolerances."""
import math

import pytest
import torch

from helpers import max_abs, rel_err

pytestmark = pytest.mark.gpu

DEV = "cuda:0"


def _randn(*shape, scale=1.0, seed=0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(torch.bfloat16)


# ----------------------------------------------------------------------------------------------- GEMM (wgmma)
GEMM_SHAPES = [
    (128, 128, 64), (256, 256, 128), (384, 896, 896), (1000, 1152, 896), (512, 512, 4864),
    (8192, 896, 896), (200, 72, 136), (130, 8, 24),
]


@pytest.mark.parametrize("bn", [0, 64, 128, 256])
@pytest.mark.parametrize("M,N,K", GEMM_SHAPES)
def test_gemm_nt(M, N, K, bn):
    from slamkit_b200 import ops
    a, b = _randn(M, K, seed=1), _randn(N, K, seed=2)
    ref = a.float() @ b.float().t()
    out = ops.gemm(a.to(DEV), b.to(DEV), force_bn=bn).cpu()
    assert rel_err(out, ref) < 4e-3, (M, N, K, bn, rel_err(out, ref))


@pytest.mark.parametrize("a_mn,b_mn", [(False, True), (True, False), (True, True)])
@pytest.mark.parametrize("M,N,K", [(256, 256, 128), (384, 896, 1152), (896, 4864, 1000), (512, 896, 8192), (200, 72, 136)])
def test_gemm_mn_major(M, N, K, a_mn, b_mn):
    """dgrad (B stored [K,N]) and wgrad (A stored [K,M], B stored [K,N]) operand layouts."""
    from slamkit_b200 import ops
    a, b = _randn(M, K, seed=3), _randn(N, K, seed=4)
    ref = a.float() @ b.float().t()
    a_dev = a.t().contiguous().to(DEV) if a_mn else a.to(DEV)
    b_dev = b.t().contiguous().to(DEV) if b_mn else b.to(DEV)
    out = ops.gemm(a_dev, b_dev, a_mn=a_mn, b_mn=b_mn).cpu()
    assert rel_err(out, ref) < 4e-3, (M, N, K, a_mn, b_mn, rel_err(out, ref))


def test_gemm_epilogues():
    from slamkit_b200 import ops
    M, N, K = 300, 264, 200
    a, b = _randn(M, K, seed=5), _randn(N, K, seed=6)
    bias, res = _randn(N, seed=7), _randn(M, N, seed=8)
    acc = a.float() @ b.float().t()
    out = ops.gemm(a.to(DEV), b.to(DEV), bias=bias.to(DEV)).cpu()
    assert rel_err(out, acc + bias.float()) < 4e-3
    out = ops.gemm(a.to(DEV), b.to(DEV), bias=bias.to(DEV), residual=res.to(DEV), round_before_res=True).cpu()
    ref = ((acc + bias.float()).to(torch.bfloat16).float() + res.float())
    assert rel_err(out, ref) < 4e-3
    out = ops.gemm(a.to(DEV), b.to(DEV), out_f32=True).cpu()
    assert out.dtype == torch.float32 and rel_err(out, acc) < 1e-5
    out = ops.gemm(a.to(DEV), b.to(DEV), bias=bias.to(DEV), act=1).cpu()
    assert rel_err(out, torch.nn.functional.gelu(acc + bias.float())) < 4e-3
    # in-place accumulate (gradient accumulation): C = bf16(acc) + C
    c = res.clone().to(DEV)
    ops.gemm(a.to(DEV), b.to(DEV), residual=c, out=c, round_before_res=True)
    assert rel_err(c.cpu(), acc.to(torch.bfloat16).float() + res.float()) < 4e-3


@pytest.mark.parametrize("M,N,K,acc", [(1152, 896, 8192, False), (896, 896, 8192, True), (512, 896, 8192, False),
                                         (384, 264, 2120, True)])
def test_gemm_splitk_wgrad(M, N, K, acc):
    """dW[M,N] (+)= dY[K,M]^T X[K,N] with the K (= tokens) loop split over idle SMs; deterministic."""
    from slamkit_b200 import ops
    dy, x = _randn(K, M, seed=11), _randn(K, N, seed=12)
    ref = dy.float().t() @ x.float()
    base = _randn(M, N, seed=13, scale=5.0)
    out = base.clone().to(DEV)
    ops.gemm_splitk(dy.to(DEV), x.to(DEV), out, a_mn=True, b_mn=True, accumulate=acc)
    want = ref.to(torch.bfloat16).float() + base.float() if acc else ref
    assert rel_err(out.cpu(), want) < 4e-3, rel_err(out.cpu(), want)
    out2 = base.clone().to(DEV)
    ops.gemm_splitk(dy.to(DEV), x.to(DEV), out2, a_mn=True, b_mn=True, accumulate=acc)
    assert torch.equal(out, out2)


@pytest.mark.parametrize("a_mn,b_mn", [(False, False), (False, True), (True, False), (True, True)])
@pytest.mark.parametrize("M,N,K,bn", [(5064, 896, 2056, 0), (4224, 1152, 2048, 0), (2560, 896, 4096, 256),
                                       (3000, 1000, 2304, 256), (4160, 1480, 2056, 256), (6000, 1000, 3000, 256),
                                       (4104, 2048, 2104, 0), (9728, 896, 2048, 0)])
def test_gemm_streamk(M, N, K, bn, a_mn, b_mn):
    """Stream-K balancing (sk_gemm_bf16_ws): partial tiles meet in the scratch, fixed-order fix-up -> same result every
    launch; all four operand layouts, ragged M / N / K edges, one to four contributors per tile, a single split unit.
    Every shape is checked to run stream-K (on 132 SMs)."""
    from slamkit_b200 import ops
    import gemm_ref as R
    a, b = _randn(M, K, seed=21).to(DEV), _randn(N, K, seed=22).to(DEV)
    a_dev = a.t().contiguous() if a_mn else a
    b_dev = b.t().contiguous() if b_mn else b
    plan = ops.gemm_plan(a_dev, b_dev, a_mn=a_mn, b_mn=b_mn, force_bn=bn, streamk=True)
    assert R.schedule_kind(plan, K) in ("streamk1", "streamk2"), plan
    out = ops.gemm(a_dev, b_dev, a_mn=a_mn, b_mn=b_mn, force_bn=bn, streamk=True)
    ref = a.float() @ b.float().t()
    assert rel_err(out, ref) < 4e-3, (M, N, K, bn, rel_err(out, ref))
    rep = R.mismatch_random(out, a, b, plan["bn"])
    assert rep is None, rep
    for _ in range(3):   # flags re-armed by the kernel; bit-identical
        out2 = ops.gemm(a_dev, b_dev, a_mn=a_mn, b_mn=b_mn, force_bn=bn, streamk=True)
        assert torch.equal(out, out2)
    assert int(ops.gemm_workspace(DEV)[-4096:].max()) == 0


def test_gemm_streamk_epilogues():
    """Bias + residual, fp32 output (the direct-store fix-up), GELU and in-place accumulation under stream-K."""
    from slamkit_b200 import ops
    import gemm_ref as R
    M, N, K = 5120, 896, 2048
    a, b = _randn(M, K, seed=5), _randn(N, K, seed=6)
    bias, res = _randn(N, seed=7), _randn(M, N, seed=8)
    acc = a.float() @ b.float().t()
    ad, bd = a.to(DEV), b.to(DEV)
    r = res.to(DEV)
    for kw in (dict(bias=bias.to(DEV), residual=r), dict(out_f32=True), dict(bias=bias.to(DEV), act=1), dict(residual=r, out=r)):
        assert R.schedule_kind(ops.gemm_plan(ad, bd, streamk=True, **kw), K) == "streamk2"
    out = ops.gemm(ad, bd, bias=bias.to(DEV), residual=res.to(DEV), round_before_res=True, streamk=True).cpu()
    ref = ((acc + bias.float()).to(torch.bfloat16).float() + res.float())
    assert rel_err(out, ref) < 4e-3
    out = ops.gemm(ad, bd, out_f32=True, streamk=True).cpu()
    assert out.dtype == torch.float32 and rel_err(out, acc) < 1e-5
    out = ops.gemm(ad, bd, bias=bias.to(DEV), act=1, streamk=True).cpu()
    assert rel_err(out, torch.nn.functional.gelu(acc + bias.float())) < 4e-3
    c = res.clone().to(DEV)
    ops.gemm(ad, bd, residual=c, out=c, round_before_res=True, streamk=True)
    assert rel_err(c.cpu(), acc.to(torch.bfloat16).float() + res.float()) < 4e-3
    # same values as the plain launch up to fp32 summation order
    plain = ops.gemm(ad, bd).float()
    sk = ops.gemm(ad, bd, streamk=True).float()
    assert rel_err(sk.cpu(), plain.cpu()) < 2e-3


def test_gemm_rejects_bad_arguments():
    from slamkit_b200 import ops, _lib
    a, b = _randn(64, 64).to(DEV), _randn(60, 64).to(DEV)  # N=60 is not a multiple of 8
    with pytest.raises(_lib.SkError):
        ops.gemm(a, b)


# ---------------------------------------------------------------------------------------------- element-wise
def test_embed_fwd_bwd():
    from slamkit_b200 import ops
    V, Vp, D, M = 502, 512, 896, 1000
    table = torch.zeros(Vp, D, dtype=torch.bfloat16)
    table[:V] = _randn(V, D, seed=1)
    g = torch.Generator().manual_seed(0)
    ids = torch.randint(0, V, (M,), generator=g)
    out = ops.embed_fwd(ids.to(DEV), table.to(DEV), V).cpu()
    assert torch.equal(out, table[ids])
    dx = _randn(M, D, seed=2)
    dtab = _randn(Vp, D, seed=3).to(DEV)
    before = dtab.cpu().float()
    ops.embed_bwd(ids.to(DEV), dx.to(DEV), dtab, V, accumulate=True)
    ref = before.clone().index_add_(0, ids, dx.float())
    assert rel_err(dtab.cpu(), ref) < 4e-3


@pytest.mark.parametrize("M,D", [(64, 896), (1000, 896), (33, 128), (7, 1024)])
def test_rmsnorm_fwd_bwd(M, D):
    from slamkit_b200 import ops
    from oracle.lm_oracle import rms_norm
    x = _randn(M, D, seed=1)
    w = (1 + 0.1 * torch.randn(D, generator=torch.Generator().manual_seed(2))).to(torch.bfloat16)
    y, rstd = ops.rmsnorm_fwd(x.to(DEV), w.to(DEV), 1e-6)
    ref = rms_norm(x, w, 1e-6)
    assert rel_err(y.cpu(), ref) < 2e-3
    assert (y.cpu() != ref).float().mean() < 0.02  # same rounding points -> almost always bit-identical
    # backward against fp32 autograd of the same function
    dy, dres = _randn(M, D, seed=3), _randn(M, D, seed=4)
    xf = x.float().requires_grad_(True)
    wf = w.float().requires_grad_(True)
    h = xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + 1e-6)
    (wf * h * dy.float()).sum().backward()
    dw = torch.zeros(1, D, dtype=torch.bfloat16, device=DEV)
    dx = ops.rmsnorm_bwd(dy.to(DEV), x.to(DEV), w.to(DEV), rstd, dres.to(DEV), dw, accumulate_dw=False)
    assert rel_err(dx.cpu(), xf.grad + dres.float()) < 6e-3
    assert rel_err(dw.cpu().view(-1), wf.grad) < 6e-3


def test_rope_matches_hf_and_inverts():
    from slamkit_b200 import ops
    from slamkit_b200.lm import rope_tables
    from oracle.lm_oracle import OracleLMConfig, apply_rope, rope_cos_sin
    B, T, H, KVH, hd = 2, 100, 3, 1, 64
    qkv = _randn(B * T, (H + 2 * KVH) * hd, seed=1)
    cos, sin = rope_tables(10000.0, hd, 256)
    out = ops.rope_(qkv.clone().to(DEV), cos.to(DEV), sin.to(DEV), T, H + KVH, hd).cpu()
    cfg = OracleLMConfig(head_dim=hd)
    pos = torch.arange(T)[None].expand(B, -1)
    c, s = rope_cos_sin(cfg, pos, torch.bfloat16)
    q = qkv[:, :H * hd].view(B, T, H, hd).transpose(1, 2)
    k = qkv[:, H * hd:(H + KVH) * hd].view(B, T, KVH, hd).transpose(1, 2)
    qr, kr = apply_rope(q, k, c, s)
    assert torch.equal(out[:, :H * hd].view(B, T, H, hd).transpose(1, 2), qr)      # bit-exact: same rounding points
    assert torch.equal(out[:, H * hd:(H + KVH) * hd].view(B, T, KVH, hd).transpose(1, 2), kr)
    assert torch.equal(out[:, (H + KVH) * hd:], qkv[:, (H + KVH) * hd:])            # v untouched
    back = ops.rope_(out.clone().to(DEV), cos.to(DEV), sin.to(DEV), T, H + KVH, hd, inverse=True).cpu()
    assert rel_err(back[:, :(H + KVH) * hd], qkv[:, :(H + KVH) * hd]) < 8e-3


def test_swiglu_fwd_bwd():
    from slamkit_b200 import ops
    M, F = 300, 4864
    gu = _randn(M, 2 * F, seed=1, scale=2.0)
    act = ops.swiglu_fwd(gu.to(DEV)).cpu()
    g, u = gu[:, :F], gu[:, F:]
    ref = torch.nn.functional.silu(g) * u  # bf16 ops, like HF
    assert rel_err(act, ref) < 2e-3
    assert (act != ref).float().mean() < 0.02
    dact = _randn(M, F, seed=2)
    gf, uf = g.float().requires_grad_(True), u.float().requires_grad_(True)
    (torch.nn.functional.silu(gf) * uf * dact.float()).sum().backward()
    dgu = ops.swiglu_bwd(gu.to(DEV), dact.to(DEV)).cpu()
    assert rel_err(dgu[:, :F], gf.grad) < 6e-3
    assert rel_err(dgu[:, F:], uf.grad) < 6e-3


def _unblock(x_blocked, F):
    """[M, 2F] in [128 gate | 128 up] column blocks -> (gate [M, F], up [M, F])"""
    v = x_blocked.view(x_blocked.shape[0], F // 128, 2, 128)
    return v[:, :, 0].reshape(-1, F), v[:, :, 1].reshape(-1, F)


@pytest.mark.parametrize("M,F,K", [(300, 256, 128), (1000, 4864, 896), (8192, 4864, 896), (130, 384, 200)])
def test_linear_swiglu_fused_matches_unfused_chain(M, F, K):
    """gate/up GEMM with SwiGLU in the epilogue == plain GEMM followed by the swiglu kernel, bit for bit; the fused
    backward (d_gu from dy * W_down without writing d_act) == dgrad GEMM followed by the swiglu backward kernel."""
    from slamkit_b200 import ops
    x, wg, wu = _randn(M, K, seed=1).to(DEV), _randn(F, K, seed=2, scale=0.05).to(DEV), _randn(F, K, seed=3, scale=0.05).to(DEV)
    gu_b, act = ops.linear_swiglu_fwd(x, ops.block_gate_up(wg, wu))
    gu_ref = ops.gemm(x, torch.cat([wg, wu], 0))                 # [M, 2F] = [gate | up]
    g, u = _unblock(gu_b, F)
    assert torch.equal(g, gu_ref[:, :F]) and torch.equal(u, gu_ref[:, F:])
    assert torch.equal(act, ops.swiglu_fwd(gu_ref))
    ref = torch.nn.functional.silu(gu_ref[:, :F]) * gu_ref[:, F:]        # bf16 ops, like HF
    assert rel_err(act.cpu(), ref.cpu()) < 2e-3
    # backward
    N = K
    dy, wd = _randn(M, N, seed=4).to(DEV), _randn(N, F, seed=5, scale=0.05).to(DEV)
    dgu_b = ops.linear_swiglu_bwd(dy, wd, gu_b)
    dact = ops.gemm(dy, wd, b_mn=True)
    dgu_ref = ops.swiglu_bwd(gu_ref, dact)
    dg, du = _unblock(dgu_b, F)
    assert torch.equal(dg, dgu_ref[:, :F]) and torch.equal(du, dgu_ref[:, F:])


@pytest.mark.parametrize("M,T,H,KVH,K,packed", [(200, 100, 3, 1, 128, False), (2048, 1024, 14, 2, 896, False), (512, 256, 4, 2, 256, True)])
def test_linear_rope_fused_matches_unfused_chain(M, T, H, KVH, K, packed):
    """QKV projection with bias + RoPE in the epilogue == GEMM(+bias) followed by the rope kernel, bit for bit."""
    from slamkit_b200 import ops
    from slamkit_b200.lm import rope_tables
    hd = 64
    N = (H + 2 * KVH) * hd
    x, w, b = _randn(M, K, seed=1).to(DEV), _randn(N, K, seed=2, scale=0.05).to(DEV), _randn(N, seed=3).to(DEV)
    cos, sin = rope_tables(10000.0, hd, 1024)
    cos, sin = cos.to(DEV), sin.to(DEV)
    pos = None
    if packed:
        g = torch.Generator().manual_seed(7)
        pos = torch.cat([torch.arange(n) for n in (100, 156, 200, 56)]).to(torch.int32).to(DEV)
        assert pos.numel() == M
    out = ops.linear_rope(x, w, b, cos, sin, T, (H + KVH) * hd, pos_ids=pos)
    ref = ops.rope_(ops.gemm(x, w, bias=b), cos, sin, T, H + KVH, hd, pos_ids=pos)
    assert torch.equal(out, ref)
    plain = ops.gemm(x, w, bias=b)
    assert torch.equal(out[:, (H + KVH) * hd:], plain[:, (H + KVH) * hd:])      # v heads untouched
    assert not torch.equal(out[:, :64], plain[:, :64])


@pytest.mark.parametrize("num_items", [0.0, 777.0])
def test_cross_entropy_fwd_bwd(num_items):
    from slamkit_b200 import ops
    from oracle.lm_oracle import compute_loss
    B, T, V, Vp = 3, 50, 502, 512
    logits = torch.zeros(B, T, Vp, dtype=torch.bfloat16)
    logits[..., :V] = _randn(B, T, V, seed=1, scale=3.0)
    logits[..., V:] = 7.0  # garbage in the padding columns must be ignored
    g = torch.Generator().manual_seed(2)
    labels = torch.randint(0, V, (B, T), generator=g)
    labels[1, 30:] = -100
    lf = logits[..., :V].float().requires_grad_(True)
    ref_loss = compute_loss(lf, labels, num_items if num_items > 0 else None)
    ref_loss.backward()
    stats, dlogits, row_nll = ops.ce_fwd_bwd(logits.view(B * T, Vp).to(DEV), labels.view(-1).to(DEV), T, V, num_items)
    stats = stats.cpu()
    assert abs(float(stats[0]) - float(ref_loss)) < 2e-6 * abs(float(ref_loss)) + 1e-6
    n_valid = int((labels[:, 1:] != -100).sum())
    assert int(stats[1]) == n_valid
    d = dlogits.cpu().view(B, T, Vp)
    assert rel_err(d[..., :V], lf.grad) < 4e-3
    assert float(d[..., V:].float().abs().max()) == 0.0
    assert float(d[:, -1].float().abs().max()) == 0.0  # last position has no target


@pytest.mark.parametrize("V,Vp,rows", [(5003, 5056, 40), (152167, 152192, 12)])
def test_ce_large_vocabulary(V, Vp, rows):
    """Text + unit vocabularies (interleaved tokeniser, ~152 k columns): the block-per-row two-pass kernel."""
    from slamkit_b200 import ops
    from oracle.lm_oracle import compute_loss
    B, T = 2, rows
    logits = torch.zeros(B, T, Vp, dtype=torch.bfloat16)
    logits[..., :V] = _randn(B, T, V, seed=4, scale=3.0)
    logits[..., V:] = 9.0
    g = torch.Generator().manual_seed(5)
    labels = torch.randint(0, V, (B, T), generator=g)
    labels[0, 3] = V - 1            # last real column
    labels[1, rows // 2:] = -100
    num_items = float((labels[:, 1:] != -100).sum())
    lf = logits[..., :V].float().requires_grad_(True)
    ref_loss = compute_loss(lf, labels, num_items)
    ref_loss.backward()
    stats, dlogits, row_nll = ops.ce_fwd_bwd(logits.view(B * T, Vp).to(DEV), labels.view(-1).to(DEV), T, V, num_items)
    assert abs(float(stats[0]) - float(ref_loss)) < 1e-5 * abs(float(ref_loss))
    assert int(stats[1]) == int(num_items)
    d = dlogits.cpu().view(B, T, Vp)
    assert rel_err(d[..., :V], lf.grad) < 4e-3, rel_err(d[..., :V], lf.grad)
    assert float(d[..., V:].float().abs().max()) == 0.0
    assert float(d[:, -1].float().abs().max()) == 0.0


# ---------------------------------------------------------------------------------------------- attention
def _attn_ref(qkv, B, T, H, KVH, causal, scale, d_o=None):
    hd = 64
    x = qkv.float().requires_grad_(True)
    q = x[:, :H * hd].view(B, T, H, hd).transpose(1, 2)
    k = x[:, H * hd:(H + KVH) * hd].view(B, T, KVH, hd).transpose(1, 2)
    v = x[:, (H + KVH) * hd:].view(B, T, KVH, hd).transpose(1, 2)
    rep = H // KVH
    k = k[:, :, None].expand(-1, -1, rep, -1, -1).reshape(B, H, T, hd)
    v = v[:, :, None].expand(-1, -1, rep, -1, -1).reshape(B, H, T, hd)
    s = (q @ k.transpose(-1, -2)) * scale
    if causal:
        s = s.masked_fill(torch.ones(T, T, dtype=torch.bool).triu(1), float("-inf"))
    p = torch.softmax(s, -1)
    o = (p @ v).transpose(1, 2).reshape(B * T, H * hd)
    lse = torch.logsumexp(s, -1)
    if d_o is not None:
        (o * d_o.float()).sum().backward()
        return o.detach(), lse.detach(), x.grad
    return o.detach(), lse.detach(), None


@pytest.mark.parametrize("B,T,H,KVH,causal", [(2, 256, 4, 2, True), (1, 1024, 14, 2, True), (2, 200, 2, 1, True),
                                              (2, 750, 12, 12, False), (1, 77, 2, 2, False)])
def test_attention_fwd_bwd(B, T, H, KVH, causal):
    from slamkit_b200 import ops
    hd = 64
    qkv = _randn(B * T, (H + 2 * KVH) * hd, seed=1)
    d_o = _randn(B * T, H * hd, seed=2)
    scale = 1.0 / math.sqrt(hd)
    o_ref, lse_ref, dqkv_ref = _attn_ref(qkv, B, T, H, KVH, causal, scale, d_o)
    o, lse = ops.attn_fwd(qkv.to(DEV), B, T, H, KVH, causal, scale)
    assert rel_err(o.cpu(), o_ref) < 5e-3, rel_err(o.cpu(), o_ref)
    assert max_abs(lse.cpu(), lse_ref) < 2e-3
    dqkv = ops.attn_bwd(qkv.to(DEV), o, d_o.to(DEV), lse, B, T, H, KVH, causal, scale).cpu()
    nq, nk = H * hd, (H + KVH) * hd
    assert rel_err(dqkv[:, :nq], dqkv_ref[:, :nq]) < 1e-2, "dq"
    assert rel_err(dqkv[:, nq:nk], dqkv_ref[:, nq:nk]) < 1e-2, "dk"
    assert rel_err(dqkv[:, nk:], dqkv_ref[:, nk:]) < 1e-2, "dv"


@pytest.mark.parametrize("B,T,H,KVH,causal", [(2, 256, 4, 2, True), (1, 1024, 14, 2, True), (2, 200, 2, 1, True),
                                              (2, 750, 4, 4, False), (1, 77, 2, 2, False), (8, 1024, 14, 2, True)])
def test_attention_tc_fwd(B, T, H, KVH, causal):
    """Fused-qkv forward entry point against the fp32 reference (one batch row at a time at the full LM shape)."""
    from slamkit_b200 import ops
    hd = 64
    qkv = _randn(B * T, (H + 2 * KVH) * hd, seed=5)
    scale = 1.0 / math.sqrt(hd)
    o, lse = ops.attn_tc_fwd(qkv.to(DEV), B, T, H, KVH, causal, scale)
    refs = [_attn_ref(qkv[b * T:(b + 1) * T], 1, T, H, KVH, causal, scale)[:2] for b in range(B)]
    o_ref = torch.cat([r[0].detach() for r in refs], 0)
    lse_ref = torch.cat([r[1].detach() for r in refs], 0)
    assert rel_err(o.cpu(), o_ref) < 5e-3, rel_err(o.cpu(), o_ref)
    assert max_abs(lse.cpu(), lse_ref) < 2e-3


@pytest.mark.parametrize("B,T,H,KVH,causal", [(2, 256, 4, 2, True), (1, 1024, 14, 2, True), (2, 200, 2, 1, True),
                                              (2, 750, 4, 4, False), (1, 77, 2, 2, False)])
def test_attention_tc_bwd(B, T, H, KVH, causal):
    from slamkit_b200 import ops
    hd = 64
    qkv = _randn(B * T, (H + 2 * KVH) * hd, seed=7)
    d_o = _randn(B * T, H * hd, seed=8)
    scale = 1.0 / math.sqrt(hd)
    _, _, dqkv_ref = _attn_ref(qkv, B, T, H, KVH, causal, scale, d_o)
    o, lse = ops.attn_tc_fwd(qkv.to(DEV), B, T, H, KVH, causal, scale)
    dqkv = ops.attn_tc_bwd(qkv.to(DEV), o, d_o.to(DEV), lse, B, T, H, KVH, causal, scale)
    dqkv2 = ops.attn_tc_bwd(qkv.to(DEV), o, d_o.to(DEV), lse, B, T, H, KVH, causal, scale)
    assert torch.equal(dqkv, dqkv2)   # deterministic
    dqkv = dqkv.cpu()
    nq, nk = H * hd, (H + KVH) * hd
    assert rel_err(dqkv[:, :nq], dqkv_ref[:, :nq]) < 1e-2, ("dq", rel_err(dqkv[:, :nq], dqkv_ref[:, :nq]))
    assert rel_err(dqkv[:, nq:nk], dqkv_ref[:, nq:nk]) < 1e-2, ("dk", rel_err(dqkv[:, nq:nk], dqkv_ref[:, nq:nk]))
    assert rel_err(dqkv[:, nk:], dqkv_ref[:, nk:]) < 1e-2, ("dv", rel_err(dqkv[:, nk:], dqkv_ref[:, nk:]))


def _packed_positions(B, T, seed):
    """position_ids of a packed batch: documents of random length (some length 1, some tile-aligned) until T is full."""
    g = torch.Generator().manual_seed(seed)
    pos = torch.zeros(B, T, dtype=torch.int64)
    for b in range(B):
        t = 0
        while t < T:
            n = int(torch.randint(1, 300, (1,), generator=g))
            if int(torch.randint(0, 4, (1,), generator=g)) == 0:
                n = 128 * int(torch.randint(1, 3, (1,), generator=g))      # a document that ends on a tile boundary
            n = min(n, T - t)
            pos[b, t:t + n] = torch.arange(n)
            t += n
    return pos


def test_seg_bounds_from_position_ids():
    from slamkit_b200 import ops
    pos = _packed_positions(3, 1000, seed=3)
    ss, se = ops.seg_bounds(pos.to(DEV))
    ss, se = ss.cpu().view(3, 1000), se.cpu().view(3, 1000)
    for b in range(3):
        starts = [t for t in range(1000) if t == 0 or pos[b, t] == 0] + [1000]
        want_s = torch.empty(1000, dtype=torch.int32); want_e = torch.empty(1000, dtype=torch.int32)
        for a, e in zip(starts[:-1], starts[1:]):
            want_s[a:e] = a; want_e[a:e] = e
        assert torch.equal(ss[b], want_s) and torch.equal(se[b], want_e)


@pytest.mark.parametrize("B,T,H,KVH", [(2, 640, 4, 2), (1, 1024, 14, 2), (2, 333, 2, 1)])
def test_attention_tc_packed_documents(B, T, H, KVH):
    """Packed batches: attention is causal inside a document and empty across documents (what the reference's varlen
    flash-attention path computes from position_ids).  fp32 reference with the explicit block-diagonal mask."""
    from slamkit_b200 import ops
    from oracle.lm_oracle import packed_mask
    hd = 64
    qkv = _randn(B * T, (H + 2 * KVH) * hd, seed=9)
    d_o = _randn(B * T, H * hd, seed=10)
    scale = 1.0 / math.sqrt(hd)
    pos = _packed_positions(B, T, seed=11)
    mask = packed_mask(pos)                                    # [B,1,T,T] bool
    x = qkv.float().requires_grad_(True)
    q = x[:, :H * hd].view(B, T, H, hd).transpose(1, 2)
    k = x[:, H * hd:(H + KVH) * hd].view(B, T, KVH, hd).transpose(1, 2)
    v = x[:, (H + KVH) * hd:].view(B, T, KVH, hd).transpose(1, 2)
    rep = H // KVH
    k = k[:, :, None].expand(-1, -1, rep, -1, -1).reshape(B, H, T, hd)
    v = v[:, :, None].expand(-1, -1, rep, -1, -1).reshape(B, H, T, hd)
    sc = ((q @ k.transpose(-1, -2)) * scale).masked_fill(~mask, float("-inf"))
    o_ref = (torch.softmax(sc, -1) @ v).transpose(1, 2).reshape(B * T, H * hd)
    lse_ref = torch.logsumexp(sc, -1).detach()
    (o_ref * d_o.float()).sum().backward()
    ss, se = ops.seg_bounds(pos.to(DEV))
    o, lse = ops.attn_tc_fwd(qkv.to(DEV), B, T, H, KVH, True, scale, seg_start=ss)
    assert rel_err(o.cpu(), o_ref.detach()) < 5e-3, rel_err(o.cpu(), o_ref.detach())
    assert max_abs(lse.cpu(), lse_ref) < 2e-3
    dqkv = ops.attn_tc_bwd(qkv.to(DEV), o, d_o.to(DEV), lse, B, T, H, KVH, True, scale, seg_start=ss, seg_end=se)
    dqkv2 = ops.attn_tc_bwd(qkv.to(DEV), o, d_o.to(DEV), lse, B, T, H, KVH, True, scale, seg_start=ss, seg_end=se)
    assert torch.equal(dqkv, dqkv2)
    dqkv = dqkv.cpu()
    nq, nk = H * hd, (H + KVH) * hd
    assert rel_err(dqkv[:, :nq], x.grad[:, :nq]) < 1e-2, ("dq", rel_err(dqkv[:, :nq], x.grad[:, :nq]))
    assert rel_err(dqkv[:, nq:nk], x.grad[:, nq:nk]) < 1e-2, ("dk", rel_err(dqkv[:, nq:nk], x.grad[:, nq:nk]))
    assert rel_err(dqkv[:, nk:], x.grad[:, nk:]) < 1e-2, ("dv", rel_err(dqkv[:, nk:], x.grad[:, nk:]))
    # one document per row == the plain causal kernel, bit for bit
    pos1 = torch.arange(T)[None].expand(B, -1).contiguous()
    s1, e1 = ops.seg_bounds(pos1.to(DEV))
    o1, lse1 = ops.attn_tc_fwd(qkv.to(DEV), B, T, H, KVH, True, scale, seg_start=s1)
    o0, lse0 = ops.attn_tc_fwd(qkv.to(DEV), B, T, H, KVH, True, scale)
    assert torch.equal(o1, o0) and torch.equal(lse1, lse0)


# ---------------------------------------------------------------------------------------------- optimiser
def test_adamw_matches_oracle_and_torch():
    from slamkit_b200 import ops
    from oracle.lm_oracle import adamw_step_
    n = 8 * 1000
    p, g = _randn(n, seed=1, scale=0.02), _randn(n, seed=2, scale=1e-3)
    m, v = _randn(n, seed=3, scale=1e-3), _randn(n, seed=4, scale=1e-3).abs()
    pd, gd, md, vd = (t.clone().to(DEV) for t in (p, g, m, v))
    po, mo, vo = p.clone(), m.clone(), v.clone()
    for step in (1, 2, 3):
        ops.adamw_step(pd, gd, md, vd, 1e-3, 0.9, 0.999, 1e-8, 0.01, step)
        adamw_step_(po, g, mo, vo, lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-8, weight_decay=0.01, step=step)
    for a, b, nm in ((pd, po, "p"), (md, mo, "m"), (vd, vo, "v")):
        # fp32 math with one bf16 rounding per step on both sides.  bf16 inputs make exact rounding ties common, so
        # fma contraction flips a few percent of results by one bf16 ulp (torch's own CPU and CUDA fused kernels
        # differ from each other the same way).
        assert (a.cpu() != b).float().mean() < 0.06, nm
        assert rel_err(a.cpu(), b) < 1e-3, nm
