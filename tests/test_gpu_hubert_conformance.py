"""Conformance of the HuBERT unit-extraction path per element, against the references of tests/hubert_ref.py.

The split-bf16 GEMM (sk_gemm_split) runs on operands whose three-product accumulator is exact in fp32, so its hi, lo and
fp32 outputs are compared bit for bit at the shapes of hubert_step.cu (mHuBERT-25Hz geometry), the strided-window conv
layers and the grouped positional conv with column compaction; every GEMM case first asserts the tile width it gets
(sk_gemm_split_plan).  Then guard bands, argument checks, the conv0 front and every stage of the real geometry (each
from the device's own previous stage, and every kernel inside each encoder layer from the device's own input to it),
k-means labels, prepared weights, and reads of never-written workspace.
References are computed in float64 on the GPU.
"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import gemm_ref as G
import hubert_ref as R

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
HERE = os.path.dirname(os.path.abspath(__file__))
LMAX = 64


# ----------------------------------------------------------------------------------------------------- the hook
def _desc(M, N, K, A, A_lo, B, B_lo, Cout, C_lo=None, *, batch=1, a_mode=0, lda=None, a_mn=0, a3d=(0, 0, 0, 0),
          ldb=None, ldc=None, out_f32=0, bias=None, bias_f32=1, res=None, res_lo=None, ldr=0, act=0, col=(0, 0),
          force_bn=0, passes=3):
    from slamkit_b200 import _lib as L
    p = lambda t: t.data_ptr() if t is not None else None
    d = L.SkGemmSplitDesc()
    d.M, d.N, d.K, d.batch, d.a_mode, d.passes = M, N, K, batch, a_mode, passes
    d.A, d.A_lo, d.lda, d.a_mn = p(A), p(A_lo), lda if lda is not None else K, a_mn
    d.a_inner, d.a_rows, d.a_row_stride, d.a_batch_stride = a3d
    d.B, d.B_lo, d.ldb = p(B), p(B_lo), ldb if ldb is not None else K
    d.C, d.C_lo, d.ldc, d.out_f32 = p(Cout), p(C_lo), ldc if ldc is not None else N, out_f32
    d.bias, d.bias_f32 = p(bias), bias_f32
    d.residual, d.residual_lo, d.ldr, d.act = p(res), p(res_lo), ldr, act
    d.col_gin, d.col_gout, d.force_bn = col[0], col[1], force_bn
    return d


def _plan(d):
    from slamkit_b200 import _lib as L
    lib = L.require_cuda()
    plan = L.SkGemmPlan()
    L.check(lib.sk_gemm_split_plan(C.byref(d), C.byref(plan)))
    return {name: int(getattr(plan, name)) for name, _ in L.SkGemmPlan._fields_}


def _run(d):
    from slamkit_b200 import _lib as L
    lib = L.require_cuda()
    L.check(lib.sk_gemm_split(C.byref(d), L.stream_ptr()))
    torch.cuda.synchronize()


def _expect_plan(d, bn):
    plan = _plan(d)
    assert plan["bn"] == bn and plan["splits"] == 1 and plan["sk_units"] == 0 and plan["tma_store"] == 0, plan
    return plan


def _ops(rows, cols, K, seed, lmax=LMAX):
    return R.split_int_operand(rows, cols, R.split_amax(K, lmax), lmax, seed, DEV)


def _check_hilo(hi, lo, want, rows_per_clip, group, what):
    for o, w, n in ((hi, want[0], "hi"), (lo, want[1], "lo")):
        rep = R.mismatch_exact(o, w, rows_per_clip, group, f"{what} {n}")
        assert rep is None, rep


# ----------------------------------------------------------------------------------------------------- a. split GEMM
# hubert_step.cu at the mHuBERT-25Hz geometry: (N, K, epilogue)
CALLS = {
    "proj": (768, 512, "bias_hilo"),
    "qkv": (2304, 768, "bias"),
    "oproj": (768, 768, "bias_res"),
    "ff1": (3072, 768, "gelu"),
    "ff2": (768, 3072, "bias_res"),
    "kmeans": (512, 768, "f32"),
}
SPLIT_M = [1, 127, 128, 129, 3000]
WIDTHS = [0, 64, 128, 256]


def split_case(M, N, K, epi, force_bn, seed=0):
    a = R.split_amax(K, LMAX)
    ah, al = _ops(M, K, K, seed)
    bh, bl = _ops(N, K, K, seed + 1)
    scale = G.acc_scale(K, a)
    g = torch.Generator(device=DEV).manual_seed(seed + 2)
    bias = torch.randn(N, generator=g, device=DEV) * scale if epi != "f32" else None
    rh = rl = None
    if epi == "bias_res":
        rh, rl = R.real_split((M, N), scale, seed + 3, DEV)
    f32 = epi == "f32"
    out = torch.empty(M, N, device=DEV, dtype=torch.float32 if f32 else torch.bfloat16)
    out_lo = None if f32 else torch.empty(M, N, device=DEV, dtype=torch.bfloat16)
    d = _desc(M, N, K, ah, al, bh, bl, out, out_lo, out_f32=int(f32), bias=bias, res=rh, res_lo=rl,
              ldr=N if rh is not None else 0, act=1 if epi == "gelu" else 0, force_bn=force_bn)
    bn = _expect_plan(d, R.pick_bn(M, N, force_bn))["bn"]
    _run(d)
    acc = R.split_exact_acc(ah, al, bh, bl)
    what = f"M={M} N={N} K={K} {epi} bn={bn}"
    if epi == "gelu":
        v = R.split_epilogue(acc, bias, out_f32=True)
        g_ = G.gelu_exact(v)
        rep = R.mismatch_bound(R.hilo(out, out_lo), g_, R.gelu_bound(v, g_), M, bn, what)
        assert rep is None, rep
    elif f32:
        rep = R.mismatch_exact(out, R.split_epilogue(acc, out_f32=True), M, bn, what)
        assert rep is None, rep
    else:
        _check_hilo(out, out_lo, R.split_epilogue(acc, bias, rh, rl), M, bn, what)


@pytest.mark.parametrize("force_bn", WIDTHS, ids=lambda b: f"bn{b or 'auto'}")
@pytest.mark.parametrize("M", SPLIT_M)
@pytest.mark.parametrize("call", list(CALLS))
def test_split_gemm_exact(call, M, force_bn):
    N, K, epi = CALLS[call]
    split_case(M, N, K, epi, force_bn)


def test_split_gemm_several_tiles_per_cta_at_bn256():
    """N 768 at M 6000: 47 x 3 = 141 tiles at BN 256 on 132 SMs, so CTAs run a second tile through the pair-slot ring
    (qkv and ff1 at M 3000 do the same at 216 and 288 tiles)."""
    split_case(6000, 768, 768, "bias_res", 256)
    split_case(6000, 768, 768, "bias_res", 0)


@pytest.mark.parametrize("K", [64, 576, 832])
@pytest.mark.parametrize("force_bn", WIDTHS, ids=lambda b: f"bn{b or 'auto'}")
def test_split_gemm_odd_kblock_counts(K, force_bn):
    """1, 9 and 13 k-blocks: the pair-slot ring wraps on an odd count."""
    split_case(3000, 768, K, "bias_hilo", force_bn)
    split_case(129, 768, K, "bias_hilo", force_bn)


# ----------------------------------------------------------------------------------------------------- b. windowed conv
@pytest.mark.parametrize("act", [0, 1], ids=["linear", "gelu"])
@pytest.mark.parametrize("Mc", [1, 63, 127, 128, 129, 750])
@pytest.mark.parametrize("k,st", [(3, 2), (2, 2)])
def test_windowed_conv_exact(k, st, Mc, act):
    B, Cc = 3, 512
    T_in = (Mc - 1) * st + k                       # the last window ends at the clip's end
    K = k * Cc
    ah, al = _ops(B * T_in, Cc, K, 10 + Mc)
    wh, wl = _ops(Cc, K, K, 11)
    out, out_lo = torch.empty(B * Mc, Cc, device=DEV, dtype=torch.bfloat16), torch.empty(B * Mc, Cc, device=DEV, dtype=torch.bfloat16)
    d = _desc(Mc, Cc, K, ah, al, wh, wl, out, out_lo, batch=B, a3d=(K, Mc, st * Cc, T_in * Cc), act=act)
    bn = _expect_plan(d, R.pick_bn(B * Mc, Cc))["bn"]
    _run(d)
    acc = R.split_exact_acc(R.window_rows(ah, B, Mc, k, st, Cc), R.window_rows(al, B, Mc, k, st, Cc), wh, wl)
    what = f"conv k={k} st={st} B={B} M={Mc} bn={bn}"
    if act:
        v = R.split_epilogue(acc, out_f32=True)
        g = G.gelu_exact(v)
        rep = R.mismatch_bound(R.hilo(out, out_lo), g, R.gelu_bound(v, g), Mc, bn, what)
        assert rep is None, rep
    else:
        _check_hilo(out, out_lo, R.split_epilogue(acc), Mc, bn, what)


# ----------------------------------------------------------------------------------------------------- c. positional conv
def posconv_case(Kpos, cg, Tf, B=2, act=0, seed=0):
    groups = 16 if cg == 48 else 4
    halo = Kpos // 2
    Tp = Tf + 2 * halo
    GP = groups * R.GROUP_PAD
    K = Kpos * R.GROUP_PAD
    xh, xl = _ops(B * Tp, GP, K, seed + Tf)
    wh, wl = _ops(GP, K, K, seed + 1)
    bias = torch.randn(GP, generator=torch.Generator(device=DEV).manual_seed(seed + 2), device=DEV) * G.acc_scale(K, 2)
    H = groups * cg
    out, out_lo = torch.empty(B * Tf, H, device=DEV, dtype=torch.bfloat16), torch.empty(B * Tf, H, device=DEV, dtype=torch.bfloat16)
    d = _desc(Tf, GP, K, xh, xl, wh, wl, out, out_lo, batch=B, a_mode=1, a3d=(GP, Tp, GP, Tp * GP), ldc=H, bias=bias,
              act=act, col=(R.GROUP_PAD, cg))
    _expect_plan(d, 64)
    _run(d)
    sh = (B, Tp, GP)
    acc = R.posconv_split_acc(xh.view(sh), xl.view(sh), wh, wl, Tf, Kpos, groups)
    what = f"posconv Kpos={Kpos} cg={cg} Tf={Tf} B={B}"
    if act:
        v = R.split_epilogue(acc, bias, out_f32=True, col_gin=R.GROUP_PAD, col_gout=cg)
        g = G.gelu_exact(v)
        rep = R.mismatch_bound(R.hilo(out, out_lo), g, R.gelu_bound(v, g), Tf, cg, what)
        assert rep is None, rep
    else:
        _check_hilo(out, out_lo, R.split_epilogue(acc, bias, col_gin=R.GROUP_PAD, col_gout=cg), Tf, cg, what)


@pytest.mark.parametrize("Tf", [1, 63, 64, 65, 127, 128, 129, 750])
@pytest.mark.parametrize("cg", [48, 64, 32, 16, 8])
@pytest.mark.parametrize("Kpos", [2, 16, 128])
def test_posconv_exact(Kpos, cg, Tf):
    posconv_case(Kpos, cg, Tf)


@pytest.mark.parametrize("Tf", [129, 750])
def test_posconv_gelu_real_groups(Tf):
    posconv_case(128, 48, Tf, B=3, act=1)


# ----------------------------------------------------------------------------------------------------- d. guard bands
def _nan_bits(t):
    return t.view(torch.int16) if t.dtype == torch.bfloat16 else t.view(torch.int32)


@pytest.mark.parametrize("call", ["proj", "kmeans"])
def test_guard_bands(call):
    """Outputs inside NaN-sentinel buffers with a pitch gap and rows past M; A and B pitched with NaN beyond K."""
    N, K, epi = CALLS[call]
    M, pad_c, pad_r = 129, 24, 7
    f32 = epi == "f32"
    ah, al = _ops(M, K, K, 3)
    bh, bl = _ops(N, K, K, 4)
    nanpad = lambda t, extra: torch.cat([t, torch.full((t.shape[0], extra), float("nan"), device=DEV, dtype=t.dtype)], 1)
    A, Al, Bh, Bl = nanpad(ah, 64), nanpad(al, 64), nanpad(bh, 72), nanpad(bl, 72)
    dt = torch.float32 if f32 else torch.bfloat16
    out = torch.full((M + pad_r, N + pad_c), float("nan"), device=DEV, dtype=dt)
    out_lo = None if f32 else torch.full((M + pad_r, N + pad_c), float("nan"), device=DEV, dtype=dt)
    sent = [_nan_bits(t).clone() for t in (out, out_lo) if t is not None]
    bias = None if f32 else torch.randn(N, device=DEV) * 100
    d = _desc(M, N, K, A, Al, Bh, Bl, out, out_lo, lda=K + 64, ldb=K + 72, ldc=N + pad_c, out_f32=int(f32), bias=bias)
    _expect_plan(d, R.pick_bn(M, N))
    _run(d)
    acc = R.split_exact_acc(ah, al, bh, bl)
    if f32:
        assert R.mismatch_exact(out[:M, :N], R.split_epilogue(acc, out_f32=True), M) is None
    else:
        _check_hilo(out[:M, :N], out_lo[:M, :N], R.split_epilogue(acc, bias), M, 64, "guard")
    for t, s in zip([t for t in (out, out_lo) if t is not None], sent):
        bits = _nan_bits(t)
        assert torch.equal(bits[:, N:], s[:, N:]), "pitch gap written"
        assert torch.equal(bits[M:], s[M:]), "rows past M written"


def test_guard_bands_batched_conv_and_compaction():
    """Batched conv output: rows past B*M stay untouched; compacted pos-conv output with a pitch gap."""
    B, Mc, k, st, Cc = 2, 130, 3, 2, 512
    T_in = (Mc - 1) * st + k
    K = k * Cc
    ah, al = _ops(B * T_in, Cc, K, 5)
    wh, wl = _ops(Cc, K, K, 6)
    out = torch.full((B * Mc + 5, Cc), float("nan"), device=DEV, dtype=torch.bfloat16)
    out_lo = out.clone()
    d = _desc(Mc, Cc, K, ah, al, wh, wl, out, out_lo, batch=B, a3d=(K, Mc, st * Cc, T_in * Cc))
    _expect_plan(d, R.pick_bn(B * Mc, Cc))
    _run(d)
    assert torch.isnan(out[B * Mc:].float()).all() and torch.isnan(out_lo[B * Mc:].float()).all()
    acc = R.split_exact_acc(R.window_rows(ah, B, Mc, k, st, Cc), R.window_rows(al, B, Mc, k, st, Cc), wh, wl)
    _check_hilo(out[:B * Mc], out_lo[:B * Mc], R.split_epilogue(acc), Mc, 64, "batched conv guard")
    # compaction into a pitched output: columns past G*cg never written
    groups, cg, Kpos, Tf = 4, 48, 16, 65
    halo, GP = Kpos // 2, groups * 64
    Tp = Tf + 2 * halo
    xh, xl = _ops(B * Tp, GP, Kpos * 64, 7)
    ph, pl = _ops(GP, Kpos * 64, Kpos * 64, 8)
    ldc = groups * cg + 16
    o = torch.full((B * Tf, ldc), float("nan"), device=DEV, dtype=torch.bfloat16)
    ol = o.clone()
    d = _desc(Tf, GP, Kpos * 64, xh, xl, ph, pl, o, ol, batch=B, a_mode=1, a3d=(GP, Tp, GP, Tp * GP), ldc=ldc,
              col=(64, cg))
    _expect_plan(d, 64)
    _run(d)
    assert torch.isnan(o[:, groups * cg:].float()).all() and torch.isnan(ol[:, groups * cg:].float()).all()
    acc = R.posconv_split_acc(xh.view(B, Tp, GP), xl.view(B, Tp, GP), ph, pl, Tf, Kpos, groups)
    _check_hilo(o[:, :groups * cg], ol[:, :groups * cg], R.split_epilogue(acc, col_gin=64, col_gout=cg), Tf, cg, "posconv guard")


# ----------------------------------------------------------------------------------------------------- e. argument checks
def test_argument_checks_launch_nothing():
    from slamkit_b200 import _lib as L
    lib = L.require_cuda()
    M, N, K = 128, 256, 512
    ah, al = _ops(M, K, K, 0)
    bh, bl = _ops(N, K, K, 1)
    out = torch.full((M, N), float("nan"), device=DEV, dtype=torch.bfloat16)
    out_lo = out.clone()
    bad = {
        "a_mode 1 without the 3-D view": _desc(M, N, K, ah, al, bh, bl, out, out_lo, a_mode=1),
        "passes 3 without lo operands": _desc(M, N, K, ah, None, bh, None, out, out_lo),
        "force_bn 192": _desc(M, N, K, ah, al, bh, bl, out, out_lo, force_bn=192),
        "force_bn 224": _desc(M, N, K, ah, al, bh, bl, out, out_lo, force_bn=224),
        "MN-major 3-D A": _desc(M, N, K, ah, al, bh, bl, out, out_lo, a_mn=1, a3d=(K, M, K, M * K)),
    }
    torch.cuda.synchronize()
    for what, d in bad.items():
        before = int(lib.sk_launch_count())
        plan = L.SkGemmPlan()
        assert lib.sk_gemm_split_plan(C.byref(d), C.byref(plan)) != 0, f"{what}: plan accepted"
        assert lib.sk_gemm_split(C.byref(d), L.stream_ptr()) != 0, f"{what}: launch accepted"
        assert int(lib.sk_launch_count()) == before, f"{what}: something was launched"
    torch.cuda.synchronize()
    assert torch.isnan(out.float()).all() and torch.isnan(out_lo.float()).all()


# ----------------------------------------------------------------------------------------------------- feature extractor
def _fe(layer=2, conv_kernel=None, conv_stride=None, max_batch=3, max_samples=160000, seed=0):
    from slamkit_b200.feature_extractor import HubertB200Config, HubertB200FeatureExtractor, random_params
    kw = {}
    if conv_kernel:
        kw = dict(conv_kernel=conv_kernel, conv_stride=conv_stride)
    cfg = HubertB200Config(layer=layer, **kw)
    p = random_params(cfg, seed)
    return HubertB200FeatureExtractor(cfg, p, device=DEV, max_batch=max_batch, max_samples=max_samples), p


def _fe_tensor(fe, name):
    """One tensor of the flat fp32 weight buffer (prepared layout), on the device."""
    lib, h = fe.lib, fe._h
    buf = C.create_string_buffer(64)
    for i in range(lib.sk_hubert_tensor_info(h, -1, None, 0, None, None, None)):
        off, r, c = C.c_int64(), C.c_int32(), C.c_int32()
        lib.sk_hubert_tensor_info(h, i, buf, 64, C.byref(off), C.byref(r), C.byref(c))
        if buf.value.decode() == name:
            return fe.weights[off.value:off.value + r.value * c.value].view(r.value, c.value), off.value
    raise KeyError(name)


def _frames(cfg, S):
    L, T = S + 2 * cfg.pad, []
    for k, s in zip(cfg.conv_kernel, cfg.conv_stride):
        L = (L - k) // s + 1
        T.append(L)
    return T


# ----------------------------------------------------------------------------------------------------- f. conv0 front
def conv0_case(fe, wav):
    cfg = fe.config
    B, S = wav.shape
    KW, ST = cfg.conv_kernel[0], cfg.conv_stride[0]
    T0 = _frames(cfg, S)[0]
    got = fe.debug_stage(wav, 100, B * T0, cfg.conv_dim).double()
    w, _ = _fe_tensor(fe, "conv0.w")
    gamma, beta = _fe_tensor(fe, "gn.g")[0][0], _fe_tensor(fe, "gn.b")[0][0]
    want, z, mag = R.conv0_reference(wav.to(DEV), w, gamma, beta, cfg.pad, KW, ST)
    C_ = cfg.conv_dim
    rep = R.mismatch_bound(got, want.reshape(-1, C_), R.conv0_bound(z, want, mag, KW).reshape(-1, C_), T0, 64,
                           f"conv0 KW={KW} ST={ST} B={B} S={S} T0={T0}")
    assert rep is None, rep


@pytest.fixture(scope="module")
def fe_real():
    return _fe()


@pytest.mark.parametrize("T0", [143, 511, 512, 513, 1023, 1025])
def test_conv0_frame_sweep(fe_real, T0):
    fe, _ = fe_real
    S = 5 * T0 - 75                                  # (S + 80 - 10) / 5 + 1 = T0
    assert _frames(fe.config, S)[0] == T0
    g = torch.Generator().manual_seed(T0)
    wav = (0.1 * torch.randn(3, S, generator=g)).clamp(-1, 1)
    wav[1, S // 2:] = 0                              # ragged clips with zero tails
    wav[2, S // 5:] = 0
    conv0_case(fe, wav)


def test_conv0_special_clips(fe_real):
    fe, _ = fe_real
    S = 16000
    g = torch.Generator().manual_seed(1)
    wav = torch.stack([torch.zeros(S),                                            # silence: var 0 -> GELU(beta)
                       torch.where(torch.rand(S, generator=g) < 0.5, -1.0, 1.0),   # full scale
                       0.5 + 1e-3 * torch.randn(S, generator=g)])                  # DC offset + small noise
    conv0_case(fe, wav)


def test_conv0_generic_kernel():
    """A (8, 4) first layer takes the generic conv0 kernel."""
    fe, _ = _fe(layer=1, conv_kernel=(8, 3, 3, 3, 3, 2, 2, 2), conv_stride=(4, 2, 2, 2, 2, 2, 2, 2), max_samples=20000)
    g = torch.Generator().manual_seed(2)
    wav = (0.1 * torch.randn(2, 12345, generator=g)).clamp(-1, 1)
    wav[1, 7000:] = 0
    conv0_case(fe, wav)


def _conv0_packed_child():
    fe, _ = _fe(layer=1, conv_kernel=(8, 3, 3, 3, 3, 2, 2, 2), conv_stride=(4, 2, 2, 2, 2, 2, 2, 2), max_samples=20000)
    g = torch.Generator().manual_seed(3)
    conv0_case(fe, (0.1 * torch.randn(2, 12345, generator=g)).clamp(-1, 1))
    fe2, _ = _fe(layer=1, max_samples=20000)
    conv0_case(fe2, (0.1 * torch.randn(2, 16000, generator=g)).clamp(-1, 1))


def test_conv0_packed_pair_variant_in_child():
    """SK_CONV0_MODE=1 (read once per process) selects the packed-pair generic kernel for every geometry."""
    env = dict(os.environ, SK_CONV0_MODE="1")
    code = (f"import sys; sys.path[:0] = [{HERE!r}, {os.path.dirname(HERE)!r}]; "
            "import test_gpu_hubert_conformance as T; T._conv0_packed_child(); print('ok')")
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "ok" in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]


# ----------------------------------------------------------------------------------------------------- g. stage isolation
@pytest.fixture(scope="module")
def stages(fe_real):
    """B = 3 ragged clips of about 10 s at the real geometry; every stage the device computes, as fp32 on the device."""
    fe, p = fe_real
    cfg = fe.config
    S = 160000
    g = torch.Generator().manual_seed(5)
    wav = (0.1 * torch.randn(3, S, generator=g)).clamp(-1, 1)
    wav[1, 131000:] = 0
    wav[2, 97000:] = 0
    T = _frames(cfg, S)
    st = {f"conv{i}": fe.debug_stage(wav, 100 + i, 3 * T[i], cfg.conv_dim) for i in range(8)}
    st["proj"] = fe.debug_stage(wav, 200, 3 * T[-1], cfg.hidden)
    st["pos"] = fe.debug_stage(wav, 201, 3 * T[-1], cfg.hidden)
    st["embed"] = fe.debug_stage(wav, 0, 3 * T[-1], cfg.hidden)
    M = 3 * T[-1]
    for l in range(cfg.layer):
        for j, cols in enumerate((3 * cfg.hidden, cfg.hidden, cfg.hidden, cfg.hidden, cfg.ffn, cfg.hidden)):
            st[f"layer{l}.{j}"] = fe.debug_stage(wav, 300 + 10 * l + j, M, cols)
        st[f"layer{l}.out"] = fe.debug_stage(wav, l + 1, M, cfg.hidden)
    return fe, wav, T, st


@pytest.mark.parametrize("i", range(1, 8))
def test_stage_conv_layer(stages, i):
    fe, wav, T, st = stages
    cfg = fe.config
    Cc, k, s = cfg.conv_dim, cfg.conv_kernel[i], cfg.conv_stride[i]
    xh, xl = R.split_f32(st[f"conv{i - 1}"])
    wh, wl = R.split_f32(_fe_tensor(fe, f"conv{i}.w")[0])
    rows = R.boundary_rows(T[i], 3, 0.1, seed=i).to(DEV)
    ah, al = R.window_rows(xh, 3, T[i], k, s, Cc)[rows], R.window_rows(xl, 3, T[i], k, s, Cc)[rows]
    ref = ah.double() @ wh.double().t() + ah.double() @ wl.double().t() + al.double() @ wh.double().t()
    g = G.gelu_exact(ref)
    bound = 1.13 * R.split_random_bound(ah, al, wh, wl, ref, hilo_out=False) + R.gelu_bound(ref, g)
    got = st[f"conv{i}"][rows]
    rep = R.mismatch_bound(got, g, bound, len(rows), 64, f"conv{i} (rows sampled; row = index into the sample)")
    assert rep is None, rep


def test_stage_projection(stages):
    fe, wav, T, st = stages
    cfg = fe.config
    x = st["conv7"].double()
    gamma, beta = _fe_tensor(fe, "fp.ln.g")[0][0], _fe_tensor(fe, "fp.ln.b")[0][0]
    ln, mean, rstd = R.layernorm_reference(x, gamma, beta, cfg.ln_eps)
    ln_err = R.layernorm_bound(x, gamma, ln, mean, rstd)
    w, _ = _fe_tensor(fe, "fp.w")
    b = _fe_tensor(fe, "fp.b")[0][0]
    wh, wl = R.split_f32(w)
    lh, ll = R.split_f32(ln.float())
    ref = ln @ R.hilo(wh, wl).t() + b.double()
    bound = ln_err @ w.double().abs().t() + R.split_random_bound(lh, ll, wh, wl, ref, extra_abs=b.double().abs()) \
        + (ln.abs() @ (w.double() - R.hilo(wh, wl)).abs().t())
    rep = R.mismatch_bound(st["proj"].double(), ref, bound, T[-1], 64, "projection")
    assert rep is None, rep


def test_stage_positional_conv(stages):
    fe, wav, T, st = stages
    cfg = fe.config
    Tf, G_, Kpos = T[-1], cfg.pos_conv_groups, cfg.pos_conv_kernel
    cg = cfg.hidden // G_
    xh, xl = R.split_f32(st["proj"])
    sh = R.regroup_pad(xh, 3, Tf, Kpos // 2, G_, cg)
    sl = R.regroup_pad(xl, 3, Tf, Kpos // 2, G_, cg)
    w, _ = _fe_tensor(fe, "pos.w")
    b = _fe_tensor(fe, "pos.b")[0][0]
    wh, wl = R.split_f32(w)
    acc = R.posconv_split_acc(sh, sl, wh, wl, Tf, Kpos, G_, exact=False)
    absacc = R.posconv_split_acc(sh.abs(), sl.abs(), wh.abs(), wl.abs(), Tf, Kpos, G_, exact=False)
    v = R.compact_columns(acc + b.double(), 64, cg)
    g = G.gelu_exact(v)
    acc_err = R.compact_columns(3 * Kpos * 64 * R.U23 * absacc + 2 * R.U24 * (acc.abs() + b.double().abs()), 64, cg)
    bound = 1.13 * acc_err + R.gelu_bound(v, g)
    rep = R.mismatch_bound(st["pos"].double(), g, bound, Tf, cg, "positional conv")
    assert rep is None, rep


def test_stage_embed_layernorm(stages):
    fe, wav, T, st = stages
    cfg = fe.config
    x = st["proj"].double() + st["pos"].double()
    gamma, beta = _fe_tensor(fe, "enc.ln.g")[0][0], _fe_tensor(fe, "enc.ln.b")[0][0]
    ref, mean, rstd = R.layernorm_reference(x, gamma, beta, cfg.ln_eps)
    bound = R.layernorm_bound(x, gamma, ref, mean, rstd, hilo_out=False)
    rep = R.mismatch_bound(st["embed"].double(), ref, bound, T[-1], 64, "embed LayerNorm (fp32 copy)")
    assert rep is None, rep


LAYER_STEPS = ["qkv", "attention", "oproj", "ln1", "ff1", "ff2", "ln2"]


@pytest.mark.parametrize("step", LAYER_STEPS)
@pytest.mark.parametrize("l", [0, 1])
def test_stage_encoder_layer(stages, l, step):
    """Every kernel of encoder layer l, from the device's own input to it (the taps of sk_hubert_debug_stage), against
    its float64 reference and its own bound (hubert_ref: linear_with_bound, attention_with_bound, layernorm_with_bound).
    The device reads each input as the hi/lo pair its fp32 tap is the exact sum of."""
    fe, wav, T, st = stages
    cfg = fe.config
    Tf, nh = T[-1], cfg.n_heads
    w = lambda n: _fe_tensor(fe, f"layers.{l}.{n}")[0]
    vec = lambda n: w(n)[0]
    pair = lambda t: R.hilo(*R.split_f32(t))
    x0 = pair(st["embed"] if l == 0 else st[f"layer{l - 1}.out"])
    tap = lambda j: pair(st[f"layer{l}.{j}"])
    if step == "qkv":
        got, (want, bound) = st[f"layer{l}.0"], R.linear_with_bound(x0, None, w("wqkv"), vec("bqkv"))
    elif step == "attention":
        got, (want, bound) = st[f"layer{l}.1"], R.attention_with_bound(tap(0), None, 3, Tf, nh, 1.0 / 8.0)
    elif step == "oproj":
        got, (want, bound) = st[f"layer{l}.2"], R.linear_with_bound(tap(1), None, w("wo"), vec("bo"), res=x0)
    elif step == "ln1":
        got, (want, bound) = st[f"layer{l}.3"], R.layernorm_with_bound(tap(2), None, vec("ln1.g"), vec("ln1.b"), cfg.ln_eps)
    elif step == "ff1":
        got, (want, bound) = st[f"layer{l}.4"], R.linear_with_bound(tap(3), None, w("ff1.w"), vec("ff1.b"), act=1)
    elif step == "ff2":
        got, (want, bound) = st[f"layer{l}.5"], R.linear_with_bound(tap(4), None, w("ff2.w"), vec("ff2.b"), res=tap(3))
    else:
        got, (want, bound) = st[f"layer{l}.out"], R.layernorm_with_bound(tap(5), None, vec("ln2.g"), vec("ln2.b"),
                                                                         cfg.ln_eps, hilo_out=False)
    rep = R.mismatch_bound(got.double(), want, bound, Tf, 64, f"layer {l} {step}")
    assert rep is None, rep


# ----------------------------------------------------------------------------------------------------- h. units
def test_units_are_the_fp64_argmin_of_the_device_features(fe_real):
    fe, p = fe_real
    S = 160000
    g = torch.Generator().manual_seed(8)
    wav = (0.1 * torch.randn(3, S, generator=g)).clamp(-1, 1)
    wav[2, 90000:] = 0
    feat = fe.features(wav).reshape(-1, fe.config.hidden)
    ids, nf = fe.units_device(wav, None)
    centers = p["kmeans.centers"].to(DEV)
    want, margin = R.kmeans_labels_with_margin(feat, centers)
    bound = R.kmeans_margin_bound(feat, centers)
    diff = (ids.reshape(-1).long() != want)
    assert bool((margin[diff] < bound[diff]).all()), (diff.nonzero()[:5].flatten().tolist(), margin[diff][:5], bound[diff][:5])
    assert int(diff.sum()) <= max(1, ids.numel() // 1000), int(diff.sum())
    assert int(ids.min()) >= 0 and int(ids.max()) < fe.config.n_units


def test_n_frames_exact(fe_real):
    fe, _ = fe_real
    S = 160000
    T = _frames(fe.config, S)[-1]
    r = torch.arange(S + 1, dtype=torch.float32)
    prod = (r / S) * T
    on_int = (prod == prod.round()).nonzero().flatten()[1:4].tolist()    # float32 products that land on an integer
    lens = [0, 1, S - 1, S, S + 1] + on_int
    wav = torch.zeros(len(lens), S)
    ids, nf = fe.units_device(wav, torch.tensor(lens))
    assert nf.cpu().tolist() == R.rel_len(torch.tensor(lens), S, T).tolist()
    _, nf0 = fe.units_device(wav[:2], None)
    assert nf0.cpu().tolist() == [T, T]


def test_kmeans_all_nan_rows_get_label_zero():
    from slamkit_b200 import _lib as L
    lib = L.require_cuda()
    g = torch.Generator(device=DEV).manual_seed(0)
    M, U, ld = 64, 500, 512
    dot = torch.randn(M, ld, generator=g, device=DEV)
    csq = torch.rand(U, generator=g, device=DEV) * 10
    dot[5] = float("nan")
    dot[40] = float("nan")
    dot[41, :U:2] = float("nan")                    # some NaN distances: the finite ones decide
    labels = torch.full((M,), -7, dtype=torch.int32, device=DEV)
    L.check(lib.sk_kmeans_argmin(L.ptr(dot), L.ptr(csq), L.ptr(labels), M, U, ld, L.stream_ptr()))
    got = labels.cpu()
    d = (csq[None, :] + -2.0 * dot[:, :U]).cpu()
    want = torch.where(torch.isnan(d), torch.tensor(float("inf")), d).argmin(1).to(torch.int32)
    assert got[5] == 0 and got[40] == 0
    fin = [i for i in range(M) if i not in (5, 40)]
    assert torch.equal(got[fin], want[fin])


def test_extract_rejects_non_finite_audio(fe_real):
    fe, _ = fe_real
    wav = 0.1 * torch.randn(2, 16000, generator=torch.Generator().manual_seed(4))
    ok = fe.extract(wav)
    wav[1, 1234] = float("nan")
    with pytest.raises(ValueError):
        fe.extract(wav)
    ids, _ = fe.units_device(wav, None)
    assert int(ids.min()) >= 0 and int(ids.max()) < fe.config.n_units
    assert np.array_equal(fe.extract(wav[:1])[0], ok[0])


# ----------------------------------------------------------------------------------------------------- i. prepared weights
def test_prepared_weights_bitwise(fe_real):
    fe, _ = fe_real
    fe.prepared.fill_(0xFF)
    fe._bind(3, 160000)
    torch.cuda.synchronize()
    n = int(fe.lib.sk_hubert_param_count(fe._h))
    half = (n * 2 + 255) // 256 * 256
    hi = fe.prepared[:n * 2].view(torch.bfloat16)
    lo = fe.prepared[half:half + n * 2].view(torch.bfloat16)
    wh, wl = R.split_f32(fe.weights)
    assert torch.equal(hi.view(torch.int16), wh.view(torch.int16)), "w_hi differs from the host split"
    assert torch.equal(lo.view(torch.int16), wl.view(torch.int16)), "w_lo differs from the host split"
    km, off = _fe_tensor(fe, "km.centers")
    U = fe.config.n_units
    assert km.shape[0] % 64 == 0 and bool((hi[off + U * km.shape[1]:off + km.numel()].float() == 0).all())
    csq = fe.prepared[2 * half:2 * half + 4 * km.shape[0]].view(torch.float32)
    ref = (km.double() ** 2).sum(1)
    assert bool(((csq.double() - ref).abs() <= km.shape[1] * R.U24 * ref + 1e-30).all())
    assert bool((csq[U:] == 0).all())


# ----------------------------------------------------------------------------------------------------- j. workspace, determinism
def test_poisoned_workspace_and_determinism(fe_real):
    """units / features on a workspace filled with 0xFF (NaN in bf16 and fp32) and on a zeroed one are bit-identical:
    no kernel reads workspace it did not write (halo rows, pad channels, conv ping-pong buffers, Upad columns)."""
    fe, _ = fe_real
    S = 160000
    g = torch.Generator().manual_seed(6)
    wav = (0.1 * torch.randn(3, S, generator=g)).clamp(-1, 1)
    wav[1, 100000:] = 0
    lens = torch.tensor([S, 100000, S])
    outs = []
    for fill in (0xFF, 0x00, 0xFF):
        fe.workspace.fill_(fill)
        ids, nf = fe.units_device(wav, lens)
        fe.workspace.fill_(fill)
        feat = fe.features(wav)
        outs.append((ids.clone(), nf.clone(), feat.clone()))
    for ids, nf, feat in outs[1:]:
        assert torch.equal(ids, outs[0][0]) and torch.equal(nf, outs[0][1])
        assert torch.equal(feat.view(torch.int32), outs[0][2].view(torch.int32))
    assert bool(torch.isfinite(outs[0][2]).all())
    # a clip alone and inside a batch of the same S
    alone = fe.features(wav[1:2])
    assert torch.equal(alone[0].view(torch.int32), outs[0][2][1].view(torch.int32))
    ids1, _ = fe.units_device(wav[2:3], None)
    assert torch.equal(ids1[0], outs[0][0][2])
