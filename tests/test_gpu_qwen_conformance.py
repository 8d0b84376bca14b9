"""Conformance of the Qwen2 layer's own kernels per element, against the references of tests/qwen_ref.py: RMSNorm forward
and backward, RoPE forward and inverse (standalone), SwiGLU forward and backward (standalone, over every bf16 gate bit
pattern), and the SwiGLU and RoPE epilogues fused into the GEMM.

Fused cases use operands that make the fp32 accumulator exact (integers, or one-hot rows that pass a chosen weight
through unchanged), then apply the element-wise reference; each one first asks the planner (sk_neox_gemm_plan) for its
tile width and epilogue warps and asserts them.  The shapes are chosen for 132 SMs.  Outputs sit between NaN guard
bands, or inside sentinel-filled pitched buffers, that must stay untouched.  Also: a dependent rmsnorm -> SwiGLU
forward -> SwiGLU backward -> rmsnorm backward chain on one stream, and the argument checks that refuse a launch."""
import ctypes as C
import os
import subprocess
import sys
import time

import numpy as np
import pytest
import torch

import gemm_ref as R
import qwen_ref as Q

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
BF = torch.bfloat16
PAD = 64
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SENT16 = 0x7FB5          # a NaN payload no kernel produces


def _lib():
    from slamkit_b200 import _lib as L
    return L, L.require_cuda()


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def _guarded(shape, dtype, fill=None):
    """(buffer, view): a device tensor of `shape` between PAD-element NaN guard bands."""
    n = int(np.prod(shape))
    buf = torch.full((n + 2 * PAD,), float("nan"), dtype=dtype, device=DEV)
    view = buf[PAD:PAD + n].view(*shape)
    if fill is not None:
        view.copy_(torch.as_tensor(np.asarray(fill), dtype=torch.float32).to(dtype).reshape(shape))
    return buf, view


def _guard_ok(buf):
    return bool(buf[:PAD].isnan().all()) and bool(buf[-PAD:].isnan().all())


def _np(t):
    return t.float().cpu().numpy()


def _dev(a, dtype=BF):
    return torch.as_tensor(np.asarray(a, np.float32)).to(dtype).to(DEV)


@pytest.fixture(scope="module", autouse=True)
def _timer():
    t0 = time.time()
    yield
    print(f"\ntest_gpu_qwen_conformance: {time.time() - t0:.1f} s")


def _plan(kind, M, N, K):
    L, lib = _lib()
    p = L.SkGemmPlan()
    L.check(lib.sk_neox_gemm_plan(kind, M, N, K, 0, C.byref(p)))
    return {f: int(getattr(p, f)) for f, _ in L.SkGemmPlan._fields_}


def _mode(kind, plan):
    """Where the tile is finished: from the wgmma registers (one-pass SwiGLU forward on 4 epilogue warps, as the header
    documents) or from the parked accumulator."""
    return "register" if kind == 4 and plan["epi_warps"] == 4 and plan["tma_store"] and plan["sk_units"] == 0 else "parked"


def _sm_note():
    _, lib = _lib()
    n = lib.sk_device_sm_count()
    return "" if n == 132 else f" (the shapes are chosen for 132 SMs; this device has {n})"


# ----------------------------------------------------------------------------------------------------- RMSNorm
RMS_D = [8, 120, 256, 896, 1000, 1024]
RMS_M = [1, 7, 8, 9, 1000, 8192]


def _rms_x(M, D, seed):
    r = np.random.default_rng(seed)
    scale = np.exp(r.uniform(-6, 3, size=(M, 1)))
    x = Q.bf16(r.normal(size=(M, D)) * scale)
    w = Q.bf16(1 + 0.3 * r.normal(size=D))
    return x, w


def _rms_fwd(x, w, eps=1e-6):
    L, lib = _lib()
    M, D = x.shape
    yb, y = _guarded((M, D), BF)
    rb, rstd = _guarded((M,), torch.float32)
    xd, wd = _dev(x), _dev(w)
    L.check(lib.sk_rmsnorm_fwd(_p(xd), _p(wd), _p(y), _p(rstd), M, D, L.f32(eps), L.stream_ptr()))
    torch.cuda.synchronize()
    assert _guard_ok(yb) and _guard_ok(rb), "rmsnorm_fwd wrote outside its outputs"
    return _np(y), _np(rstd)


@pytest.mark.parametrize("M", RMS_M)
@pytest.mark.parametrize("D", RMS_D)
def test_rmsnorm_fwd_per_element(D, M):
    x, w = _rms_x(M, D, seed=D * 7 + M)
    y, rstd = _rms_fwd(x, w)
    rep = Q.check_rmsnorm_fwd(y, rstd, x, w, 1e-6)
    assert rep == [], "\n".join(rep)
    print(f"D={D} M={M}: {Q.rmsnorm_two_candidates(x, w, 1e-6)} of {x.size} outputs had two candidates")


def _rms_bwd(dy, x, w, rstd, dres, dw_old, accumulate):
    L, lib = _lib()
    M, D = x.shape
    xb, dx = _guarded((M, D), BF)
    wb, dw = _guarded((D,), BF, dw_old)
    partial = torch.empty(lib.sk_rmsnorm_bwd_blocks() * D, dtype=torch.float32, device=DEV)
    ops = [_dev(dy), _dev(x), _dev(w), torch.as_tensor(np.asarray(rstd, np.float32)).to(DEV),
           _dev(dres) if dres is not None else None]
    L.check(lib.sk_rmsnorm_bwd(*(_p(t) for t in ops), _p(dx), _p(dw), _p(partial), M, D, int(accumulate),
                               L.stream_ptr()))
    torch.cuda.synchronize()
    assert _guard_ok(xb) and _guard_ok(wb), "rmsnorm_bwd wrote outside its outputs"
    return _np(dx), _np(dw)


@pytest.mark.parametrize("M", RMS_M)
@pytest.mark.parametrize("D", RMS_D)
def test_rmsnorm_bwd_bit_exact(D, M):
    """Exact operands (power-of-two rstd, integer grids, row sums of g * x multiples of D): dx with and without dres,
    dw written and accumulated, bit for bit.  At M = 8192 the grid-stride row loop wraps (4 * SMs * 8 rows per pass)."""
    dy, x, w, rstd, dres = Q.exact_rmsnorm_bwd_operands(M, D, seed=D + M)
    old = Q.bf16(np.random.default_rng(M).integers(-64, 65, size=D).astype(np.float32))
    for d_res in (None, dres):
        for acc in (False, True):
            dx, dw = _rms_bwd(dy, x, w, rstd, d_res, old, acc)
            want_dx, want_dw = Q.rmsnorm_bwd_exact(dy, x, w, rstd, d_res, old if acc else None)
            rep = Q.check_exact(dx, want_dx, f"dx dres={d_res is not None}") + \
                Q.check_exact(dw, want_dw, f"dw accumulate={acc}")
            assert rep == [], "\n".join(rep)


@pytest.mark.parametrize("D,M", [(896, 8192), (1000, 1000), (120, 9), (1024, 7), (8, 1000)])
def test_rmsnorm_bwd_random_with_forward_rstd(D, M):
    """Random operands and the forward's own rstd: dx within the derived bound, dw within its column-sum bound."""
    _, lib = _lib()
    x, w = _rms_x(M, D, seed=5 * D + M)
    _, rstd = _rms_fwd(x, w)
    r = np.random.default_rng(D)
    dy, dres = Q.bf16(r.normal(size=(M, D))), Q.bf16(r.normal(size=(M, D)))
    old = Q.bf16(r.normal(size=D))
    dx, dw = _rms_bwd(dy, x, w, rstd, dres, old, True)
    blocks = min(lib.sk_rmsnorm_bwd_blocks(), (M + 7) // 8)
    rep = Q.check_rmsnorm_bwd(dx, dw, dy, x, w, rstd, dres, old, blocks)
    assert rep == [], "\n".join(rep)


# ----------------------------------------------------------------------------------------------------- RoPE
def _rope_run(qkv, cos, sin, pos_ids, T, n_rot, hd, rot, inverse, maxpos):
    """qkv [M, ld] inside a sentinel-filled buffer with 24 more columns (the pitch) and 8 more rows."""
    L, lib = _lib()
    M, width = qkv.shape
    big = torch.full((M + 8, width + 24), SENT16, dtype=torch.int16, device=DEV).view(BF)
    view = big[:M, :width]
    view.copy_(qkv.to(DEV))
    pos = pos_ids.to(torch.int32).to(DEV) if pos_ids is not None else None
    c, s = cos.to(DEV), sin.to(DEV)
    if rot == hd:
        rc = lib.sk_rope(_p(view), _p(c), _p(s), _p(pos), M, T, big.stride(0), n_rot, hd, int(inverse), maxpos,
                         L.stream_ptr())
    else:
        rc = lib.sk_rope_partial(_p(view), _p(c), _p(s), _p(pos), M, T, big.stride(0), n_rot, hd, rot, int(inverse),
                                 maxpos, L.stream_ptr())
    L.check(rc)
    torch.cuda.synchronize()
    out = big.cpu()
    outside = torch.ones(out.shape, dtype=torch.bool)
    outside[:M, :width] = False
    assert bool((out.view(torch.int16)[outside] == SENT16).all()), "rope wrote outside the qkv rows"
    return out[:M, :width]


ROPE_CASES = [(hd, hd) for hd in range(16, 129, 16)] + [(64, 32), (64, 16)]


@pytest.mark.parametrize("packed", [False, True], ids=["rowpos", "pos_ids"])
@pytest.mark.parametrize("hd,rot", ROPE_CASES, ids=[f"hd{h}-rot{r}" for h, r in ROPE_CASES])
def test_rope_fwd_and_inverse_bit_exact(hd, rot, packed):
    """14 q + 2 k heads rotate (GQA), 2 v heads and 16 padding columns must stay bit-identical; positions from packed
    documents with values below 0 and at or above max_pos (clamped), or row % T."""
    from slamkit_b200.lm import rope_tables
    H, KVH, M, T, maxpos = 14, 2, 1000, 250, 300
    n_rot = H + KVH
    g = torch.Generator().manual_seed(hd * 3 + rot)
    qkv = torch.randn(M, (H + 2 * KVH) * hd + 16, generator=g).to(BF)
    cos, sin = rope_tables(10000.0, rot, maxpos)
    pos_ids = None
    if packed:
        pos_ids = torch.cat([torch.arange(n) for n in (400, 250, 7, 343)])
        pos_ids[[3, 500, 900]] = torch.tensor([-1, -300, 10 ** 6])
    pos = Q.rope_positions(M, T, maxpos, pos_ids)
    for inverse in (False, True):
        got = _rope_run(qkv, cos, sin, pos_ids, T, n_rot, hd, rot, inverse, maxpos)
        rep = Q.check_rope(got, Q.rope_ref(qkv, cos, sin, pos, n_rot, hd, rot, inverse), f"rope inverse={inverse}")
        assert rep == [], "\n".join(rep)


# ----------------------------------------------------------------------------------------------------- SwiGLU
UPS = [1.0, -1.5, 0.0078125, 3072.0, 0.0]
DACTS = [1.0, 0.375, -2.0, 0.0010004043579101562, 5.0]


def _swiglu_standalone(gate, up, dact):
    L, lib = _lib()
    M, F = gate.shape
    gu = torch.cat([_dev(gate), _dev(up)], 1).contiguous()
    ab, act = _guarded((M, F), BF)
    db, dgu = _guarded((M, 2 * F), BF)
    dd = _dev(dact)
    L.check(lib.sk_swiglu_fwd(_p(gu), _p(act), M, F, L.stream_ptr()))
    L.check(lib.sk_swiglu_bwd(_p(gu), _p(dd), _p(dgu), M, F, L.stream_ptr()))
    torch.cuda.synchronize()
    assert _guard_ok(ab) and _guard_ok(db), "swiglu wrote outside its outputs"
    d = _np(dgu)
    return _np(act), d[:, :F], d[:, F:]


def test_swiglu_every_bf16_gate():
    """All 65,536 gate bit patterns (±0, subnormals, ±inf, NaNs) against five up / d_act values each: act, d_gate and
    d_up within the bound, NaN exactly where torch gives NaN.  Gates whose sigmoid is an fp32 subnormal (-88.5, -88,
    -87.5) are where a flush-to-zero reciprocal shows."""
    g = Q.all_bf16()
    G = np.tile(g, (len(UPS), 1))
    U_ = np.broadcast_to(np.array(UPS, np.float32)[:, None], G.shape).copy()
    D_ = np.broadcast_to(Q.bf16(np.array(DACTS, np.float32))[:, None], G.shape).copy()
    act, dg, du = _swiglu_standalone(G, U_, D_)
    rep = Q.check_swiglu_fwd(act, G, U_) + Q.check_swiglu_bwd(dg, du, G, U_, D_)
    assert rep == [], "\n".join(rep)


@pytest.mark.parametrize("M,F", [(3, 616), (1, 8), (7, 24), (1000, 4864), (129, 4856)])
def test_swiglu_shapes(M, F):
    """M * F / 8 odd (the forward's second vector per thread runs past the end), F % 16 == 8."""
    r = np.random.default_rng(M * F)
    G, U_, D_ = (Q.bf16(r.normal(size=(M, F)) * s) for s in (4.0, 2.0, 1.0))
    act, dg, du = _swiglu_standalone(G, U_, D_)
    rep = Q.check_swiglu_fwd(act, G, U_) + Q.check_swiglu_bwd(dg, du, G, U_, D_)
    assert rep == [], "\n".join(rep)


# ----------------------------------------------------------------------------------------------------- fused epilogues
def _unblock(x, F):
    v = x.view(x.shape[0], F // 128, 2, 128)
    return v[:, :, 0].reshape(-1, F), v[:, :, 1].reshape(-1, F)


def _finite_bf16_weights(rows, cols):
    """[rows, cols] bf16 holding every finite bf16 value once (rows * cols >= 65,280), the rest zero."""
    v = Q.all_bf16()
    v = v[np.isfinite(v)]
    out = np.zeros(rows * cols, np.float32)
    out[:len(v)] = v
    return out.reshape(rows, cols)


def swiglu_fwd_case(M, F, sweep, expect_warps):
    """Gate/up GEMM with the SwiGLU forward epilogue.  sweep: one-hot x rows pass the gate weights through unchanged,
    so the gates take every finite bf16 value; else integer operands.  gu exact, act within the SwiGLU bound."""
    from slamkit_b200 import ops
    K = 128
    plan = _plan(4, M, 2 * F, K)
    assert (plan["bn"], plan["epi_warps"]) == (256, expect_warps), f"SwiGLU forward plan {plan}{_sm_note()}"
    if sweep:
        x = torch.zeros(M, K, dtype=BF)
        x[torch.arange(M), torch.arange(M) % K] = 1.0
        wg = torch.from_numpy(_finite_bf16_weights(F, K)).to(BF)
        wu = R.int_operand(F, K, 8, 2)
    else:
        x, wg, wu = R.int_operand(M, K, 8, 1), R.int_operand(F, K, 8, 2), R.int_operand(F, K, 8, 3)
    acc = x.double() @ torch.cat([wg, wu], 0).double().t()
    gu_want = R.epilogue(acc)
    gu_b, act = ops.linear_swiglu_fwd(x.to(DEV), ops.block_gate_up(wg.to(DEV), wu.to(DEV)))
    g, u = _unblock(gu_b, F)
    rep = R.mismatch_exact(torch.cat([g, u], 1).cpu(), gu_want, 256, f"gu M={M} F={F}")
    assert rep is None, rep
    G, U_ = gu_want[:, :F].numpy(), gu_want[:, F:].numpy()
    rep = Q.check_swiglu_fwd(_np(act), G, U_, f"fused act M={M} F={F}")
    assert rep == [], "\n".join(rep)
    return plan


def swiglu_bwd_case(M, F, sweep, expect_warps):
    """d_gu from d_act = dy * W_down (integer operands: d_act exact) and a saved gu that holds every bf16 gate bit
    pattern (sweep) or random values."""
    from slamkit_b200 import ops
    N = 128
    plan = _plan(5, M, F, N)
    assert (plan["bn"], plan["epi_warps"]) == (256, expect_warps), f"SwiGLU backward plan {plan}{_sm_note()}"
    dy, wd = R.int_operand(M, N, 8, 4), R.int_operand(N, F, 8, 5)
    r = np.random.default_rng(M + F)
    if sweep:
        G = np.resize(Q.all_bf16(), (M, F))
    else:
        G = Q.bf16(r.normal(size=(M, F)) * 4)
    U_ = Q.bf16(r.normal(size=(M, F)) * 2)
    gu = ops.block_gate_up(_dev(G).t().contiguous(), _dev(U_).t().contiguous()).t().contiguous()   # [M, 2F] blocked
    dgu = ops.linear_swiglu_bwd(dy.to(DEV), wd.to(DEV), gu)
    dact = R.epilogue(dy.double() @ wd.double()).numpy()
    dg, du = _unblock(dgu, F)
    rep = Q.check_swiglu_bwd(_np(dg), _np(du), G, U_, dact, f"fused M={M} F={F}")
    assert rep == [], "\n".join(rep)
    return plan


FUSED_M = [1, 2, 7, 64, 65, 127, 128, 129, 1000, 8192]


@pytest.mark.parametrize("F", [4864, 640])
@pytest.mark.parametrize("M", FUSED_M)
def test_fused_swiglu_fwd_register(M, F):
    swiglu_fwd_case(M, F, False, 4)


@pytest.mark.parametrize("F", [4864, 640])
@pytest.mark.parametrize("M", FUSED_M)
def test_fused_swiglu_bwd_8_warps(M, F):
    swiglu_bwd_case(M, F, False, 8)


def test_fused_swiglu_every_gate():
    swiglu_fwd_case(128, 512, True, 4)
    swiglu_bwd_case(8, 8192 + 128, True, 8)


ROPE_FUSED = {   # width -> (M, N, K, rope_cols): chosen so that the planner picks that width on 132 SMs
    128: (100, 1152, 896, 1024),
    192: (8192, 1152, 896, 1024),        # the benchmark's QKV projection
    256: (640, 4096, 256, 3584),
}


def rope_fused_case(width, expect_warps):
    from slamkit_b200 import ops
    from slamkit_b200.lm import rope_tables
    M, N, K, rope_cols = ROPE_FUSED[width]
    plan = _plan(6, M, N, K)
    assert (plan["bn"], plan["epi_warps"]) == (width, expect_warps), f"RoPE epilogue plan {plan}{_sm_note()}"
    maxpos = 512
    x, w = R.int_operand(M, K, 8, 11), R.int_operand(N, K, 8, 12)
    bias = R.real_operand((N,), R.acc_scale(K, 8), 13)
    cos, sin = rope_tables(1000000.0, 64, maxpos)
    lens = [M // 3, M // 3 + 5, M - 2 * (M // 3) - 5]
    pos_ids = torch.cat([torch.arange(n) * 3 for n in lens])     # packed documents, some past the table
    pos_ids[0] = -7
    out = ops.linear_rope(x.to(DEV), w.to(DEV), bias.to(DEV), cos.to(DEV), sin.to(DEV), 1, rope_cols,
                          pos_ids=pos_ids.to(torch.int32).to(DEV)).cpu()
    pre = R.epilogue(R.exact_acc(x, w), bias).to(BF)
    want = Q.rope_ref(pre, cos, sin, Q.rope_positions(M, 1, maxpos, pos_ids), rope_cols // 64, 64)
    rep = R.mismatch_exact(out, want.float(), width, f"qkv + rope, {width}-wide tiles")
    assert rep is None, rep
    return plan


@pytest.mark.parametrize("width", list(ROPE_FUSED))
def test_fused_rope(width):
    rope_fused_case(width, 8 if width == 256 else 4)


# ----------------------------------------------------------------------------------------------------- env variants
ENV_VARIANTS = {
    "SK_GEMM_EW=8": ("8", [("swiglu_fwd", (8192, 4864)), ("swiglu_fwd", (129, 640)), ("swiglu_fwd_sweep", None)]),
    "SK_GEMM_EW=4": ("4", [("swiglu_bwd", (8192, 4864)), ("swiglu_bwd", (65, 640)), ("swiglu_bwd_sweep", None),
                           ("rope", 256)]),
}


def env_child(name):
    """Runs in a child process with SK_GEMM_EW set (the launcher reads it once per process)."""
    val, cases = ENV_VARIANTS[name]
    w = int(val)
    for kind, arg in cases:
        if kind == "swiglu_fwd":
            swiglu_fwd_case(*arg, False, w)
        elif kind == "swiglu_fwd_sweep":
            swiglu_fwd_case(128, 512, True, w)
        elif kind == "swiglu_bwd":
            swiglu_bwd_case(*arg, False, w)
        elif kind == "swiglu_bwd_sweep":
            swiglu_bwd_case(8, 8192 + 128, True, w)
        else:
            rope_fused_case(arg, w)
    print(f"{name}: {len(cases)} fused cases conform")


def _child(code, env_val):
    env = dict(os.environ)
    if env_val is not None:
        env["SK_GEMM_EW"] = env_val
    pre = f"import sys; sys.path[:0] = [{ROOT!r}, {HERE!r}]; import test_gpu_qwen_conformance as t; "
    return subprocess.run([sys.executable, "-c", pre + code], env=env, cwd=ROOT, capture_output=True, text=True,
                          timeout=900)


@pytest.mark.parametrize("name", list(ENV_VARIANTS))
def test_env_selected_variants(name):
    r = _child(f"t.env_child({name!r})", ENV_VARIANTS[name][0])
    print(r.stdout)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-4000:]


# ----------------------------------------------------------------------------------------------------- coverage
def plan_combos():
    """(epilogue, width, warps, register/parked) of every fused case above, in this process's environment."""
    out = set()
    for M in FUSED_M:
        for F in (4864, 640):
            p = _plan(4, M, 2 * F, 128)
            out.add(("swiglu_fwd", p["bn"], p["epi_warps"], _mode(4, p)))
            p = _plan(5, M, F, 128)
            out.add(("swiglu_bwd", p["bn"], p["epi_warps"], _mode(5, p)))
    for M, N, K, _ in ROPE_FUSED.values():
        p = _plan(6, M, N, K)
        out.add(("rope", p["bn"], p["epi_warps"], _mode(6, p)))
    return out


# The RoPE epilogue never runs 64-wide tiles: sk_linear_rope has no forced width, and the planner only takes 64 over
# 128 when it costs 25 % less, which a 64-wide tiling of the same rows (at least as many waves) never does.
EXPECTED = {("swiglu_fwd", 256, 4, "register"), ("swiglu_fwd", 256, 8, "parked"), ("swiglu_bwd", 256, 8, "parked"),
            ("swiglu_bwd", 256, 4, "parked"), ("rope", 128, 4, "parked"), ("rope", 192, 4, "parked"),
            ("rope", 256, 8, "parked"), ("rope", 256, 4, "parked")}


def test_coverage_table():
    """Prints the (width, warps, register / parked) combinations each fused epilogue reaches in this suite, with the
    SK_GEMM_EW variants asked in child processes, and fails if one is missing."""
    seen = {c + ("default",) for c in plan_combos()}
    for name, (val, _) in ENV_VARIANTS.items():
        r = _child("print(repr(sorted(t.plan_combos())))", val)
        assert r.returncode == 0, r.stderr[-4000:]
        seen |= {c + (name,) for c in eval(r.stdout.strip().splitlines()[-1])}
    print(f"\nfused epilogue: width x epilogue warps (where the tile is finished) [environment]{_sm_note()}")
    for c in sorted(seen):
        print(f"  {c[0]:11s} {c[1]:4d} x {c[2]} ({c[3]}) [{c[4]}]")
    missing = EXPECTED - {c[:4] for c in seen}
    assert not missing, f"never planned: {sorted(missing)}{_sm_note()}"


# ----------------------------------------------------------------------------------------------------- launch chain
def _chain(sync):
    from slamkit_b200 import ops
    M, d, F = 1000, 896, 4864
    g = torch.Generator(device=DEV).manual_seed(3)
    x = (torch.randn(M, d, generator=g, device=DEV) * 2).to(BF)
    w = (1 + 0.1 * torch.randn(d, generator=g, device=DEV)).to(BF)
    wgu = (torch.randn(2 * F, d, generator=g, device=DEV) * 0.05).to(BF)
    wd = (torch.randn(d, F, generator=g, device=DEV) * 0.05).to(BF)
    torch.cuda.synchronize()
    out = []
    s = torch.cuda.synchronize if sync else (lambda: None)
    dres = torch.zeros(M, d, dtype=BF, device=DEV)
    h, rstd = ops.rmsnorm_fwd(x, w, 1e-6)
    s()
    gu, act = ops.linear_swiglu_fwd(h, wgu)
    s()
    dgu = ops.linear_swiglu_bwd(h, wd, gu)
    s()
    dw = torch.zeros(d, dtype=BF, device=DEV)
    dx = ops.rmsnorm_bwd(dgu.view(-1)[:M * d].view(M, d), x, w, rstd, dres, dw, accumulate_dw=False)
    torch.cuda.synchronize()
    for t in (h, rstd, gu, act, dgu, dx, dw):
        out.append(t.clone())
    return out


def test_dependent_chain_on_one_stream():
    """rmsnorm_fwd -> linear_swiglu_fwd (reads h) -> linear_swiglu_bwd (reads gu) -> rmsnorm_bwd (reads rstd), back to
    back with programmatic dependent launch: equal to the same chain with a synchronise after every launch, and two
    runs bit-identical."""
    a, b, c = _chain(False), _chain(True), _chain(False)
    names = ["h", "rstd", "gu", "act", "dgu", "dx", "dw"]
    for n, x, y, z in zip(names, a, b, c):
        assert torch.equal(x.view(torch.uint8), y.view(torch.uint8)), f"{n}: chained != synchronised"
        assert torch.equal(x.view(torch.uint8), z.view(torch.uint8)), f"{n}: two runs differ"


# ----------------------------------------------------------------------------------------------------- argument checks
def _bad_calls():
    L, lib = _lib()
    buf = torch.zeros(1 << 20, dtype=BF, device=DEV)
    f = torch.zeros(1 << 16, dtype=torch.float32, device=DEV)
    p, pf, st = _p(buf), _p(f), L.stream_ptr()
    eps = L.f32(1e-6)
    return {
        "rmsnorm_fwd D%8": lambda: lib.sk_rmsnorm_fwd(p, p, p, pf, 4, 20, eps, st),
        "rmsnorm_fwd D>1024": lambda: lib.sk_rmsnorm_fwd(p, p, p, pf, 4, 1032, eps, st),
        "rmsnorm_bwd D%8": lambda: lib.sk_rmsnorm_bwd(p, p, p, pf, None, p, p, pf, 4, 20, 0, st),
        "rmsnorm_bwd D>1024": lambda: lib.sk_rmsnorm_bwd(p, p, p, pf, None, p, p, pf, 4, 1032, 0, st),
        "rope head_dim%16": lambda: lib.sk_rope(p, p, p, None, 8, 8, 128, 2, 40, 0, 64, st),
        "rope rot=48": lambda: lib.sk_rope_partial(p, p, p, None, 8, 8, 128, 2, 64, 48, 0, 64, st),
        "rope rot=16 at hd 128": lambda: lib.sk_rope_partial(p, p, p, None, 8, 8, 256, 2, 128, 16, 0, 64, st),
        "rope T>max_pos": lambda: lib.sk_rope(p, p, p, None, 8, 100, 128, 2, 64, 0, 64, st),
        "linear_swiglu_fwd F%128": lambda: lib.sk_linear_swiglu_fwd(64, 200, 64, p, p, p, p, st),
        "linear_swiglu_bwd F%128": lambda: lib.sk_linear_swiglu_bwd(64, 64, 200, p, p, p, p, st),
    }


@pytest.mark.parametrize("bad", ["rmsnorm_fwd D%8", "rmsnorm_fwd D>1024", "rmsnorm_bwd D%8", "rmsnorm_bwd D>1024",
                                 "rope head_dim%16", "rope rot=48", "rope rot=16 at hd 128", "rope T>max_pos",
                                 "linear_swiglu_fwd F%128", "linear_swiglu_bwd F%128"])
def test_rejects_bad_arguments(bad):
    _, lib = _lib()
    calls = _bad_calls()
    torch.cuda.synchronize()
    n0 = lib.sk_launch_count()
    assert calls[bad]() != 0, f"{bad}: accepted"
    assert lib.sk_launch_count() == n0, f"{bad}: launched a kernel"
    assert lib.sk_last_error().decode()
