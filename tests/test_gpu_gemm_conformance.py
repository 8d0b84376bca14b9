"""Conformance of the wgmma GEMM (gemm_tcgen05.cu) per element, against the exact references of tests/gemm_ref.py.

Integer operands make the fp32 accumulator exact, so outputs are compared bit for bit; each case first asks the launcher
(ops.gemm_plan) which schedule it runs and asserts it is the one the case names.  Covered: every schedule (plain tiles
of 64 / 128 / 256 columns, split-K, stream-K with one and with several contributors per tile, column-unit stream-K and
8 epilogue warps, which environment variables select) x every operand major x every epilogue the schedule takes;
stale workspace state; the decode step's calls at M = 1 .. 129; batch invariance of the forward GEMM; pitched operands
with NaN padding and an output inside a sentinel-filled buffer; dependent GEMMs launched back to back; argument checks.
"""
import functools
import os
import subprocess
import sys

import pytest
import torch

import gemm_ref as R

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)

MAJORS = [(False, False), (False, True), (True, False), (True, True)]
MAJOR_IDS = ["KK", "KM", "MK", "MM"]   # (A, B): K-major or MN-major
# schedule kind -> (M, N, K, force_bn, scratch).  Ragged M, N and K everywhere; the shapes were chosen for 132 SMs and
# every case asserts the schedule it gets.
SCHEDULES = {
    "plain64": (328, 264, 200, 64, False),
    "plain128": (328, 264, 200, 128, False),
    "plain256": (328, 264, 200, 256, False),
    "splitk": (200, 264, 2112, 0, True),
    "streamk1": (4160, 1480, 2056, 256, True),    # 33 x 6 tiles: 11 units over 22 groups, one contributor per tile
    "streamk2": (5064, 896, 2056, 256, True),     # 40 x 4 tiles: 7 units over 28 groups, three contributors per tile
}
EPILOGUES = ["none", "bias", "bias_res_r", "bias_res", "res_r", "res", "inplace_r", "inplace", "f32", "f32_bias_res", "gelu"]
SPLITK_EPILOGUES = ["none", "inplace_r", "inplace"]   # split-K takes plain and in-place bf16 outputs only
AMAX = 8


def _matrix():
    for kind in SCHEDULES:
        for epi in (SPLITK_EPILOGUES if kind == "splitk" else EPILOGUES):
            for major, mid in zip(MAJORS, MAJOR_IDS):
                yield pytest.param(kind, major, epi, id=f"{kind}-{mid}-{epi}")


@functools.lru_cache(maxsize=4)
def _data(M, N, K, seed=0):
    """Integer A [M,K], B [N,K], real bias [N] and residual [M,N] on the accumulator's scale, exact accumulator."""
    a = R.int_operand(M, K, AMAX, seed, DEV)
    b = R.int_operand(N, K, AMAX, seed + 1, DEV)
    scale = R.acc_scale(K, AMAX)
    bias = R.real_operand((N,), scale, seed + 2, DEV)
    res = R.real_operand((M, N), scale, seed + 3, DEV)
    return a, b, bias, res, R.exact_acc(a, b)


def _layout(t, mn):
    return t.t().contiguous() if mn else t


def _epilogue_args(epi, bias, res):
    """-> (gemm kwargs, reference kwargs, in-place?)"""
    table = {
        "none": ({}, {}),
        "bias": ({"bias": bias}, {"bias": bias}),
        "bias_res_r": ({"bias": bias, "residual": res, "round_before_res": True},
                       {"bias": bias, "residual": res, "round_before_res": True}),
        "bias_res": ({"bias": bias, "residual": res}, {"bias": bias, "residual": res}),
        "res_r": ({"residual": res, "round_before_res": True}, {"residual": res, "round_before_res": True}),
        "res": ({"residual": res}, {"residual": res}),
        "inplace_r": ({"round_before_res": True}, {"residual": res, "round_before_res": True}),
        "inplace": ({}, {"residual": res}),
        "f32": ({"out_f32": True}, {"out_f32": True}),
        "f32_bias_res": ({"out_f32": True, "bias": bias, "residual": res}, {"out_f32": True, "bias": bias, "residual": res}),
        "gelu": ({"bias": bias, "act": 1}, None),
    }
    kw, ref = table[epi]
    return dict(kw), ref, epi.startswith("inplace")


def run_case(kind, major, epi, shape=None, expect=None):
    """One matrix case: plan check (the schedule kind is `kind`, or one of `expect`), launch, bit-exact (GELU: bounded)
    comparison.  Returns the plan."""
    from slamkit_b200 import ops
    M, N, K, bn, ws = shape or SCHEDULES[kind]
    a, b, bias, res, acc = _data(M, N, K)
    a_mn, b_mn = major
    ad, bd = _layout(a, a_mn), _layout(b, b_mn)
    kw, ref_kw, inplace = _epilogue_args(epi, bias, res)
    kw.update(a_mn=a_mn, b_mn=b_mn, force_bn=bn, streamk=ws)
    if inplace:
        kw["out"] = kw["residual"] = res.clone()
    plan = ops.gemm_plan(ad, bd, **kw)
    got = R.schedule_kind(plan, K)
    assert got in (expect or (kind,)), f"{kind} {major} {epi}: the launcher plans {got}: {plan}"
    out = ops.gemm(ad, bd, **kw)
    what = f"{kind} a_mn={a_mn} b_mn={b_mn} {epi}"
    if epi == "gelu":
        rep = R.mismatch_gelu(out, acc.float() + bias.float(), plan["bn"], what)
    else:
        assert out.dtype == (torch.float32 if epi.startswith("f32") else torch.bfloat16)
        rep = R.mismatch_exact(out, R.epilogue(acc, **ref_kw), plan["bn"], what)
    assert rep is None, rep
    return plan


# --------------------------------------------------------------------------------------------------- schedule matrix
@pytest.mark.parametrize("kind,major,epi", list(_matrix()))
def test_schedule_matrix(kind, major, epi):
    run_case(kind, major, epi)


def test_schedule_coverage():
    """The matrix above reaches every schedule kind with every operand major (printed as a table)."""
    from slamkit_b200 import ops
    hit = {}
    for p in _matrix():
        kind, major, epi = p.values
        M, N, K, bn, ws = SCHEDULES[kind]
        a, b, bias, res, _ = _data(M, N, K)
        kw, _, inplace = _epilogue_args(epi, bias, res)
        if inplace:
            kw["out"] = kw["residual"] = res
        plan = ops.gemm_plan(_layout(a, major[0]), _layout(b, major[1]), a_mn=major[0], b_mn=major[1], force_bn=bn,
                             streamk=ws, **kw)
        hit.setdefault((R.schedule_kind(plan, K), major), []).append(epi)
    kinds = list(SCHEDULES)
    print("\nschedule kind x operand major (A,B): epilogues run")
    for kind in kinds:
        print(f"  {kind:9s} " + "  ".join(f"{mid}:{len(hit.get((kind, mj), []))}" for mj, mid in zip(MAJORS, MAJOR_IDS)))
    missing = [(k, mid) for k in kinds for mj, mid in zip(MAJORS, MAJOR_IDS) if (k, mj) not in hit]
    assert not missing, f"schedule kinds never run: {missing}"


@pytest.mark.parametrize("kind", list(SCHEDULES))
@pytest.mark.parametrize("major", MAJORS, ids=MAJOR_IDS)
def test_random_data_per_element(kind, major):
    """bf16 normal operands (not integers): per-element bound of fp32 accumulation + output rounding."""
    from slamkit_b200 import ops
    M, N, K, bn, ws = SCHEDULES[kind]
    g = torch.Generator(device=DEV).manual_seed(5)
    a = torch.randn(M, K, generator=g, device=DEV).to(torch.bfloat16)
    b = torch.randn(N, K, generator=g, device=DEV).to(torch.bfloat16)
    ad, bd = _layout(a, major[0]), _layout(b, major[1])
    kw = dict(a_mn=major[0], b_mn=major[1], force_bn=bn, streamk=ws)
    plan = ops.gemm_plan(ad, bd, **kw)
    assert R.schedule_kind(plan, K) == kind, plan
    rep = R.mismatch_random(ops.gemm(ad, bd, **kw), a, b, plan["bn"], what=f"{kind} {major}")
    assert rep is None, rep


# --------------------------------------------------------------------------------------------------- stale state
@pytest.mark.parametrize("kind", ["splitk", "streamk1", "streamk2"])
def test_alternating_inputs_on_one_workspace(kind):
    """A / B, then A' / B', then A / B again on the shared scratch, back to back: a fix-up or reduction that read a
    partial before it was written would pick up the other input set's values."""
    from slamkit_b200 import ops
    M, N, K, bn, _ = SCHEDULES[kind]
    sets = [_data(M, N, K, seed=0), _data(M, N, K, seed=100)]
    outs = []
    for i in (0, 1, 0, 1):
        a, b = sets[i][0], sets[i][1]
        assert R.schedule_kind(ops.gemm_plan(a, b, force_bn=bn, streamk=True), K) == kind
        outs.append((i, ops.gemm(a, b, force_bn=bn, streamk=True)))
    for n, (i, out) in enumerate(outs):
        rep = R.mismatch_exact(out, R.epilogue(sets[i][4]), bn or 128, f"{kind} launch {n} (input set {i})")
        assert rep is None, rep
    assert int(ops.gemm_workspace(DEV)[-4096:].max()) == 0, "stream-K flag words not re-armed"


# --------------------------------------------------------------------------------------------------- decode-sized M
DECODE_M = [1, 2, 7, 8, 63, 64, 65, 127, 128, 129]


def _ints(rows, cols, seed, amax=AMAX):
    return R.int_operand(rows, cols, amax, seed, DEV)


@pytest.mark.parametrize("M", DECODE_M)
def test_decode_qkv_rope(M):
    """QKV projection + bias + RoPE (N = 1152, K = 896) with per-row positions, some past the table (clamped)."""
    from slamkit_b200 import ops
    from slamkit_b200.lm import rope_tables
    N, K, maxpos, rope_cols = 1152, 896, 256, 1024
    x, w = _ints(M, K, 1), _ints(N, K, 2)
    bias = R.real_operand((N,), R.acc_scale(K, AMAX), 3, DEV)
    cos, sin = (t.to(DEV) for t in rope_tables(10000.0, 64, maxpos))
    g = torch.Generator().manual_seed(M)
    pos = torch.randint(0, maxpos, (M,), generator=g)
    pos[-1] = maxpos + 37                         # clamped to maxpos - 1
    if M > 1:
        pos[0] = maxpos - 1
    if M > 2:
        pos[1] = maxpos
    pos = pos.to(torch.int32).to(DEV)
    out = ops.linear_rope(x, w, bias, cos, sin, 1, rope_cols, pos_ids=pos)
    rep = R.mismatch_exact(out, R.rope_epilogue(R.exact_acc(x, w), bias, cos, sin, pos, rope_cols), 256, f"qkv+rope M={M}")
    assert rep is None, rep


@pytest.mark.parametrize("M", DECODE_M)
def test_decode_oproj_residual(M):
    """o-projection + residual into a separate output (896 x 896, rounded before the add, like the forward pass)."""
    from slamkit_b200 import ops
    ao, wo = _ints(M, 896, 4), _ints(896, 896, 5)
    x = R.real_operand((M, 896), R.acc_scale(896, AMAX), 6, DEV)
    out = ops.gemm(ao, wo, residual=x, round_before_res=True)
    rep = R.mismatch_exact(out, R.epilogue(R.exact_acc(ao, wo), residual=x, round_before_res=True), 256, f"o-proj M={M}")
    assert rep is None, rep


@pytest.mark.parametrize("M", DECODE_M)
def test_decode_swiglu(M):
    """gate/up projection with SwiGLU in the epilogue (F = 4864): gu exact, act bit-equal to the unfused kernel."""
    from slamkit_b200 import ops
    F, K = 4864, 896
    h, wg, wu = _ints(M, K, 7), _ints(F, K, 8), _ints(F, K, 9)
    gu_b, act = ops.linear_swiglu_fwd(h, ops.block_gate_up(wg, wu))
    gu_want = R.epilogue(R.exact_acc(h, torch.cat([wg, wu], 0)))
    gu = torch.cat([v.reshape(M, F) for v in gu_b.view(M, F // 128, 2, 128).unbind(2)], 1)   # [gate | up]
    rep = R.mismatch_exact(gu, gu_want, 256, f"gate/up M={M}")
    assert rep is None, rep
    assert torch.equal(act, ops.swiglu_fwd(gu))


@pytest.mark.parametrize("round_before_res", [True, False], ids=["rbr1", "rbr0"])
@pytest.mark.parametrize("M", DECODE_M)
def test_decode_down_proj_inplace_splitk(M, round_before_res):
    """Down projection added in place with scratch (N = 896, K = 4864): split-K, both rounding points."""
    from slamkit_b200 import ops
    act, wd = _ints(M, 4864, 10), _ints(896, 4864, 11)
    x = R.real_operand((M, 896), R.acc_scale(4864, AMAX), 12, DEV)
    xm = x.clone()
    kw = dict(residual=xm, out=xm, round_before_res=round_before_res, streamk=True)
    assert R.schedule_kind(ops.gemm_plan(act, wd, **kw), 4864) == "splitk"
    ops.gemm(act, wd, **kw)
    want = R.epilogue(R.exact_acc(act, wd), residual=x, round_before_res=round_before_res)
    rep = R.mismatch_exact(xm, want, 128, f"down-proj M={M} round_before_res={round_before_res}")
    assert rep is None, rep


SENT16 = 0x7FB5          # a NaN payload no kernel produces


@pytest.mark.parametrize("N", [512, 152192])
@pytest.mark.parametrize("M", DECODE_M)
def test_decode_head_pitched(M, N):
    """LM head into logits of pitch ldl > N: the [:M, :N] block exact, every other element of the buffer untouched."""
    from slamkit_b200 import ops
    K, ldl = 896, N + 64
    h, w = _ints(M, K, 13), _ints(N, K, 14)
    buf = torch.full((M + 1, ldl), SENT16, dtype=torch.int16, device=DEV).view(torch.bfloat16)
    out = buf[:M, :N]
    ops.gemm(h, w, out=out)
    rep = R.mismatch_exact(out, R.epilogue(R.exact_acc(h, w)), 256, f"head M={M} N={N}")
    assert rep is None, rep
    outside = torch.ones(buf.shape, dtype=torch.bool, device=DEV)
    outside[:M, :N] = False
    assert bool((buf.view(torch.int16)[outside] == SENT16).all()), "the head wrote outside [:M, :N]"


# --------------------------------------------------------------------------------------------------- batch invariance
@pytest.mark.parametrize("N", [896, 1152])
def test_batch_invariance(N):
    """Row i of gemm(A[:m], B) == row i of gemm(A, B) bit for bit for every m (the forward GEMMs take no scratch, so a
    sequence's logits do not depend on the batch around it), although the tile width changes with m."""
    from slamkit_b200 import ops
    g = torch.Generator(device=DEV).manual_seed(N)
    A = torch.randn(6000, 896, generator=g, device=DEV).to(torch.bfloat16)
    B = torch.randn(N, 896, generator=g, device=DEV).to(torch.bfloat16)
    full = ops.gemm(A, B)
    rep = R.mismatch_random(full, A, B, 256, what="full batch")
    assert rep is None, rep
    bns = set()
    for m in (1, 2, 7, 64, 65, 128, 129, 300, 1000, 1500, 2048, 3000, 4224, 5999):
        bns.add(ops.gemm_plan(A[:m], B)["bn"])
        part = ops.gemm(A[:m], B)
        rep = R.mismatch_exact(part, full[:m], 256, f"rows of a batch of {m} vs 6000")
        assert rep is None, rep
    assert len(bns) >= 2, bns          # the invariance holds across tile widths


# --------------------------------------------------------------------------------------------------- guard bands
def _pitched(t, pad_cols, pad_rows, fill=float("nan")):
    """t as a view into a larger buffer whose extra columns and rows hold `fill`."""
    r, c = t.shape
    buf = torch.full((r + pad_rows, c + pad_cols), fill, dtype=t.dtype, device=t.device)
    buf[:r, :c] = t
    return buf[:r, :c]


GUARD_CASES = [("plain128", False), ("plain256", False), ("plain64", True), ("plain256", True), ("splitk", False),
               ("streamk2", False), ("streamk2", True)]


@pytest.mark.parametrize("major", MAJORS, ids=MAJOR_IDS)
@pytest.mark.parametrize("kind,out_f32", GUARD_CASES, ids=[f"{k}-{'f32' if f else 'bf16'}" for k, f in GUARD_CASES])
def test_guard_bands_and_pitches(kind, out_f32, major):
    """A, B and the residual at pitches wider than their rows with NaN in the padding (and NaN rows past K for MN-major
    operands, past M / N otherwise); C inside a sentinel-filled buffer with ldr != ldc: the result is exact and no byte
    outside [:M, :N] changes, on the TMA-store path and the direct-store (fp32) path."""
    from slamkit_b200 import ops
    M, N, K, bn, ws = SCHEDULES[kind]
    a, b, bias, res, acc = _data(M, N, K)
    a_mn, b_mn = major
    ad = _pitched(_layout(a, a_mn), 24, 64)
    bd = _pitched(_layout(b, b_mn), 40, 64)
    odt = torch.float32 if out_f32 else torch.bfloat16
    sent = torch.tensor([SENT16], dtype=torch.int16).view(torch.bfloat16).item() if not out_f32 else float("nan")
    big = torch.full((M + 24, N + 64), sent, dtype=odt, device=DEV)
    before = big.clone()
    out = big[16:16 + M, 8:8 + N]
    kw = dict(a_mn=a_mn, b_mn=b_mn, force_bn=bn, streamk=ws, out=out, out_f32=out_f32)
    if kind == "splitk":   # in place: the residual is the output (ldr == ldc by construction)
        out.copy_(res.to(odt))
        before[16:16 + M, 8:8 + N] = out
        kw.update(residual=out, round_before_res=True)
        want = R.epilogue(acc, residual=res, round_before_res=True)
    else:
        rp = _pitched(res, 8, 8)
        assert rp.stride(0) != out.stride(0)
        kw.update(bias=bias, residual=rp, round_before_res=True)
        want = R.epilogue(acc, bias, res, round_before_res=True, out_f32=out_f32)
    plan = ops.gemm_plan(ad, bd, **kw)
    assert R.schedule_kind(plan, K) == kind and plan["tma_store"] == (0 if out_f32 or kind == "splitk" else 1), plan
    ops.gemm(ad, bd, **kw)
    rep = R.mismatch_exact(out, want, plan["bn"], f"{kind} pitched")
    assert rep is None, rep
    bits = (lambda t: t.view(torch.int32)) if out_f32 else (lambda t: t.view(torch.int16))
    changed = bits(big) != bits(before)
    changed[16:16 + M, 8:8 + N] = False
    assert not bool(changed.any()), f"{int(changed.sum())} elements outside [:M, :N] were written, first {changed.nonzero()[:4].tolist()}"


# --------------------------------------------------------------------------------------------------- launch chains
def test_chain_read_after_write_and_write_after_read():
    """y1 = x W1^T; y2 = y1 W2^T (reads y1); y3 = y2 W3^T (reads y2); then y2 is overwritten by an unrelated GEMM
    while nothing waits on the host: y3 must see the y2 of the chain, and y1 -> y2 -> y3 each the previous output."""
    from slamkit_b200 import ops
    x, w1 = _ints(512, 128, 20, 4), _ints(256, 128, 21, 4)
    w2, w3 = _ints(256, 256, 22, 1), _ints(384, 256, 23, 1)
    z, wz = _ints(512, 640, 24), _ints(256, 640, 25)
    r1 = R.epilogue(R.exact_acc(x, w1))
    r2 = R.epilogue(R.exact_acc(r1.to(torch.bfloat16), w2))
    r3 = R.epilogue(R.exact_acc(r2.to(torch.bfloat16), w3))
    rz = R.epilogue(R.exact_acc(z, wz))
    y1 = torch.full((512, 256), 7.0, dtype=torch.bfloat16, device=DEV)   # stale contents a premature read would see
    y2 = torch.full((512, 256), -5.0, dtype=torch.bfloat16, device=DEV)
    torch.cuda.synchronize()
    ops.gemm(x, w1, out=y1, force_bn=64)
    ops.gemm(y1, w2, out=y2, force_bn=256)
    y3 = ops.gemm(y2, w3)
    ops.gemm(z, wz, out=y2)                       # write-after-read of y2
    for name, got, want in (("y3", y3, r3), ("y1", y1, r1), ("y2 overwritten", y2, rz)):
        rep = R.mismatch_exact(got, want, 256, name)
        assert rep is None, rep


def test_chain_decode_residual_ping_pong():
    """The decode step's residual stream over 6 layers, no host synchronisation: xm = bf16(bf16(ao Wo^T) + x), then
    xm += bf16(act Wd^T) in place with split-K, then x and xm swap."""
    from slamkit_b200 import ops
    B, d, F, L = 8, 896, 4864, 6
    aos = [_ints(B, d, 30 + l) for l in range(L)]
    wos = [_ints(d, d, 40 + l) for l in range(L)]
    acts = [_ints(B, F, 50 + l) for l in range(L)]
    wds = [_ints(d, F, 60 + l) for l in range(L)]
    acc_o = [R.exact_acc(a, w) for a, w in zip(aos, wos)]
    acc_d = [R.exact_acc(a, w) for a, w in zip(acts, wds)]
    x0 = R.real_operand((B, d), R.acc_scale(F, AMAX), 70, DEV)
    bufs = [x0.clone(), torch.empty_like(x0)]
    assert R.schedule_kind(ops.gemm_plan(acts[0], wds[0], residual=bufs[1], out=bufs[1], round_before_res=True,
                                         streamk=True), F) == "splitk"
    torch.cuda.synchronize()
    cur = 0
    for l in range(L):
        x, xm = bufs[cur], bufs[1 - cur]
        ops.gemm(aos[l], wos[l], residual=x, out=xm, round_before_res=True)
        ops.gemm(acts[l], wds[l], residual=xm, out=xm, round_before_res=True, streamk=True)
        cur = 1 - cur
    want = x0.float()
    for l in range(L):
        xm = R.epilogue(acc_o[l], residual=want, round_before_res=True)
        want = R.epilogue(acc_d[l], residual=xm, round_before_res=True)
    rep = R.mismatch_exact(bufs[cur], want, 128, f"residual stream after {L} layers")
    assert rep is None, rep


# --------------------------------------------------------------------------------------------------- env variants
ENV_VARIANTS = {
    # column-unit stream-K: 5 x 19 tiles, a unit is a column of 5 tiles
    "SK_STREAMK=2": (("SK_STREAMK", "2"), (640, 4864, 2056, 256, True), "colunits",
                     ["none", "bias_res_r", "res", "inplace", "f32", "gelu"]),
    # 8 epilogue warps on the plain 256-wide tiles
    "SK_GEMM_EW=8": (("SK_GEMM_EW", "8"), SCHEDULES["plain256"], "ew8",
                     ["none", "bias", "bias_res_r", "bias_res", "res_r", "inplace", "gelu"]),
}


def env_child(name):
    """Runs in a child process with the variable set: the integer matrix for that variant's shape."""
    _, shape, check, epis = ENV_VARIANTS[name]
    n = 0
    for major in MAJORS:
        for epi in epis:
            expect = ("streamk1", "streamk2") if check == "colunits" else ("plain256",)
            plan = run_case(name, major, epi, shape=shape, expect=expect)
            if check == "colunits":
                assert plan["sk_colunits"] == 1 and plan["sk_units"] > 0, plan
            elif plan["tma_store"]:
                assert plan["epi_warps"] == 8, plan
            n += 1
    print(f"{name}: {n} cases bit-exact")


@pytest.mark.parametrize("name", list(ENV_VARIANTS))
def test_env_selected_variants(name):
    (var, val), *_ = ENV_VARIANTS[name]
    env = dict(os.environ)
    env[var] = val
    code = (f"import sys; sys.path[:0] = [{ROOT!r}, {HERE!r}]; import test_gpu_gemm_conformance as t; "
            f"t.env_child({name!r})")
    r = subprocess.run([sys.executable, "-c", code], env=env, cwd=ROOT, capture_output=True, text=True, timeout=900)
    print(r.stdout)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-4000:]


# --------------------------------------------------------------------------------------------------- argument checks
def _raw_call(lib, L, fn, args):
    import ctypes as C
    M, N, K, pa, lda, am, pb, ldb, bm, pc, ldc, f32, pbias, pres, ldr, rbr, act, fbn = args
    if fn == "plan":
        plan = L.SkGemmPlan()
        return lib.sk_gemm_plan(M, N, K, pa, lda, am, pb, ldb, bm, pc, ldc, f32, pbias, pres, ldr, rbr, act, fbn,
                                C.c_void_p(0), C.c_int64(0), C.byref(plan))
    return lib.sk_gemm_bf16(M, N, K, pa, lda, am, pb, ldb, bm, pc, ldc, f32, pbias, pres, ldr, rbr, act, fbn, L.stream_ptr())


BAD_ARGS = {
    "lda<K": dict(lda=248), "lda<M(a_mn)": dict(a_mn=1, lda=248), "ldb<K": dict(ldb=248), "ldb<N(b_mn)": dict(b_mn=1, ldb=248),
    "ldc<N": dict(ldc=248), "ldr<N": dict(ldr=248), "A+2B": dict(A=2), "B+2B": dict(B=2), "C+2B": dict(C=2),
    "residual+8B": dict(residual=8), "bias+2B": dict(bias=2), "M=0": dict(M=0), "N=0": dict(N=0), "K=0": dict(K=0),
    "N%8": dict(N=252),
}


@pytest.mark.parametrize("bad", list(BAD_ARGS))
def test_rejects_bad_arguments(bad):
    """Pitches below the row width, misaligned pointers and empty problems return an error and launch nothing."""
    import ctypes as C
    from slamkit_b200 import _lib as L
    lib = L.require_cuda()
    buf = torch.zeros(4, 256 * 256 + 64, dtype=torch.bfloat16, device=DEV)
    bias = torch.zeros(512, dtype=torch.bfloat16, device=DEV)
    base = dict(M=256, N=256, K=256, A=0, lda=256, a_mn=0, B=0, ldb=256, b_mn=0, C=0, ldc=256, residual=0, ldr=256,
                bias=0)
    ptr = {"A": buf[0], "B": buf[1], "C": buf[2], "residual": buf[3], "bias": bias}

    def args(mod):
        v = dict(base, **mod)
        p = {k: C.c_void_p(ptr[k].data_ptr() + (mod.get(k, 0) if k in mod else 0)) for k in ptr}
        return (v["M"], v["N"], v["K"], p["A"], v["lda"], v["a_mn"], p["B"], v["ldb"], v["b_mn"], p["C"], v["ldc"], 0,
                p["bias"], p["residual"], v["ldr"], 1, 0, 0)

    assert _raw_call(lib, L, "plan", args({})) == 0 and _raw_call(lib, L, "gemm", args({})) == 0
    torch.cuda.synchronize()
    n0 = lib.sk_launch_count()
    bad_args = args(BAD_ARGS[bad])
    assert _raw_call(lib, L, "plan", bad_args) != 0, f"{bad}: accepted by the planner"
    assert _raw_call(lib, L, "gemm", bad_args) != 0, f"{bad}: accepted"
    assert lib.sk_launch_count() == n0, f"{bad}: launched a kernel"
    assert lib.sk_last_error().decode()
