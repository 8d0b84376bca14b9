"""CPU self-test of tests/vocoder_ref.py: an emulation of vocoder_conv_kernel with its phase, tile and tap structure passes
the exact and bounded checks, and each injected defect of the vocoder path is flagged at its location."""
import math

import pytest
import torch
import torch.nn.functional as F

import vocoder_ref as V

BM = V.BM


# ----------------------------------------------------------------------------------------------------- kernel emulation
def emulate(x, w, bias, geo, slope, valid, up, res=None, mode=0, sum_in=None, divide=0, defect=None, exact=True):
    """vocoder_conv_kernel on the CPU: prepared taps per phase, time tiles of BM q values with the halo staged once
    (leaky ReLU, then the hi / lo split), one shifted slice of the stage per tap, three products, then the epilogue.
    exact: accumulate in float64 (equal to the kernel's fp32 sums on exact operands); else fp32."""
    acc_t = torch.float64 if exact else torch.float32
    taps, bases = [], []
    for r, js in enumerate(geo.phases):
        bases.append(len(taps))
        for j in js:
            jj = min(j + 1, geo.k - 1) if defect == "tap_off_by_one" else j
            taps.append(w[:, :, jj].t() if geo.transposed else w[:, :, jj])
    if defect == "swap_tap_bases":
        bases[0], bases[1] = bases[1], bases[0]
    in_off0, in_step = (0, -1) if geo.transposed else (-geo.pad, geo.dil)
    out_mul, out_off = (geo.rate, -geo.pad) if geo.transposed else (1, 0)
    T_in, Cout = x.shape[0], taps[0].shape[0]
    out = torch.zeros(geo.T_out, Cout, dtype=torch.float32)
    live_all = V.position_mask(valid, up, geo.T_out)
    for r, js in enumerate(geo.phases):
        nt = len(js)
        off_min = in_off0 + min(0, (nt - 1) * in_step)
        arows = BM + (nt - 1) * abs(in_step)
        for q0 in range(0, geo.Q, BM):
            g = torch.arange(arows) + q0 + off_min
            ok = (g >= 0) & (g < T_in)
            rows = torch.zeros(arows, x.shape[1])
            rows[ok] = x[g[ok]].float()
            if defect == "leaky_after_split":
                h, l = V.split_f32(rows)
                h, l = V.leaky32(h, slope), V.leaky32(l, slope)
            else:
                h, l = V.split_f32(V.leaky32(rows, slope))
            if defect == "missing_halo_row" and q0 == BM:
                h[-1] = 0
                l[-1] = 0
            acc = torch.zeros(BM, Cout, dtype=acc_t)
            for m in range(nt):
                W = taps[min(bases[r] + m, len(taps) - 1)]
                wh, wl = V.split_f32(W)
                if defect == "drop_hi_lo_chunk":      # channel tile 1, input chunk 0
                    wl = wl.clone()
                    wl[geo.BN:2 * geo.BN, :V.KC] = 0
                s = in_off0 + m * in_step - off_min
                ah, al = h[s:s + BM].to(acc_t), l[s:s + BM].to(acc_t)
                wh, wl = wh.to(acc_t), wl.to(acc_t)
                acc = acc + ah @ wh.t() + ah @ wl.t() + al @ wh.t()
                if defect == "add_lo_lo":
                    acc = acc + al @ wl.t()
            q = torch.arange(q0, min(q0 + BM, geo.Q))
            o = q * out_mul + r + out_off
            sel = (o >= 0) & (o < geo.T_out)
            q, o = q[sel], o[sel]
            v = acc[q - q0].float() + bias.float()
            if res is not None:
                v = v + res[o].float()
            if mode == 2 and defect != "mode2_overwrites":
                v = sum_in[o].float() + v
            if divide > 0 and defect != "no_divide":
                v = v / torch.tensor(float(divide))
            live = torch.ones_like(o, dtype=torch.bool) if defect == "mask_not_zeroed" else live_all[o]
            out[o] = torch.where(live[:, None], v, torch.zeros_like(v))
    return out


def exact_case(k=5, transposed=False, rate=1, dil=2, T_in=300, Cin=48, Cout=64, slope=0.1, mode=0, divide=0, up=1,
               seed=0, mask_edges=True):
    geo = V.Geometry(k, transposed, rate, dil, T_in, Cout)
    K = len(geo.phases[0]) * Cin
    x, t = V.exact_activation(T_in, Cin, V.exact_amax(K, 0.6), 0.6, slope, seed)
    wshape = (Cin, Cout, k) if transposed else (Cout, Cin, k)
    w = V.exact_values(wshape, V.exact_amax(K, 0.6), 0.6, seed + 1)
    g = torch.Generator().manual_seed(seed + 2)
    bias = torch.randn(Cout, generator=g)
    valid = (torch.rand(geo.T_out // up, generator=g) < 0.9).to(torch.uint8)
    if mask_edges:
        for o in (0, 127, 128, 255, 256, geo.T_out - 1):
            if o < geo.T_out:
                valid[o // up] = 0
    res = torch.randn(geo.T_out, Cout, generator=g) if mode or seed % 2 else None
    sum_in = torch.randn(geo.T_out, Cout, generator=g) if mode == 2 else None
    live = V.position_mask(valid, up, geo.T_out)
    want = V.exact_epilogue(V.split_exact_acc(t, w, geo), bias, live, res, mode, sum_in, divide)
    args = dict(x=x, w=w, bias=bias, geo=geo, slope=slope, valid=valid, up=up, res=res, mode=mode, sum_in=sum_in,
                divide=divide)
    return args, want


CASES = {
    "conv k5 d2": dict(),
    "conv k11 d5 slope 1 mode 2": dict(k=11, dil=5, slope=1.0, mode=2, divide=3, Cin=20, Cout=28),
    "convT u5 k11": dict(k=11, transposed=True, rate=5, dil=1, T_in=60, Cin=52, Cout=32, up=5),
    "convT u4 k8 mode 1": dict(k=8, transposed=True, rate=4, dil=1, T_in=70, Cin=16, Cout=96, up=4, mode=1),
    "convT u2 k2": dict(k=2, transposed=True, rate=2, dil=1, T_in=129, Cin=4, Cout=16, up=2),
}


@pytest.mark.parametrize("name", list(CASES))
def test_clean_emulation_passes(name):
    args, want = exact_case(**CASES[name])
    out = emulate(**args)
    rep = V.mismatch_exact(out, want, args["geo"], name)
    assert rep is None, rep


def _flagged(name, defect, **kw):
    args, want = exact_case(**dict(CASES[name], **kw))
    rep = V.mismatch_exact(emulate(**args, defect=defect), want, args["geo"], f"{name} with {defect}")
    assert rep is not None, f"{defect} was not flagged on {name}"
    return rep


def test_tap_defects_are_flagged():
    for name in ("convT u5 k11", "convT u4 k8 mode 1"):
        rep = _flagged(name, "tap_off_by_one")
        assert "phases [0, 1" in rep, rep
        rep = _flagged(name, "swap_tap_bases")
        assert "phases [0, 1]" in rep, rep


def test_missing_halo_row_is_flagged_in_its_tile():
    for name in ("conv k5 d2", "conv k11 d5 slope 1 mode 2"):
        rep = _flagged(name, "missing_halo_row", mask_edges=False)
        assert "flagged tiles [1]" in rep, rep


def test_product_defects_are_flagged():
    rep = _flagged("convT u4 k8 mode 1", "drop_hi_lo_chunk")
    assert "channel tiles [1]" in rep, rep
    for name in CASES:
        _flagged(name, "add_lo_lo")


def test_leaky_after_split_is_flagged():
    _flagged("conv k5 d2", "leaky_after_split")
    _flagged("convT u5 k11", "leaky_after_split")


def test_epilogue_defects_are_flagged():
    args, want = exact_case(**CASES["conv k5 d2"])
    rep = V.mismatch_exact(emulate(**args, defect="mask_not_zeroed"), want, args["geo"])
    masked = ~V.position_mask(args["valid"], 1, args["geo"].T_out)
    assert rep is not None and f"{int(masked.sum()) * 64} of" in rep, rep
    _flagged("conv k11 d5 slope 1 mode 2", "mode2_overwrites")
    _flagged("conv k11 d5 slope 1 mode 2", "no_divide")


def test_exact_operands_hold_their_contract():
    x, t = V.exact_activation(500, 64, 3, 0.7, 0.1, seed=4)
    assert bool((x < 0).any()) and bool((t != 0).any())
    h, l = V.split_f32(t)
    assert torch.equal(h, h.round()) and bool((l != 0).any())
    geo = V.Geometry(11, False, 1, 5, 300, 64)
    w = V.exact_values((64, 512, 11), 1, 1.0, seed=5)
    x2, t2 = V.exact_activation(300, 512, 1, 1.0, 1.0, seed=6)
    with pytest.raises(AssertionError, match="not exact"):
        V.split_exact_acc(t2, w, geo)


# ----------------------------------------------------------------------------------------------------- random mode
def test_random_bound_holds_and_sees_a_dropped_product():
    g = torch.Generator().manual_seed(3)
    for k, tr, u, d, Cin, Cout in ((7, False, 1, 3, 96, 64), (8, True, 4, 1, 64, 32), (3, False, 1, 1, 32, 128)):
        T_in = 200
        geo = V.Geometry(k, tr, u, d, T_in, Cout)
        x = torch.randn(T_in, Cin, generator=g)
        w = torch.randn((Cin, Cout, k) if tr else (Cout, Cin, k), generator=g) / (Cin * k) ** 0.5
        bias = torch.randn(Cout, generator=g) * 0.1
        res = torch.randn(geo.T_out, Cout, generator=g)
        sum_in = torch.randn(geo.T_out, Cout, generator=g)
        valid = torch.ones(geo.T_out // u, dtype=torch.uint8)
        valid[3] = 0
        live = V.position_mask(valid, u, geo.T_out)
        want, bound = V.layer_bound(x, w, bias, geo, 0.1, live, res, 2, sum_in, 3)
        args = dict(x=x, w=w, bias=bias, geo=geo, slope=0.1, valid=valid, up=u, res=res, mode=2, sum_in=sum_in, divide=3)
        rep = V.mismatch_bound(emulate(**args, exact=False), want, bound, geo, "fp32 emulation")
        assert rep is None, rep
    # one input chunk (all of Cin = 32) of channel tile 1 without its hi*lo product
    rep = V.mismatch_bound(emulate(**args, exact=False, defect="drop_hi_lo_chunk"), want, bound, geo)
    assert rep is not None and "channel tiles [1]" in rep, rep


def test_post_bound_holds():
    g = torch.Generator().manual_seed(8)
    C, n, start = 16, 300, 40
    S = torch.randn(start + n + 40, C, generator=g)
    w = torch.randn(1, C, 7, generator=g) / 5
    b = torch.tensor([0.05])
    want, bound = V.post_bound(S, w, b, start, n)
    a = torch.zeros(n) + 0.0
    seg = S[start - 3:start + n + 3]
    lk = torch.where(seg > 0, seg, seg * torch.tensor(0.01, dtype=torch.float32))
    for c in range(C):
        for k in range(7):
            a = a + w[0, c, k] * lk[k:k + n, c]
    out = torch.tanh(a + b)
    bad = ((out.double() - want).abs() > bound)
    assert not bool(bad.any())
    assert bool(((out.double() + 4 * bound - want).abs() > bound).any())


# ----------------------------------------------------------------------------------------------------- durations
def _dur_sd(E, H, seed=0):
    g = torch.Generator().manual_seed(seed)
    sd = {"dict.weight": torch.randn(50, E, generator=g)}
    for n, s in (("conv1.0", (H, E, 3)), ("conv2.0", (H, H, 3))):
        sd[f"dur_predictor.{n}.weight"] = torch.randn(s, generator=g) / (s[1] * 3) ** 0.5
        sd[f"dur_predictor.{n}.bias"] = 0.05 * torch.randn(H, generator=g)
    for n in ("ln1", "ln2"):
        sd[f"dur_predictor.{n}.weight"] = 1 + 0.1 * torch.randn(H, generator=g)
        sd[f"dur_predictor.{n}.bias"] = 0.1 * torch.randn(H, generator=g)
    sd["dur_predictor.proj.weight"] = 0.5 * torch.randn(1, H, generator=g) / H ** 0.5
    sd["dur_predictor.proj.bias"] = torch.tensor([0.9])
    return sd


def _dur_emulation(units, sd, eps=1e-5):
    """dur_kernel in fp32 (sums in torch's order, not the kernel's)."""
    p = lambda n: sd["dur_predictor." + n].float()
    x = sd["dict.weight"].float()[units].t()[None]
    ln = lambda a, gm, bt: F.layer_norm(a, a.shape[-1:], gm, bt, eps)
    h1 = ln(F.conv1d(x, p("conv1.0.weight"), p("conv1.0.bias"), padding=1)[0].t().clamp_min(0), p("ln1.weight"), p("ln1.bias"))
    h2 = ln(F.conv1d(h1.t()[None], p("conv2.0.weight"), p("conv2.0.bias"), padding=1)[0].t().clamp_min(0),
            p("ln2.weight"), p("ln2.bias"))
    return (h2 * p("proj.weight").reshape(-1)).sum(-1) + p("proj.bias")


def test_dur_predictor_bound_holds():
    for E, H in ((64, 32), (128, 100)):
        sd = _dur_sd(E, H)
        units = torch.randint(0, 50, (33,), generator=torch.Generator().manual_seed(1))
        v, e = V.dur_predictor_bound(units, sd)
        got = _dur_emulation(units, sd)
        assert bool(((got.double() - v).abs() <= e).all())
        assert float(e.max()) < 5e-2   # a worst-case bound: three LayerNorm rstd factors amplify it


def _half_integer_logds():
    """fp32 v whose fl32(exp(v)) - 1 is exactly n + 0.5 for several n."""
    out = []
    for n in range(1, 9):
        v = torch.tensor(math.log(n + 1.5), dtype=torch.float32)
        for _ in range(64):
            pre = torch.exp(v) - 1
            if float(pre) == n + 0.5:
                out.append(v.clone())
                break
            v = torch.nextafter(v, torch.tensor(math.inf if float(pre) < n + 0.5 else -math.inf))
    assert len(out) >= 4
    return torch.stack(out)


def test_rounding_rule_is_checked():
    v = torch.cat([_half_integer_logds(), torch.linspace(-2, 3, 50)])
    pre = torch.exp(v) - 1
    rint = torch.round(pre).clamp_min(1).long()
    assert V.mismatch_durations(rint, v, pre) is None
    assert V.mismatch_durations(rint, v) is None
    away = torch.floor(pre + 0.5).clamp_min(1).long()
    rep = V.mismatch_durations(away, v, pre)
    assert rep is not None, "round-half-away was not flagged"


# ----------------------------------------------------------------------------------------------------- expansion
def _expand_emulation(pk, units, durs, emb, defect=None):
    """expand_kernel: binary search of the row over starts, then of the unit over the inclusive prefix of durations."""
    T0, starts, frames = pk["T0"], pk["starts"], pk["frames"]
    x0 = torch.zeros(T0, emb.shape[1])
    valid = torch.zeros(T0, dtype=torch.uint8)
    cums = [torch.cumsum(d, 0) for d in durs]
    for f in range(T0):
        b = max([i for i, s in enumerate(starts) if s <= f], default=-1)
        if b < 0 or f - starts[b] >= frames[b]:
            continue
        local, c = f - starts[b], cums[b]
        a, z = 0, len(c) - 1
        while a < z:
            mid = (a + z) // 2
            if (c[mid] >= local if defect == "boundary_shift" else c[mid] > local):
                z = mid
            else:
                a = mid + 1
        valid[f] = 1
        x0[f] = emb[units[b][a]]
    return x0, valid


def test_expansion_defect_is_flagged():
    g = torch.Generator().manual_seed(2)
    emb = torch.randn(20, 8, generator=g)
    units = [torch.randint(0, 20, (n,), generator=g) for n in (1, 33, 5)]
    durs = [torch.randint(1, 4, (len(u),), generator=g) for u in units]
    pk = V.pack_rows(units, durs, 3, emb)
    assert pk["T0"] == sum(int(d.sum()) for d in durs) + 4 * 3
    x0, valid = _expand_emulation(pk, units, durs, emb)
    assert V.mismatch_frames(x0, valid, pk) is None
    x0, valid = _expand_emulation(pk, units, durs, emb, defect="boundary_shift")
    rep = V.mismatch_frames(x0, valid, pk)
    assert rep is not None and "row 1, frame" in rep, rep
