"""Conformance of the HiFi-GAN unit vocoder per element, against the references of tests/vocoder_ref.py.

Each convolution layer is reached through the sk_vocoder_conv hook, which runs it exactly as sk_vocoder_run does (the
same weight preparation and launcher).  On exact split operands the three-product accumulator is exact in fp32, so the
outputs are compared bit for bit across tile widths, kernels, dilations, the polyphase transposed convs, the time-tile
edges, the epilogue modes and masked frames.  Real-width layers of the benchmark geometry are checked against float64
under a per-element bound, and the whole benchmark network is run layer by layer (each layer checked from the device's
own input to it), with sk_vocoder_run's waveform checked against conv_post of the chain's last sum.  Then the duration
predictor and the durations prefix, guard bands, launch chains and argument checks.
References are computed in float64 on the GPU.
"""
import ctypes as C

import pytest
import torch

import vocoder_ref as V

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
DENSITY = 0.6


# ----------------------------------------------------------------------------------------------------- the hook
def _desc(x, w, bias, geo, slope, valid, up, y=None, res=None, sm=None, mode=0, divide=0, prep=None):
    from slamkit_b200.vocoder import SkVocoderConvDesc
    p = lambda t: t.data_ptr() if t is not None else None
    d = SkVocoderConvDesc()
    d.T_in, d.Cin, d.Cout, d.k = geo.T_in, w.shape[0] if geo.transposed else w.shape[1], geo.Cout, geo.k
    d.transposed, d.rate, d.dilation, d.slope = int(geo.transposed), geo.rate, geo.dil, slope
    d.x, d.weight, d.bias, d.valid, d.up, d.mode = p(x), p(w), p(bias), p(valid), up, mode
    d.y, d.res, d.sum, d.divide = p(y), p(res), p(sm), divide
    d.prep, d.prep_bytes = p(prep), prep.numel() if prep is not None else 0
    return d


def _prep(geo, Cin):
    return torch.empty(V.prep_bytes(geo.Cout, Cin, geo.k), dtype=torch.uint8, device=DEV)


def _hook(x, w, bias, geo, slope, valid, up, y=None, res=None, sm=None, mode=0, divide=0, sync=True):
    from slamkit_b200 import _lib as L
    lib = L.require_cuda()
    prep = _prep(geo, x.shape[1])
    L.check(lib.sk_vocoder_conv(C.byref(_desc(x, w, bias, geo, slope, valid, up, y, res, sm, mode, divide, prep)),
                                L.stream_ptr()))
    if sync:
        torch.cuda.synchronize()
    return prep


def _valid(geo, up, seed, edges=True):
    g = torch.Generator().manual_seed(seed)
    valid = (torch.rand(geo.T_out // up, generator=g) < 0.9).to(torch.uint8)
    if edges:   # frames holding the first / last position and the positions around time-tile edges
        for o in (0, BM - 1, BM, 2 * BM - 1, 2 * BM, geo.T_out - 1):
            if o < geo.T_out:
                valid[o // up] = 0
    return valid


BM = V.BM


# ----------------------------------------------------------------------------------------------------- a. exact sweep
NT_OF = {16: 1, 28: 1, 32: 2, 48: 2, 64: 4, 96: 4, 256: 4, 512: 4}
COUTS = list(NT_OF)
CINS = [4, 16, 20, 32, 48, 52, 128, 512]
QS = [1, 127, 128, 129, 255, 257]


def _cases():
    cases = []
    for i in range(24):
        k, dil = [3, 5, 7, 11][i % 4], [1, 2, 3, 5][(i // 4) % 4]
        mode = [0, 1, 2][(i // 2) % 3]
        cases.append(dict(k=k, transposed=False, rate=1, dil=dil, T_in=QS[i % 6], Cin=CINS[(3 * i + 1) % 8],
                          Cout=COUTS[i % 8], slope=[1.0, 0.1][(i // 3) % 2], mode=mode,
                          divide=[0, 1, 3][(i // 5) % 3] if mode else 0, res=bool(mode or i % 2), seed=i))
    pairs = [(5, 11), (4, 8), (2, 4), (4, 4), (5, 5), (2, 2)]
    for i in range(12):
        u, k = pairs[i % 6]
        pad = (k - u) // 2
        mode = [0, 1, 2][i % 3]
        cases.append(dict(k=k, transposed=True, rate=u, dil=1, T_in=max(1, QS[(i + 1) % 6] - -(-pad // u)),
                          Cin=CINS[(5 * i + 2) % 8], Cout=COUTS[(i + 3) % 8], slope=0.1, mode=mode,
                          divide=[0, 3, 1][i % 3] if mode == 2 else 0, res=bool(i % 2 or mode), seed=100 + i))
    cases.append(dict(k=11, transposed=False, rate=1, dil=5, T_in=4100, Cin=128, Cout=64, slope=0.1, mode=2, divide=3,
                      res=True, seed=200))
    cases.append(dict(k=11, transposed=True, rate=5, dil=1, T_in=900, Cin=512, Cout=256, slope=0.1, mode=0, divide=0,
                      res=False, seed=201))
    return cases


CASES = _cases()


def _cid(c):
    kind = f"T{c['rate']}" if c["transposed"] else f"d{c['dil']}"
    return f"k{c['k']}{kind}-T{c['T_in']}-{c['Cin']}x{c['Cout']}-s{c['slope']}-m{c['mode']}/{c['divide']}-{c['seed']}"


def exact_case(c):
    geo = V.Geometry(c["k"], c["transposed"], c["rate"], c["dil"], c["T_in"], c["Cout"])
    assert V.pick_nt(c["Cout"]) == NT_OF[c["Cout"]]
    Cin = c["Cin"]
    K = len(geo.phases[0]) * Cin
    x, t = V.exact_activation(c["T_in"], Cin, V.exact_amax(K, DENSITY), DENSITY, c["slope"], c["seed"], DEV)
    wshape = (Cin, geo.Cout, geo.k) if geo.transposed else (geo.Cout, Cin, geo.k)
    w = V.exact_values(wshape, V.exact_amax(K, DENSITY), DENSITY, c["seed"] + 1, DEV)
    g = torch.Generator(device=DEV).manual_seed(c["seed"] + 2)
    bias = torch.randn(geo.Cout, generator=g, device=DEV)
    up = c["rate"] if geo.transposed else next(u for u in (4, 2, 1) if geo.T_out % u == 0)
    valid = _valid(geo, up, c["seed"]).to(DEV)
    res = torch.randn(geo.T_out, geo.Cout, generator=g, device=DEV) if c["res"] else None
    sm = torch.randn(geo.T_out, geo.Cout, generator=g, device=DEV) if c["mode"] == 2 else \
        torch.full((geo.T_out, geo.Cout), float("nan"), device=DEV)
    live = V.position_mask(valid, up, geo.T_out)
    want = V.exact_epilogue(V.split_exact_acc(t, w, geo), bias, live, res, c["mode"], sm.clone(), c["divide"])
    return geo, dict(x=x, w=w, bias=bias, geo=geo, slope=c["slope"], valid=valid, up=up, res=res), sm, want


@pytest.mark.parametrize("c", CASES, ids=[_cid(c) for c in CASES])
def test_exact_layer(c):
    geo, args, sm, want = exact_case(c)
    y = torch.full((geo.T_out, geo.Cout), 777.0, device=DEV)
    if c["mode"] == 0:
        _hook(**args, y=y)
        out = y
    else:
        _hook(**args, y=y, sm=sm, mode=c["mode"], divide=c["divide"])
        out = sm
        assert bool((y == 777.0).all()), "y was written in a sum mode"
    rep = V.mismatch_exact(out, want, geo, _cid(c))
    assert rep is None, rep
    live = V.position_mask(args["valid"], args["up"], geo.T_out).to(DEV)
    assert bool((out[~live] == 0).all()) and bool((args["x"] != 0).any())


# ----------------------------------------------------------------------------------------------------- b. random layers
# real-width layers of the benchmark geometry (test_gpu_vocoder.BENCH_CFG): (Cin, Cout, k, transposed, rate, dil, T_in)
REAL = [
    (128, 512, 7, False, 1, 1, 300),
    (512, 256, 11, True, 5, 1, 120),
    (256, 256, 11, False, 1, 5, 600),
    (256, 256, 3, False, 1, 1, 600),
    (256, 128, 8, True, 4, 1, 150),
    (128, 128, 7, False, 1, 3, 600),
    (64, 32, 8, True, 4, 1, 300),
    (32, 32, 11, False, 1, 5, 1200),
    (32, 16, 4, True, 2, 1, 1200),
    (16, 16, 7, False, 1, 3, 2400),
]


@pytest.mark.parametrize("layer", REAL, ids=[f"{l[0]}x{l[1]}-k{l[2]}{'T' if l[3] else 'd'}{l[4] if l[3] else l[5]}" for l in REAL])
def test_random_layer_vs_fp64(layer):
    Cin, Cout, k, tr, u, d, T_in = layer
    geo = V.Geometry(k, tr, u, d, T_in, Cout)
    g = torch.Generator(device=DEV).manual_seed(Cin * 7 + k)
    x = torch.randn(T_in, Cin, generator=g, device=DEV)
    w = torch.randn((Cin, Cout, k) if tr else (Cout, Cin, k), generator=g, device=DEV) * (0.5 / (Cin * k) ** 0.5)
    bias = 0.05 * torch.randn(Cout, generator=g, device=DEV)
    up = u if tr else 4
    valid = _valid(geo, up, k).to(DEV)
    live = V.position_mask(valid, up, geo.T_out)
    res = torch.randn(geo.T_out, Cout, generator=g, device=DEV)
    sm = torch.randn(geo.T_out, Cout, generator=g, device=DEV)
    want, bound = V.layer_bound(x, w, bias, geo, 0.1, live, res, 2, sm.clone(), 3)
    _hook(x, w, bias, geo, 0.1, valid, up, res=res, sm=sm, mode=2, divide=3)
    rep = V.mismatch_bound(sm, want, bound, geo, "real-width layer")
    assert rep is None, rep


# ----------------------------------------------------------------------------------------------------- c. stage chain
@pytest.fixture(scope="module")
def bench():
    import test_gpu_vocoder as TV
    from slamkit_b200.vocoder import HifiGanB200Vocoder, fold_weight_norm
    sd = TV._random_state_dict(TV.BENCH_CFG, seed=11)
    voc = HifiGanB200Vocoder(TV.BENCH_CFG, sd, device=DEV, max_rows=4, max_frames=512)
    folded = {k: v.to(DEV) for k, v in fold_weight_norm(sd).items()}
    return TV.BENCH_CFG, voc, folded


def test_stage_chain_and_waveform(bench):
    cfg, voc, W = bench
    g = torch.Generator().manual_seed(4)
    lens = [7, 19, 3]
    codes = torch.stack([torch.cat([torch.randint(0, 500, (n,), generator=g), torch.full((19 - n,), -1)]) for n in lens])
    counts = torch.tensor(lens, dtype=torch.int32)
    dur, _, frames, _ = voc.durations(codes, counts)
    durs = [dur[b, :n].cpu() for b, n in enumerate(lens)]
    units = [codes[b, :n] for b, n in enumerate(lens)]
    assert [int(d.sum()) for d in durs] == frames.cpu().tolist()
    G0 = int(voc.lib.sk_vocoder_gap(voc._h))
    pk = V.pack_rows(units, durs, G0, W["dict.weight"].cpu())
    T0, x0, valid = pk["T0"], pk["x0"].to(DEV), pk["valid"].to(DEV)
    nk = len(cfg["resblock_kernel_sizes"])
    C0 = cfg["upsample_initial_channel"]
    U_total = voc.upsampling
    act, U, ch = T0 * C0, 1, C0
    for u in cfg["upsample_rates"]:
        U, ch = U * u, ch // 2
        act = max(act, T0 * U * ch)
    bufs = [torch.zeros(act, device=DEV) for _ in range(4)]
    Xb, Yb, Tb, Sb = bufs
    view = lambda b, T, Cc: b[:T * Cc].view(T, Cc)
    failures = []

    def layer(name, x, T_in, Cout, k, tr, u, dil, slope, y, res, sm, mode, divide, up):
        geo = V.Geometry(k, tr, u, dil, T_in, Cout)
        live = V.position_mask(valid, up, geo.T_out)
        want, bound = V.layer_bound(x.clone(), W[name + ".weight"], W[name + ".bias"], geo, slope, live,
                                    None if res is None else res.clone(), mode,
                                    None if sm is None else sm.clone(), divide)
        _hook(x, W[name + ".weight"], W[name + ".bias"], geo, slope, valid, up, y=y, res=res, sm=sm, mode=mode,
              divide=divide, sync=False)
        out = y if mode == 0 else sm
        rep = V.mismatch_bound(out, want, bound, geo, name, [s * up for s in pk["starts"]])
        if rep:
            failures.append(rep)

    S = view(Sb, T0, C0)
    layer("conv_pre", x0, T0, C0, 7, False, 1, 1, 1.0, S, None, None, 0, 0, 1)
    U, ch = 1, C0
    for i, (u, k) in enumerate(zip(cfg["upsample_rates"], cfg["upsample_kernel_sizes"])):
        T_in, U, ch = T0 * U, U * u, ch // 2
        T = T0 * U
        S_in = view(Sb, T_in, ch * 2)
        X, Y, Tm, S = view(Xb, T, ch), view(Yb, T, ch), view(Tb, T, ch), view(Sb, T, ch)
        layer(f"ups.{i}", S_in, T_in, ch, k, True, u, 1, 0.1, X, None, None, 0, 0, U)
        for j, (rk, dl) in enumerate(zip(cfg["resblock_kernel_sizes"], cfg["resblock_dilation_sizes"])):
            cur = X
            p = f"resblocks.{i * nk + j}"
            for a in range(3):
                layer(f"{p}.convs1.{a}", cur, T, ch, rk, False, 1, dl[a], 0.1, Tm, None, None, 0, 0, U)
                if a < 2:
                    layer(f"{p}.convs2.{a}", Tm, T, ch, rk, False, 1, 1, 0.1, Y, cur, None, 0, 0, U)
                    cur = Y
                else:
                    layer(f"{p}.convs2.{a}", Tm, T, ch, rk, False, 1, 1, 0.1, None, cur, S, 1 if j == 0 else 2,
                          nk if j == nk - 1 else 0, U)
        assert not failures, "\n".join(failures[:3])
    assert U == U_total
    wave, wl = voc.vocode_batch(codes, counts)
    for b in range(len(lens)):
        n = int(wl[b])
        want, bound = V.post_bound(S, W["conv_post.weight"], W["conv_post.bias"], pk["starts"][b] * U, n)
        rep = V.mismatch_wave(wave[b, :n], want, bound, U, f"row {b} waveform vs conv_post of the chain")
        assert rep is None, rep


# ----------------------------------------------------------------------------------------------------- d. durations
def _dur_cfg(E, H):
    return dict(resblock_kernel_sizes=[3], resblock_dilation_sizes=[[1, 1, 1]], upsample_rates=[2],
                upsample_kernel_sizes=[4], upsample_initial_channel=16, model_in_dim=E, num_embeddings=100,
                embedding_dim=E, dur_predictor_params=dict(encoder_embed_dim=E, var_pred_hidden_dim=H,
                                                           var_pred_kernel_size=3, var_pred_dropout=0.5))


@pytest.mark.parametrize("H", [32, 100, 128, 1024])
def test_durations_vs_fp64(H):
    import test_gpu_vocoder as TV
    from slamkit_b200.vocoder import HifiGanB200Vocoder, fold_weight_norm
    cfg = _dur_cfg(128, H)
    sd = TV._random_state_dict(cfg, seed=H)
    voc = HifiGanB200Vocoder(cfg, sd, device=DEV, max_rows=8, max_frames=4096)
    W = {k: v.to(DEV) for k, v in fold_weight_norm(sd).items()}
    lens = [1, 2, 3, 31, 32, 33, 65]
    g = torch.Generator().manual_seed(H + 1)
    codes = torch.full((len(lens), 65), -1, dtype=torch.int64)
    for b, n in enumerate(lens):
        codes[b, :n] = torch.randint(0, 100, (n,), generator=g)
    dur, logd, frames, status = voc.durations(codes, torch.tensor(lens, dtype=torch.int32))
    torch.cuda.synchronize()
    assert int(status.sum()) == 0
    for b, n in enumerate(lens):
        v, e = V.dur_predictor_bound(codes[b, :n].to(DEV), W)
        bad = ~((logd[b, :n].double() - v).abs() <= e)
        assert not bool(bad.any()), f"H={H} row {b} ({n} units): log_dur off at units {bad.nonzero().flatten()[:8].tolist()}"
        rep = V.mismatch_durations(dur[b, :n], logd[b, :n], what=f"H={H} row {b}")
        assert rep is None, rep
        assert int(frames[b]) == int(dur[b, :n].long().sum()), f"row {b}: frames != sum of durations"


# ----------------------------------------------------------------------------------------------------- e. buffers
def _small_exact(mode=0, divide=0, seed=0):
    c = dict(k=3, transposed=False, rate=1, dil=1, T_in=300, Cin=32, Cout=64, slope=0.1, mode=mode, divide=divide,
             res=True, seed=seed)
    return exact_case(c)


def test_nan_sum_guard_bands_and_repeat():
    margin = 1024
    geo, args, sm, want = _small_exact(mode=1, divide=3)
    n = geo.T_out * geo.Cout
    sbuf = torch.full((n + 2 * margin,), float("nan"), device=DEV)
    ybuf = torch.full((n + 2 * margin,), 12345.0, device=DEV)
    s_out, y_out = sbuf[margin:margin + n].view(geo.T_out, geo.Cout), ybuf[margin:margin + n].view(geo.T_out, geo.Cout)
    _hook(**args, y=y_out, sm=s_out, mode=1, divide=3)
    assert bool(torch.isfinite(s_out).all()), "mode 1 read the NaN-poisoned sum"
    assert V.mismatch_exact(s_out, want, geo, "mode 1 over NaN") is None
    assert bool(torch.isnan(sbuf[:margin]).all()) and bool(torch.isnan(sbuf[margin + n:]).all())
    assert bool((ybuf == 12345.0).all()), "y was written in mode 1"
    first = s_out.clone()
    _hook(**args, y=y_out, sm=s_out, mode=1, divide=3)
    assert torch.equal(first, s_out), "two runs differ"
    geo, args, sm, want = _small_exact(mode=0, seed=3)
    _hook(**args, y=y_out)
    assert V.mismatch_exact(y_out, want, geo, "mode 0 in a guarded buffer") is None
    assert bool((ybuf[:margin] == 12345.0).all()) and bool((ybuf[margin + n:] == 12345.0).all())


def test_back_to_back_launches():
    g = torch.Generator(device=DEV).manual_seed(9)
    T = 400
    ga, gb = V.Geometry(7, False, 1, 3, T, 64), V.Geometry(8, True, 4, 1, T, 32)
    x = torch.randn(T, 48, generator=g, device=DEV)
    wa = torch.randn(64, 48, 7, generator=g, device=DEV) / 18
    wb = torch.randn(64, 32, 8, generator=g, device=DEV) / 22
    ba, bb = torch.randn(64, generator=g, device=DEV), torch.randn(32, generator=g, device=DEV)
    va, vb = torch.ones(T, dtype=torch.uint8, device=DEV), torch.ones(T, dtype=torch.uint8, device=DEV)
    vb[7] = 0
    outs = []
    for sync in (True, False):
        mid = torch.full((T, 64), float("nan"), device=DEV)
        out = torch.full((4 * T, 32), float("nan"), device=DEV)
        keep = [_hook(x, wa, ba, ga, 1.0, va, 1, y=mid, sync=sync),
                _hook(mid, wb, bb, gb, 0.1, vb, 4, y=out, sync=sync)]
        torch.cuda.synchronize()
        del keep
        outs.append((mid, out))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
    want, bound = V.layer_bound(outs[1][0], wb, bb, gb, 0.1, V.position_mask(vb, 4, 4 * T))
    assert V.mismatch_bound(outs[1][1], want, bound, gb, "second of two back-to-back launches") is None


# ----------------------------------------------------------------------------------------------------- f. argument checks
def test_argument_checks_launch_nothing():
    from slamkit_b200 import _lib as L
    lib = L.require_cuda()
    geo, args, sm, want = _small_exact()
    x, w, bias, valid = args["x"], args["w"], args["bias"], args["valid"]
    y = torch.full((geo.T_out, geo.Cout), 777.0, device=DEV)
    prep = _prep(geo, x.shape[1])
    big = torch.zeros(V.prep_bytes(512, 512, 32), dtype=torch.uint8, device=DEV)
    ok = lambda **kw: _desc(**dict(dict(x=x, w=w, bias=bias, geo=geo, slope=0.1, valid=valid, up=1, y=y, prep=prep), **kw))

    def edit(d, **kw):
        for k, v in kw.items():
            setattr(d, k, v)
        return d

    bad = {
        "Cin not a multiple of 4": edit(ok(), Cin=30),
        "Cout not a multiple of 4": edit(ok(), Cout=62),
        "kernel 33": edit(ok(prep=big), k=33),
        "even kernel of a conv": edit(ok(), k=4),
        "transposed with k - rate odd": edit(ok(), transposed=1, rate=2, k=3),
        "transposed with rate > k": edit(ok(), transposed=1, rate=4, k=2),
        "mode 3": edit(ok(), mode=3),
        "mode 0 with divide": edit(ok(), divide=2),
        "mode 0 without y": ok(y=None),
        "mode 2 without sum": edit(ok(), mode=2),
        "null x": ok(x=None),
        "null valid": ok(valid=None),
        "up not dividing T_out": edit(ok(), up=7),
        "prep too small": edit(ok(), prep_bytes=prep.numel() - 1),
        "halo over the shared-memory limit": edit(ok(prep=big), k=31, dilation=15),
    }
    torch.cuda.synchronize()
    for what, d in bad.items():
        before = int(lib.sk_launch_count())
        assert lib.sk_vocoder_conv(C.byref(d), L.stream_ptr()) != 0, f"{what}: accepted"
        assert int(lib.sk_launch_count()) == before, f"{what}: something was launched"
    torch.cuda.synchronize()
    assert bool((y == 777.0).all())
    before = int(lib.sk_launch_count())
    assert lib.sk_vocoder_conv(C.byref(ok()), L.stream_ptr()) == 0
    assert int(lib.sk_launch_count()) == before + 2   # prepare + conv
    torch.cuda.synchronize()


def _config(**kw):
    from slamkit_b200.vocoder import SkVocoderConfig
    E = kw.get("E", 128)
    c = SkVocoderConfig()
    c.num_embeddings, c.embedding_dim, c.model_in_dim = 100, E, E
    c.upsample_initial_channel = kw.get("C0", 512)
    c.n_upsamples = 1
    c.upsample_rates[0], c.upsample_kernel_sizes[0] = 2, 4
    c.n_resblocks = 1
    c.resblock_kernel_sizes[0] = kw.get("rk", 3)
    for a in range(3):
        c.resblock_dilations[0][a] = kw.get("dil", 1)
    c.dur_predictor, c.dur_hidden, c.dur_kernel = int("H" in kw), kw.get("H", 0), 3
    c.max_rows, c.max_frames = 2, 64
    return c


def test_create_refuses_what_run_cannot_launch():
    from slamkit_b200 import _lib as L
    lib = L.load()

    def create(**kw):
        h = C.c_void_p()
        rc = lib.sk_vocoder_create(C.byref(_config(**kw)), C.byref(h))
        if rc == 0:
            lib.sk_vocoder_destroy(h)
        return rc, lib.sk_last_error().decode()

    # kernel 31 at dilation 15: a 450-row halo fits 16-channel tiles, not 64-channel ones
    assert create(rk=31, dil=15, C0=32)[0] == 0
    rc, msg = create(rk=31, dil=15, C0=512)
    assert rc != 0 and "ResBlock kernel 31 at dilation 15" in msg and "shared memory" in msg, msg
    # the duration predictor's shared memory: (5 E + 3 H + 32) x 4 bytes <= 48 KB
    assert create(E=2048, H=128)[0] == 0
    rc, msg = create(E=2400, H=128)
    assert rc != 0 and "embedding_dim 2400" in msg and "shared memory" in msg, msg
    rc, msg = create(E=128, H=2048)
    assert rc != 0 and "var_pred_hidden_dim" in msg, msg
