"""Conformance of the gradient path of the train step: the kernels that turn dlogits into parameter updates for every
model family (Qwen2, pre- and post-LN OPT, GPT-NeoX, OPT with fp32 master weights).

Cross-entropy gradients are compared per element with float64 softmax - onehot under the bound of
tests/grad_ref.py; table gradients, column sums, LayerNorm dw / db, gradient norms, the fp32 AdamW and the small
kernels bit for bit against exact references.  Outputs sit between NaN guard bands that must stay untouched."""
import ctypes as C
import json
import time
import types

import numpy as np
import pytest
import torch

import grad_ref as R

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
BF = torch.bfloat16
PAD = 64


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
        view.copy_(torch.as_tensor(fill, dtype=dtype).reshape(shape))
    return buf, view


def _guard_ok(buf):
    return bool(buf[:PAD].isnan().all()) and bool(buf[-PAD:].isnan().all())


def _np(t):
    return t.float().cpu().numpy()


_KEEP = []   # device operands built inline as call arguments: kept alive until the test's launches have finished


def _dev(a, dtype):
    t = (a if isinstance(a, torch.Tensor) else torch.as_tensor(np.asarray(a))).to(dtype).to(DEV)
    _KEEP.append(t)
    return t


@pytest.fixture(autouse=True)
def _keep_operands():
    yield
    torch.cuda.synchronize()
    _KEEP.clear()


@pytest.fixture(scope="module", autouse=True)
def _timer():
    t0 = time.time()
    yield
    print(f"\ntest_gpu_grad_conformance: {time.time() - t0:.1f} s")


# ----------------------------------------------------------------------------------------------------- A. cross entropy
CE_SHAPES = [(2, 8, 64, 16), (502, 512, 256, 64), (513, 520, 64, 32), (8192, 8192, 48, 24), (152167, 152168, 8, 8)]


def _ce_inputs(V, ldl, M, T, seed):
    g = torch.Generator().manual_seed(seed)
    logits = (torch.randn(M, ldl, generator=g) * 3).to(BF)
    logits[:, V:] = float("nan")                              # padding columns are never read as logits
    labels = torch.randint(0, V, (M,), generator=g)
    labels[3::7] = -100
    labels[5] = V
    labels[6] = V + 1
    return logits, labels


def _ce_expect(logits, labels, T, V, ldl, gs, row_weight=None):
    x = _np(logits)
    d, nll, valid, lse, spread, p, g = R.ce_reference(np.nan_to_num(x, nan=-1e30), labels.numpy(), T, V, gs, row_weight)
    kern = "warp" if ldl <= 512 else "block"
    return d, nll, valid, R.ce_bound(kern, p, d, lse, spread, ldl, g), lse


@pytest.mark.parametrize("V,ldl,M,T", CE_SHAPES)
def test_ce_gradient_per_element(V, ldl, M, T):
    L, lib = _lib()
    logits, labels = _ce_inputs(V, ldl, M, T, V)
    n_items = 37.0
    dbuf, dl = _guarded((M, ldl), BF)
    partial = torch.empty(2 * lib.sk_ce_blocks(M), device=DEV)
    row_nll = torch.full((M,), float("nan"), device=DEV)
    stats = torch.zeros(3, device=DEV)
    lg, lb = logits.to(DEV), labels.to(DEV)
    L.check(lib.sk_ce_fwd_bwd(_p(lg), _p(lb), _p(dl), _p(partial), _p(row_nll), _p(stats), M, T, V, ldl, L.f32(n_items),
                              L.f32(1.0), L.stream_ptr()))
    torch.cuda.synchronize()
    assert _guard_ok(dbuf)
    gs = float(np.float32(1.0) / np.float32(n_items))
    d, nll, valid, bound, lse = _ce_expect(logits, labels, T, V, ldl, gs)
    errs = R.check_ce_grad(_np(dl), d, valid, V, bound)
    assert not errs, "\n".join(errs)
    rn = row_nll.cpu().numpy()
    assert bool((rn[~valid] == 0).all())
    tol = 1e-4 * (1 + np.abs(lse))
    assert bool((np.abs(rn - nll) <= tol).all()), float(np.abs(rn - nll).max())
    st = stats.cpu().numpy()
    assert st[1] == valid.sum()
    assert abs(st[2] - nll.sum()) <= tol.sum() and abs(st[0] - nll.sum() / n_items) <= tol.sum() / n_items


@pytest.mark.parametrize("V,ldl,M,T", [CE_SHAPES[1], CE_SHAPES[3]])
def test_ce_row_weight_and_mean_reduction(V, ldl, M, T):
    L, lib = _lib()
    logits, labels = _ce_inputs(V, ldl, M, T, 7)
    w = torch.linspace(-2.0, 3.0, M)
    lg, lb = logits.to(DEV), labels.to(DEV)
    partial = torch.empty(2 * lib.sk_ce_blocks(M), device=DEV)
    stats = torch.zeros(3, device=DEV)
    dl = torch.empty(M, ldl, dtype=BF, device=DEV)
    L.check(lib.sk_ce_fwd_bwd_weighted(_p(lg), _p(lb), _p(dl), _p(partial), None, _p(_dev(w, torch.float32)), _p(stats), M, T, V, ldl,
                                       L.f32(1.0), L.f32(1.0), L.stream_ptr()))
    d, _, valid, bound, _ = _ce_expect(logits, labels, T, V, ldl, 1.0, w.numpy())
    errs = R.check_ce_grad(_np(dl), d, valid, V, bound)
    assert not errs, "\n".join(errs)
    # mean over valid targets: the unscaled bf16 gradient, then bf16(fp32(c * (1 / n_valid))) by scale_by_inv_count
    dloss = 0.75
    L.check(lib.sk_ce_fwd_bwd(_p(lg), _p(lb), _p(dl), _p(partial), None, _p(stats), M, T, V, ldl, L.f32(0.0), L.f32(dloss),
                              L.stream_ptr()))
    d, _, valid, bound, _ = _ce_expect(logits, labels, T, V, ldl, dloss)
    sc = np.float32(1.0) / np.float32(valid.sum())
    lo = R.bf16((R.bf16_from64(d - bound) * sc).astype(np.float32))
    hi = R.bf16((R.bf16_from64(d + bound) * sc).astype(np.float32))
    got = _np(dl)
    bad = ~((got >= lo) & (got <= hi))
    assert not bad.any(), R.locate(bad, got, d * float(sc), "mean dlogits")[:6]
    assert float(stats[1]) == valid.sum()


def test_ce_chunked_head_rows():
    """The chunked lm_head's CE: a full chunk at row 0 and a ragged one at row0 = 32, gradient written over the logits."""
    L, lib = _lib()
    V, ldl, M, T = 8192, 8192, 48, 24
    logits, labels = _ce_inputs(V, ldl, M, T, 11)
    lb = labels.to(DEV)
    partial = torch.full((2 * M,), float("nan"), device=DEV)
    out = torch.empty(M, ldl, dtype=BF, device=DEV)
    gs = float(np.float32(0.5) / np.float32(29.0))
    for r0, rows in ((0, 32), (32, 16)):
        chunk = logits[r0:r0 + rows].to(DEV)
        L.check(lib.sk_ce_chunk(_p(chunk), _p(lb), _p(chunk), _p(partial), r0, rows, M, T, V, ldl, L.f32(gs), L.stream_ptr()))
        out[r0:r0 + rows] = chunk
    stats = torch.zeros(3, device=DEV)
    L.check(lib.sk_ce_finalize(_p(partial), M, L.f32(29.0), _p(stats), L.stream_ptr()))
    d, nll, valid, bound, lse = _ce_expect(logits, labels, T, V, ldl, gs)
    errs = R.check_ce_grad(_np(out), d, valid, V, bound)
    assert not errs, "\n".join(errs)
    pr = partial.cpu().numpy().reshape(M, 2)
    assert np.array_equal(pr[:, 1], valid.astype(np.float32))
    assert bool((np.abs(pr[:, 0] - nll) <= 1e-4 * (1 + np.abs(lse))).all())
    assert float(stats[1]) == valid.sum()


# ----------------------------------------------------------------------------------------------------- B. table gradients
def _scratch(rows, D):
    s = torch.full((2 * rows * D,), float("nan"), device=DEV)         # 64-bit words; the launcher clears them
    _KEEP.append(s)
    return s


@pytest.mark.parametrize("case", ["random", "one_id", "accumulate"])
def test_token_table_bf16_bit_exact(case):
    L, lib = _lib()
    M, D, V, Vp = 8192, 768, 502, 512
    dx = R.grid_values((M, D), 14, 255, 3)
    r = np.random.default_rng(4)
    ids = r.integers(0, V, size=M) if case != "one_id" else np.full(M, 7)
    ids[:3] = [-100, V, V + 1]                                  # skipped
    old = R.bf16(R.grid_values((Vp, D), 10, 200, 5)) if case == "accumulate" else None
    tbuf, tab = _guarded((Vp, D), BF, old if old is not None else np.zeros((Vp, D), np.float32))
    L.check(lib.sk_embed_bwd(_p(_dev(ids, torch.int64)), _p(_dev(dx, BF)), _p(_scratch(Vp, D)), _p(tab), M, D, V, Vp,
                             int(old is not None), L.stream_ptr()))
    torch.cuda.synchronize()
    assert _guard_ok(tbuf)
    rows = np.where((ids >= 0) & (ids < V), ids, -1)
    assert np.array_equal(R.table_fix_sum(rows, dx, Vp), R.index_add64(rows, dx, Vp))   # the grid makes it exact
    errs = R.check_exact(_np(tab), R.table_grad_bf16(rows, dx, Vp, old), "dE")
    assert not errs, "\n".join(errs)


def test_embed_forward_maps_skipped_ids_to_row_zero():
    """The forward reads row 0 for ids outside [0, V) (the reference would index out of range), the backward skips
    them: pad / ignore ids contribute nothing to any row."""
    L, lib = _lib()
    V, D = 502, 64
    E = torch.randn(V, D).to(BF).to(DEV)
    ids = torch.tensor([-100, V, V + 1, 5], dtype=torch.int64, device=DEV)
    out = torch.empty(4, D, dtype=BF, device=DEV)
    L.check(lib.sk_embed_fwd(_p(ids), _p(E), _p(out), 4, D, V, L.stream_ptr()))
    assert torch.equal(out[:3], E[0].expand(3, D)) and torch.equal(out[3], E[5])


@pytest.mark.parametrize("pos_kind", ["none", "packed", "clamped"])
@pytest.mark.parametrize("accumulate", [0, 1])
def test_position_table_bf16_bit_exact(pos_kind, accumulate):
    L, lib = _lib()
    B, T, D, n_pos = 4, 512, 768, 514
    M = B * T
    dx = R.grid_values((M, D), 16, 255, 6)
    if pos_kind == "none":
        pos = None
    elif pos_kind == "packed":
        pos = np.concatenate([np.concatenate([np.arange(n) for n in (100, 1, 411)])] * B).astype(np.int32)
    else:
        pos = (np.arange(M) % 700 - 3).astype(np.int32)        # past the table -> last row; below -2 -> row 0
    old = R.bf16(R.grid_values((n_pos, D), 9, 100, 7)) if accumulate else np.zeros((n_pos, D), np.float32)
    tbuf, tab = _guarded((n_pos, D), BF, old)
    L.check(lib.sk_opt_pos_bwd(_p(_dev(pos, torch.int32) if pos is not None else None), _p(_dev(dx, BF)),
                               _p(_scratch(n_pos, D)), _p(tab), M, T, D, n_pos, accumulate, L.stream_ptr()))
    torch.cuda.synchronize()
    assert _guard_ok(tbuf)
    rows = R.opt_pos_rows(pos, M, T, n_pos)
    errs = R.check_exact(_np(tab), R.table_grad_bf16(rows, dx, n_pos, old if accumulate else None), "dP")
    assert not errs, "\n".join(errs)


@pytest.mark.parametrize("keep", [0, 1])
def test_fp32_tables_with_tied_head_bit_exact(keep):
    L, lib = _lib()
    M, T, D, V, Vp, n_pos = 4096, 512, 768, 502, 512, 2050
    dx = R.grid_values((M, D), 30, 1 << 20, 8)                  # fp32 rows on a 2^-30 grid
    ids = np.random.default_rng(9).integers(0, V, size=M)
    ids[:64] = 11
    ids[64:67] = [-100, V, V + 1]
    head = R.bf16(R.grid_values((Vp, D), 12, 255, 10))
    old = R.grid_values((Vp, D), 24, 1 << 16, 11)
    tbuf, tab = _guarded((Vp, D), torch.float32, old)
    L.check(lib.sk_table_bwd_f32(_p(_dev(ids, torch.int64)), None, _p(_dev(dx, torch.float32)), _p(_scratch(Vp, D)), _p(tab),
                                 _p(_dev(head, BF)), M, T, D, V, Vp, keep, L.stream_ptr()))
    rows = np.where((ids >= 0) & (ids < V), ids, -1)
    want = R.table_grad_f32(rows, dx, Vp, head=head, old=old if keep else None)
    errs = R.check_exact(_np(tab), want, "dE fp32")
    pbuf, ptab = _guarded((n_pos, D), torch.float32, np.zeros((n_pos, D), np.float32))
    L.check(lib.sk_table_bwd_f32(None, None, _p(_dev(dx, torch.float32)), _p(_scratch(n_pos, D)), _p(ptab), None, M, T, D,
                                 n_pos, n_pos, keep, L.stream_ptr()))
    torch.cuda.synchronize()
    assert _guard_ok(tbuf) and _guard_ok(pbuf)
    errs += R.check_exact(_np(ptab), R.table_grad_f32(R.opt_pos_rows(None, M, T, n_pos), dx, n_pos), "dP fp32")
    assert not errs, "\n".join(errs)


@pytest.mark.parametrize("pos_kind", ["packed", "clamped"])
def test_fp32_position_table_with_position_ids(pos_kind):
    L, lib = _lib()
    B, T, D, n_pos = 4, 512, 768, 514
    M = B * T
    dx = R.grid_values((M, D), 30, 1 << 20, 12)
    if pos_kind == "packed":
        pos = np.concatenate([np.concatenate([np.arange(n) for n in (100, 1, 411)])] * B).astype(np.int32)
    else:
        pos = (np.arange(M) % 700 - 3).astype(np.int32)        # past the table -> last row; below -2 -> row 0
    old = R.grid_values((n_pos, D), 24, 1 << 16, 13)
    pbuf, ptab = _guarded((n_pos, D), torch.float32, old)
    L.check(lib.sk_table_bwd_f32(None, _p(_dev(pos, torch.int32)), _p(_dev(dx, torch.float32)), _p(_scratch(n_pos, D)),
                                 _p(ptab), None, M, T, D, n_pos, n_pos, 1, L.stream_ptr()))
    torch.cuda.synchronize()
    assert _guard_ok(pbuf)
    errs = R.check_exact(_np(ptab), R.table_grad_f32(R.opt_pos_rows(pos, M, T, n_pos), dx, n_pos, old=old), "dP fp32")
    assert not errs, "\n".join(errs)


def test_fixed_point_documented_range():
    """A 2^-40 term counts, terms at or below 2^-41 vanish, and sums reach just below 2^23 exactly."""
    L, lib = _lib()
    D = 8
    vals = np.array([2.0 ** -40, 2.0 ** -41, 2.0 ** -42, 3 * 2.0 ** -41, 2.0 ** 22 - 0.25, 2.0 ** 22 - 0.25, -2.0 ** -40, 1.0],
                    np.float32)
    dx = np.tile(vals[:, None], (1, D))
    ids = np.array([0, 1, 2, 3, 4, 4, 5, 6])
    tab = torch.zeros(8, D, device=DEV)
    L.check(lib.sk_table_bwd_f32(_p(_dev(ids, torch.int64)), None, _p(_dev(dx, torch.float32)), _p(_scratch(8, D)), _p(tab),
                                 None, 8, 8, D, 8, 8, 0, L.stream_ptr()))
    got = _np(tab)[:, 0]
    assert got[:7].tolist() == [2.0 ** -40, 0.0, 0.0, 2.0 ** -39, 2.0 ** 23 - 0.5, -2.0 ** -40, 1.0]


def test_fp32_table_precision_at_opt125m_magnitudes(monkeypatch):
    """The fp32 table gradient inherits the fixed point's 2^-41 rounding per term.  Measured on the residual gradient
    of one opt-125m forward-backward at [8, 512] (bf16 autocast, loss / num_items): per-element error of the kernel's
    token and position table gradients against float64, next to torch's fp32 index_add_ on the same rows."""
    from oracle import opt_oracle as O
    from oracle.lm_oracle import compute_loss
    L, lib = _lib()
    c = O.OracleOptConfig()                                    # opt-125m geometry, vocabulary 502
    p = {k: v.to(DEV) for k, v in O.init_params(c, seed=1, dtype=torch.float32).items()}
    B, T = 8, 512
    g = torch.Generator().manual_seed(2)
    ids = torch.randint(2, 502, (B, T), generator=g)
    ids[:, 0] = 1
    captured = []
    shim = types.SimpleNamespace(**{k: getattr(O.F, k) for k in dir(O.F) if not k.startswith("__")})

    def embedding(idx, table):
        out = torch.nn.functional.embedding(idx, table)
        if not captured:
            out.retain_grad()
            captured.append(out)
        return out
    shim.embedding = embedding
    monkeypatch.setattr(O, "F", shim)
    leaves = {k: v.clone().requires_grad_(True) for k, v in p.items()}
    ids_d = ids.to(DEV)
    with torch.autocast("cuda", dtype=torch.bfloat16):
        logits = O.forward_logits(leaves, c, ids_d)
        loss = compute_loss(logits, ids_d, float(B * (T - 1)))
    loss.backward()
    dres = captured[0].grad.float().reshape(B * T, -1).contiguous()      # d loss / d (embed_tokens + embed_positions)
    M, D = dres.shape
    report = {"dres_median_abs": float(dres.abs().median())}
    for name, idx, n_rows in (("token", ids.reshape(-1).numpy(), c.vocab_size),
                              ("position", R.opt_pos_rows(None, M, T, c.max_positions + 2), c.max_positions + 2)):
        tab = torch.zeros(n_rows, D, device=DEV)
        L.check(lib.sk_table_bwd_f32(_p(_dev(idx, torch.int64)) if name == "token" else None, None, _p(dres),
                                     _p(_scratch(n_rows, D)), _p(tab), None, M, T, D, n_rows, n_rows, 0, L.stream_ptr()))
        x = dres.cpu().numpy()
        ref = R.index_add64(idx, x, n_rows)
        tor = torch.zeros(n_rows, D).index_add_(0, torch.from_numpy(idx.astype(np.int64)), torch.from_numpy(x)).numpy()
        used = np.unique(idx)
        ek = np.abs(_np(tab)[used] - ref[used]).ravel()
        et = np.abs(tor[used] - ref[used]).ravel()
        ratio = float(np.median(ek)) / max(float(np.median(et)), 2.0 ** -149)
        report[name] = {"kernel_median": float(np.median(ek)), "torch_median": float(np.median(et)),
                        "kernel_max": float(ek.max()), "torch_max": float(et.max()), "ratio": ratio,
                        "grad_median_abs": float(np.median(np.abs(ref[used])))}
    print("fp32 table gradient precision:", json.dumps(report))
    for name in ("token", "position"):
        assert report[name]["ratio"] <= 4.0, report
        assert report[name]["kernel_max"] <= 2 * report[name]["torch_max"], report


# ----------------------------------------------------------------------------------------------------- C. colsum, LN
@pytest.mark.parametrize("M", [1, 7, 8192, 16384])
@pytest.mark.parametrize("N,ld", [(1152, 1152), (2304, 2312), (3 * 1024 + 8, 3 * 1024 + 8), (1000, 1000)])
def test_colsum_bit_exact(M, N, ld):
    L, lib = _lib()
    x = np.random.default_rng(M + N).integers(-8, 9, size=(M, ld)).astype(np.float32)
    x[:, N:] = np.nan                                          # columns past N are never read
    old = R.bf16(np.random.default_rng(1).integers(-100, 100, size=N).astype(np.float32))
    part = torch.empty(lib.sk_colsum_splits() * N, device=DEV)
    for acc in (0, 1):
        obuf, out = _guarded((N,), BF, old)
        L.check(lib.sk_colsum(_p(_dev(x, BF)), _p(out), _p(part), M, N, ld, acc, L.stream_ptr()))
        torch.cuda.synchronize()
        assert _guard_ok(obuf)
        errs = R.check_exact(_np(out), R.colsum_ref(x[:, :N], old if acc else None), f"colsum acc={acc}")
        assert not errs, "\n".join(errs)


def _ln_inputs(M, D, seed):
    r = np.random.default_rng(seed)
    x = r.integers(-16, 17, size=(M, D)).astype(np.float32)
    dy = r.integers(-8, 9, size=(M, D)).astype(np.float32)
    w = r.integers(-4, 5, size=D).astype(np.float32)
    mean = (r.integers(-4, 5, size=M) * 0.5).astype(np.float32)
    rstd = (2.0 ** -r.integers(0, 4, size=M)).astype(np.float32)
    return x, dy, w, mean, rstd


LN_D = [768, 896, 1024, 1032, 1536, 1544, 2048]


@pytest.mark.parametrize("D", LN_D)
@pytest.mark.parametrize("M", [7, 4096])
def test_layernorm_bwd_bf16_and_dual(D, M):
    L, lib = _lib()
    x, dy, w, mean, rstd = _ln_inputs(M, D, D + M)
    _, dy2, w2, _, _ = _ln_inputs(M, D, D + M + 1)
    dres = R.bf16(np.random.default_rng(3).integers(-64, 64, size=(M, D)).astype(np.float32) * 0.125)
    blocks = lib.sk_layernorm_bwd_blocks()
    old = R.bf16(np.arange(D, dtype=np.float32) % 17)
    dx = torch.empty(M, D, dtype=BF, device=DEV)
    bufs = [_guarded((D,), BF, old) for _ in range(4)]
    part = torch.empty(4 * blocks * D, device=DEV)
    args = [_p(_dev(a, t)) for a, t in ((x, BF), (w, BF), (mean, torch.float32), (rstd, torch.float32))]
    L.check(lib.sk_layernorm_bwd(_p(_dev(dy, BF)), args[0], args[1], args[2], args[3], _p(_dev(dres, BF)), _p(dx),
                                 _p(bufs[0][1]), _p(bufs[1][1]), _p(part), _p(part[blocks * D:]), M, D, 1, L.stream_ptr()))
    torch.cuda.synchronize()
    rdx, rdw, rdb = R.ln_bwd_ref(dy, x, w, mean, rstd)
    errs = R.check_exact(_np(bufs[0][1]), R.bf16((rdw.astype(np.float32) + old).astype(np.float32)), "dw")
    errs += R.check_exact(_np(bufs[1][1]), R.bf16((rdb.astype(np.float32) + old).astype(np.float32)), "db")
    errs += R.check_bf16_interval(_np(dx), rdx + dres, R.ln_dx_bound(dy, x, w, mean, rstd) + 2 * R.U * np.abs(rdx + dres),
                                  "dx")
    # dual LayerNorm (GPT-NeoX): dx from w1 dy1 + w2 dy2, four weight gradients, accumulate off
    bufs2 = [_guarded((D,), BF, old) for _ in range(4)]
    L.check(lib.sk_layernorm2_bwd(_p(_dev(dy, BF)), _p(_dev(dy2, BF)), args[0], args[1], _p(_dev(w2, BF)), args[2], args[3],
                                  None, _p(dx), *[_p(b[1]) for b in bufs2], _p(part), M, D, 0, L.stream_ptr()))
    torch.cuda.synchronize()
    r2 = R.ln_bwd_ref(dy, x, w, mean, rstd, dy2=dy2, w2=w2)
    for name, b, ref in zip(("dw1", "db1", "dw2", "db2"), bufs2, r2[1:]):
        errs += R.check_exact(_np(b[1]), R.bf16(ref.astype(np.float32)), name)
    errs += R.check_bf16_interval(_np(dx), r2[0], R.ln_dx_bound(dy, x, w, mean, rstd, dy2, w2) + 2 * R.U * np.abs(r2[0]),
                                  "dx dual")
    assert all(_guard_ok(b[0]) for b in bufs + bufs2)
    assert not errs, "\n".join(errs)


@pytest.mark.parametrize("D", LN_D)
@pytest.mark.parametrize("M,dres_mode", [(7, "none"), (4096, "alias"), (1100, "separate")])
def test_layernorm_bwd_f32(D, M, dres_mode):
    L, lib = _lib()
    x, dy, w, mean, rstd = _ln_inputs(M, D, 3 * D + M)
    blocks = lib.sk_layernorm_bwd_blocks()
    rin = np.random.default_rng(5).integers(-1000, 1000, size=(M, D)).astype(np.float32) * np.float32(2.0 ** -10)
    dres_out = _dev(rin if dres_mode == "alias" else np.zeros((M, D), np.float32), torch.float32)
    dres_in = {"none": None, "alias": dres_out, "separate": _dev(rin, torch.float32)}[dres_mode]
    d16 = torch.empty(M, D, dtype=BF, device=DEV)
    old = (np.arange(D) % 13).astype(np.float32)
    wb, dw = _guarded((D,), torch.float32, old)
    bb, db = _guarded((D,), torch.float32, old)
    part = torch.empty(2 * blocks * D, device=DEV)
    L.check(lib.sk_layernorm_bwd_f32(_p(_dev(dy, BF)), _p(_dev(x, torch.float32)), _p(_dev(w, torch.float32)),
                                     _p(_dev(mean, torch.float32)), _p(_dev(rstd, torch.float32)), _p(dres_in), _p(dres_out),
                                     _p(d16), _p(dw), _p(db), _p(part), M, D, 1, L.stream_ptr()))
    torch.cuda.synchronize()
    rdx, rdw, rdb = R.ln_bwd_ref(dy, x, w, mean, rstd)
    base = np.zeros_like(rdx) if dres_mode == "none" else rin.astype(np.float64)
    errs = R.check_exact(_np(dw), (rdw.astype(np.float32) + old).astype(np.float32), "dw")
    errs += R.check_exact(_np(db), (rdb.astype(np.float32) + old).astype(np.float32), "db")
    got = _np(dres_out)
    bound = R.ln_dx_bound(dy, x, w, mean, rstd) + 2 * R.U * np.abs(base + rdx)
    off = np.abs(got - (base + rdx)) > bound
    errs += R.locate(off, got, base + rdx, "dres_out")
    errs += R.check_exact(_np(d16), R.bf16(got), "dres16 = bf16(dres_out)")
    assert _guard_ok(wb) and _guard_ok(bb)
    assert not errs, "\n".join(errs)


# ----------------------------------------------------------------------------------------------------- D. norm and clip
def _norm_layout(n_layers=24):
    """268 tensors: a 24-layer list of 11 tensors each (more tensors than the finalize block has threads) between an
    embedding, a tensor split over five chunks, an all-zero tensor and an 8-element one."""
    sizes = [512 * 64]
    for _ in range(n_layers):
        sizes += [64, 64 * 96, 96, 64 * 64, 64, 64 * 256, 64 * 128, 64, 32, 32, 64]
    sizes += [70000, 64, 0 + 8]
    return sizes


def _run_norm(lib, L, flat, sizes, max_norm, dtype, emulate=1):
    offs, n, cs, cl, tb = R.chunk_tables(sizes, 16384)
    partial = torch.empty(len(cs), device=DEV)
    stats = torch.zeros(3, device=DEV)
    a = [_p(_dev(v, t)) for v, t in ((cs, torch.int64), (cl, torch.int32), (tb, torch.int32))]
    if dtype == BF:
        L.check(lib.sk_grad_norm(_p(flat), a[0], a[1], len(cs), a[2], len(sizes), _p(partial), L.f32(max_norm), emulate,
                                 _p(stats), L.stream_ptr()))
    else:
        L.check(lib.sk_grad_norm_f32(_p(flat), a[0], a[1], len(cs), a[2], len(sizes), _p(partial), L.f32(max_norm),
                                     _p(stats), L.stream_ptr()))
    return stats.cpu(), partial.cpu(), (cs, cl)


def _chunk_sumsq(flat, tables):
    """Exact per-chunk sums of squares of integer gradients (what sumsq_chunks_kernel writes to `partial`)."""
    f = flat.double()
    return torch.tensor([float((f[s:s + n] ** 2).sum()) for s, n in zip(*tables)], dtype=torch.float32)


def _norm_grads(sizes, dtype, seed, zero_all=False):
    offs, n, _, _, _ = R.chunk_tables(sizes, 16384)
    flat = torch.zeros(n, dtype=dtype)
    g = torch.Generator().manual_seed(seed)
    parts = []
    for i, (o, s) in enumerate(zip(offs, sizes)):
        v = torch.zeros(s) if zero_all or i == len(sizes) - 2 else torch.randint(-3, 4, (s,), generator=g).float()
        flat[o:o + s] = v.to(dtype)
        parts.append(flat[o:o + s].clone())
    return flat, parts


@pytest.mark.parametrize("dtype", [BF, torch.float32])
@pytest.mark.parametrize("max_norm", [0.5, 0.0, -1.0, "at_total", 1e9])
def test_grad_norm_and_coefficient_bit_exact(dtype, max_norm):
    L, lib = _lib()
    sizes = _norm_layout()
    assert len(sizes) > 256
    flat, parts = _norm_grads(sizes, dtype, 1)
    norms, total, _ = R.clip_grad_norm_ref(parts, 1.0)
    mn = float(total) if max_norm == "at_total" else max_norm
    _, _, coef = R.clip_grad_norm_ref(parts, mn)
    st, partial, tables = _run_norm(lib, L, flat.to(DEV), sizes, mn, dtype)
    # the per-tensor norms stay inside gradnorm_finalize_kernel; what it reads, the per-chunk sums of squares, is exact
    assert torch.equal(partial, _chunk_sumsq(flat, tables))
    assert float(st[0]) == float(total), (float(st[0]), float(total))
    assert float(st[1]) == float(coef), (float(st[1]), float(coef))
    ex = torch.linalg.vector_norm(torch.stack([torch.linalg.vector_norm(p.float()) for p in parts]))
    assert float(st[2]) == float(ex)
    if dtype == BF:   # emulate_bf16 = 0: the fp32 norms of the bf16 values
        st0 = _run_norm(lib, L, flat.to(DEV), sizes, mn, dtype, emulate=0)[0]
        assert float(st0[0]) == float(ex)


@pytest.mark.parametrize("dtype", [BF, torch.float32])
@pytest.mark.parametrize("bad", ["zero", "inf", "nan"])
def test_nonfinite_and_zero_totals_then_adamw_match_torch(dtype, bad):
    """clip_grad_norm_(error_if_nonfinite=False) followed by fused AdamW, as HF Trainer runs them."""
    L, lib = _lib()
    sizes = [64, 4096, 64]
    flat, parts = _norm_grads(sizes, dtype, 2, zero_all=(bad == "zero"))
    if bad != "zero":
        flat[64 + 5] = float(bad)
        parts[1][5] = float(bad)
    norms, total, coef = R.clip_grad_norm_ref(parts, 0.5)
    fl = flat.to(DEV)
    st = _run_norm(lib, L, fl, sizes, 0.5, dtype)[0]
    same = lambda a, b: (np.isnan(a) and np.isnan(b)) or a == b
    assert same(float(st[0]), float(total)) and same(float(st[1]), float(coef)), (st.tolist(), float(total), float(coef))
    # AdamW with the coefficient read from stats
    n = flat.numel()
    params = torch.linspace(-1, 1, n)
    hp = dict(lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-8, weight_decay=0.0)
    tp = torch.nn.Parameter(params.to(dtype).to(DEV).clone())
    tp.grad = fl.clone() * coef.to(DEV).to(dtype)
    opt = torch.optim.AdamW([tp], lr=hp["lr"], betas=(hp["beta1"], hp["beta2"]), eps=hp["eps"], weight_decay=0.0, fused=True)
    opt.step()
    m = torch.zeros(n, dtype=dtype, device=DEV)
    v = torch.zeros(n, dtype=dtype, device=DEV)
    p = params.to(dtype).to(DEV).clone()
    stats = st.to(DEV)
    if dtype == BF:
        L.check(lib.sk_adamw_step(_p(p), _p(fl), _p(m), _p(v), C.c_int64(n), L.f32(hp["lr"]), L.f32(0.9), L.f32(0.999),
                                  L.f32(1e-8), L.f32(0.0), 1, _p(stats), L.stream_ptr()))
        nan_k, nan_t = p.isnan(), tp.detach().isnan()
        assert torch.equal(nan_k, nan_t)
    else:
        shadow = torch.empty(n, dtype=BF, device=DEV)
        L.check(lib.sk_adamw_master_step(_p(p), _p(shadow), _p(fl), _p(m), _p(v), C.c_int64(n), L.f32(hp["lr"]), L.f32(0.9),
                                         L.f32(0.999), L.f32(1e-8), L.f32(0.0), 1, _p(stats), L.stream_ptr()))
        a, b = p.cpu(), tp.detach().cpu()
        assert torch.equal(a.isnan(), b.isnan())
        assert torch.equal(torch.nan_to_num(a), torch.nan_to_num(b))


# ----------------------------------------------------------------------------------------------------- E. AdamW
def _adam_state(n, seed):
    r = np.random.default_rng(seed)
    p = r.normal(0, 1, n).astype(np.float32)
    g = r.normal(0, 1e-2, n).astype(np.float32)
    g[:8] = [0.0, -0.0, 1e-40, -1e-42, 1e30, -1e30, 1e-3, 0.0]      # zero, subnormal, huge
    m = r.normal(0, 1e-3, n).astype(np.float32)
    v = np.abs(r.normal(0, 1e-5, n)).astype(np.float32)
    v[6:8] = 0.0
    return p, g, m, v


@pytest.mark.parametrize("n", [8, 3 * 132 * 8 * 256 * 4 + 8])
@pytest.mark.parametrize("step,wd,coef", [(1, 0.0, 1.0), (2, 0.1, 0.375), (10000, 0.01, 1.0)])
def test_adamw_master_bit_exact(n, step, wd, coef):
    L, lib = _lib()
    p, g, m, v = _adam_state(n, n + step)
    d = [_dev(a, torch.float32) for a in (p, g, m, v)]
    sbuf, shadow = _guarded((n,), BF)
    stats = torch.tensor([1.0, coef, 1.0], device=DEV)
    L.check(lib.sk_adamw_master_step(_p(d[0]), _p(shadow), _p(d[1]), _p(d[2]), _p(d[3]), C.c_int64(n), L.f32(1e-3), L.f32(0.9),
                                     L.f32(0.999), L.f32(1e-8), L.f32(wd), step, _p(stats), L.stream_ptr()))
    torch.cuda.synchronize()
    want = R.adamw_master(p, g, m, v, lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-8, wd=wd, step=step, coef=coef)
    errs = []
    for name, got, w in zip(("param", "exp_avg", "exp_avg_sq", "shadow"), (d[0], d[2], d[3], shadow), want):
        errs += R.check_exact(_np(got), w, name)
    assert _guard_ok(sbuf)
    assert not errs, "\n".join(errs)


@pytest.mark.parametrize("step,wd,coef", [(1, 0.0, 1.0), (3, 0.1, 0.3), (10000, 0.0, 1.0)])
def test_adamw_bf16_per_element(step, wd, coef):
    L, lib = _lib()
    n = 1 << 20
    p, g, m, v = (R.bf16(a) for a in _adam_state(n, step))
    g[:8] = R.bf16(np.array([0.0, -0.0, 1e-40, -1e-39, 1e-3, -1e-3, 1e-3, 0.0], np.float32))   # zero, subnormal
    d = [_dev(a, BF) for a in (p, g, m, v)]
    stats = torch.tensor([1.0, coef, 1.0], device=DEV)
    L.check(lib.sk_adamw_step(_p(d[0]), _p(d[1]), _p(d[2]), _p(d[3]), C.c_int64(n), L.f32(1e-3), L.f32(0.9), L.f32(0.999),
                              L.f32(1e-8), L.f32(wd), step, _p(stats), L.stream_ptr()))
    hp = dict(lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-8, wd=wd, step=step)
    refs = R.adamw_bf16_ref(p, g, m, v, coef=coef, **hp)
    gb = R.bf16((g * np.float32(coef)).astype(np.float32)) if coef != 1.0 else g
    bounds = R.adamw_bf16_bound(p, gb, m, v, **hp)
    errs = []
    for name, got, ref, b in zip(("param", "exp_avg", "exp_avg_sq"), (d[0], d[2], d[3]), refs, bounds):
        errs += R.check_bf16_interval(_np(got), ref, b, name)
    assert not errs, "\n".join(errs)


@pytest.mark.parametrize("arch,master", [("opt", False), ("opt", True), ("qwen2", False)])
def test_optimizer_step_weight_decay_groups(arch, master):
    """sk_lm_optimizer_step with weight_decay > 0: one clipped AdamW launch per tensor over its ALIGN_ELEMS-padded range,
    weight decay 0 for the [1, n] tensors (biases and norm weights).  The fp32 master branch is compared bit for bit
    with grad_ref.adamw_groups, the bf16 branch per element per tensor; the padding between tensors stays 0."""
    from slamkit_b200.lm import B200AdamW, B200UnitLM, LMConfig, OptLMConfig
    # OPT's fc1 bias (ffn = 264) is not a multiple of ALIGN_ELEMS (64), so its launch covers padding; every Qwen2 tensor
    # size is a multiple of 64 (hidden = heads * 64, ffn a multiple of 128), so that layout has none
    if arch == "opt":
        cfg = OptLMConfig(vocab_size=502, hidden=128, n_layers=2, n_heads=2, ffn=264, max_positions=128)
    else:
        cfg = LMConfig(vocab_size=502, hidden=128, n_layers=2, n_heads=2, n_kv_heads=1, head_dim=64, ffn=256)
    model = B200UnitLM(cfg, device=DEV, max_batch=1, max_seq=64, trainable=True, master_weights=master)
    layout = sorted(model.tensors.values())
    assert any(r == 1 for _, r, _ in layout) and any(r > 1 for _, r, _ in layout)
    n = model.n_params
    inside = np.zeros(n, bool)
    for off, rows, cols in layout:
        inside[off:off + rows * cols] = True
    assert inside.all() == (arch == "qwen2")
    r = np.random.default_rng(5)
    fill = lambda a: np.where(inside, a, 0.0).astype(np.float32)
    p, g, m, v = (fill(r.normal(0, 0.5, n)), fill(r.normal(0, 1e-2, n)), fill(r.normal(0, 1e-3, n)),
                  fill(np.abs(r.normal(0, 1e-5, n))))
    hp = dict(lr=1e-2, beta1=0.9, beta2=0.999, eps=1e-8, step=1)
    # lr * wd = 1 %: about two bf16 ulps of a parameter, so a decayed [1, n] tensor shows in the bf16 branch as well
    opt = B200AdamW(model, lr=hp["lr"], weight_decay=1.0, max_grad_norm=0.5)
    if master:
        for buf, a in ((model.params32, p), (model.grads32, g), (opt.exp_avg, m), (opt.exp_avg_sq, v)):
            buf.copy_(torch.from_numpy(a))
        model.params.fill_(float("nan"))                       # the step rewrites the whole bf16 shadow
    else:
        p, g, m, v = (R.bf16(a) for a in (p, g, m, v))
        for buf, a in ((model.params, p), (model.grads, g), (opt.exp_avg, m), (opt.exp_avg_sq, v)):
            buf.copy_(torch.from_numpy(a).to(BF))
    opt.step()
    torch.cuda.synchronize()
    coef = float(opt.stats[1])
    assert 0.0 < coef < 1.0                                    # the clip applies inside every per-tensor launch
    errs = []
    if master:
        want = R.adamw_groups(p, g, m, v, layout, wd=1.0, coef=coef, **hp)
        for name, got, w in zip(("params32", "exp_avg", "exp_avg_sq", "shadow"),
                                (model.params32, opt.exp_avg, opt.exp_avg_sq, model.params), want):
            errs += R.check_exact(_np(got), w, name)
    else:
        got = [_np(t) for t in (model.params, opt.exp_avg, opt.exp_avg_sq)]
        for off, rows, cols in layout:
            s = slice(off, off + -(-rows * cols // 64) * 64)
            t_hp = dict(hp, wd=0.0 if rows == 1 else 1.0)
            refs = R.adamw_bf16_ref(p[s], g[s], m[s], v[s], coef=coef, **t_hp)
            gb = R.bf16((g[s] * np.float32(coef)).astype(np.float32))
            bounds = R.adamw_bf16_bound(p[s], gb, m[s], v[s], **t_hp)
            for name, gt, ref, b in zip(("param", "exp_avg", "exp_avg_sq"), got, refs, bounds):
                errs += R.check_bf16_interval(gt[s], ref, b, f"{name} of [{rows}, {cols}] at {off}")
        for name, gt in zip(("param", "exp_avg", "exp_avg_sq"), got):
            errs += R.locate(gt[~inside] != 0, gt[~inside], np.zeros(int((~inside).sum())), f"{name} padding")
    assert not errs, "\n".join(errs[:40])


# ----------------------------------------------------------------------------------------------------- F. small kernels
def test_relu_bwd_bit_exact():
    L, lib = _lib()
    n = 4096 + 8
    a = torch.randn(n).to(BF)
    specials = torch.tensor([0.0, -0.0, 1e-40, -1e-40, float("nan"), float("inf"), -float("inf"), 1.0]).to(BF)
    a[:8] = specials
    g = torch.randn(n).to(BF)
    gbuf, gv = _guarded((n,), BF, g.float().numpy())
    L.check(lib.sk_relu_bwd(_p(gv), _p(_dev(a, BF)), C.c_int64(n), L.stream_ptr()))
    torch.cuda.synchronize()
    want = torch.ops.aten.threshold_backward(g, a, 0)                # autograd's ReLU backward: a NaN activation passes g
    assert float(want[4]) == float(g[4])
    assert torch.equal(gv.cpu().view(torch.int16), want.view(torch.int16))
    assert _guard_ok(gbuf)


@pytest.mark.parametrize("keep", [0, 1])
def test_widen_grads_with_guard_bands(keep):
    L, lib = _lib()
    lens = [8, 16384, 16384, 9992, 64]
    starts, o = [], 0
    for ln in lens:
        o += 64                                                  # a guard band before every chunk
        starts.append(o)
        o += ln
    n = o + 64
    # finite sentinels, different in the two buffers: a vector widened into a band writes 1.0 (keep = 0) or 8.0 (keep = 1)
    # over the 7.0 there, so an overrun before or after any chunk changes bits of g32
    g16 = torch.full((n,), 1.0, dtype=BF)
    g32 = torch.full((n,), 7.0)
    old = torch.randint(-1000, 1000, (n,)).float() * 2.0 ** -8
    for s, ln in zip(starts, lens):
        g16[s:s + ln] = (torch.randn(ln) * 1e-3).to(BF)
        g32[s:s + ln] = old[s:s + ln]
    d16, d32 = g16.to(DEV), g32.to(DEV)
    L.check(lib.sk_widen_grads(_p(d16), _p(d32), _p(_dev(starts, torch.int64)), _p(_dev(lens, torch.int32)), len(lens), keep,
                               L.stream_ptr()))
    want = g32.clone()
    for s, ln in zip(starts, lens):
        want[s:s + ln] = (old[s:s + ln] + g16[s:s + ln].float()) if keep else g16[s:s + ln].float()
    got = d32.cpu()
    assert torch.equal(got.view(torch.int32), want.view(torch.int32))   # chunks widened, the bands untouched


def test_master_widen_chunks_cover_linear_weights_and_biases_only():
    from oracle import opt_oracle as O
    from oracle import opt_amp_oracle as A
    from slamkit_b200.lm import B200UnitLM, OptLMConfig
    L, lib = _lib()
    c = O.OracleOptConfig(vocab_size=502, hidden=128, n_layers=2, n_heads=2, ffn=256, max_positions=128)
    m = B200UnitLM(OptLMConfig(vocab_size=502, hidden=128, n_layers=2, n_heads=2, ffn=256, max_positions=128),
                   device=DEV, max_batch=1, max_seq=64, trainable=True, master_weights=True)
    m.load_hf_state_dict(A.init_params_fp32(c, seed=0))
    cs = (C.c_int64 * 4096)()
    cl = (C.c_int32 * 4096)()
    k = lib.sk_lm_widen_chunks(m._h, cs, cl, 4096)
    assert k > 0
    covered = np.zeros(int(m.grads.numel()), bool)
    for i in range(k):
        assert cs[i] % 8 == 0 and cl[i] % 8 == 0
        covered[cs[i]:cs[i] + cl[i]] = True
    for name, (off, rows, cols) in m.tensors.items():
        linear = name.split(".")[-1] in ("wqkv", "bqkv", "wo", "bo", "w1", "b1", "w2", "b2")
        seg = covered[off:off + rows * cols]
        assert bool(seg.all()) if linear else not bool(seg.any()), name


# ----------------------------------------------------------------------------------------------------- G. chains, runs, refusals
def test_pdl_chains_see_previous_writes_and_runs_are_identical():
    L, lib = _lib()
    M, N = 4096, 1152
    x = _dev(np.random.default_rng(0).integers(-8, 9, size=(M, N)), BF)
    part = torch.empty(lib.sk_colsum_splits() * N, device=DEV)
    outs = []
    for _ in range(2):
        out = torch.zeros(N, dtype=BF, device=DEV)
        for _ in range(3):                                       # back to back, each accumulating the previous result
            L.check(lib.sk_colsum(_p(x), _p(out), _p(part), M, N, N, 1, L.stream_ptr()))
        outs.append(out.clone())
    s = x.float().sum(0).cpu().numpy()
    want = np.zeros_like(s)
    for _ in range(3):
        want = R.bf16(s + want)
    assert not R.check_exact(_np(outs[0]), want, "3 x colsum")
    assert torch.equal(outs[0].view(torch.int16), outs[1].view(torch.int16))
    # table gradient with heavy collisions: two runs give identical bytes
    M, D, V = 8192, 768, 502
    dx = _dev(np.random.default_rng(1).normal(0, 1e-3, size=(M, D)).astype(np.float32), torch.float32)
    ids = _dev(np.random.default_rng(2).integers(0, 4, size=M), torch.int64)
    runs = []
    for _ in range(2):
        t = torch.zeros(512, D, device=DEV)
        L.check(lib.sk_table_bwd_f32(_p(ids), None, _p(dx), _p(_scratch(512, D)), _p(t), None, M, M, D, V, 512, 0,
                                     L.stream_ptr()))
        runs.append(t.cpu())
    assert torch.equal(runs[0].view(torch.int32), runs[1].view(torch.int32))


def test_argument_checks_refuse_without_launching():
    L, lib = _lib()
    x = torch.zeros(1024, dtype=BF, device=DEV)
    f = torch.zeros(4096, device=DEV)
    before = lib.sk_launch_count()
    s = L.stream_ptr()
    assert lib.sk_ce_fwd_bwd(_p(x), _p(x), _p(x), _p(f), None, _p(f), 4, 4, 10, 12, L.f32(1), L.f32(1), s) == -1   # ldl % 8
    assert lib.sk_ce_fwd_bwd(_p(x), _p(x), _p(x), _p(f), None, _p(f), 4, 4, 17, 16, L.f32(1), L.f32(1), s) == -1   # V > ldl
    assert lib.sk_ce_chunk(_p(x), _p(x), _p(x), _p(f), 3, 4, 6, 2, 8, 8, L.f32(1), s) == -1                  # past M
    assert lib.sk_ce_fwd_bwd_weighted(_p(x), _p(x), _p(x), _p(f), None, None, _p(f), 4, 4, 8, 8, L.f32(1), L.f32(1), s) == -1
    assert lib.sk_embed_bwd(_p(x), _p(x), _p(f), _p(x), 4, 12, 8, 8, 0, s) == -1                                  # D % 8
    assert lib.sk_opt_pos_bwd(None, _p(x), _p(f), _p(x), 4, 4, 12, 8, 0, s) == -1
    assert lib.sk_table_bwd_f32(None, None, _p(f), _p(f), _p(f), _p(x), 4, 4, 8, 8, 8, 0, s) == -1           # head w/o ids
    assert lib.sk_relu_bwd(_p(x), _p(x), C.c_int64(12), s) == -1
    assert lib.sk_colsum(_p(x), _p(x), _p(f), 4, 12, 12, 0, s) == -1
    assert lib.sk_layernorm_bwd(_p(x), _p(x), _p(x), _p(f), _p(f), None, _p(x), _p(x), _p(x), _p(f), _p(f), 4, 2056, 0, s) == -1
    assert lib.sk_layernorm_bwd_f32(_p(x), _p(f), _p(f), _p(f), _p(f), None, _p(f), _p(x), _p(f), _p(f), _p(f), 0, 8, 0, s) == -1
    assert lib.sk_adamw_step(_p(x), _p(x), _p(x), _p(x), C.c_int64(12), L.f32(1), L.f32(0.9), L.f32(0.9), L.f32(1e-8),
                             L.f32(0), 1, None, s) == -1
    assert lib.sk_adamw_master_step(_p(f), _p(x), _p(f), _p(f), _p(f), C.c_int64(8), L.f32(1), L.f32(0.9), L.f32(0.9),
                                    L.f32(1e-8), L.f32(0), 0, None, s) == -1                                   # step 0
    assert lib.sk_launch_count() == before
