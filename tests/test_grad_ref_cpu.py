"""CPU checks of tests/grad_ref.py: each checker accepts a faithful model of its kernel and flags an injected defect
(one bf16 ulp, a dropped scatter collision, a position row off by one, a tail vector not written, `accumulate`
ignored, the clip coefficient applied twice or not at all, a no-decay tensor decayed, an exp two bf16 ulps off in the
CE gradient; exps within CUDA expf's 2 fp32 ulps are inside the CE bound by construction)."""
import numpy as np
import pytest
import torch

import grad_ref as R


def _ulp_up(a, idx):
    """a with one element moved up by one bf16 ulp."""
    b = a.copy()
    t = torch.from_numpy(b[idx:idx + 1].copy()).to(torch.bfloat16)
    t = (t.view(torch.int16) + 1).view(torch.bfloat16).float().numpy()
    b[idx] = t[0]
    return b


def _ce_model(logits, labels, T, V, gs, exp=np.exp):
    """fp32 model of the warp CE kernel's gradient: exp, sum, reciprocal, product and scale in fp32, one bf16 rounding."""
    x = logits.astype(np.float32)
    M, ldl = x.shape
    d, _, valid, _, _, _, _ = R.ce_reference(logits, labels, T, V, gs)
    v = x[:, :V]
    mx = v.max(axis=1, keepdims=True)
    e = exp((v - mx).astype(np.float32)).astype(np.float32)
    inv = (np.float32(1) / e.sum(axis=1, dtype=np.float32, keepdims=True)).astype(np.float32)
    p = np.zeros((M, ldl), np.float32)
    p[:, :V] = e * inv
    tgt = np.where(valid, labels[np.minimum(np.arange(M) + 1, M - 1)], 0)
    p[np.arange(M)[valid], tgt[valid]] -= np.float32(1)
    out = R.bf16((p * np.float32(gs)).astype(np.float32))
    out[~valid] = 0
    return out


def _ce_case(seed=0, M=64, T=16, V=502, ldl=512):
    r = np.random.default_rng(seed)
    logits = R.bf16(r.normal(0, 3, size=(M, ldl)).astype(np.float32))
    labels = r.integers(0, V, size=M)
    labels[5] = -100
    labels[9] = V
    return logits, labels, T, V, ldl, 1.0 / 37.0


def _ce_check(got, logits, labels, T, V, ldl, gs):
    d, _, valid, lse, spread, p, g = R.ce_reference(logits, labels, T, V, gs)
    return R.check_ce_grad(got, d, valid, V, R.ce_bound("warp", p, d, lse, spread, ldl, g))


def test_ce_checker_accepts_fp32_model_and_flags_defects():
    logits, labels, T, V, ldl, gs = _ce_case()
    good = _ce_model(logits, labels, T, V, gs)
    assert _ce_check(good, logits, labels, T, V, ldl, gs) == []
    # one bf16 ulp on one element
    bad = good.copy()
    bad[3] = _ulp_up(good[3], 17)
    assert _ce_check(bad, logits, labels, T, V, ldl, gs)
    # an exp approximation two bf16 ulps off (relative 2^-7) on every term.  An exp within 2 fp32 ulps of the true value
    # cannot be flagged: the warp bound allows CUDA's expf its documented 2-ulp error, so exp implementations that close
    # are indistinguishable to this checker
    approx = _ce_model(logits, labels, T, V, gs, exp=lambda a: np.exp(a) * (1 + np.sign(np.sin(1e3 * a)) * 2.0 ** -7))
    assert _ce_check(approx, logits, labels, T, V, ldl, gs)
    # a padding column written, and an ignored row (label -100 at row 4) given a gradient
    bad = good.copy()
    bad[0, V + 1] = 1e-3
    assert _ce_check(bad, logits, labels, T, V, ldl, gs)
    bad = good.copy()
    bad[4, 3] = 1e-3
    assert _ce_check(bad, logits, labels, T, V, ldl, gs)


def test_bf16_from64_rounds_once():
    # 1 + 2^-8 + 2^-30 lies just above a bf16 tie: one rounding goes up, float32-then-bf16 would round to even (down)
    x = np.array([1 + 2.0 ** -8 + 2.0 ** -30, -(1 + 2.0 ** -8 + 2.0 ** -30), 1 + 2.0 ** -8, 3.0])
    assert R.bf16_from64(x).tolist() == [1 + 2.0 ** -7, -(1 + 2.0 ** -7), 1.0, 3.0]


# ------------------------------------------------------------------------------------------------ table gradients
def test_table_reference_is_index_add_on_the_grid_and_flags_defects():
    M, D, V = 300, 16, 7
    dx = R.grid_values((M, D), 12, 255, 1)
    ids = np.random.default_rng(2).integers(-1, V + 2, size=M)
    ids[:40] = 3                                               # collisions
    want = R.table_grad_bf16(ids, dx, V)
    assert np.array_equal(R.table_fix_sum(ids, dx, V), R.index_add64(ids, dx, V))
    assert R.check_exact(want, R.bf16(R.index_add64(ids, dx, V).astype(np.float32)), "grid") == []
    # one dropped collision
    keep = np.ones(M, bool)
    keep[7] = False
    assert R.check_exact(R.table_grad_bf16(ids[keep], dx[keep], V), want, "dropped")
    # one bf16 ulp
    bad = want.copy()
    bad[3] = _ulp_up(want[3], 5)
    assert R.check_exact(bad, want, "ulp")
    # a position row off by one
    T, n_pos = 50, 40
    rows = R.opt_pos_rows(None, M, T, n_pos)
    assert rows.max() == n_pos - 1 and rows.min() == 2
    good = R.table_grad_bf16(rows, dx, n_pos)
    assert R.check_exact(R.table_grad_bf16(np.minimum(rows + 1, n_pos - 1), dx, n_pos), good, "pos+1")
    # fp32 path: the head and the kept gradient are added in the documented order
    head = R.bf16(R.grid_values((V, D), 6, 100, 3))
    old = R.grid_values((V, D), 20, 1000, 4)
    f = R.table_grad_f32(ids, dx, V, head=head, old=old)
    assert np.array_equal(f, (old + (head + R.index_add64(ids, dx, V).astype(np.float32))).astype(np.float32))
    assert R.check_exact(R.table_grad_f32(ids, dx, V, head=head), f, "keep ignored")


def test_fixed_point_range():
    dx = np.array([[2.0 ** -40], [2.0 ** -41], [np.nextafter(np.float32(2.0 ** -41), 0)], [2.0 ** -41 * 3]], np.float32)
    s = R.table_fix_sum(np.arange(4), dx, 4)[:, 0]
    assert s.tolist() == [2.0 ** -40, 0.0, 0.0, 2.0 ** -39]   # rint: 0.5 -> 0, 1.5 -> 2
    big = np.full((2, 1), 2.0 ** 22 - 0.25, np.float32)     # the largest float32 below 2^22
    assert R.table_fix_sum(np.zeros(2), big, 1)[0, 0] == 2.0 ** 23 - 0.5


# ------------------------------------------------------------------------------------------------ column sums / widen
def test_colsum_reference_flags_tail_and_accumulate_defects():
    r = np.random.default_rng(0)
    x = r.integers(-8, 9, size=(100, 40)).astype(np.float32)
    old = R.bf16(r.integers(-50, 50, size=40).astype(np.float32))
    want = R.colsum_ref(x, old)
    assert R.check_exact(want, R.bf16((x.sum(0) + old).astype(np.float32)), "colsum") == []
    tail = want.copy()
    tail[32:] = old[32:]                                       # the last vector of 8 not written
    assert R.check_exact(tail, want, "tail")
    assert R.check_exact(R.colsum_ref(x), want, "accumulate ignored")


def test_ln_bwd_reference_and_bound():
    r = np.random.default_rng(1)
    M, D = 6, 64
    x = r.integers(-8, 9, size=(M, D)).astype(np.float32)
    dy = r.integers(-4, 5, size=(M, D)).astype(np.float32)
    w = r.integers(-3, 4, size=D).astype(np.float32)
    mean = np.full(M, 0.5)
    rstd = np.full(M, 0.25)
    dx, dw, db = R.ln_bwd_ref(dy, x, w, mean, rstd)
    assert np.array_equal(db, dy.sum(0)) and np.array_equal(dw, (dy * (x - 0.5) * 0.25).sum(0))
    b = R.ln_dx_bound(dy, x, w, mean, rstd)
    assert (b > 0).all() and (b < 1e-4 * (np.abs(dx) + 1)).all()


# ------------------------------------------------------------------------------------------------ norm, clip, AdamW
def test_clip_reference_matches_torch_and_nan_is_kept():
    gs = [torch.tensor([3.0, 4.0]), torch.tensor([12.0]), torch.zeros(5)]
    norms, total, coef = R.clip_grad_norm_ref(gs, 0.5)
    tgs = [g.clone().requires_grad_(False) for g in gs]
    params = [torch.nn.Parameter(torch.zeros_like(g)) for g in gs]
    for p, g in zip(params, tgs):
        p.grad = g.clone()
    t_total = torch.nn.utils.clip_grad_norm_(params, 0.5)
    assert float(total) == float(t_total) == 13.0 and [float(n) for n in norms] == [5.0, 12.0, 0.0]
    assert float(params[0].grad[0]) == float((3.0 * coef).item())
    _, _, c = R.clip_grad_norm_ref([torch.tensor([float("nan"), 1.0])], 0.5)
    assert torch.isnan(c)
    _, _, c = R.clip_grad_norm_ref([torch.tensor([float("inf"), 1.0])], 0.5)
    assert float(c) == 0.0
    _, _, c = R.clip_grad_norm_ref(gs, 0.0)
    assert float(c) == 1.0


def _adam_case(n=64, seed=0):
    r = np.random.default_rng(seed)
    p = r.normal(0, 1, n).astype(np.float32)
    g = r.normal(0, 1e-2, n).astype(np.float32)
    m = r.normal(0, 1e-3, n).astype(np.float32)
    v = np.abs(r.normal(0, 1e-5, n)).astype(np.float32)
    return p, g, m, v


HP = dict(lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-8, step=3)


def test_adamw_master_matches_torch_fused_formula_and_flags_clip_defects():
    p, g, m, v = _adam_case()
    want = R.adamw_master(p, g, m, v, wd=0.1, coef=0.25, **HP)
    tp, tg, tm, tv = (torch.from_numpy(a.copy()) for a in (p, g, m, v))
    from oracle.lm_oracle import adamw_step_
    adamw_step_(tp, tg * torch.tensor(0.25), tm, tv, weight_decay=0.1, **HP)
    # the oracle evaluates in torch fp32 tensors with its own grouping; both agree to the last ulp or so
    assert np.allclose(want[0], tp.numpy(), rtol=2e-7, atol=0)
    twice = R.adamw_master(p, (g * np.float32(0.25)).astype(np.float32), m, v, wd=0.1, coef=0.25, **HP)
    none = R.adamw_master(p, g, m, v, wd=0.1, coef=1.0, **HP)
    for bad in (twice, none):
        assert R.check_exact(bad[0], want[0], "params") and R.check_exact(bad[1], want[1], "exp_avg")
    assert np.array_equal(want[3], R.bf16(want[0]))


def test_decay_groups_flag_a_decayed_norm_weight():
    """The optimizer step's decay groups: a [1, n] tensor moves as with weight decay 0."""
    p, g, m, v = _adam_case(128, 3)
    layout = [(0, 4, 16), (64, 1, 64)]                         # (offset, rows, cols): a matrix and a norm weight
    want = R.adamw_groups(p, g, m, v, layout, wd=0.1, **HP)
    assert np.array_equal(want[0][64:], R.adamw_master(p[64:], g[64:], m[64:], v[64:], wd=0.0, **HP)[0])
    decayed = R.adamw_master(p, g, m, v, wd=0.1, **HP)
    assert R.check_exact(decayed[0], want[0], "norm weight decayed")


def test_adamw_bf16_bound_is_located():
    p, g, m, v = _adam_case(4096, 5)
    p, g, m, v = (R.bf16(a) for a in (p, g, m, v))
    rp, rm, rv = R.adamw_bf16_ref(p, g, m, v, wd=0.0, **HP)
    bp, bm, bv = R.adamw_bf16_bound(p, g, m, v, wd=0.0, **HP)
    # the slack admits two bf16 values only near rounding boundaries
    assert R.check_bf16_interval(R.bf16(rp.astype(np.float32)), rp, bp, "p") == []
    two = R.bf16_from64(rp - bp) != R.bf16_from64(rp + bp)
    assert two.mean() < 0.01
    bad = R.bf16(rp.astype(np.float32))
    bad = _ulp_up(bad, int(np.argmin(two)))
    assert R.check_bf16_interval(bad, rp, bp, "p")
