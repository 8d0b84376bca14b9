"""References and checkers for the HuBERT unit-extraction path (waveform -> features -> k-means ids), per element.

Exact split mode.  The HuBERT GEMMs run split-bf16: every operand x is a pair (hi, lo) of bf16 tensors and a GEMM
accumulates A_hi B_hi + A_hi B_lo + A_lo B_hi in fp32 -- deliberately without A_lo B_lo.  Here A_hi and B_hi hold small
integers and A_lo, B_lo hold small integers times 2^-8, all exact in bf16.  Every product then lies on the 2^-8 grid
and, as long as K (amax_hi bmax_hi + amax_hi bmax_lo + amax_lo bmax_hi) < 2^16, every partial sum is below 2^16 on that
grid: 24 significant bits, exact in fp32 whatever the tile width or summation order.  The float64 three-product sum is
therefore the kernel's accumulator bit for bit (split_exact_acc asserts these preconditions), and an added lo*lo product
(integers times 2^-16) or a missing hi*lo product changes it.  `split_epilogue` then emulates the GEMM epilogue in fp32
at the kernel's rounding points (gemm_tcgen05.cu: epi_bias_act, epi_residual and the hi/lo store):
    v = acc + bias(fp32);  v = act(v);  v = v + res_hi;  v = v + res_lo;  hi = bf16(v), lo = bf16(v - hi)  (or fp32 v)
so hi, lo and fp32 outputs compare bit for bit.  GELU outputs are bounded like gemm_ref.mismatch_gelu instead.

Layouts (what the GEMM's 3-D A view and column compaction mean):
  * windowed conv (conv layers 1..7): row m of clip b reads A[b][m*st*C : m*st*C + k*C] of the channels-last
    activation; output row b*M + m.
  * grouped positional conv (a_mode 1) on the staging layout xp [B, Tf + 2*halo, G*64]: output (b, t, g, c) =
    sum_{j, ci} xp[b, t + j, g*64 + ci] W[g*64 + c, j*64 + ci]; accumulator column g*64 + c goes to output column
    g*cg + c when c < cg and is dropped otherwise; the fp32 bias is read at the padded column g*64 + c.
  * regroup_pad: [B*Tf, G*cg] -> [B, Tf + 2*halo, G*64] with zero halo rows and zero pad channels.
  * rel_len: n_frames = ceil(float32(lens) / S * T) in float32, clamped to [0, T].

Per-element bounds for real data (docstrings of the *_bound functions give the derivations): the conv0 + GroupNorm +
GELU front, LayerNorm on hi/lo inputs, the split GEMM on real operands, and a whole post-LN encoder layer computed from
the device's own input to it (encoder_layer_reference: first-order propagation of every kernel's own bound).  Every
mismatch report names (clip, frame, 128-row tile, column group), so a failure points at the part of the schedule that
produced it.
"""
from __future__ import annotations

from typing import Optional

import torch

import attn_ref as A
import gemm_ref as G

BM = 128
BK = 64
GROUP_PAD = 64
LO_SCALE = 2.0 ** -8
EXACT_SPLIT_LIMIT = 2.0 ** 16
U23 = 2.0 ** -23
U24 = 2.0 ** -24


# ----------------------------------------------------------------------------------------------------- operands
def split_int_operand(rows: int, cols: int, amax: int, lmax: int, seed: int, device="cpu"):
    """(hi, lo) bf16 [rows, cols]: hi uniform integers in [-amax, amax], lo uniform integers in [-lmax, lmax] * 2^-8."""
    g = torch.Generator(device=device).manual_seed(seed)
    hi = torch.randint(-amax, amax + 1, (rows, cols), generator=g, device=device).to(torch.bfloat16)
    lo = (torch.randint(-lmax, lmax + 1, (rows, cols), generator=g, device=device).double() * LO_SCALE).to(torch.bfloat16)
    return hi, lo


def split_amax(K: int, lmax: int = 64) -> int:
    """Largest hi amplitude that keeps the split accumulator exact at this K with lo integers up to lmax:
    K (a^2 + 2 a lmax 2^-8) < 2^16 (K = 8192 -> 2)."""
    a = 1
    while K * ((a + 1) ** 2 + 2 * (a + 1) * lmax * LO_SCALE) < EXACT_SPLIT_LIMIT:
        a += 1
    assert K * (a * a + 2 * a * lmax * LO_SCALE) < EXACT_SPLIT_LIMIT, f"no exact amplitude at K={K}, lmax={lmax}"
    return a


def real_split(shape, scale: float, seed: int, device="cpu"):
    """(hi, lo) bf16 split of normal fp32 values of the given scale (a residual as the kernels store one)."""
    g = torch.Generator(device=device).manual_seed(seed)
    x = torch.randn(shape, generator=g, device=device) * scale
    return split_f32(x)


def split_f32(x: torch.Tensor):
    """fp32 -> (hi, lo) bf16 as split_f32_kernel / split_store: hi = bf16(x), lo = bf16(x - hi)."""
    x = x.float()
    hi = x.to(torch.bfloat16)
    lo = (x - hi.float()).to(torch.bfloat16)
    return hi, lo


def hilo(hi: torch.Tensor, lo: torch.Tensor) -> torch.Tensor:
    return hi.double() + lo.double()


def split_exact_acc(ah: torch.Tensor, al: torch.Tensor, bh: torch.Tensor, bl: torch.Tensor) -> torch.Tensor:
    """float64 [M, N] = Ah Bh^T + Ah Bl^T + Al Bh^T (no Al Bl^T); asserts that the kernel's fp32 sums are exact."""
    K = ah.shape[1]
    m = lambda t: float(t.float().abs().max()) if t.numel() else 0.0
    worst = K * (m(ah) * m(bh) + m(ah) * m(bl) + m(al) * m(bh))
    assert worst < EXACT_SPLIT_LIMIT, f"split accumulation is not exact: K={K} worst partial sum {worst}"
    for t in (ah, bh):
        assert torch.equal(t.float(), t.float().round()), "hi operands must be integers"
    for t in (al, bl):
        assert torch.equal(t.double() / LO_SCALE, (t.double() / LO_SCALE).round()), "lo operands must be on the 2^-8 grid"
    ah, al, bh, bl = ah.double(), al.double(), bh.double(), bl.double()
    return ah @ bh.t() + ah @ bl.t() + al @ bh.t()


# ----------------------------------------------------------------------------------------------------- epilogue
def split_epilogue(acc: torch.Tensor, bias: Optional[torch.Tensor] = None, res_hi: Optional[torch.Tensor] = None,
                   res_lo: Optional[torch.Tensor] = None, out_f32: bool = False, col_gin: int = 0, col_gout: int = 0):
    """fp32 emulation of the split GEMM's epilogue (no activation); acc exact in fp32.  Returns (hi, lo) fp32-valued
    bf16 numbers, or the fp32 value when out_f32.  With col_gin the bias is added at the accumulator column and the
    columns are compacted before the residual (read at the output column)."""
    v = acc.float()
    if bias is not None:
        v = v + bias.float()
    if col_gin:
        v = compact_columns(v, col_gin, col_gout)
    if res_hi is not None:
        v = v + res_hi.float()
    if res_lo is not None:
        v = v + res_lo.float()
    if out_f32:
        return v
    hi = G.bf16_round(v)
    return hi, G.bf16_round(v - hi)


def compact_columns(v: torch.Tensor, gin: int, gout: int) -> torch.Tensor:
    """[rows, G*gin] -> [rows, G*gout]: keep the first gout columns of every group of gin."""
    rows, n = v.shape
    return v.reshape(rows, n // gin, gin)[:, :, :gout].reshape(rows, -1)


def pick_bn(M_total: int, N: int, force_bn: int = 0, a_mode: int = 0, nsm: int = 132) -> int:
    """Tile width the launcher picks for a split / batched GEMM (sk_pick_bn without the 192 / 224 fit, which these
    GEMMs never take): 256, displaced by 128 or 64 when that costs >= 25 % less; a_mode 1 is always 64."""
    if a_mode == 1:
        return 64
    if force_bn in (64, 128, 256):
        return force_bn

    def cost(bn):
        tiles = -(-M_total // BM) * -(-N // bn)
        tc = 100 if bn >= 256 else (61 if bn == 128 else 54)
        return -(-tiles // nsm) * tc

    best, best_cost = 256, cost(256)
    for bn in (128, 64):
        if cost(bn) * 100 < best_cost * 75:
            best, best_cost = bn, cost(bn)
    return best


# ----------------------------------------------------------------------------------------------------- layouts
def window_rows(a: torch.Tensor, B: int, M: int, k: int, st: int, C: int) -> torch.Tensor:
    """Windowed-conv A operand: a is the channels-last activation [B, T_in * C] (any shape with B leading rows);
    row b*M + m is a[b, m*st*C : m*st*C + k*C]."""
    flat = a.reshape(B, -1)
    w = flat.unfold(1, k * C, st * C)
    assert w.shape[1] >= M, f"clip too short for {M} windows"
    return w[:, :M].reshape(B * M, k * C)


def posconv_windows(xp: torch.Tensor, Tf: int, Kpos: int, g: int) -> torch.Tensor:
    """Grouped positional-conv A operand of group g: row b*Tf + t is xp[b, t:t+Kpos, g*64:(g+1)*64] flattened in (tap,
    channel) order -- the k-block kb of a_mode 1 is staging row t + kb."""
    B = xp.shape[0]
    x = xp[:, :, g * GROUP_PAD:(g + 1) * GROUP_PAD]              # [B, Tp, 64]
    w = x.unfold(1, Kpos, 1)                                      # [B, Tp - Kpos + 1, 64, Kpos]
    return w[:, :Tf].permute(0, 1, 3, 2).reshape(B * Tf, Kpos * GROUP_PAD)


def posconv_split_acc(xp_hi, xp_lo, w_hi, w_lo, Tf: int, Kpos: int, groups: int, exact: bool = True) -> torch.Tensor:
    """float64 accumulator [B*Tf, groups*64] of the grouped positional conv (three products, padded columns)."""
    outs = []
    for g in range(groups):
        ah, al = posconv_windows(xp_hi, Tf, Kpos, g), posconv_windows(xp_lo, Tf, Kpos, g)
        bh, bl = w_hi[g * GROUP_PAD:(g + 1) * GROUP_PAD], w_lo[g * GROUP_PAD:(g + 1) * GROUP_PAD]
        if exact:
            outs.append(split_exact_acc(ah, al, bh, bl))
        else:
            ah, al, bh, bl = ah.double(), al.double(), bh.double(), bl.double()
            outs.append(ah @ bh.t() + ah @ bl.t() + al @ bh.t())
    return torch.cat(outs, dim=1)


def regroup_pad(x: torch.Tensor, B: int, T: int, halo: int, groups: int, cg: int, cgp: int = GROUP_PAD) -> torch.Tensor:
    """[B*T, groups*cg] -> [B, T + 2*halo, groups*cgp], zero halo rows and zero pad channels (regroup_pad_kernel)."""
    out = torch.zeros(B, T + 2 * halo, groups, cgp, dtype=x.dtype, device=x.device)
    out[:, halo:halo + T, :, :cg] = x.reshape(B, T, groups, cg)
    return out.reshape(B, T + 2 * halo, groups * cgp)


def rel_len(lens, S: int, T: int) -> torch.Tensor:
    """n_frames = ceil(float32(lens) / S * T) in float32 arithmetic (hubert_feature_extractor.py:46), clamped."""
    if lens is None:
        return torch.full((1,), T, dtype=torch.int32)
    r = (torch.as_tensor(lens).float() / torch.tensor(float(S), dtype=torch.float32)) * torch.tensor(float(T), dtype=torch.float32)
    return torch.ceil(r).clamp(0, T).to(torch.int32)


# ----------------------------------------------------------------------------------------------------- bounds
def gelu_bound(v: torch.Tensor, g: torch.Tensor, hilo_out: bool = True) -> torch.Tensor:
    """|kernel GELU - exact GELU| at pre-activation v: the Abramowitz-Stegun erf (1.5e-7 absolute, times |v|/2) plus
    the approximate rcp / ex2 of the folded form (relative 2^-21 of a tail below |v|/2), 4e-7 |v| together, a few fp32
    roundings (2^-22 |g|) and the hi/lo representation (2^-17 |g|, or one bf16 ulp for a bf16 output)."""
    v, g = v.double().abs(), g.double().abs()
    rep = 2.0 ** -17 * g if hilo_out else G.ulp_bf16(g)
    return 4e-7 * v + 2.0 ** -22 * g + rep + 1e-30


def conv0_reference(wav: torch.Tensor, w: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, pad: int, KW: int,
                    ST: int, eps: float = 1e-5, n_stat: Optional[int] = None):
    """float64 conv0 (1 -> C, no bias) + GroupNorm(C groups, over time, biased variance) + exact GELU.
    -> (gelu out [B, T0, C], pre-activation z, |shift| + sum_j |w_j scale x_j| (the operand magnitude A of the FMA
    chain)).  n_stat: frames the statistics use (T0 = all; a smaller value emulates a defective statistics pass)."""
    x = torch.nn.functional.pad(wav.double(), (pad, pad))
    win = x.unfold(1, KW, ST)                                     # [B, T0, KW]
    wd = w.double().reshape(-1, KW)                               # [C, KW]
    y = win @ wd.t()                                              # [B, T0, C]
    T0 = y.shape[1]
    ys = y[:, :(n_stat or T0)]
    mean = ys.mean(dim=1, keepdim=True)
    var = ys.var(dim=1, unbiased=False, keepdim=True)
    sc = gamma.double() / torch.sqrt(var + eps)
    sh = beta.double() - mean * sc
    z = y * sc + sh
    mag = sh.abs() + win.abs() @ wd.abs().t() * sc.abs()
    return G.gelu_exact(z), z, mag


def conv0_bound(z: torch.Tensor, g: torch.Tensor, mag: torch.Tensor, KW: int) -> torch.Tensor:
    """Per-element bound of the conv0 front (hubert_kernels.cu): the GroupNorm scale and shift are formed in fp64 and
    rounded to fp32 (2^-24 relative each); the taps are pre-multiplied by the scale in fp32 (2^-24 relative each) and
    the KW-tap chain of fp32 FMAs is seeded with the shift (one rounding per FMA, each of at most the running magnitude).
    All of these are relative to the chain's operand magnitude mag = |shift| + sum_j |w_j scale x_j|, so
    |dz| <= (KW + 3) 2^-24 mag.  For a clip with a DC offset, z is a small difference of two large terms (y scale and
    shift = beta - mean scale); mag contains |mean scale|, which is that cancellation term.  GELU's slope is below 1.13,
    then gelu_bound adds the approximate erf and the hi/lo representation."""
    dz = (KW + 3) * U24 * mag.double()
    return 1.13 * dz + gelu_bound(z, g)


def layernorm_reference(x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, eps: float, unbiased: bool = False):
    """float64 LayerNorm over the last dim of x (float64 sum of the hi/lo inputs).  -> (out, mean, rstd)."""
    x = x.double()
    mean = x.mean(dim=-1, keepdim=True)
    var = x.var(dim=-1, unbiased=unbiased, keepdim=True)
    rstd = 1.0 / torch.sqrt(var + eps)
    return (x - mean) * rstd * gamma.double() + beta.double(), mean, rstd


def layernorm_bound(x: torch.Tensor, gamma: torch.Tensor, out: torch.Tensor, mean: torch.Tensor, rstd: torch.Tensor,
                    hilo_out: bool = True) -> torch.Tensor:
    """Per-element bound of layernorm_hilo_kernel (one warp per row, D <= 1024): the input is a_hi + a_lo (+ b_hi +
    b_lo) in fp32 (2^-24 |x| for the added input); the fp32 sums run 32 terms per lane, then a 5-level shuffle tree:
    depth <= 40, so |d sum| <= 40 2^-24 sum|.|; hence the mean is off by dm <= 40 2^-24 mean|x| + 2^-24 |x|, and the
    variance by 40 2^-24 var + dm^2 (the cross term cancels), so rstd is off by 21 2^-24 rstd plus rsqrtf's 2 ulp.
    (x - mean) rstd gamma + beta adds four roundings.  Together
      |d out| <= |gamma| rstd (dm + |x - mean| 28 2^-24) + 4 2^-24 (|out| + |beta|-sized terms) + representation,
    the representation being 2^-17 |out| for a hi/lo output and nothing for the fp32 copy."""
    x = x.double()
    ax = x.abs()
    dm = 40 * U24 * ax.mean(dim=-1, keepdim=True) + U24 * ax.amax(dim=-1, keepdim=True)
    d = gamma.double().abs() * rstd * (dm + (x - mean).abs() * 28 * U24)
    d = d + 4 * U24 * (out.abs() + (x - mean).abs() * rstd * gamma.double().abs())
    if hilo_out:
        d = d + 2.0 ** -17 * out.abs()
    return d + 1e-30


def split_random_bound(ah, al, bh, bl, ref: torch.Tensor, hilo_out: bool = True, extra_abs: Optional[torch.Tensor] = None):
    """Per-element bound of a split GEMM on real operands against the float64 three-product sum `ref`: fp32
    accumulation of the 3K products in any order (3K 2^-23 sum|products|, as gemm_ref.random_bound), up to three
    epilogue roundings (bias, residual hi, residual lo: 3 2^-24 |v|, with extra_abs = |bias| + |residual| terms) and the
    hi/lo representation (2^-17 |v|)."""
    K = ah.shape[1]
    A, Al, Bh, Bl = ah.double().abs(), al.double().abs(), bh.double().abs(), bl.double().abs()
    absacc = A @ Bh.t() + A @ Bl.t() + Al @ Bh.t()
    v = ref.double().abs()
    d = 3 * K * U23 * absacc + 3 * U24 * (v + (extra_abs if extra_abs is not None else 0.0))
    if hilo_out:
        d = d + 2.0 ** -17 * v
    return d + 1e-30


# ----------------------------------------------------------------------------------------------------- checker
def report_rows(bad: torch.Tensor, out: torch.Tensor, want: torch.Tensor, rows_per_clip: int, col_group: int, what: str,
                limit: int = 6) -> Optional[str]:
    """None when nothing is flagged, else a message with the count and the first mismatches as
    (clip, frame, 128-row tile, column group)."""
    n = int(bad.sum())
    if n == 0:
        return None
    idx = bad.nonzero()[:limit].tolist()
    lines = [f"{what}: {n} of {bad.numel()} elements differ; first (clip, frame, tile row, column group | col): got / want"]
    for r, c in idx:
        b, m = divmod(r, rows_per_clip)
        lines.append(f"  (clip {b}, frame {m}, tile {m // BM}, group {c // col_group} | col {c}): "
                     f"{float(out[r, c])!r} / {float(want[r, c])!r}")
    rows = bad.any(dim=1).nonzero().flatten()
    cols = bad.any(dim=0).nonzero().flatten()
    clips = sorted({int(r) // rows_per_clip for r in rows.tolist()})
    lines.append(f"  flagged clips {clips[:8]}, rows [{int(rows.min())}, {int(rows.max())}], "
                 f"columns [{int(cols.min())}, {int(cols.max())}]")
    return "\n".join(lines)


def mismatch_exact(out: torch.Tensor, want: torch.Tensor, rows_per_clip: int, col_group: int = 64,
                   what: str = "split gemm") -> Optional[str]:
    """Element-wise equality (NaN never equals anything); out and want 2-D."""
    assert out.shape == want.shape, (out.shape, want.shape)
    o, w = out.float(), want.float().to(out.device)
    return report_rows(o != w, o, w, rows_per_clip, col_group, what)


def mismatch_bound(out: torch.Tensor, want: torch.Tensor, bound: torch.Tensor, rows_per_clip: int, col_group: int = 64,
                   what: str = "split gemm") -> Optional[str]:
    """|out - want| <= bound per element (NaN fails)."""
    assert out.shape == want.shape, (out.shape, want.shape)
    o, w = out.double(), want.double().to(out.device)
    bad = ~((o - w).abs() <= bound.to(out.device))
    return report_rows(bad, o, w, rows_per_clip, col_group, what)


def boundary_rows(T: int, B: int, frac: float = 0.1, seed: int = 0) -> torch.Tensor:
    """Row indices (into [B*T]) that a per-element check of a large stage covers: every row within 2 of a 128-row tile
    edge or a clip edge, plus a random `frac` of the rest."""
    keep = set()
    for b in range(B):
        for t in list(range(0, T, BM)) + [T]:
            for d in (-2, -1, 0, 1):
                if 0 <= t + d < T:
                    keep.add(b * T + t + d)
    g = torch.Generator().manual_seed(seed)
    rnd = (torch.rand(B * T, generator=g) < frac).nonzero().flatten().tolist()
    keep.update(rnd)
    return torch.tensor(sorted(keep), dtype=torch.long)


def kmeans_labels_with_margin(feat: torch.Tensor, centers: torch.Tensor):
    """float64 distances |c|^2 - 2 x.c (sklearn's argmin form) -> (first argmin, top-2 margin)."""
    d = (centers.double() ** 2).sum(1)[None, :] - 2.0 * feat.double() @ centers.double().t()
    top2 = torch.topk(d, 2, dim=1, largest=False).values
    return torch.argmin(d, dim=1), top2[:, 1] - top2[:, 0]


def kmeans_margin_bound(feat: torch.Tensor, centers: torch.Tensor) -> torch.Tensor:
    """Per-row bound of the fp32 distance the device compares: the split GEMM's dot product (3H 2^-23 sum|x c| via
    split_random_bound, times 2) plus the fp32 |c|^2 (H 2^-24 |c|^2) and the final fp32 add; twice that separates two
    labels."""
    H = feat.shape[1]
    ax, ac = feat.double().abs(), centers.double().abs()
    dot_err = 2 * (3 * H * U23) * (ax @ ac.t()).amax(dim=1)
    csq_err = H * U24 * (centers.double() ** 2).sum(1).max()
    return 2 * (dot_err + csq_err) + 1e-12


# ----------------------------------------------------------------------------------------------------- encoder layer
# A post-LN encoder layer of the device (hubert_step.cu), from its input x (hb[0]):
#   qkv = x Wqkv^T + bqkv;  a = attention(qkv);  t1 = a Wo^T + bo + x;  h1 = LN1(t1);
#   f = GELU(h1 W1^T + b1);  t2 = f W2^T + b2 + h1;  out = LN2(t2)  (the fp32 copy of LN2's hi/lo output is the stage).
# sk_hubert_debug_stage taps every one of these intermediates, so each kernel is checked from the device's own inputs
# against its own bound: a worst-case bound propagated through a whole layer grows by sum|W| per linear and would no
# longer see a wrong head or residual.  The helpers below take optional input bounds (e_x) for first-order propagation;
# the device tests pass none.
def linear_with_bound(x: torch.Tensor, e_x, w: torch.Tensor, b: torch.Tensor, act: int = 0,
                      res: Optional[torch.Tensor] = None, e_res=None):
    """y = act(x W^T + b) (+ res) in float64 for the device's split linear (hubert_step.cu linear_split), and its bound:
    propagated e_x |W|^T; the split GEMM's own error 3K 2^-23 |x||W| (fp32 accumulation of the three products) +
    2^-16 |x||W| (the dropped x_lo W_lo) + |x| |W - (W_hi + W_lo)| (the weights' pair rounding); bias and residual adds
    (2^-24 each); GELU as gelu_bound after a slope of 1.13; the hi/lo representation 2^-17 |y|."""
    wd = w.double()
    wh, wl = split_f32(w)
    K = x.shape[1]
    ax = x.abs()
    v = x @ wd.t() + b.double()
    e = (e_x @ wd.abs().t() if e_x is not None else 0.0) + (3 * K * U23 + 2.0 ** -16) * (ax @ wd.abs().t()) \
        + ax @ (wd - hilo(wh, wl)).abs().t() + 2 * U24 * (v.abs() + b.double().abs())
    if act:
        g = G.gelu_exact(v)
        return g, 1.13 * e + gelu_bound(v, g)
    if res is not None:
        v = v + res
        e = e + (e_res if e_res is not None else 0.0) + 2 * U24 * (v.abs() + res.abs())
    return v, e + 2.0 ** -17 * v.abs()


def layernorm_with_bound(t: torch.Tensor, e_t: Optional[torch.Tensor], gamma: torch.Tensor, beta: torch.Tensor, eps: float,
                         hilo_out: bool = True):
    """LayerNorm of t in float64 and its bound: layernorm_bound for the kernel itself, plus the first-order change of
    the output under an input change dt:  n = (t - mean) rstd,  dn = rstd (dt - mean(dt)) - n rstd mean(n dt), so
    |d out| <= |gamma| rstd (e + mean(e) + |n| mean(|n| e))."""
    out, mean, rstd = layernorm_reference(t, gamma, beta, eps)
    if e_t is None:
        return out, layernorm_bound(t, gamma, out, mean, rstd, hilo_out)
    n = ((t - mean) * rstd).abs()
    prop = gamma.double().abs() * rstd * (e_t + e_t.mean(-1, keepdim=True) + n * (n * e_t).mean(-1, keepdim=True))
    return out, prop + layernorm_bound(t, gamma, out, mean, rstd, hilo_out)


def attention_with_bound(qkv: torch.Tensor, e_qkv: Optional[torch.Tensor], B: int, T: int, H: int, scale: float):
    """Bidirectional attention of the fused [B*T, 3H*64] projection per clip, in float64, and its bound: the split
    kernel's own contract bound (attn_ref.fwd_reference, split) at the reference q, k, v, plus the first-order change
    under input changes: with P = softmax(s), ds_ij <= DS_ij = scale (e_q_i |k_j| + |q_i| e_k_j),
    dO_i = sum_j P_ij dv_j + sum_j P_ij ds_ij (v_j - O_i), so |dO_i| <= P e_v + (P * DS)(|v| + |O_i|)."""
    hd = A.HD
    split3 = lambda x: [x[:, i * H * hd:(i + 1) * H * hd].reshape(B, T, H, hd) for i in range(3)]
    q, k, v = split3(qkv)
    lo, hi = A.bounds(B, T, False)
    O, _, bo, _ = A.fwd_reference(q.cpu(), k.cpu(), v.cpu(), lo, hi, scale, causal=False, split=True)
    O, bo = O.to(qkv.device), bo.to(qkv.device)
    if e_qkv is None:
        return O.reshape(B * T, H * hd), bo.reshape(B * T, H * hd)
    eq, ek, ev = split3(e_qkv)
    prop = torch.zeros_like(O)
    for b in range(B):
        for h in range(H):
            qh, kh, vh = q[b, :, h], k[b, :, h], v[b, :, h]
            P = torch.softmax((qh @ kh.t()) * scale, dim=-1)
            DS = scale * (eq[b, :, h] @ kh.abs().t() + qh.abs() @ ek[b, :, h].t())
            W = P * DS
            prop[b, :, h] = P @ ev[b, :, h] + W @ vh.abs() + W.sum(-1, keepdim=True) * O[b, :, h].abs()
    return O.reshape(B * T, H * hd), (bo + prop).reshape(B * T, H * hd)
