"""References and checkers for the HiFi-GAN unit vocoder (vocoder.cu), per element.

Layer geometry (what one launch of vocoder_conv_kernel computes).  A conv (kernel k, dilation d, padding
pad = (k - 1) d / 2) maps x [T, Cin] to y [T, Cout] with one phase: output row o = q reads input rows q - pad + m d for
taps m.  A ConvTranspose1d (stride u, padding pad = (k - u) / 2) runs polyphase: phase r in [0, u) uses the taps
j = r, r + u, r + 2u, ... (tap m of the phase is j = r + m u), output row o = q u + r - pad reads input row q - m, and
q runs over [0, Q) with Q = T_in + ceil(pad / u).  Time tiles are BM = 128 values of q; channel tiles are BN = 16 NT
output channels, NT = 4, 2 or 1 for Cout >= 64, >= 32, else.

Exact split mode.  The kernel stages t = leaky_relu(x, slope) in fp32 and splits it as hi = bf16(t), lo = bf16(t - hi);
prepare_kernel splits the weights the same way; the products are hi*hi + hi*lo + lo*hi (no lo*lo) in fp32.
`exact_values` builds t = hi + lo with hi a small nonzero integer and lo an integer times 2^-12 below half a bf16 ulp of
hi (so bf16(t) == hi and t - hi == lo exactly), or t = 0; `exact_activation` returns x = 10 t where t < 0 under slope
0.1, and fl32(x * 0.1f) == t exactly (0.1f is 0.1 (1 + 1.5e-8), well inside half an ulp).  Every product then lies on
the 2^-12 grid and, while sum |products| over taps x Cin stays below 2^24 * 2^-12 (`split_exact_acc` asserts it per
output), every partial sum is exact in fp32 in any order: the float64 three-product sum is the kernel's accumulator
bit for bit.  An added lo*lo (2^-24 grid, summed over many terms) or a missing hi*lo changes it.  `exact_epilogue`
then emulates the epilogue in fp32 at the kernel's rounding points,
    v = acc + bias;  v = v + res;  (mode 2) v = sum + v;  (divide) v = v / divide;  0 where the frame is masked,
so outputs compare bit for bit.

Random mode, the chain bounds and the duration predictor are bounded per element; the *_bound docstrings derive them.
Mismatch reports name (row, position in row, 128-row time tile, phase, channel tile), so a failure points at the part
of the schedule that produced it.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence

import torch
import torch.nn.functional as F

import hubert_ref as R

BM = 128
KC = 32
CPAD = 64
LO_EXP = 12
LO_Q = 2.0 ** -LO_EXP
LO_MAX = 7                        # |lo| <= 7 * 2^-12 < 2^-9: half a bf16 ulp just below 1
EXACT_LIMIT = 2.0 ** 24 * LO_Q    # sum |products| on the 2^-12 grid that fp32 holds exactly
U23 = 2.0 ** -23
U24 = 2.0 ** -24
SLOPE_F32 = float(torch.tensor(0.1, dtype=torch.float32))


# ----------------------------------------------------------------------------------------------------- geometry
def pick_nt(Cout: int) -> int:
    return 4 if Cout >= 64 else (2 if Cout >= 32 else 1)


def prep_bytes(Cout: int, Cin: int, k: int) -> int:
    """Scratch sk_vocoder_conv needs for the split weights: hi and lo bf16 [k][round_up(Cout, 64)][round_up(Cin, 32)]."""
    return 2 * 2 * k * (-(-Cout // CPAD) * CPAD) * (-(-Cin // KC) * KC)


class Geometry:
    """Phase / tap / tile structure of one layer (run_layer's ConvParams)."""

    def __init__(self, k: int, transposed: bool, rate: int, dil: int, T_in: int, Cout: int):
        self.k, self.transposed, self.rate, self.dil, self.T_in, self.Cout = k, bool(transposed), rate, dil, T_in, Cout
        if transposed:
            self.pad = (k - rate) // 2
            self.T_out = T_in * rate
            self.Q = T_in + -(-self.pad // rate)
            self.phases = [list(range(r, k, rate)) for r in range(rate)]
        else:
            self.pad = (k * dil - dil) // 2
            self.T_out = T_in
            self.Q = T_in
            self.phases = [list(range(k))]
        self.BN = 16 * pick_nt(Cout)

    def locate(self, o: int):
        """(time tile, phase) of output row o."""
        if self.transposed:
            q, r = divmod(o + self.pad, self.rate)
            return q // BM, r
        return o // BM, 0

    def describe(self) -> str:
        kind = f"convT u={self.rate}" if self.transposed else f"conv d={self.dil}"
        return f"{kind} k={self.k} T_in={self.T_in} Q={self.Q} Cout={self.Cout} NT={pick_nt(self.Cout)}"


def conv_ref(t: torch.Tensor, w: torch.Tensor, geo: Geometry) -> torch.Tensor:
    """float64 layer without bias: t [T_in, Cin], torch-layout weights -> [T_out, Cout]."""
    a = t.double().t()[None]
    if geo.transposed:
        y = F.conv_transpose1d(a, w.double(), stride=geo.rate, padding=geo.pad)
    else:
        y = F.conv1d(a, w.double(), dilation=geo.dil, padding=geo.pad)
    return y[0].t()


def position_mask(valid: torch.Tensor, up: int, T_out: int) -> torch.Tensor:
    return valid.bool().repeat_interleave(up)[:T_out]


# ----------------------------------------------------------------------------------------------------- exact operands
def bf16(x: torch.Tensor) -> torch.Tensor:
    return x.float().to(torch.bfloat16).float()


def split_f32(x: torch.Tensor):
    """The kernel's split of an fp32 value: hi = bf16(x), lo = bf16(x - hi) (both returned as fp32)."""
    x = x.float()
    hi = bf16(x)
    return hi, bf16(x - hi)


def leaky32(x: torch.Tensor, slope: float) -> torch.Tensor:
    """The staging's leaky ReLU in fp32: x > 0 ? x : x * slope (slope as fp32)."""
    x = x.float()
    return torch.where(x > 0, x, x * torch.tensor(slope, dtype=torch.float32, device=x.device))


def exact_values(shape, amax: int, density: float, seed: int, device="cpu") -> torch.Tensor:
    """fp32 t = hi + lo: hi uniform nonzero integers in [-amax, amax] with probability `density` (else t = 0), lo
    uniform integers in [-7, 7] times 2^-12.  Asserts bf16(t) == hi and t - hi == bf16(t - hi)."""
    g = torch.Generator().manual_seed(seed)
    mag = torch.randint(1, amax + 1, shape, generator=g).double()
    sign = torch.randint(0, 2, shape, generator=g).double() * 2 - 1
    keep = (torch.rand(shape, generator=g) < density).double()
    hi = mag * sign * keep
    lo = torch.randint(-LO_MAX, LO_MAX + 1, shape, generator=g).double() * LO_Q * keep
    t = (hi + lo).float()
    h, l = split_f32(t)
    assert torch.equal(h.double(), hi) and torch.equal(l.double(), lo), "exact operand does not split as built"
    return t.to(device)


def exact_activation(T: int, C: int, amax: int, density: float, slope: float, seed: int, device="cpu"):
    """(x, t): x fp32 [T, C] whose staged value leaky32(x, slope) is exactly the exact operand t."""
    t = exact_values((T, C), amax, density, seed)
    if slope == 1.0:
        x = t.clone()
    else:
        assert slope == 0.1, "exact activations are built for slope 1 and 0.1"
        x = torch.where(t < 0, t.double() * 10, t.double()).float()
        assert torch.equal(x.double(), torch.where(t < 0, t.double() * 10, t.double())), "10 t is not exact in fp32"
    assert torch.equal(leaky32(x, slope), t), "leaky_relu(x) does not reproduce t exactly"
    return x.to(device), t.to(device)


def exact_amax(K: int, density: float) -> int:
    """Largest hi amplitude (at most 2, so that lo*lo stays within a few ulps of the output and an added lo*lo shows)
    whose expected sum |products| over K = taps x Cin stays well inside the exact limit."""
    a = 1
    while K * (a + 1) ** 2 * density * density * 2.0 < EXACT_LIMIT and a < 2:
        a += 1
    return a


def split_exact_acc(t: torch.Tensor, w: torch.Tensor, geo: Geometry) -> torch.Tensor:
    """float64 [T_out, Cout] three-product accumulator of the layer on exact operands (t the staged activation, w the
    torch-layout weights); asserts that the kernel's fp32 sums are exact."""
    ah, al = split_f32(t)
    wh, wl = split_f32(w)
    for v in (ah, wh):
        assert torch.equal(v, v.round()), "hi operands must be integers"
    for v in (al, wl):
        assert torch.equal(v.double() / LO_Q, (v.double() / LO_Q).round()), "lo operands must be on the 2^-12 grid"
    mag = conv_ref(ah.abs(), wh.abs() + wl.abs(), geo) + conv_ref(al.abs(), wh.abs(), geo)
    worst = float(mag.max()) if mag.numel() else 0.0
    assert worst < EXACT_LIMIT, f"split accumulation is not exact: sum |products| reaches {worst} ({geo.describe()})"
    return conv_ref(ah, wh, geo) + conv_ref(ah, wl, geo) + conv_ref(al, wh, geo)


def exact_epilogue(acc: torch.Tensor, bias: torch.Tensor, live: torch.Tensor, res: Optional[torch.Tensor] = None,
                   mode: int = 0, sum_in: Optional[torch.Tensor] = None, divide: int = 0) -> torch.Tensor:
    """fp32 emulation of the epilogue at the kernel's rounding points; acc exact in fp32; live [T_out] bool."""
    v = acc.float() + bias.float().to(acc.device)
    if res is not None:
        v = v + res.float()
    if mode == 2:
        v = sum_in.float() + v
    if divide > 0:
        v = v / torch.tensor(float(divide), dtype=torch.float32, device=v.device)
    return torch.where(live[:, None].to(v.device), v, torch.zeros_like(v))


# ----------------------------------------------------------------------------------------------------- random mode
def layer_bound(x: torch.Tensor, w: torch.Tensor, bias: torch.Tensor, geo: Geometry, slope: float, live: torch.Tensor,
                res: Optional[torch.Tensor] = None, mode: int = 0, sum_in: Optional[torch.Tensor] = None, divide: int = 0):
    """(want, bound): the layer in float64 from the fp32 input x (leaky_relu with the exact slope) and a per-element
    bound of the kernel against it.
      * staging: t = fl(x * 0.1f) is t (1 + d) with |d| <= 2^-24 + 1.5e-8 < 2^-23 (0.1f is 0.1 (1 + 1.5e-8));
      * the split: |t - (hi + lo)| <= 2^-16 |t| (lo = bf16(t - hi) rounds a residual of at most 2^-8 |t| to 8 bits),
        the same for the weights, and the dropped lo*lo is at most 2^-8 |t| 2^-8 |w| = 2^-16 |t||w|: each product is
        off by at most (3 2^-16 + 2^-22) |t||w|;
      * the fp32 accumulation of 3K products (K = taps x Cin) in whatever order the mma chain takes: 3K 2^-23 times the
        sum of |products| <= 1.01 sum |t||w| (as hubert_ref.split_random_bound);
      * the epilogue: up to three adds (bias, residual, running sum), 2^-24 of each result, and the divide (2^-24).
    Masked positions are exactly 0 (bound 0)."""
    t = torch.where(x.double() > 0, x.double(), x.double() * slope)
    acc = conv_ref(t, w, geo)
    mag = conv_ref(t.abs(), w.abs(), geo)
    K = len(geo.phases[0]) * x.shape[1]
    e = (3 * 2.0 ** -16 + 2.0 ** -22) * mag + 3 * K * U23 * 1.01 * mag
    v = acc + bias.double()
    run = v.abs()
    if res is not None:
        v = v + res.double()
        run = run + v.abs()
    if mode == 2:
        v = sum_in.double() + v
        run = run + v.abs()
    e = e + U24 * run
    if divide > 0:
        v = v / divide
        e = e / divide + U24 * v.abs()
    lv = live[:, None].to(v.device)
    return torch.where(lv, v, torch.zeros_like(v)), torch.where(lv, e + 1e-30, torch.zeros_like(e))


def post_bound(S: torch.Tensor, w: torch.Tensor, b: torch.Tensor, start: int, n: int):
    """(want, bound) of conv_post + tanh for one row of n samples starting at position `start` of S [T, C] (fp32, the
    device's last ResBlock mean).  post_kernel sums 7 C products w * leaky(v) in fp32 (leaky: fl(0.01f v), off by
    2^-24 + 2.3e-8 < 2^-23 relative), one rounding per step (two without FMA contraction), so the sum is off by at most
    2 (7C + 1) 2^-24 (sum |w leaky(v)| + |b|) plus 2^-23 sum |w leaky(v)|; tanh has slope <= 1 and tanhf is within
    2 ulp (4 2^-24 |y|)."""
    C = S.shape[1]
    seg = S[start - 3:start + n + 3].double()
    t = torch.where(seg > 0, seg, 0.01 * seg)
    a = F.conv1d(t.t()[None], w.double())[0, 0] + b.double()
    mag = F.conv1d(t.abs().t()[None], w.double().abs())[0, 0]
    y = torch.tanh(a)
    e = 2 * (7 * C + 1) * U24 * (mag + b.double().abs()) + U23 * mag + 4 * U24 * y.abs() + 1e-38
    return y, e


# ----------------------------------------------------------------------------------------------------- durations
def _chain_conv3(x: torch.Tensor, w: torch.Tensor, b: torch.Tensor, chunk: int = 8):
    """(y, e) of dur_kernel's conv (k = 3, padding 1) on x [n, C]: y [n, H] in float64 and the rounding bound of its fp32
    chain a = b; a += w[h, c, k] x[i - 1 + k, c] (c outer, k inner): every step rounds once to its running sum s and,
    without FMA contraction, once more to its product, so |e| <= 2^-24 (sum_steps |s| + sum |products|)."""
    n, C = x.shape
    xp = F.pad(x.double(), (0, 0, 1, 1))
    win = xp.unfold(0, 3, 1)                                                  # [n, C, 3]
    wd = w.double()
    ys, es = [], []
    for i0 in range(0, n, chunk):
        P = (wd[None] * win[i0:i0 + chunk, None]).flatten(2)                  # [c, H, C * 3] in (c, k) order
        s = b.double()[None, :, None] + torch.cumsum(P, dim=2)
        ys.append(s[:, :, -1])
        es.append(U24 * (s.abs().sum(2) + P.abs().sum(2)))
    return torch.cat(ys), torch.cat(es)


def dur_predictor_bound(units: torch.Tensor, sd: Dict[str, torch.Tensor], eps: float = 1e-5):
    """(v, bound) of dur_kernel's pre-rounding log-duration for one row of units, float64, from the fp32 weights.
    Each conv (k = 3, padding 1; the row is zero-padded at both ends, conv2 on the LayerNorm-1 outputs) is bounded by
    its own fp32 chain (_chain_conv3) plus, for conv2, the LayerNorm-1 error propagated through |w|; ReLU has slope <= 1;
    each LayerNorm (block_sum: a 5-level shuffle tree, then at most 32 warp partials in order, depth <= 37) is bounded by
    hubert_ref.layernorm_with_bound, which covers a sum depth of 40 and adds the first-order change under its input's
    error; the projection rounds z = LN2 * pw (2^-24 |z|), sums H terms with block_sum (depth 37) and adds the bias:
    38 2^-24 sum |z| + sum |pw| e + 2^-24 |v|."""
    p = "dur_predictor."
    g = lambda n: sd[p + n].double()
    x = sd["dict.weight"].double()[units.long()]                             # [n, E]
    a1, e1 = _chain_conv3(x, g("conv1.0.weight"), g("conv1.0.bias"))
    h1, eh1 = R.layernorm_with_bound(a1.clamp_min(0), e1, g("ln1.weight"), g("ln1.bias"), eps, hilo_out=False)
    a2, e2 = _chain_conv3(h1, g("conv2.0.weight"), g("conv2.0.bias"))
    e2 = e2 + F.conv1d(eh1.t()[None], g("conv2.0.weight").abs(), padding=1)[0].t()
    h2, eh2 = R.layernorm_with_bound(a2.clamp_min(0), e2, g("ln2.weight"), g("ln2.bias"), eps, hilo_out=False)
    pw = g("proj.weight").reshape(-1)
    z = h2 * pw
    v = z.sum(-1) + g("proj.bias").reshape(-1)
    e = (eh2 * pw.abs()).sum(-1) + 39 * U24 * z.abs().sum(-1) + U24 * v.abs()
    return v, e + 1e-30


def durations_from_logd(v: torch.Tensor) -> torch.Tensor:
    """torch.clamp(torch.round(torch.exp(v) - 1), min=1) on float64 values (round half to even)."""
    return torch.round(torch.exp(v.double()) - 1).clamp_min(1).long()


def mismatch_durations(dur: torch.Tensor, v: torch.Tensor, pre: Optional[torch.Tensor] = None, tol: float = 16 * U24,
                       what: str = "durations") -> Optional[str]:
    """dur == max(1, rint(exp(v) - 1)) per unit.  With `pre`, the exact fp32 value that was rounded, every unit is
    compared (rint rounds half to even); without it, units whose exp(v) - 1 lies within `tol` relative (expf's and the
    subtraction's rounding) of a half-integer are skipped, since the device's fp32 value may fall on either side."""
    dur = dur.long().cpu()
    if pre is not None:
        want = torch.round(pre.double().cpu()).clamp_min(1).long()
        keep = torch.ones_like(dur, dtype=torch.bool)
    else:
        ev = torch.exp(v.double().cpu())
        x = ev - 1
        keep = (x - x.floor() - 0.5).abs() > tol * ev + 1e-12
        want = torch.round(x).clamp_min(1).long()
    bad = keep & (dur != want)
    n = int(bad.sum())
    if n == 0:
        return None
    idx = bad.nonzero().flatten()[:6].tolist()
    return f"{what}: {n} of {dur.numel()} units differ; first (unit: got / want): " + \
        ", ".join(f"{i}: {int(dur[i])} / {int(want[i])}" for i in idx)


# ----------------------------------------------------------------------------------------------------- packing
def pack_rows(units: Sequence[torch.Tensor], durs: Sequence[torch.Tensor], G0: int, emb: torch.Tensor,
              spk: Optional[torch.Tensor] = None, sty: Optional[torch.Tensor] = None) -> Dict:
    """The packed unit-frame timeline of a batch: G0 zero frames, row 0's frames (unit i repeated dur[i] times), G0
    zero frames, row 1, ...  Returns T0, starts, frames, valid uint8 [T0], unit index per frame (-1 in gaps), row per
    frame (-1 in gaps) and x0 fp32 [T0, in_dim] = [embedding | speaker 0 | style 0] of each frame's unit, zero in gaps."""
    frames = [int(d.sum()) for d in durs]
    starts, s = [], G0
    for f in frames:
        starts.append(s)
        s += f + G0
    T0 = s
    in_dim = emb.shape[1] * (1 + (spk is not None) + (sty is not None))
    x0 = torch.zeros(T0, in_dim, dtype=torch.float32)
    valid = torch.zeros(T0, dtype=torch.uint8)
    unit_at = torch.full((T0,), -1, dtype=torch.long)
    row_at = torch.full((T0,), -1, dtype=torch.long)
    for b, (u, d) in enumerate(zip(units, durs)):
        idx = torch.repeat_interleave(torch.arange(len(u)), d.long().cpu())
        sl = slice(starts[b], starts[b] + frames[b])
        unit_at[sl], row_at[sl], valid[sl] = idx, b, 1
        parts = [emb.float().cpu()[u.long().cpu()[idx]]]
        for extra in (spk, sty):
            if extra is not None:
                parts.append(extra.float().cpu()[0][None].expand(len(idx), -1))
        x0[sl] = torch.cat(parts, dim=1)
    return dict(T0=T0, starts=starts, frames=frames, valid=valid, x0=x0, unit_at=unit_at, row_at=row_at)


def mismatch_frames(x0: torch.Tensor, valid: torch.Tensor, pk: Dict, what: str = "expansion") -> Optional[str]:
    """x0 / valid of a packed timeline against pack_rows' `pk`, bit for bit; reports (row, frame in row, unit)."""
    bad = (x0.float().cpu() != pk["x0"]).any(dim=1) | (valid.cpu() != pk["valid"])
    n = int(bad.sum())
    if n == 0:
        return None
    lines = [f"{what}: {n} of {bad.numel()} frames differ; first (row, frame in row, unit | timeline frame):"]
    for f in bad.nonzero().flatten()[:6].tolist():
        b = int(pk["row_at"][f])
        loc = f"row {b}, frame {f - pk['starts'][b]}, unit {int(pk['unit_at'][f])}" if b >= 0 else "gap"
        lines.append(f"  ({loc} | {f})")
    return "\n".join(lines)


# ----------------------------------------------------------------------------------------------------- checkers
def _rows_of(o: int, row_starts: Optional[List[int]]):
    if not row_starts:
        return "-", o
    b = max(i for i, s in enumerate(row_starts) if s <= o) if o >= row_starts[0] else -1
    return (b, o - row_starts[b]) if b >= 0 else ("gap", o)


def report(bad: torch.Tensor, out: torch.Tensor, want: torch.Tensor, geo: Geometry, what: str,
           row_starts: Optional[List[int]] = None, limit: int = 6) -> Optional[str]:
    """None when nothing is flagged, else the count, the first mismatches as (row, position, time tile, phase, channel
    tile) and the flagged tiles, phases and channel tiles.  row_starts: first output position of each packed row."""
    n = int(bad.sum())
    if n == 0:
        return None
    idx = bad.nonzero()
    lines = [f"{what} [{geo.describe()}]: {n} of {bad.numel()} elements differ; first "
             "(row, position, tile, phase, channel tile | o, c): got / want"]
    for o, c in idx[:limit].tolist():
        tile, ph = geo.locate(o)
        b, pos = _rows_of(o, row_starts)
        lines.append(f"  (row {b}, position {pos}, tile {tile}, phase {ph}, channel tile {c // geo.BN} | o {o}, c {c}): "
                     f"{float(out[o, c])!r} / {float(want[o, c])!r}")
    locs = [geo.locate(o) for o in idx[:, 0].unique().tolist()]
    tiles = sorted({t for t, _ in locs})
    phases = sorted({p for _, p in locs})
    ctiles = sorted({c // geo.BN for c in idx[:, 1].unique().tolist()})
    lines.append(f"  flagged tiles {tiles[:12]}, phases {phases[:12]}, channel tiles {ctiles[:12]}")
    return "\n".join(lines)


def mismatch_exact(out: torch.Tensor, want: torch.Tensor, geo: Geometry, what: str = "vocoder conv",
                   row_starts: Optional[List[int]] = None) -> Optional[str]:
    """Element-wise equality (NaN never equals anything); out and want [T_out, Cout]."""
    assert out.shape == want.shape, (out.shape, want.shape)
    o, w = out.float(), want.float().to(out.device)
    return report((o != w).cpu(), o.cpu(), w.cpu(), geo, what, row_starts)


def mismatch_bound(out: torch.Tensor, want: torch.Tensor, bound: torch.Tensor, geo: Geometry,
                   what: str = "vocoder conv", row_starts: Optional[List[int]] = None) -> Optional[str]:
    """|out - want| <= bound per element (NaN fails; a zero bound demands exact zeros)."""
    assert out.shape == want.shape, (out.shape, want.shape)
    o, w = out.double(), want.double().to(out.device)
    bad = ~((o - w).abs() <= bound.to(out.device))
    return report(bad.cpu(), o.cpu(), w.cpu(), geo, what, row_starts)


def mismatch_wave(wave: torch.Tensor, want: torch.Tensor, bound: torch.Tensor, U: int, what: str = "waveform") -> Optional[str]:
    """One row's samples against want within bound; reports (sample, frame, position in frame)."""
    bad = ~((wave.double().cpu() - want.double().cpu()).abs() <= bound.double().cpu())
    n = int(bad.sum())
    if n == 0:
        return None
    idx = bad.nonzero().flatten()
    lines = [f"{what}: {n} of {bad.numel()} samples exceed the bound; first (sample, frame, offset): got / want"]
    for p in idx[:6].tolist():
        lines.append(f"  ({p}, frame {p // U}, offset {p % U}): {float(wave[p])!r} / {float(want[p])!r}")
    lines.append(f"  flagged frames {sorted({p // U for p in idx.tolist()})[:12]}")
    return "\n".join(lines)
