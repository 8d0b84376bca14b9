"""GPU checks of fp32 OPT inference (`B200UnitLM(..., fp32_inference=True)`, `sk_lm_set_fp32`): the forward pass, the
scores and the decoding of a float32 OPT checkpoint, as the reference runs one (fp32 weights, no autocast).

The forward pass, the log-likelihoods (with and without ignore_tokens) and greedy generation are checked against the
reference's own UnitLM on a float32 checkpoint (tests/golden/opt_fp32_tiny.npz).  The rest is measured against fp64:
the OPT restatement of oracle/opt_oracle.py run on fp64 parameters, fp64 log_softmax, and the fp64 attention reference of
tests/attn_ref.py.  The causal split-bf16 attention is also checked bit
for bit on inputs whose three-product sums are exact (integer hi operands, lo operands on a power-of-two grid).  The bounds are stated next to each check; the fp32 path must be
at least 100 times closer to fp64 than the bf16 path on the same weights."""
import ctypes as C
import json
import math
import os

import pytest
import torch

import attn_ref as A
from oracle import opt_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
BF = torch.bfloat16


def _lib():
    from slamkit_b200 import _lib as L
    return L, L.require_cuda()


def _p(t, off=0):
    return C.c_void_p(t.data_ptr() + off * t.element_size()) if t is not None else C.c_void_p(0)


def _lm_cfg(c):
    from slamkit_b200.lm import OptLMConfig
    return OptLMConfig(vocab_size=c.vocab_size, hidden=c.hidden, n_layers=c.n_layers, n_heads=c.n_heads, ffn=c.ffn,
                       max_positions=c.max_positions, ln_eps=c.ln_eps, tie_embeddings=c.tie_embeddings)


def _models(c, seed, B, T, std=0.02, bf16=False):
    """fp32 inference model (and optionally the bf16 one) on the same seeded fp32 parameters."""
    from slamkit_b200.lm import B200UnitLM
    p = O.init_params(c, seed=seed, std=std, dtype=torch.float32)
    m = B200UnitLM(_lm_cfg(c), device=DEV, max_batch=B, max_seq=T, trainable=False, fp32_inference=True)
    m.load_hf_state_dict(p)
    m16 = None
    if bf16:
        m16 = B200UnitLM(_lm_cfg(c), device=DEV, max_batch=B, max_seq=T, trainable=False)
        m16.load_hf_state_dict(p)
    return m, m16, p


def _fp64_logits(p, c, ids):
    p64 = {k: v.to(DEV, torch.float64) for k, v in p.items()}
    with torch.no_grad():
        return O.forward_logits(p64, c, ids.to(DEV))


def _fp64_token_nll(z, ids, pad=0, ban=None):
    z = z.clone()
    if ban:
        z[..., ban] = float("-inf")
    lp = torch.log_softmax(z[:, :-1], -1)
    y = ids[:, 1:].to(z.device)
    nll = -lp.gather(-1, y.clamp(min=0).unsqueeze(-1)).squeeze(-1)
    mask = y != pad
    return torch.where(mask, nll, torch.zeros_like(nll)), mask


def _right_padded(B, T, V, seed, min_len=8):
    g = torch.Generator().manual_seed(seed)
    lens = torch.randint(min_len, T + 1, (B,), generator=g)
    lens[0] = T
    ids = torch.randint(2, V, (B, T), generator=g)
    ids[:, 0] = 1
    ids[torch.arange(T)[None] >= lens[:, None]] = 0
    return ids, lens


C125 = dict(vocab_size=502, hidden=768, n_layers=12, n_heads=12, ffn=3072, max_positions=2048)
SMALL = dict(vocab_size=502, hidden=256, n_layers=3, n_heads=4, ffn=1024, max_positions=512)

# Per-token NLL bound of the fp32 path against fp64 at the opt-125m geometry.  Each split product drops lo*lo (relative
# 2^-16 of |a||b|) and each pair rounds its value to ~2^-17 relative; through 12 layers and a 502-way log_softmax with
# O(1) logits this stays below 1e-4 per token with a wide margin.
NLL_BOUND = 1e-4


# ------------------------------------------------------------------------------------------------ 1. reference golden
# tests/golden/opt_fp32_tiny.npz: the reference's own UnitLM on a float32 checkpoint (oracle/make_opt_fp32_golden.py)
def test_reference_golden(golden_dir):
    from test_opt_fp32_cpu import golden_fp32
    from slamkit_b200.lm import B200UnitLM
    z, c, p = golden_fp32(golden_dir)
    m = B200UnitLM(_lm_cfg(c), device=DEV, max_batch=4, max_seq=c.max_positions, trainable=False, fp32_inference=True)
    m.load_hf_state_dict(p)
    ids = torch.from_numpy(z["logits/ids"]).to(DEV)
    want = torch.from_numpy(z["logits/z"]).to(DEV)
    got = m.forward(ids).logits
    rel = float((got.double() - want.double()).norm() / want.double().norm())
    tokens = torch.from_numpy(z["loglik/tokens"])
    ignore = z["loglik/ignore"].tolist()
    errs = {}
    for key, mean_nll, ign in (("sum", False, None), ("mean", True, None), ("sum_ign", False, ignore),
                               ("mean_ign", True, ignore)):
        ll = m.sequence_log_likelihood(tokens, mean_nll, ign)
        assert ll.dtype == torch.float32
        errs[key] = float((ll.cpu().double() - torch.from_numpy(z["loglik/" + key]).double()).abs().max())
    print(f"golden: logits rel-L2 {rel:.3e}, log-likelihood errors {errs}")
    assert rel < 1e-4
    n = int((tokens[:, 1:] != 0).sum(-1).max())
    for key, e in errs.items():
        assert e < (1e-4 if key.startswith("mean") else 1e-4 * n), key
    prompt = torch.from_numpy(z["gen/prompt"])
    want_seq = torch.from_numpy(z["gen/out"])[0]
    margin = torch.from_numpy(z["gen/margin"])
    out = m.generate(prompt, max_new_tokens=len(margin), do_sample=False)[0].cpu()
    P = prompt.shape[1]
    for i in range(len(margin)):
        if float(margin[i]) <= 1e-4:
            break                              # a near tie: the continuation may legitimately differ from here on
        assert int(out[P + i]) == int(want_seq[P + i]), i


# ---------------------------------------------------------------------------------------- 2. fp64 oracle at real width
def test_opt125m_token_nll_vs_fp64_and_bf16_gap():
    c = O.OracleOptConfig(**C125)
    B, T = 8, 512
    m, m16, p = _models(c, 3, B, T, bf16=True)
    ids, lens = _right_padded(B, T, c.vocab_size, 4)
    ids_d = ids.to(DEV)
    ref = _fp64_logits(p, c, ids)
    want, mask = _fp64_token_nll(ref, ids)
    ll, tok = m.sequence_log_likelihood(ids_d, mean_nll=False, return_token_nll=True)
    assert ll.dtype == torch.float32 and tok.dtype == torch.float32
    logits = m.forward(ids_d).logits
    assert logits.dtype == torch.float32
    valid = torch.arange(T, device=DEV)[None] < lens.to(DEV)[:, None]
    zerr = (logits.double() - ref)[valid].norm() / ref[valid].norm()
    err32 = (tok.double() - want).abs()[mask]
    _, tok16 = m16.sequence_log_likelihood(ids_d, mean_nll=False, return_token_nll=True)
    err16 = (tok16.double() - want).abs()[mask]
    print(f"fp32 path: logits rel-L2 {float(zerr):.3e}, token NLL max {float(err32.max()):.3e} mean "
          f"{float(err32.mean()):.3e}; bf16 path: max {float(err16.max()):.3e} mean {float(err16.mean()):.3e}")
    assert float(zerr) < 1e-4
    assert float(err32.max()) < NLL_BOUND
    assert float(err32.mean()) * 100 <= float(err16.mean())
    assert float(err32.max()) * 100 <= float(err16.max())
    # the sum over a row's tokens, in fp32 and in a fixed order
    want_ll = -(want * mask).sum(-1)
    assert float((ll.double() - want_ll).abs().max()) < NLL_BOUND * T


# ------------------------------------------------------------------------------------------------------- 3. tie rule
def test_fp32_scores_resolve_pairs_that_bf16_ties():
    """Pairs whose fp64 mean NLLs differ by more than the fp32 bound but by less than half a bf16 step: the fp32 path
    orders each as fp64 does; the bf16 path ties at least one (its scores round to the same bf16 value)."""
    c = O.OracleOptConfig(**SMALL)
    B, T = 48, 96
    m, m16, p = _models(c, 5, B, T, std=0.05, bf16=True)
    ids, _ = _right_padded(B, T, c.vocab_size, 6, min_len=T // 2)
    want_tok, mask = _fp64_token_nll(_fp64_logits(p, c, ids), ids)
    want = -(want_tok.sum(-1) / mask.sum(-1))
    got = m.sequence_log_likelihood(ids.to(DEV), mean_nll=True).double()
    got16 = m16.sequence_log_likelihood(ids.to(DEV), mean_nll=True)
    assert float((got - want).abs().max()) < NLL_BOUND
    def half_step(x):                                      # half the bf16 spacing at |x|
        return 2.0 ** (math.floor(math.log2(abs(float(x)))) - 8)

    pairs = [(i, j) for i in range(B) for j in range(i + 1, B)
             if 4 * NLL_BOUND < abs(float(want[i] - want[j])) < min(half_step(want[i]), half_step(want[j]))]
    assert len(pairs) >= 10, len(pairs)
    for i, j in pairs:
        assert (got[i] > got[j]) == (want[i] > want[j]), (i, j)
    assert any(bool(got16[i] == got16[j]) for i, j in pairs)


# ------------------------------------------------------------------------------ 4. causal split attention conformance
def _causal_split(hi, lo, B, T, H, o_hi=None, o_lo=None):
    L, lib = _lib()
    o_hi = torch.empty(B * T, H * 64, dtype=BF, device=DEV) if o_hi is None else o_hi
    o_lo = torch.empty_like(o_hi) if o_lo is None else o_lo
    L.check(lib.sk_attn_tc_fwd_split_causal(_p(hi), _p(lo), _p(o_hi), _p(o_lo), B, T, H, hi.stride(0), o_hi.stride(0),
                                            L.f32(0.125), L.stream_ptr()))
    return o_hi, o_lo


def _fused(parts, B, T, H, ld=None, fill=float("nan")):
    """[B*T, ld] hi and lo projections (q | k | v heads), padding columns filled with NaN."""
    ld = ld or 3 * H * 64
    out = []
    for half in (0, 1):
        x = torch.full((B * T, ld), fill, dtype=BF)
        x[:, :3 * H * 64] = torch.cat([parts[half], parts[2 + half], parts[4 + half]], 2).reshape(B * T, -1).to(BF)
        out.append(x.to(DEV))
    return out


@pytest.mark.parametrize("T", [1, 63, 64, 65, 127, 128, 129, 1000, 2048])
@pytest.mark.parametrize("B,H", [(2, 12), (1, 4), (3, 2)])
def test_causal_split_uniform_exact(T, B, H):
    """q = 0: row t's output is fl(sum_{s<=t} (Vh + Vl)) * fl(1/(t+1)); the sum is exact (|sum| < 2^17, step 2^-6), so
    the (hi, lo) output is compared bit for bit.  Inputs at a pitch with NaN padding; outputs inside NaN guard bands."""
    z = torch.zeros(B, T, H, 64)
    k_hi = A.int_values((B, T, H, 64), 4, T)
    v_hi = A.int_values((B, T, H, 64), 16, T + 1)
    v_lo = A.int_values((B, T, H, 64), 16, T + 2) / 64.0
    ssum = (v_hi.double() + v_lo.double()).cumsum(1).float()
    inv = torch.ones(()) / torch.arange(1, T + 1, dtype=torch.float32)
    o = ssum * inv[None, :, None, None]
    want_hi = A.bf16(o)
    want_lo = A.bf16(o - want_hi)
    hi, lo = _fused((z, z, k_hi, torch.zeros_like(k_hi), v_hi, v_lo), B, T, H, ld=3 * H * 64 + 64)
    guard = 96
    ob = torch.full((B * T + 2, H * 64 + guard), float("nan"), dtype=BF, device=DEV)
    ob_lo = ob.clone()
    o_hi = ob[1:B * T + 1, :H * 64]
    o_lo = ob_lo[1:B * T + 1, :H * 64]
    _causal_split(hi, lo, B, T, H, o_hi, o_lo)
    A_hi, A_lo = A.heads(o_hi, B, T, H), A.heads(o_lo, B, T, H)
    for got, want, what in ((A_hi, want_hi, "hi"), (A_lo, want_lo, "lo")):
        bad = A.mismatch_exact(got, want, f"causal split uniform {what} T={T}")
        assert bad is None, str(bad)
    outside = torch.ones(ob.shape, dtype=torch.bool, device=DEV)
    outside[1:B * T + 1, :H * 64] = False
    for buf in (ob, ob_lo):
        assert bool(buf[outside].isnan().all()), "a write outside the output"


def _causal_split_onehot(B, T, H, seed):
    """attn_ref.split_onehot under the causal mask: integer hi operands, lo operands that feed the Qh Kl and Ql Kh
    products (Ql non-zero only where Kl is zero and vice versa), v on the 2^-6 grid, so every score is exact and each
    row's softmax is one-hot on its target: key t ("latest" heads, the diagonal) or key 0 ("earliest" heads).
    Returns the six [B, T, H, 64] operands and the expected (o_hi, o_lo)."""
    modes = A.modes_for(H)
    lo, hi = A.bounds(B, T, True)
    tgt = A.onehot_targets(lo, hi, modes)
    q = A.onehot_q(tgt, modes)
    k = A.onehot_k(B, T, H)
    q_hi, q_lo = q.clone(), torch.zeros_like(q)
    sg = torch.tensor([1.0 if m == "latest" else -1.0 for m in modes])
    p = torch.tensor([2.0 ** (10 + 4 * d) for d in range(4)])
    q_lo[..., 4:8] = sg[:, None] * p
    q_hi[..., 4:8] = q[..., 4:8] - q_lo[..., 4:8]
    k_hi, k_lo = k.clone(), torch.zeros_like(k)
    k_lo[..., :4] = -1.0
    k_hi[..., :4] = k[..., :4] + 1.0
    for t in (q_hi, q_lo, k_hi, k_lo):
        assert A.is_bf16(t)
    v_hi = A.int_values((B, T, H, 64), 16, seed)
    v_lo = A.int_values((B, T, H, 64), 16, seed + 1) / 64.0
    o = A.expect_onehot_fwd(v_hi + v_lo, tgt, 1)[0]
    o_hi = A.bf16(o)
    return (q_hi, q_lo, k_hi, k_lo, v_hi, v_lo), (o_hi, A.bf16(o - o_hi))


@pytest.mark.parametrize("T", [1, 63, 64, 65, 127, 128, 129, 1000, 2048])
@pytest.mark.parametrize("B,H", [(2, 12), (1, 4), (3, 2)])
def test_causal_split_onehot_exact(T, B, H):
    """All three products carry signal (Qh Kh, Qh Kl, Ql Kh); outputs compared bit for bit."""
    parts, (want_hi, want_lo) = _causal_split_onehot(B, T, H, seed=T + H)
    hi, lo = _fused(parts, B, T, H)
    o_hi, o_lo = _causal_split(hi, lo, B, T, H)
    for got, want, what in ((A.heads(o_hi, B, T, H), want_hi, "hi"), (A.heads(o_lo, B, T, H), want_lo, "lo")):
        bad = A.mismatch_exact(got, want, f"causal split one-hot {what} T={T}")
        assert bad is None, str(bad)


def test_causal_split_random_per_element():
    B, T, H = 2, 333, 4
    g = torch.Generator().manual_seed(41)
    parts = []
    for _ in range(3):
        x = torch.randn(B, T, H, 64, generator=g) * 2.0
        xh = A.bf16(x)
        parts += [xh, A.bf16(x - xh)]
    hi, lo = _fused(parts, B, T, H)
    o_hi, o_lo = _causal_split(hi, lo, B, T, H)
    got = A.heads(o_hi, B, T, H).double() + A.heads(o_lo, B, T, H).double()
    q, k, v = parts[0] + parts[1], parts[2] + parts[3], parts[4] + parts[5]
    lo_b, hi_b = A.bounds(B, T, True)
    O_, _, bo, _ = A.fwd_reference(q, k, v, lo_b, hi_b, 0.125, True, split=True)
    bad = A.mismatch_bound(got, O_, bo, "causal split random hi + lo")
    assert bad is None, str(bad)


@pytest.mark.parametrize("t", [127, 255, 1023])
def test_causal_split_future_and_batch_isolation(t):
    """NaN in the keys and values of rows > t, where t + 1 is a multiple of the 128-row query tile, and in another
    batch row leaves rows <= t unchanged: no key tile past a query tile's diagonal is read.  Inside the diagonal tile the
    future keys are read and masked to a zero weight, so a NaN value there would reach the output through 0 * NaN; real
    K / V are finite, and this test does not cover that case."""
    B, T, H = 3, 1100, 4
    g = torch.Generator().manual_seed(t)
    parts = []
    for _ in range(3):
        x = torch.randn(B, T, H, 64, generator=g)
        xh = A.bf16(x)
        parts += [xh, A.bf16(x - xh)]
    hi, lo = _fused(parts, B, T, H)
    base = [x.clone() for x in _causal_split(hi, lo, B, T, H)]
    for x in (hi, lo):
        xv = x.view(B, T, -1)
        xv[0, t + 1:, H * 64:] = float("nan")                # future keys and values of row 0
        xv[2] = float("nan")                                  # all of batch row 2
    got = _causal_split(hi, lo, B, T, H)
    rows0 = torch.arange(t + 1, device=DEV)
    rows1 = T + torch.arange(T, device=DEV)
    for g_, b_ in zip(got, base):
        assert torch.equal(g_[rows0], b_[rows0]), "a future key reached an earlier row"
        assert torch.equal(g_[rows1], b_[rows1]), "another batch row reached row 1"


# -------------------------------------------------------------------------------------------------- 5. fp32 scoring
def _scoring_case(V, B, T, seed):
    g = torch.Generator().manual_seed(seed)
    ldl = (V + 63) // 64 * 64 + 64
    z = torch.randn(B * T, V, generator=g, dtype=torch.float64) * 4
    buf = torch.full((B * T, ldl), float("nan"), dtype=torch.float32)    # columns >= V are NaN: never read
    buf[:, :V] = z.float()
    ids = torch.randint(1, V, (B, T), generator=g)
    ids[1, T // 2:] = 0                                                  # right padding (pad id 0)
    ids[2, 1:] = 0                                                       # an empty row: NaN with mean_nll
    ban = torch.randperm(V, generator=g)[:V // 5].tolist()
    ids[3, 5] = ban[0]                                                   # a banned target: +inf
    return z, buf.to(DEV), ids, ban, ldl


@pytest.mark.parametrize("V", [502, 8192, 8193, 9000])
@pytest.mark.parametrize("mean_nll", [False, True])
@pytest.mark.parametrize("banned", [False, True])
def test_seq_loglik_f32_vs_fp64(V, mean_nll, banned):
    from slamkit_b200.generation import ban_bitmask
    L, lib = _lib()
    B, T = 6, 40
    z, buf, ids, ban, ldl = _scoring_case(V, B, T, V + int(mean_nll))
    ban = ban if banned else []
    bits = ban_bitmask(ban, V).to(DEV) if ban else None
    ids_d = ids.to(DEV)

    def run():
        tok = torch.empty(B * (T - 1), dtype=torch.float32, device=DEV)
        ll = torch.empty(B, dtype=torch.float32, device=DEV)
        L.check(lib.sk_seq_loglik_f32(_p(buf), ldl, V, _p(ids_d), B, T, 0, _p(bits), int(mean_nll), _p(tok), _p(ll),
                                      L.stream_ptr()))
        return tok.view(B, T - 1).cpu(), ll.cpu()

    tok, ll = run()
    tok2, ll2 = run()
    assert torch.equal(tok, tok2) and torch.equal(ll.view(torch.int32), ll2.view(torch.int32))
    want, mask = _fp64_token_nll(z.view(B, T, V).float().double(), ids, ban=ban or None)
    fin = torch.isfinite(want)
    assert torch.equal(torch.isfinite(tok), fin)
    # fp32 log_softmax: |error| <= a few ulps of max |z| and of log(sum)
    assert float((tok.double() - want)[fin].abs().max()) < 2e-5
    assert bool((tok[~mask] == 0).all())
    s = (want * mask).sum(-1)
    n = mask.sum(-1)
    w_ll = -(s / n) if mean_nll else -s
    for b in range(B):
        if mean_nll and int(n[b]) == 0:
            assert math.isnan(float(ll[b]))
        elif not math.isfinite(float(w_ll[b])):
            assert float(ll[b]) == float(w_ll[b])
        else:
            assert abs(float(ll[b]) - float(w_ll[b])) < 2e-5 * max(1, int(n[b]))


# -------------------------------------------------------------------------------------------------------- 6. decoding
def test_prefill_and_decode_follow_the_full_forward():
    from slamkit_b200.lm import DecodeSession
    c = O.OracleOptConfig(**SMALL)
    B, T, k = 4, 120, 6
    m, _, _ = _models(c, 7, B, T + k)
    ids, lens = _right_padded(B, T + k, c.vocab_size, 8, min_len=k + 10)
    full = m.forward(ids.to(DEV)).logits.clone()
    plens = lens - k
    prompt = ids.clone()
    prompt[torch.arange(T + k)[None] >= plens[:, None]] = 0
    sess = DecodeSession(m, B, T + k, k, 0)
    sess.kv.view(torch.float32).fill_(float("nan"))          # positions at or past lens are never read
    got = [sess.prefill(prompt[:, :T], plens).clone()]
    for i in range(k - 1):
        pos = (plens + i).to(torch.int32)
        got.append(sess.step(ids.gather(1, pos[:, None].long())[:, 0].to(DEV), pos.to(DEV)).clone())
    scale = float(full.abs().max())
    for i, g_ in enumerate(got):
        want = full[torch.arange(B, device=DEV), (plens - 1 + i).to(DEV)]
        assert g_.dtype == torch.float32
        assert float((g_ - want).abs().max()) <= 2e-5 * max(1.0, scale), i


def _decode_run(m, ids, lens, T_cache, k, graph):
    from slamkit_b200.lm import DecodeSession
    B = ids.shape[0]
    sess = DecodeSession(m, B, T_cache, k, 0)
    sess.prefill(ids, lens)
    tok = torch.zeros(B, dtype=torch.long, device=DEV)
    pos = torch.zeros(B, dtype=torch.int32, device=DEV)
    outs, g = [], None
    for i in range(k):
        tok.copy_(((lens * 7 + i * 13) % 400 + 2).to(DEV))
        pos.copy_((lens + i).to(DEV))
        if graph and i > 0:
            if g is None:
                g, cur, side = torch.cuda.CUDAGraph(), torch.cuda.current_stream(), torch.cuda.Stream()
                side.wait_stream(cur)
                with torch.cuda.stream(side):
                    g.capture_begin()
                    sess.step(tok, pos)
                    g.capture_end()
                cur.wait_stream(side)
            g.replay()
        else:
            sess.step(tok, pos)
        outs.append(sess.logits.clone())
    return outs


def test_decode_graph_replay_and_batch_invariance():
    c = O.OracleOptConfig(**SMALL)
    B, T, k = 8, 70, 5
    m, _, _ = _models(c, 9, B, T + k)
    ids, lens = _right_padded(B, T, c.vocab_size, 10)
    eager = _decode_run(m, ids, lens, T + k, k, False)
    replay = _decode_run(m, ids, lens, T + k, k, True)
    for a, b in zip(eager, replay):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32)), "graph replay differs from eager"
    alone = _decode_run(m, ids[3:4], lens[3:4], T + k, k, False)
    for a, b in zip(alone, eager):
        assert torch.equal(a[0].view(torch.int32), b[3].view(torch.int32)), "row 3 alone differs from row 3 in the batch"


@pytest.mark.parametrize("case", ["greedy", "temp0.8-top_k25", "top_p0.9", "bans-greedy", "bans-temp1.3-top_k40"])
def test_select_next_f32_matches_host_rules(case):
    from decode_ref import expected_token
    from test_gpu_generate import SAMPLER_CASES
    from slamkit_b200.generation import ban_bitmask
    L, lib = _lib()
    c = dict(SAMPLER_CASES[case])
    bans = c.pop("bans", False)
    B, V = 48, 502
    g = torch.Generator().manual_seed(len(case))
    logits = torch.randn(B, V, generator=g) * 3.0
    logits[0, 5] = logits[0, 9] = logits[0].max() + 1             # tied maxima: greedy takes the lower id
    logits[2, 7] = logits[2].max() + 2 ** -20                     # an fp32 margin that bf16 could not hold
    banned = torch.randperm(V, generator=g)[:V // 3].tolist() if bans else []
    banned = [i for i in banned if i not in (5, 7, 9)]
    u = torch.rand(B, generator=g)
    ldl = 512
    dl = torch.full((B, ldl), float("nan"))
    dl[:, :V] = logits
    dl = dl.to(DEV)
    cfg = L.SkSampling(seed=1, top_p=float(c.get("top_p", 1.0)), temperature=float(c.get("temperature", 1.0)),
                       do_sample=int(c["do_sample"]), top_k=int(c.get("top_k", 0)), n_eos=0, pad_token_id=0,
                       max_length=1 << 30)
    st = {k: torch.zeros(B, dtype=torch.int32, device=DEV) for k in ("pos", "finished", "n_gen")}
    tokens, out = torch.zeros(B, dtype=torch.long, device=DEV), torch.full((B, 1), -1, dtype=torch.long, device=DEV)
    step = torch.zeros(2, dtype=torch.int32, device=DEV)
    state = L.SkDecodeState(tokens.data_ptr(), st["pos"].data_ptr(), st["finished"].data_ptr(), st["n_gen"].data_ptr(),
                            out.data_ptr(), step.data_ptr(), 1, 0)
    ban = ban_bitmask(banned, V).to(DEV) if banned else None
    L.check(lib.sk_select_next_f32(_p(dl), ldl, V, B, _p(ban), C.byref(cfg), _p(u.to(DEV)), C.byref(state), L.stream_ptr()))
    got = out[:, 0].cpu().tolist()
    skipped = 0
    for b in range(B):
        want, dist = expected_token(logits[b], c["do_sample"], c.get("temperature", 1.0), c.get("top_k"), c.get("top_p"),
                                    banned, float(u[b]))
        if dist < 1e-6:
            skipped += 1
            continue
        assert got[b] == want, (b, got[b], want)
    if not c["do_sample"]:
        assert got[0] == 5 and got[2] == 7
    assert skipped <= 2


def test_generate_greedy_follows_fp64():
    """Cached greedy generate of the fp32 model takes the fp64 argmax at every step whose top-1 / top-2 margin exceeds
    the logits bound."""
    c = O.OracleOptConfig(**SMALL)
    m, _, p = _models(c, 11, 2, 64, std=0.05)
    prompt = torch.tensor([[1, 17, 33, 5, 250, 9, 41, 77]])
    out = m.generate(prompt, max_new_tokens=12, do_sample=False, eos_token_id=[])
    seq = out[0].cpu()
    for t in range(prompt.shape[1], seq.shape[0]):
        z = _fp64_logits(p, c, seq[None, :t])[0, -1]
        top = torch.topk(z, 2).values
        if float(top[0] - top[1]) > 1e-4:
            assert int(seq[t]) == int(z.argmax()), t


# -------------------------------------------------------------------------------------------------------- 7. refusals
def test_refusals_launch_nothing():
    from slamkit_b200 import _lib as L
    from slamkit_b200.lm import B200UnitLM, LMConfig, NeoxLMConfig
    lib = L.require_cuda()
    c = O.OracleOptConfig(**SMALL)
    m, _, _ = _models(c, 1, 2, 32)
    ids = torch.ones(2, 8, dtype=torch.long, device=DEV)
    stats = torch.zeros(3, device=DEV)
    row = torch.zeros(16, device=DEV)
    f32 = torch.zeros(m.n_params, device=DEV)
    m.forward(ids)
    calls = [
        lambda: lib.sk_lm_forward_backward(m._h, _p(ids), _p(ids), None, 2, 8, L.f32(0), L.f32(1), 0, _p(stats),
                                           L.stream_ptr()),
        lambda: lib.sk_lm_forward_rows(m._h, _p(ids), _p(ids), None, 2, 8, _p(row), _p(stats), L.stream_ptr()),
        lambda: lib.sk_lm_backward_weighted(m._h, _p(ids), _p(ids), None, 2, 8, _p(row), 0, _p(stats), L.stream_ptr()),
        lambda: lib.sk_lm_optimizer_step(m._h, _p(f32), _p(f32), L.f32(1e-3), L.f32(0.9), L.f32(0.999), L.f32(1e-8),
                                         L.f32(0), 1, L.f32(1), 0, _p(stats), L.stream_ptr()),
        lambda: lib.sk_lm_set_master(m._h, _p(m.params32), _p(f32)),
        lambda: lib.sk_lm_forward(m._h, _p(ids), _p(ids), None, 2, 8, L.f32(0), _p(stats), L.stream_ptr()),
    ]
    for fn in calls:
        with pytest.raises(L.SkError, match="fp32 inference|sk_lm_set_fp32"):
            L.check(fn())
    assert lib.sk_lm_logits(m._h) is None
    master = B200UnitLM(_lm_cfg(c), device=DEV, max_batch=2, max_seq=32, master_weights=True)
    qwen = B200UnitLM(LMConfig(vocab_size=502, hidden=128, n_layers=1, n_heads=2, n_kv_heads=1, head_dim=64, ffn=256),
                      device=DEV, max_batch=2, max_seq=32, trainable=False)
    neox = B200UnitLM(NeoxLMConfig(vocab_size=502, hidden=128, n_layers=1, n_heads=2, ffn=512, max_positions=64,
                                   rot_dims=16),
                      device=DEV, max_batch=2, max_seq=32, trainable=False)
    prep = torch.empty(int(lib.sk_lm_fp32_prepared_bytes(m._h)), dtype=torch.uint8, device=DEV)
    n0 = lib.sk_launch_count()
    for h, msg in ((master._h, "master"), (qwen._h, "OPT decoder only"), (neox._h, "OPT decoder only")):
        with pytest.raises(L.SkError, match=msg):
            L.check(lib.sk_lm_set_fp32(h, _p(f32), _p(prep), C.c_int64(prep.numel()), L.stream_ptr()))
    for fn in calls:
        with pytest.raises(L.SkError):
            L.check(fn())
    assert lib.sk_launch_count() == n0, "a refused call launched a kernel"
    with pytest.raises(NotImplementedError):
        master.generate(torch.ones(1, 4, dtype=torch.long), max_new_tokens=3)


# -------------------------------------------------------------------------------------------------------------- 8. CLI
def _trained_float32_checkpoint(tmp_path):
    """A GSLM checkpoint trained by cli/train.py with torch_dtype=float32 (fp32 master weights), as users produce one."""
    from cli import train
    from test_gpu_opt import _opt_train_args, _tiny_opt_dir
    from test_gpu_round2 import _write_tokens
    base = _tiny_opt_dir(tmp_path / "base", twist=False)
    tok = str(tmp_path / "tok.jsonl")
    _write_tokens(tok, 24, 1)
    args = [a.replace("torch_dtype=bfloat16", "torch_dtype=float32") for a in _opt_train_args(base, False)]
    train.main([f"data.train_path={tok}", f"data.val_path={tok}", *args, "+training_args.max_steps=4",
                f"training_args.output_dir={tmp_path}/ck"])
    return tmp_path / "ck"


def test_cli_eval_scores_and_generates_a_float32_checkpoint(tmp_path):
    import sys
    sys.path.insert(0, os.path.dirname(__file__))
    import cli.eval as E
    from cli.extract_features import build_tokeniser
    from slamkit_b200 import metrics as M
    from slamkit_b200.config import load_config
    from slamkit_b200.lm import B200UnitLM
    from slamkit_b200.lm import checkpoint_is_fp32
    from slamkit_b200.speech_lm import B200SpeechLM
    from test_gpu_eval import _write_clips
    from test_gpu_vocoder import _textless_checkpoint
    from flac_writer import write_flac
    ck = _trained_float32_checkpoint(tmp_path)
    assert checkpoint_is_fp32(json.load(open(ck / "config.json")))
    assert B200UnitLM.from_pretrained(str(ck), device=DEV, trainable=False).fp32
    assert not B200UnitLM.from_pretrained(str(ck), device=DEV, trainable=True).fp32
    g = torch.Generator().manual_seed(13)
    sw = tmp_path / "swuggy"
    _write_clips(sw, [f"{d}/{i}_w.wav" for d in ("a", "b") for i in range(4)], g)
    common = [f"model.pretrained_model={ck}", "+synthetic_weights=true", "batch_size=2", "num_workers=2"]
    argv = common + ["metric=swuggy_inter", f"metric.data_path={sw}"]
    res = E.main(argv)
    cfg = load_config("eval", argv)
    model = E.load_model(cfg, DEV)
    assert model.fp32
    slm = B200SpeechLM(model, build_tokeniser(cfg, DEV))
    assert model.sequence_log_likelihood(torch.ones(2, 9, dtype=torch.long), True).dtype == torch.float32
    assert res == M.swuggy(slm, str(sw), None, True, 2, 2, True, True)
    data = tmp_path / "prompts"
    data.mkdir()
    for i, n in enumerate((36000, 20000, 52000)):
        pcm = (0.2 * torch.randn(n, generator=g).clamp(-4, 4) / 4 * 32767).round().long().numpy()[:, None]
        write_flac(str(data / f"p{i}.flac"), pcm)
    mp, cp = _textless_checkpoint(tmp_path)
    out = tmp_path / "gen"
    res = E.main(common + ["metric=generate", "vocoder=vocoder_hubert_25", f"vocoder.model_path={mp}",
                           f"vocoder.config_path={cp}", f"metric.data_path={data}/*.flac", "metric.prompt_length=2",
                           f"metric.out_path={out}", "metric.generate_kwargs.do_sample=false",
                           "metric.generate_kwargs.max_new_tokens=16"])
    gens = res["generate"]
    assert len(gens) == 3
    assert sorted(os.listdir(out)) == sorted(f"generate_{i}.wav" for i, w in enumerate(gens) if w.numel() > 0)
