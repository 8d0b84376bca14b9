"""Conformance of decode.cu, the kernels behind `generate`: the fp32-cache decode attention (`sk_attn_decode_split`),
token selection (`sk_select_next`, `sk_select_next_f32`) with its Philox draws and decode state, and the KV-cache
writes of prefill and decode steps.

References: tests/attn_ref.py (fp32 decode one-hot / uniform expectations, exact, and the random-mode bound against
fp64) and tests/decode_ref.py (HF's selection rules, constructed rows with an exact answer, Philox4x32-10)."""
import ctypes as C

import numpy as np
import pytest
import torch

import attn_ref as A
import decode_ref as D

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
BF = torch.bfloat16


def _lib():
    from slamkit_b200 import _lib as L
    return L, L.require_cuda()


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


# ---------------------------------------------------------------------------------------- A. fp32-cache decode attention
LENS = [1, 63, 64, 65, 127, 128, 129, 1000, 2048]


def _lens(B, H, T_cache):
    choices = [n for n in LENS if n <= T_cache] + ([T_cache] if T_cache not in LENS else [])
    return torch.tensor([choices[(b * 5 + H) % len(choices)] for b in range(B)], dtype=torch.int32)


def _fused_q(x, H, fill=float("nan")):
    """[B, 3 H 64] bf16 on the device: the query heads as the first columns of a fused projection (ldq = 3 H 64)."""
    B = x.shape[0]
    buf = torch.full((B, 3 * H * 64), fill, dtype=BF)
    buf[:, :H * 64] = x.reshape(B, -1).to(BF)
    return buf.to(DEV)


def _cache(x, lens):
    """fp32 [B, H, Tc, 64] on the device with NaN at t >= lens[b]: those slots are never read."""
    c = x.clone().float()
    for b in range(c.shape[0]):
        c[b, :, int(lens[b]):] = float("nan")
    return c.to(DEV)


def _decode_split(q_hi, q_lo, kc, vc, lens, B, H, T_cache, ldq=None, ldo=None):
    """Runs sk_attn_decode_split; outputs at pitch ldo = H 64 + 64 with NaN sentinel columns.  Returns (o_hi, o_lo)
    as [B, H, 64] float on the CPU and the raw output buffers."""
    L, lib = _lib()
    ldq = ldq or 3 * H * 64
    ldo = ldo or H * 64 + 64
    partial = torch.empty(int(lib.sk_attn_decode_partial_bytes(B, H, T_cache)) // 4, device=DEV)
    ob = torch.full((B, ldo), float("nan"), dtype=BF, device=DEV)
    ob_lo = ob.clone()
    lens_d = lens.to(DEV)
    L.check(lib.sk_attn_decode_split(_p(q_hi), _p(q_lo), ldq, _p(kc), _p(vc), _p(lens_d), _p(ob), _p(ob_lo), ldo,
                                     _p(partial), B, H, T_cache, L.f32(0.125), L.stream_ptr()))
    torch.cuda.synchronize()
    for buf in (ob, ob_lo):
        assert bool(buf[:, H * 64:].isnan().all()), "a write past the heads of the output row"
    return (ob[:, :H * 64].float().cpu().view(B, H, 64), ob_lo[:, :H * 64].float().cpu().view(B, H, 64)), (ob, ob_lo)


def _causal_rows(q_hi, q_lo, k, v, lens, rows):
    """Row lens[b] - 1 of sk_attn_tc_fwd_split_causal over the same keys (T = lens[b]): the query row is the decode
    query, earlier rows q = 0.  k / v are split into their exact bf16 pairs."""
    L, lib = _lib()
    H = q_hi.shape[1]
    out = {}
    for b in rows:
        n = int(lens[b])
        z = torch.zeros(n, H, 64)
        qh, ql = z.clone(), z.clone()
        qh[n - 1], ql[n - 1] = q_hi[b], q_lo[b]
        kk, vv = k[b, :, :n].permute(1, 0, 2), v[b, :, :n].permute(1, 0, 2)
        kh, vh = A.bf16(kk), A.bf16(vv)
        kl, vl = kk - kh, vv - vh
        assert A.is_bf16(kl) and A.is_bf16(vl)
        hi = torch.cat([qh, kh, vh], 1).reshape(n, -1).to(BF).to(DEV)
        lo = torch.cat([ql, kl, vl], 1).reshape(n, -1).to(BF).to(DEV)
        o_hi = torch.empty(n, H * 64, dtype=BF, device=DEV)
        o_lo = torch.empty_like(o_hi)
        L.check(lib.sk_attn_tc_fwd_split_causal(_p(hi), _p(lo), _p(o_hi), _p(o_lo), 1, n, H, 3 * H * 64, H * 64,
                                                L.f32(0.125), L.stream_ptr()))
        out[b] = (o_hi[n - 1].float().cpu().view(H, 64), o_lo[n - 1].float().cpu().view(H, 64))
    return out


@pytest.mark.parametrize("T_cache", [2048, 130])
@pytest.mark.parametrize("B", [1, 5, 64])
@pytest.mark.parametrize("H", [2, 12, 16])
def test_decode_split_exact_modes(H, B, T_cache):
    """One-hot (latest / earliest per head) and uniform outputs bit for bit, bit-identical on a second run, and equal
    bit for bit to the causal split-bf16 kernel's row over the same keys."""
    lens = _lens(B, H, T_cache)
    (q_hi, q_lo, k, v), (w_hi, w_lo) = A.decode_split_onehot(B, H, T_cache, lens, A.modes_for(H), seed=H + B)
    qh, ql, kc, vc = _fused_q(q_hi, H), _fused_q(q_lo, H), _cache(k, lens), _cache(v, lens)
    (o_hi, o_lo), raw = _decode_split(qh, ql, kc, vc, lens, B, H, T_cache)
    for got, want, what in ((o_hi, w_hi, "hi"), (o_lo, w_lo, "lo")):
        bad = A.mismatch_exact(got[:, None], want[:, None], f"decode split one-hot {what} H={H} B={B} Tc={T_cache}")
        assert bad is None, str(bad)
    _, raw2 = _decode_split(qh, ql, kc, vc, lens, B, H, T_cache)
    for a, b in zip(raw, raw2):
        assert torch.equal(a.view(torch.int16), b.view(torch.int16)), "not bit-identical run to run"
    rows = range(min(B, 5))
    for b, (c_hi, c_lo) in _causal_rows(q_hi, q_lo, k, v, lens, rows).items():
        assert torch.equal(c_hi, o_hi[b]) and torch.equal(c_lo, o_lo[b]), f"one-hot row {b} differs from the causal kernel"

    (k, v), (w_hi, w_lo) = A.decode_split_uniform(B, H, T_cache, lens, seed=H * B)
    z = torch.zeros(B, H, 64)
    (o_hi, o_lo), _ = _decode_split(_fused_q(z, H), _fused_q(z, H), _cache(k, lens), _cache(v, lens), lens, B, H, T_cache)
    for got, want, what in ((o_hi, w_hi, "hi"), (o_lo, w_lo, "lo")):
        bad = A.mismatch_exact(got[:, None], want[:, None], f"decode split uniform {what} H={H} B={B} Tc={T_cache}")
        assert bad is None, str(bad)
    for b, (c_hi, c_lo) in _causal_rows(z, z, k, v, lens, rows).items():
        assert torch.equal(c_hi, o_hi[b]) and torch.equal(c_lo, o_lo[b]), f"uniform row {b} differs from the causal kernel"


@pytest.mark.parametrize("T_cache", [2048, 130])
@pytest.mark.parametrize("B", [1, 5, 64])
@pytest.mark.parametrize("H", [2, 12, 16])
def test_decode_split_random_within_bound(H, B, T_cache):
    """Random split query, fp32 K / V that are not bf16 values: o_hi + o_lo within the fp32-decode bound of fp64."""
    lens = _lens(B, H, T_cache)
    g = torch.Generator().manual_seed(1000 + H * B + T_cache)
    x = torch.randn(B, H, 64, generator=g) * 3
    q_hi = A.bf16(x)
    q_lo = A.bf16(x - q_hi)
    k = torch.randn(B, H, T_cache, 64, generator=g)
    v = torch.randn(B, H, T_cache, 64, generator=g)
    (o_hi, o_lo), _ = _decode_split(_fused_q(q_hi, H), _fused_q(q_lo, H), _cache(k, lens), _cache(v, lens), lens, B, H,
                                    T_cache)
    O, bo = A.decode_f32_reference(q_hi + q_lo, k, v, lens, 0.125)
    bad = A.mismatch_bound((o_hi.double() + o_lo.double())[:, None], O[:, None], bo[:, None],
                           f"decode split random H={H} B={B} Tc={T_cache}")
    assert bad is None, str(bad)


def test_decode_split_refusals():
    """A null argument, ldq % 8 != 0 and an odd ldo are refused with -1 and launch nothing."""
    L, lib = _lib()
    B, H, Tc = 2, 2, 130
    q = torch.zeros(B, 3 * H * 64, dtype=BF, device=DEV)
    kc = torch.zeros(B, H, Tc, 64, device=DEV)
    lens = torch.ones(B, dtype=torch.int32, device=DEV)
    o = torch.zeros(B, H * 64 + 2, dtype=BF, device=DEV)
    part = torch.empty(int(lib.sk_attn_decode_partial_bytes(B, H, Tc)) // 4, device=DEV)

    def call(q_hi=q, ldq=3 * H * 64, ldo=H * 64):
        return lib.sk_attn_decode_split(_p(q_hi), _p(q), ldq, _p(kc), _p(kc), _p(lens), _p(o), _p(o), ldo, _p(part), B,
                                        H, Tc, L.f32(0.125), L.stream_ptr())
    assert call() == 0
    torch.cuda.synchronize()
    n0 = lib.sk_launch_count()
    assert call(q_hi=None) == -1
    assert call(ldq=3 * H * 64 - 4) == -1
    assert call(ldo=H * 64 + 1) == -1
    assert lib.sk_launch_count() == n0, "a refused call launched a kernel"


# ---------------------------------------------------------------------------------------- B. token selection
V_SHAPES = [2, 3, 31, 33, 511, 513, 152167]
KINDS = ["bf16", "f32"]


class _State:
    """SkDecodeState over device tensors; `out` is followed by a guard that no call may write."""

    def __init__(self, B, max_new, pos=None, finished=None, n_gen=None, tokens=None):
        L, _ = _lib()
        i32 = lambda x: torch.tensor(x, dtype=torch.int32, device=DEV) if x is not None else \
            torch.zeros(B, dtype=torch.int32, device=DEV)
        self.pos, self.finished, self.n_gen = i32(pos), i32(finished), i32(n_gen)
        self.tokens = torch.tensor(tokens if tokens is not None else [0] * B, dtype=torch.long, device=DEV)
        self.out_buf = torch.full((B * max_new + 16,), -7, dtype=torch.long, device=DEV)
        self.out = self.out_buf[:B * max_new].view(B, max_new)
        self.step = torch.zeros(2, dtype=torch.int32, device=DEV)
        self.st = L.SkDecodeState(self.tokens.data_ptr(), self.pos.data_ptr(), self.finished.data_ptr(),
                                  self.n_gen.data_ptr(), self.out.data_ptr(), self.step.data_ptr(), max_new, 0)


def _logits_dev(rows, kind, pad=7):
    """[B, V + pad] device logits (bf16 or fp32) with NaN pad columns on even rows and +inf on odd rows."""
    B, V = rows.shape
    buf = torch.empty(B, V + pad)
    buf[0::2, V:] = float("nan")
    buf[1::2, V:] = float("inf")
    buf[:, :V] = rows
    return buf.to(BF if kind == "bf16" else torch.float32).to(DEV), V + pad


def _cfg(do_sample=False, temperature=1.0, top_k=0, top_p=1.0, seed=1, eos=(), pad=0, max_length=1 << 30):
    L, _ = _lib()
    e = list(eos) + [0] * (8 - len(eos))
    return L.SkSampling(seed=seed, top_p=float(top_p), temperature=float(temperature), do_sample=int(do_sample),
                        top_k=int(top_k), n_eos=len(eos), eos=(C.c_int32 * 8)(*e), pad_token_id=pad,
                        max_length=max_length)


def _select(kind, logits, ldl, V, B, cfg, state, ban=None, uniforms=None):
    L, lib = _lib()
    fn = lib.sk_select_next if kind == "bf16" else lib.sk_select_next_f32
    L.check(fn(_p(logits), ldl, V, B, _p(ban), C.byref(cfg), _p(uniforms), C.byref(state.st), L.stream_ptr()))


def _run_case(kind, c: D.SelCase):
    """Two rows of the case (NaN and +inf pads); returns the two selected tokens and the state."""
    from slamkit_b200.generation import ban_bitmask
    V = c.logits.numel()
    logits, ldl = _logits_dev(c.logits[None].repeat(2, 1), kind)
    st = _State(2, 1)
    ban = ban_bitmask(c.banned, V).to(DEV) if c.banned else None
    cfg = _cfg(c.do_sample, c.temperature, c.top_k, c.top_p)
    _select(kind, logits, ldl, V, 2, cfg, st, ban, torch.full((2,), c.u, device=DEV))
    return st.out[:, 0].tolist(), st


@pytest.mark.parametrize("V", V_SHAPES)
@pytest.mark.parametrize("kind", KINDS)
def test_select_constructed_rows(kind, V):
    """Every constructed row of decode_ref at this vocabulary size selects its exact token."""
    failed = []
    for c in D.constructed_cases(V):
        D.check_case(c)
        got, st = _run_case(kind, c)
        if got != [c.want] * 2:
            failed.append((c.name, got, c.want))
        assert st.step.tolist() == [1, 0] and st.pos.tolist() == [1, 1] and st.n_gen.tolist() == [1, 1]
        assert st.tokens.tolist() == got and int((st.out_buf[2:] != -7).sum()) == 0
    assert not failed, failed


@pytest.mark.parametrize("case", ["greedy-signed-zero", "top_k-signed-zero", "top_p-signed-zero"])
@pytest.mark.parametrize("V", [4, 152167])
@pytest.mark.parametrize("kind", KINDS)
def test_select_signed_zeros_are_equal(kind, V, case):
    """-0.0 and +0.0 are one value: greedy takes the lower id, top-k keeps both signs at the k-th value, and top-p
    drops the members of a zero tie group in id order."""
    c = next(x for x in D.signed_zero_cases(V) if x.name == case)
    got, _ = _run_case(kind, c)
    assert got == [c.want] * 2, (got, c.want)


@pytest.mark.parametrize("kind", KINDS)
def test_philox_draws_are_predicted(kind):
    """uniforms = NULL over 256 equal logits: token = floor(u * 256) exactly, with u the CPU Philox draw of (seed,
    step, row), for B = 300 rows (more than one wave of CTAs) over several steps, and a seed with a high word."""
    B, V, steps = 300, 256, 3
    logits, ldl = _logits_dev(torch.full((B, V), 1.5), kind)
    for seed in (1234, 0x9E3779B97F4A7C15):
        st = _State(B, steps)
        cfg = _cfg(True, seed=seed)
        for s in range(steps):
            _select(kind, logits, ldl, V, B, cfg, st)
        got = st.out.cpu().numpy()
        for s in range(steps):
            u = D.philox_uniform(seed, s, range(B))
            want = np.floor(u.astype(np.float64) * 256).astype(np.int64)
            assert np.array_equal(got[:, s], want), (seed, s, int((got[:, s] != want).sum()))


def _state_model(st, toks, k, cfg_eos, max_new, max_length, pad):
    """CPU statement of one call's state update (decode.cu select_next_kernel) at step k."""
    for b in range(len(toks)):
        p = st["pos"][b]
        if st["finished"][b] or p + 1 >= max_length:
            st["finished"][b] = 1
            if k < max_new:
                st["out"][b][k] = pad
            continue
        t = toks[b][k]
        if k < max_new:
            st["out"][b][k] = t
        st["n_gen"][b] += 1
        st["tokens"][b] = t
        st["pos"][b] = p + 1
        if t in cfg_eos:
            st["finished"][b] = 1


@pytest.mark.parametrize("n_eos", [1, 3, 8])
@pytest.mark.parametrize("kind", KINDS)
def test_select_state_over_launches(kind, n_eos):
    """Six launches with max_new = 4 over rows that run on, finish on eos at the first step, reach max_length through
    pos, start finished, and draw an eos at the fourth step; eos ids past n_eos are ignored; a banned id with the
    largest logit and V % 32 != 0."""
    from slamkit_b200.generation import ban_bitmask
    B, V, max_new, calls, ML, pad = 6, 40, 4, 6, 100, 3
    eos = [20 + i for i in range(n_eos)]
    cfg = _cfg(True, eos=eos, pad=pad, max_length=ML)
    for i in range(n_eos, 8):
        cfg.eos[i] = 10                                    # row 0's token, beyond n_eos: never an eos
    rows = torch.full((B, V), D.FILL)
    for b, t in enumerate([10, 11, 20, 12, 14]):
        rows[b, t] = 0.0
    rows[5, 13] = rows[5, eos[-1]] = 0.0                   # two equal tokens: u < 1/2 -> 13, u >= 1/2 -> the eos
    rows[0, 33] = 100.0                                    # banned
    ban = ban_bitmask([33, 39], V).to(DEV)
    logits, ldl = _logits_dev(rows, kind)
    init = dict(pos=[5, 6, 7, 97, 9, 10], finished=[0, 0, 0, 0, 1, 0], n_gen=[0, 0, 0, 0, 3, 0],
                tokens=[100, 101, 102, 103, 104, 105])
    st = _State(B, max_new, **init)
    model = {k: list(v) for k, v in init.items()}
    model["out"] = [[-7] * max_new for _ in range(B)]
    toks = [[10] * calls, [11] * calls, [20] * calls, [12] * calls, [14] * calls,
            [13, 13, 13, eos[-1], eos[-1], eos[-1]]]
    for k in range(calls):
        u = torch.full((B,), 0.25)
        if k >= 3:
            u[5] = 0.75
        _select(kind, logits, ldl, V, B, cfg, st, ban, u.to(DEV))
        _state_model(model, toks, k, set(eos), max_new, ML, pad)
        assert st.step.tolist() == [k + 1, 0], (k, st.step.tolist())
        for name in ("pos", "finished", "n_gen", "tokens"):
            assert getattr(st, name).tolist() == model[name], (k, name, getattr(st, name).tolist(), model[name])
        assert st.out.tolist() == model["out"], (k, st.out.tolist(), model["out"])
        assert int((st.out_buf[B * max_new:] != -7).sum()) == 0, "a write past out[B, max_new]"
    assert model["finished"] == [0, 0, 1, 1, 1, 1] and model["n_gen"] == [6, 6, 1, 2, 3, 4]


# ---------------------------------------------------------------------------------------- C. KV-cache writes
def _qwen_session(B, T_cache):
    from oracle import lm_oracle as O
    from slamkit_b200.lm import B200UnitLM, DecodeSession, LMConfig
    c = O.OracleLMConfig(vocab_size=502, hidden=256, n_layers=2, n_heads=4, n_kv_heads=2, head_dim=64, ffn=256)
    p = O.init_params(c, seed=21, std=0.05)
    m = B200UnitLM(LMConfig(vocab_size=502, hidden=256, n_layers=2, n_heads=4, n_kv_heads=2, head_dim=64, ffn=256),
                   device=DEV, max_batch=B, max_seq=T_cache, trainable=False)
    m.load_hf_state_dict(p)
    return c, p, m, DecodeSession(m, B, T_cache, 4)


def _qwen_layer0_kv(c, p, ids, pos):
    """fp32 layer-0 K (after RoPE) and V of tokens ids [N] at positions pos [N] -> [N, KVH, 64] each."""
    from oracle import lm_oracle as O
    h = "lm.model.layers.0."
    x = p["lm.model.embed_tokens.weight"].float()[ids]
    y = O.rms_norm(x, p[h + "input_layernorm.weight"].float(), c.rms_eps)
    k = y @ p[h + "self_attn.k_proj.weight"].float().t() + p[h + "self_attn.k_proj.bias"].float()
    v = y @ p[h + "self_attn.v_proj.weight"].float().t() + p[h + "self_attn.v_proj.bias"].float()
    k = k.view(-1, c.n_kv_heads, 64)
    cos, sin = O.rope_cos_sin(c, pos[None], torch.float32)
    k = (k * cos[0][:, None]) + (O.rotate_half(k) * sin[0][:, None])
    return k, v.view(-1, c.n_kv_heads, 64)


def _opt_session(B, T_cache):
    from oracle import opt_oracle as O
    from slamkit_b200.lm import B200UnitLM, DecodeSession, OptLMConfig
    c = O.OracleOptConfig(vocab_size=502, hidden=256, n_layers=2, n_heads=4, ffn=512, max_positions=512)
    p = O.init_params(c, seed=22, std=0.05, dtype=torch.float32)
    m = B200UnitLM(OptLMConfig(vocab_size=502, hidden=256, n_layers=2, n_heads=4, ffn=512, max_positions=512,
                               ln_eps=c.ln_eps, tie_embeddings=c.tie_embeddings),
                   device=DEV, max_batch=B, max_seq=T_cache, trainable=False, fp32_inference=True)
    m.load_hf_state_dict(p)
    return c, p, m, DecodeSession(m, B, T_cache, 4)


def _opt_layer0_kv(c, p, ids, pos):
    """fp64 layer-0 K and V of tokens ids [N] at positions pos [N] -> ([N, H, 64] each, their error scale)."""
    pre, h = "lm.model.decoder.", "lm.model.decoder.layers.0."
    d = lambda n: p[n].double()
    x = d(pre + "embed_tokens.weight")[ids] + d(pre + "embed_positions.weight")[pos + 2]
    y = torch.nn.functional.layer_norm(x, (c.hidden,), d(h + "self_attn_layer_norm.weight"),
                                       d(h + "self_attn_layer_norm.bias"), c.ln_eps)
    out, mag = [], []
    for w in ("k_proj", "v_proj"):
        W = d(h + f"self_attn.{w}.weight")
        out.append((y @ W.t() + d(h + f"self_attn.{w}.bias")).view(-1, c.n_heads, 64))
        mag.append((y.abs() @ W.abs().t()).view(-1, c.n_heads, 64))
    return out, mag


def _planes(sess, m, B, T_cache):
    """The cache as [L, 2, B, KVH, T_cache, 64] (the documented layout) of its own dtype."""
    n_layers, kvh = m.config.n_layers, getattr(m.config, "n_kv_heads", None) or m.config.n_heads
    dt = torch.float32 if m.fp32 else BF
    n = n_layers * 2 * B * kvh * T_cache * 64
    assert sess.kv.numel() == n * (4 if m.fp32 else 2)
    return sess.kv.view(dt).view(n_layers, 2, B, kvh, T_cache, 64)


def _bits(x):
    return x.view(torch.int32) if x.dtype == torch.float32 else x.view(torch.int16)


@pytest.mark.parametrize("model", ["qwen2-gqa", "opt-fp32"])
def test_kv_cache_writes(model):
    """Prefill fills slots t < lens[b] of every (layer, K|V, row, kv head) with the layer's K / V and leaves the NaN
    sentinel elsewhere; each decode step changes exactly the slot at pos[b].  Layer 0 against a CPU reference: within
    bf16 rounding (Qwen2, K after RoPE) or fp32-grade with values that are not bf16 values (fp32 OPT)."""
    B, T, T_cache, steps = 3, 40, 70, 3
    c, p, m, sess = (_qwen_session if model == "qwen2-gqa" else _opt_session)(B, T_cache)
    cache = _planes(sess, m, B, T_cache)
    cache.fill_(float("nan"))
    lens = torch.tensor([40, 17, 1])
    g = torch.Generator().manual_seed(5)
    ids = torch.randint(2, 502, (B, T), generator=g)
    ids[torch.arange(T)[None] >= lens[:, None]] = 0

    def ref(tok, pos):
        if model == "qwen2-gqa":
            k, v = _qwen_layer0_kv(c, p, tok, pos)
            return (k, v), (None, None)
        return _opt_layer0_kv(c, p, tok, pos)

    def check_layer0(b, t, tok):
        (k, v), (mk, mv) = ref(torch.tensor([tok]), torch.tensor([t]))
        for which, want, mag in ((0, k[0], mk), (1, v[0], mv)):
            got = cache[0, which, b, :, t].double().cpu()
            if model == "qwen2-gqa":
                tol = 2.0 ** -6 * want.abs().amax(-1, keepdim=True).double() + 2.0 ** -8 * want.abs().double()
            else:
                tol = 2.0 ** -16 * (mag[0] + want.abs())
            err = (got - want.double()).abs()
            assert bool((err <= tol).all()), (model, "KV"[which], b, t, float((err - tol).max()))

    sess.prefill(ids, lens)
    torch.cuda.synchronize()
    snap = cache.clone()
    for b in range(B):
        n = int(lens[b])
        assert bool(cache[:, :, b, :, n:].isnan().all()), f"row {b}: a slot at or past lens was written"
        assert not bool(cache[:, :, b, :, :n].isnan().any()), f"row {b}: a slot below lens was not written"
        for t in range(n):
            check_layer0(b, t, int(ids[b, t]))
    if m.fp32:
        filled = torch.cat([cache[:, :, b, :, :int(lens[b])].reshape(-1) for b in range(B)])
        assert float((A.bf16(filled.cpu()) != filled.cpu()).float().mean()) > 0.9, "the fp32 cache holds bf16 values"
    pos = (lens).to(torch.int32)
    for s in range(steps):
        tok = torch.randint(2, 502, (B,), generator=g)
        sess.step(tok.to(DEV), pos.to(DEV))
        torch.cuda.synchronize()
        changed = (_bits(cache) != _bits(snap)).any(-1)           # [L, 2, B, KVH, T_cache]
        for b in range(B):
            want = torch.zeros(T_cache, dtype=torch.bool)
            want[int(pos[b])] = True
            got = changed[:, :, b].cpu()
            assert bool((got == want).all()), f"step {s} row {b}: changed slots other than pos {int(pos[b])}"
            check_layer0(b, int(pos[b]), int(tok[b]))
        snap = cache.clone()
        pos = pos + 1
