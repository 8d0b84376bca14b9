"""Data-parallel conformance on one GPU: the peer-memory all-reduce (csrc/p2p_comm.cu) against the exact reference of
tests/p2p_ref.py at every world size, and `GradSync`'s overlapped bucket reduction against a run without it.

Part A emulates W ranks on one device: W plain bf16 allocations with sentinel guard bands stand in for the ranks'
gradient buffers and W `sk_p2p_alloc` arrays are their flag arrays.  Every launch goes through the C ABI on one stream in
an order in which no kernel ever has to wait: `sk_p2p_signal` for every rank and slot, then `sk_p2p_allreduce_bf16` of
each rank, then `sk_p2p_wait`.  Each rank reads only its own share and no other rank writes it, so the result is exact.
Before every allreduce or wait launch the flag words it will spin on are read back and must be ready; otherwise the test
fails without launching, so no case can reach a spin, whatever the kernel under test does.

Part B runs `GradSync(overlap=True)` with a faked two-rank world on one GPU: the real side stream, the real backward
events of `sk_lm_forward_backward` / `sk_lm_backward_weighted` and the real bucket loop, with a stand-in collective that
doubles each bucket (a bf16 multiply, or the peer-memory kernel with both ranks on the one buffer: g + g = 2g).  The
gradients must then be exactly twice those of the same run without `GradSync`: a bucket reduced before its layer's
gradients are final would differ."""
import ctypes as C

import numpy as np
import pytest
import torch

import p2p_ref as R

DEV = "cuda:0"
pytestmark = pytest.mark.gpu

CTAS = (1, 7, 148, 1184, 100_000)          # 148 / 1184: GradSync's defaults for overlapped buckets / the tail
# Qwen2.5-0.5B (d 896, ffn 4864, 14 : 2 heads, vocab 502): one layer's tensors, 64-element aligned, and the tail
QWEN_LAYER = 14_912_384
QWEN_TAIL = 896 + 512 * 896
STREAM_WORDS = 128                          # chunks per CTA and grid step of the reduce kernel (P2P_THREADS)


def _lib():
    from slamkit_b200 import _lib as L
    lib = L.require_cuda()
    lib.sk_p2p_flag_bytes.restype = C.c_int64
    lib.sk_launch_count.restype = C.c_int64
    return lib


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


class _DevWords:
    """int32 view of a raw device allocation, for torch (CUDA array interface)."""

    def __init__(self, ptr, n):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": "<i4", "data": (ptr, False), "version": 3,
                                         "strides": None}


class Ranks:
    """W emulated ranks: W flag arrays from sk_p2p_alloc (kept for many rounds: flags are never reset) and the model
    of what they must hold."""

    def __init__(self, world, fill=0):
        self.lib, self.world = _lib(), world
        assert self.lib.sk_p2p_flag_bytes() == R.FLAG_WORDS * 4
        self.ptrs = []
        for _ in range(world):
            p = C.c_void_p()
            assert self.lib.sk_p2p_alloc(C.c_int64(R.FLAG_WORDS * 4), C.byref(p)) == 0, self.lib.sk_last_error()
            self.ptrs.append(p.value)
        self.words = [torch.as_tensor(_DevWords(p, R.FLAG_WORDS), device=DEV) for p in self.ptrs]
        assert all(w.data_ptr() == p for w, p in zip(self.words, self.ptrs))
        if fill:
            for w in self.words:
                w[:R.counter_word(0)].fill_(int(np.uint32(fill).view(np.int32)))
        self.model = R.FlagModel(world, fill)
        assert R.flag_diff(self.host(), self.model.f) == []
        self.flags = (C.c_void_p * world)(*self.ptrs)
        self.err = torch.zeros(1, dtype=torch.int32).pin_memory()
        self.err_ptr = C.c_void_p(self.err.data_ptr())
        self.epoch = fill
        self.next_slot = 0

    def free(self):
        for p in self.ptrs:
            self.lib.sk_p2p_free(C.c_void_p(p))
        self.ptrs = []

    def host(self):
        torch.cuda.synchronize()
        return torch.stack(self.words).cpu().numpy().view(np.uint32)

    def require_ready(self, rank, words, epoch, what):
        """The rule of the suite: a launch that would spin on a word that is not ready is not made."""
        own = self.words[rank].cpu().numpy().view(np.uint32)
        missing = R.unready(own, words, epoch)
        if missing:
            pytest.fail(f"{what} of rank {rank} (epoch {epoch:#x}) would wait for {missing[:6]}; not launched")

    def round(self, bufs, ranges, ctas=148, epoch=None):
        """One reduction: ranges [(slot, off, n)] of the W buffers (torch bf16 tensors), reduced with `ctas` CTAs."""
        lib, W = self.lib, self.world
        self.epoch = (self.epoch + 1) & 0xFFFFFFFF if epoch is None else epoch
        e = self.epoch
        ptrs = (C.c_void_p * W)(*[b.data_ptr() for b in bufs])
        s = _stream()
        for slot, _, _ in ranges:
            for r in range(W):
                assert lib.sk_p2p_signal(self.flags, r, W, slot, C.c_uint32(e), s) == 0, lib.sk_last_error()
                self.model.signal(r, slot, e)
        for r in range(W):
            for slot, off, n in ranges:
                self.require_ready(r, R.allreduce_spins(r, W, slot), e, f"allreduce of slot {slot}")
                assert lib.sk_p2p_allreduce_bf16(ptrs, self.flags, r, W, C.c_int64(off), C.c_int64(n), slot, C.c_uint32(e),
                                                 int(ctas), self.err_ptr, s) == 0, lib.sk_last_error()
                self.model.allreduce(r, slot, e)
        lo = min(sl for sl, _, _ in ranges)
        k = max(sl for sl, _, _ in ranges) + 1 - lo
        for r in range(W):
            self.require_ready(r, R.wait_spins(r, W, lo, k), e, f"wait on slots [{lo}, {lo + k})")
            assert lib.sk_p2p_wait(self.flags, r, W, lo, k, C.c_uint32(e), self.err_ptr, s) == 0, lib.sk_last_error()
        torch.cuda.synchronize()
        assert int(self.err[0]) == 0
        diff = R.flag_diff(self.host(), self.model.f)
        assert diff == [], diff

    def slots(self, k):
        out = [(self.next_slot + i) % R.SLOTS for i in range(k)]
        self.next_slot = (self.next_slot + k) % R.SLOTS
        return out


_RANKS = {}


@pytest.fixture(scope="module")
def ranks():
    def get(W):
        if W not in _RANKS:
            _RANKS[W] = Ranks(W)
        return _RANKS[W]
    yield get
    for rk in _RANKS.values():
        rk.free()
    _RANKS.clear()


def _upload(ins):
    return [torch.from_numpy(x.view(np.int16)).to(DEV).view(torch.bfloat16) for x in ins]


def _download(bufs):
    torch.cuda.synchronize()
    return [b.view(torch.int16).cpu().numpy().view(np.uint16) for b in bufs]


def _inputs(W, size, off, n, seed, special=False):
    """W buffers of `size` elements: sentinel NaN patterns (a different one per rank) around the range [off, off + n)"""
    rng = np.random.default_rng(seed)
    ins = []
    body = R.special_columns(W, n, rng) if special else [R.gradient_like(rng, n) for _ in range(W)]
    for r in range(W):
        x = np.full(size, 0x7FA0 + r, dtype=np.uint16)
        x[off:off + n] = body[r]
        ins.append(x)
    return ins


def _cases(W):
    """(name, off, n, size) per world size: one chunk, W-1 chunks, around the CTA stride, a real tail, a real bucket"""
    s = STREAM_WORDS * W
    return [("one chunk", 8, 8, 24),
            ("W-1 chunks", 0, 8 * (W - 1), 8 * (W - 1) + 8),
            ("stride-1", 8 * 3, 8 * (s - 1), 8 * (s + 5)),
            ("stride+1", 8 * 5, 8 * (s + 1), 8 * (s + 9)),
            ("3 strides-1", 8, 8 * (3 * s - 1), 8 * 3 * s + 8),
            ("3 strides+1", 8 * 7, 8 * (3 * s + 1), 8 * (3 * s + 17)),
            ("qwen tail at the buffer end", 8 * 9, QWEN_TAIL, 8 * 9 + QWEN_TAIL),
            ("two-layer qwen bucket", 0, 2 * QWEN_LAYER, 2 * QWEN_LAYER + 64)]


# ---------------------------------------------------------------------------------------------------- part A
@pytest.mark.parametrize("W", range(2, 9))
def test_allreduce_matches_the_rank_order_reference(ranks, W):
    """<2>, <4>, <8> and the generic <0> instance (3, 5, 6, 7 ranks) over every range shape: bit-exact, identical on all
    ranks, guard bands untouched, whatever the number of CTAs."""
    rk = ranks(W)
    for ci, (name, off, n, size) in enumerate(_cases(W)):
        ins = _inputs(W, size, off, n, seed=100 * W + ci)
        want = R.allreduce_ref(ins, off, n)
        pristine = _upload(ins)
        ctas_list = CTAS if n <= 8 * 4096 else (148, 1184)
        first = None
        for ctas in ctas_list:
            bufs = [b.clone() for b in pristine]
            rk.round(bufs, [(rk.slots(1)[0], off, n)], ctas)
            if first is None:
                errs = R.check_allreduce(_download(bufs), ins, off, n, want)
                assert errs == [], f"W={W} {name} ctas={ctas}: {errs[:6]}"
                first = bufs
            else:
                same = all(torch.equal(a.view(torch.int16), b.view(torch.int16)) for a, b in zip(bufs, first))
                assert same, f"W={W} {name}: the result with {ctas} CTAs differs from the one with {ctas_list[0]}"
        del pristine, first, bufs


@pytest.mark.parametrize("W", range(2, 9))
def test_allreduce_rounding_and_ieee_edges(ranks, W):
    """Cancellations where the fp32 order decides the bf16 result, signed zeros, +-inf and inf - inf, NaN, bf16
    subnormals and sums that round up to inf at the top of the bf16 range."""
    rk = ranks(W)
    off, n = 8 * 3, 8 * (STREAM_WORDS * W + 5) * 2
    ins = _inputs(W, off + n + 16, off, n, seed=W, special=True)
    for ctas in (1, 148):
        bufs = _upload(ins)
        rk.round(bufs, [(rk.slots(1)[0], off, n)], ctas)
        outs = _download(bufs)
        errs = R.check_allreduce(outs, ins, off, n)
        assert errs == [], f"W={W} ctas={ctas}: {errs[:6]}"
        if W >= 3:      # the inputs really tell the rank order apart
            assert not np.array_equal(outs[0][off:off + n], R.allreduce_ref(ins, off, n, list(range(W))[::-1]))
        got = R.bf16_to_f32(outs[0][off:off + n])
        assert np.isnan(got).any() and np.isinf(got).any() and (np.signbit(got) & (got == 0)).any()


def _plan_ranges(layer_sizes, tail, lpb):
    from slamkit_b200.trainer import plan_buckets
    starts = [int(sum(layer_sizes[:l])) for l in range(len(layer_sizes) + 1)]
    buckets, t = plan_buckets(starts, starts[-1] + tail, lpb)
    return R.bucket_plan_slots(buckets, t), starts[-1] + tail


@pytest.mark.parametrize("W", [2, 3, 8])
def test_a_bucket_plan_over_many_slots_then_the_next_epoch(W):
    """GradSync's ranges of a 24-layer layout, one layer per bucket, in slots 231..255 (slot 255 included), then the
    same ranges again at epoch + 1 on the same flag arrays, which are never reset."""
    rk = Ranks(W)
    try:
        ranges, size = _plan_ranges([64 * (300 + 7 * l) for l in range(24)], 896 + 64 * 502, 1)
        assert len(ranges) == 25
        first = R.SLOTS - len(ranges)
        for rnd in range(2):
            ins = _inputs(W, size + 64, 0, size, seed=7 * W + rnd)
            bufs = _upload(ins)
            rk.round(bufs, [(first + k, lo, hi - lo) for k, (lo, hi) in enumerate(ranges)], ctas=148)
            errs = R.check_ranges(_download(bufs), ins, [(lo, hi - lo) for lo, hi in ranges])
            assert errs == [], f"round {rnd}: {errs[:6]}"
        assert rk.epoch == 2
    finally:
        rk.free()


def test_epoch_wrap():
    """A round at epoch 0xFFFFFFFF on flags left at 0xFFFFFFFE by earlier rounds, then one at 0: the wrap-safe compare."""
    W = 5
    rk = Ranks(W, fill=0xFFFFFFFE)
    try:
        off, n = 16, 8 * (STREAM_WORDS * W + 3)
        for epoch in (0xFFFFFFFF, 0):
            ins = _inputs(W, off + n + 8, off, n, seed=epoch & 7)
            bufs = _upload(ins)
            rk.round(bufs, [(255, off, n)], ctas=7, epoch=epoch)
            assert R.check_allreduce(_download(bufs), ins, off, n) == []
        f = rk.host()
        assert f[0, R.ready_word(255, 1)] == 0 and f[1, R.done_word(255, 0)] == 0
    finally:
        rk.free()


def test_trace_hook_does_not_change_results(ranks):
    W = 4
    rk = ranks(W)
    lib = rk.lib
    off, n = 8, 8 * (STREAM_WORDS * W * 2 + 1)
    ins = _inputs(W, off + n + 8, off, n, seed=11)
    want = R.allreduce_ref(ins, off, n)
    stamps = torch.zeros((R.SLOTS + 1) * 4, dtype=torch.int64, device=DEV)
    assert lib.sk_p2p_set_trace(C.c_void_p(stamps.data_ptr())) == 0
    try:
        bufs = _upload(ins)
        slot = rk.slots(1)[0]
        rk.round(bufs, [(slot, off, n)], ctas=148)
    finally:
        assert lib.sk_p2p_set_trace(None) == 0
    assert R.check_allreduce(_download(bufs), ins, off, n, want) == []
    st = stamps.view(R.SLOTS + 1, 4).cpu()
    assert bool((st[slot] > 0).all()) and bool((st[R.SLOTS, :2] > 0).all()), st[slot]
    # switched off: the next round leaves the stamps alone
    before = stamps.clone()
    bufs = _upload(ins)
    rk.round(bufs, [(rk.slots(1)[0], off, n)], ctas=148)
    assert torch.equal(stamps, before)
    assert R.check_allreduce(_download(bufs), ins, off, n, want) == []


def test_refusals_change_nothing(ranks):
    """Each refused call names its reason, launches nothing and leaves buffers and flags as they were."""
    W = 3
    rk = ranks(W)
    lib = rk.lib
    ins = _inputs(W, 64, 8, 32, seed=5)
    bufs = _upload(ins)
    ptrs = (C.c_void_p * W)(*[b.data_ptr() for b in bufs])
    flags_before = rk.host()
    e = C.c_uint32(rk.epoch + 1)
    s = _stream()
    i64 = C.c_int64
    null_flags = (C.c_void_p * W)(rk.ptrs[0], None, rk.ptrs[2])
    odd_bufs = (C.c_void_p * W)(bufs[0].data_ptr(), bufs[1].data_ptr() + 2, bufs[2].data_ptr())

    def ar(rank=0, world=W, off=8, n=32, slot=0, bf=ptrs, fl=rk.flags):
        return lib.sk_p2p_allreduce_bf16(bf, fl, rank, world, i64(off), i64(n), slot, e, 148, rk.err_ptr, s)

    big = (C.c_void_p * 9)(*(list(rk.ptrs) * 3))
    calls = [
        ("world 1", lambda: ar(world=1)),
        ("world 9", lambda: ar(world=9, bf=(C.c_void_p * 9)(*([bufs[0].data_ptr()] * 9)), fl=big)),
        ("world 1", lambda: lib.sk_p2p_signal(rk.flags, 0, 1, 0, e, s)),
        ("world 9", lambda: lib.sk_p2p_wait(big, 0, 9, 0, 1, e, rk.err_ptr, s)),
        ("rank 3", lambda: ar(rank=3)),
        ("rank -1", lambda: ar(rank=-1)),
        ("rank 3", lambda: lib.sk_p2p_signal(rk.flags, 3, W, 0, e, s)),
        ("rank 3", lambda: lib.sk_p2p_wait(rk.flags, 3, W, 0, 1, e, rk.err_ptr, s)),
        ("flag array of rank 1", lambda: ar(fl=null_flags)),
        ("flag array of rank 1", lambda: lib.sk_p2p_signal(null_flags, 0, W, 0, e, s)),
        ("flag array of rank 1", lambda: lib.sk_p2p_wait(null_flags, 0, W, 0, 1, e, rk.err_ptr, s)),
        ("buffer of rank 1", lambda: ar(bf=odd_bufs)),
        ("multiple of 8", lambda: ar(off=4)),
        ("multiple of 8", lambda: ar(n=28)),
        ("bad range", lambda: ar(n=0)),
        ("bad range", lambda: ar(n=-8)),
        ("bad range", lambda: ar(off=-8)),
        ("slot -1", lambda: ar(slot=-1)),
        ("slot 256", lambda: ar(slot=256)),
        ("slot -1", lambda: lib.sk_p2p_signal(rk.flags, 0, W, -1, e, s)),
        ("slot 256", lambda: lib.sk_p2p_signal(rk.flags, 0, W, 256, e, s)),
        ("slots [250, +7)", lambda: lib.sk_p2p_wait(rk.flags, 0, W, 250, 7, e, rk.err_ptr, s)),
        ("slots [256, +1)", lambda: lib.sk_p2p_wait(rk.flags, 0, W, 256, 1, e, rk.err_ptr, s)),
        ("slots [0, +0)", lambda: lib.sk_p2p_wait(rk.flags, 0, W, 0, 0, e, rk.err_ptr, s)),
        ("slots [-1, +2)", lambda: lib.sk_p2p_wait(rk.flags, 0, W, -1, 2, e, rk.err_ptr, s)),
        ("slots [1, +2147483647)", lambda: lib.sk_p2p_wait(rk.flags, 0, W, 1, 2**31 - 1, e, rk.err_ptr, s)),
        ("range too long", lambda: ar(n=8 * 2**31)),
    ]
    for want, call in calls:
        n0 = lib.sk_launch_count()
        rc = call()
        msg = lib.sk_last_error().decode()
        assert rc != 0 and want in msg, (want, rc, msg)
        assert lib.sk_launch_count() == n0, f"{want}: refused but launched"
    torch.cuda.synchronize()
    assert R.flag_diff(rk.host(), flags_before) == []
    assert all(np.array_equal(a, b) for a, b in zip(_download(bufs), ins))
    assert int(rk.err[0]) == 0


# ---------------------------------------------------------------------------------------------------- part B
DECODERS = ["qwen2 tied", "qwen2 untied", "opt", "opt post-ln proj", "neox"]


def _model(kind):
    from slamkit_b200.lm import B200UnitLM, LMConfig, NeoxLMConfig, OptLMConfig, OptPostLnLMConfig
    if kind.startswith("qwen2"):
        cfg = LMConfig(vocab_size=502, hidden=128, n_layers=4, n_heads=2, n_kv_heads=1, head_dim=64, ffn=256,
                       max_positions=256, tie_embeddings=kind == "qwen2 tied")
    elif kind == "opt":
        cfg = OptLMConfig(vocab_size=502, hidden=128, n_layers=4, n_heads=2, ffn=256, max_positions=256)
    elif kind == "opt post-ln proj":
        cfg = OptPostLnLMConfig(vocab_size=502, hidden=128, n_layers=4, n_heads=2, ffn=256, max_positions=256, proj_dim=64)
    else:
        cfg = NeoxLMConfig(vocab_size=502, hidden=128, n_layers=5, n_heads=2, ffn=512, max_positions=256, rot_dims=16)
    return B200UnitLM(cfg, device=DEV, max_batch=4, max_seq=64, seed=1)


def _batches():
    g = torch.Generator().manual_seed(3)
    out = []
    for _ in range(2):
        ids = torch.randint(2, 502, (2, 48), generator=g)
        lab = ids.clone()
        lab[1, 40:] = -100
        out.append((ids, lab))
    return out


def _steps(m):
    from slamkit_b200 import _lib as L
    (i1, l1), (i2, l2) = _batches()
    n_items = float((l1 != -100).sum() + (l2 != -100).sum())

    def one():
        m.forward_backward(i1, l1, num_items_in_batch=n_items)

    def two():
        m.forward_backward(i1, l1, num_items_in_batch=n_items)
        m.forward_backward(i2, l2, num_items_in_batch=n_items, accumulate=True)

    def dpo():
        B, T = i1.shape
        m._ensure(B, T)
        ids, lab = i1.to(DEV), l1.to(DEV)
        row_nll = torch.empty(B * T, device=DEV, dtype=torch.float32)
        row_w = torch.tensor([0.75, -0.5], device=DEV)[:, None].expand(B, T).contiguous().view(-1)
        L.check(m.lib.sk_lm_forward_rows(m._h, L.ptr(ids), L.ptr(lab), None, B, T, L.ptr(row_nll), L.ptr(m.stats),
                                         L.stream_ptr()))
        L.check(m.lib.sk_lm_backward_weighted(m._h, L.ptr(ids), L.ptr(lab), None, B, T, L.ptr(row_w), 0, L.ptr(m.stats),
                                              L.stream_ptr()))

    return {"one micro-batch": one, "two micro-batches": two, "DPO rows pair": dpo}


class _PairAllReduce:
    """Stand-in collective: the peer-memory kernel for ranks 0 and 1, both on the one gradient buffer (g + g = 2g), in
    the slots of one GradSync step; the READY words are published from the host before the step and `wait` is never
    called."""

    def __init__(self, grads, sync, rk):
        self.grads, self.sync, self.rk = grads, sync, rk
        self.bufs = (C.c_void_p * 2)(grads.data_ptr(), grads.data_ptr())
        self.n_slots = len(sync.buckets) + 1

    def publish(self, epoch):
        rk = self.rk
        for slot in range(self.n_slots):
            for r in (0, 1):
                rk.words[r][R.ready_word(slot, 1 - r)] = int(np.uint32(epoch).view(np.int32))
                rk.model.f[r, R.ready_word(slot, 1 - r)] = epoch
        for slot in range(self.n_slots):
            for r in (0, 1):
                rk.require_ready(r, R.allreduce_spins(r, 2, slot), epoch, f"allreduce of slot {slot}")
        self.epoch, self.slot, self.ranges = epoch, 0, []

    def __call__(self, t, group=None):
        assert torch.cuda.current_stream() == self.sync.comm          # enqueued on GradSync's side stream
        lo = (t.data_ptr() - self.grads.data_ptr()) // 2
        assert t.dtype == torch.bfloat16 and t.is_contiguous() and self.slot < self.n_slots
        ctas = self.sync.ctas_tail if lo == self.sync.tail[0] else self.sync.ctas_overlap
        for r in (0, 1):
            assert self.rk.lib.sk_p2p_allreduce_bf16(self.bufs, self.rk.flags, r, 2, C.c_int64(lo), C.c_int64(t.numel()),
                                                     self.slot, C.c_uint32(self.epoch), int(ctas), self.rk.err_ptr,
                                                     _stream()) == 0, self.rk.lib.sk_last_error()
            self.rk.model.allreduce(r, self.slot, self.epoch)
        self.ranges.append((lo, lo + t.numel()))
        self.slot += 1


@pytest.mark.parametrize("standin", ["bf16 multiply", "peer-memory kernel"])
@pytest.mark.parametrize("kind", DECODERS)
def test_overlapped_gradsync_reduces_only_final_gradients(kind, standin, monkeypatch):
    import torch.distributed as dist
    from slamkit_b200.trainer import GradSync
    m = _model(kind)
    steps = _steps(m)
    refs = {}
    for name, fn in steps.items():
        m.grads.zero_()
        fn()
        torch.cuda.synchronize()
        refs[name] = m.grads.clone()
        assert bool((refs[name] != 0).any()) and not bool(refs[name].isnan().any())
    monkeypatch.setattr(dist, "is_initialized", lambda: True)
    monkeypatch.setattr(dist, "get_world_size", lambda group=None: 2)
    monkeypatch.setattr(dist, "get_rank", lambda group=None: 0)
    rk = Ranks(2) if standin == "peer-memory kernel" else None
    try:
        for lpb in (1, 2):
            sync = GradSync(m, layers_per_bucket=lpb, overlap=True, comm="nccl")
            assert sync.world == 2 and sync.overlap and sync.backend == "nccl" and len(sync.events) == m.config.n_layers + 1
            for name, fn in steps.items():
                m.grads.zero_()
                if rk is None:
                    monkeypatch.setattr(dist, "all_reduce", lambda t, group=None: t.mul_(2))
                else:
                    pair = _PairAllReduce(m.grads, sync, rk)
                    rk.epoch += 1
                    pair.publish(rk.epoch)
                    monkeypatch.setattr(dist, "all_reduce", pair)
                torch.cuda.synchronize()
                fn()
                sync.reduce()
                torch.cuda.synchronize()
                want = refs[name] * 2
                bad = (m.grads.view(torch.int16) != want.view(torch.int16)).nonzero().flatten()
                where = sorted({n for n, (o, r, c) in m.tensors.items() for i in bad[:64].tolist() if o <= i < o + r * c})
                assert bad.numel() == 0, (f"{kind}, {name}, {lpb} layer(s) per bucket: {bad.numel()} elements are not "
                                          f"2x the gradient, in {where}; buckets {sync.buckets}, tail {sync.tail}")
                if rk is not None:
                    assert pair.slot == pair.n_slots
                    assert pair.ranges == [(lo, hi) for _, lo, hi in sync.buckets] + [sync.tail]
                    assert int(rk.err[0]) == 0 and R.flag_diff(rk.host(), rk.model.f) == []
            assert m.lib.sk_lm_set_backward_events(m._h, None, 0) == 0      # before this GradSync's events go
    finally:
        if rk is not None:
            rk.free()
