"""The model of the peer-memory all-reduce (tests/p2p_ref.py) against itself and against injected defects, on the CPU.

The GPU conformance suite (test_gpu_dp_conformance.py) trusts these checkers to tell a conforming kernel from a wrong one,
so each of them is shown here to pass the protocol as the kernels document it and to flag every defect it is there for:
a sum in another order, one bf16 ulp, a share boundary moved by one chunk, a touched guard element, a READY or DONE word
written to the wrong [slot][rank], and a counter left non-zero."""
import numpy as np
import pytest

import p2p_ref as R


def _copies(world, size, seed, special=False):
    rng = np.random.default_rng(seed)
    if special:
        return R.special_columns(world, size, rng)
    return [R.gradient_like(rng, size) for _ in range(world)]


def _run(ins, off, n, **kw):
    outs = [x.copy() for x in ins]
    for r in range(len(ins)):
        R.simulate_allreduce(outs, r, off, n, **kw)
    return outs


def test_bf16_rounding_is_round_to_nearest_even():
    x = np.array([1.0, 1.0 + 2 ** -8, 1.0 + 3 * 2 ** -8, 1.0 + 2 ** -8 + 2 ** -20, -0.0, np.inf, -np.inf,
                  3.3895313892515355e38, 3.3961775292304286e38, 2.0 ** -133, 2.0 ** -134], dtype=np.float32)
    got = R.f32_to_bf16(x)
    assert [int(v) for v in got] == [0x3F80, 0x3F80, 0x3F82, 0x3F81, 0x8000, 0x7F80, 0xFF80, 0x7F7F, 0x7F80, 0x0001, 0x0000]
    assert np.isnan(R.bf16_to_f32(R.f32_to_bf16(np.array([np.nan], dtype=np.float32))))[0]
    # every bf16 pattern survives the round trip
    allb = np.arange(65536, dtype=np.uint32).astype(np.uint16)
    f = R.bf16_to_f32(allb)
    back = R.f32_to_bf16(f)
    fin = ~np.isnan(f)
    assert np.array_equal(back[fin], allb[fin]) and np.isnan(R.bf16_to_f32(back[~fin])).all()


def test_wrap_safe_ready_predicate():
    assert R.ready(5, 5) and R.ready(6, 5) and not R.ready(4, 5)
    assert R.ready(0, 0xFFFFFFFF) and not R.ready(0xFFFFFFFF, 0) and R.ready(0, 0)       # across the wrap
    assert R.ready(0x7FFFFFFF, 0) and not R.ready(0x80000000, 0)                         # half the ring ahead / behind


@pytest.mark.parametrize("world", range(2, 9))
def test_shares_partition_the_chunks(world):
    for nchunks in (1, world - 1, world, world + 1, 128 * world - 1, 1000003):
        s = R.shares(nchunks, world)
        assert s[0][0] == 0 and s[-1][1] == nchunks
        assert all(s[r][1] == s[r + 1][0] and s[r][0] <= s[r][1] for r in range(world - 1))
        assert max(h - l for l, h in s) == -(-nchunks // world)          # the launcher sizes its grid for this


@pytest.mark.parametrize("world", [2, 3, 5, 8])
@pytest.mark.parametrize("special", [False, True])
def test_protocol_model_conforms_to_its_checker(world, special):
    size, off, n = 4096 + 64, 24, 4096
    ins = _copies(world, size, world, special)
    outs = _run(ins, off, n)
    assert R.check_allreduce(outs, ins, off, n) == []
    # the reference is the rank-order fp32 sum, rounded once
    want = R.bf16_to_f32(ins[0][off:off + n])
    with np.errstate(over="ignore", invalid="ignore"):
        for x in ins[1:]:
            want = want + R.bf16_to_f32(x[off:off + n])
    assert np.array_equal(R.f32_to_bf16(want)[~np.isnan(want)], outs[0][off:off + n][~np.isnan(want)])


def test_special_columns_cover_the_edges():
    ins = _copies(5, 1024, 1, special=True)
    s = R.bf16_to_f32(R.allreduce_ref(ins, 0, 1024))
    assert np.isnan(s).any() and np.isposinf(s).any() and np.isneginf(s).any()
    assert (np.signbit(s) & (s == 0)).any() and (~np.signbit(s) & (s == 0)).any()
    assert ((s != 0) & (np.abs(s) < 2.0 ** -126)).any()                          # subnormal sums
    assert (R.allreduce_ref(ins, 0, 1024) == 0x7F7F).any()                        # bf16 max that does not round up


@pytest.mark.parametrize("world", [3, 4, 7, 8])
def test_checker_flags_a_sum_in_another_order(world):
    size = 2048
    ins = _copies(world, size, 3, special=True)
    rev = list(range(world))[::-1]
    assert not np.array_equal(R.allreduce_ref(ins, 0, size), R.allreduce_ref(ins, 0, size, rev))
    outs = _run(ins, 0, size, order=rev)
    assert any("want" in e for e in R.check_allreduce(outs, ins, 0, size))
    # dropping the last rank's term
    outs = _run(ins, 0, size, order=list(range(world - 1)))
    assert R.check_allreduce(outs, ins, 0, size)


def test_checker_flags_one_ulp_and_a_touched_guard():
    world, size, off, n = 4, 512, 64, 256
    ins = _copies(world, size, 4)
    outs = _run(ins, off, n)
    assert R.check_allreduce(outs, ins, off, n) == []
    for r, e in ((0, off), (3, off + n - 1), (2, off + 77)):
        bad = [x.copy() for x in outs]
        bad[r][e] ^= 1                                                            # one bf16 ulp
        errs = R.check_allreduce(bad, ins, off, n)
        assert any(f"rank {r}: element {e}" in x for x in errs) and any("differs from rank 0" in x for x in errs)
    for e in (0, off - 1, off + n, size - 1):
        bad = [x.copy() for x in outs]
        bad[1][e] ^= 0x8000
        assert any("outside" in x and f"first {e}" in x for x in R.check_allreduce(bad, ins, off, n)), e
    # several ranges of one round
    outs2 = [x.copy() for x in ins]
    for r in range(world):
        R.simulate_allreduce(outs2, r, 0, 32)
        R.simulate_allreduce(outs2, r, 128, 64)
    assert R.check_ranges(outs2, ins, [(0, 32), (128, 64)]) == []
    outs2[2][100] ^= 1
    assert R.check_ranges(outs2, ins, [(0, 32), (128, 64)]) == ["rank 2: 1 elements outside the reduced ranges changed, first 100"]


@pytest.mark.parametrize("world", [2, 3, 8])
@pytest.mark.parametrize("which", ["end+1", "end-1", "start+1", "start-1"])
def test_checker_flags_a_share_boundary_moved_by_one_chunk(world, which):
    size, n = 8 * 300, 8 * 300
    ins = _copies(world, size, 5)
    r = 1 if world > 2 else 0
    edge, d = (1, +1) if which.startswith("end") else (0, +1)
    d = +1 if which.endswith("+1") else -1
    if which.startswith("start") and r == 0:
        r = 1

    def moved(nchunks, w):
        s = [list(x) for x in R.shares(nchunks, w)]
        s[r][edge] += d
        return [tuple(x) for x in s]

    outs = _run(ins, 0, n, share=moved)
    assert R.check_allreduce(outs, ins, 0, n), which


def test_flag_model_protocol_and_defects():
    world, epoch = 4, 7
    m = R.FlagModel(world)
    slots = [0, 5, 255]
    for s in slots:
        for r in range(world):
            m.signal(r, s, epoch)
    for r in range(world):
        for s in slots:
            assert R.unready(m.f[r], R.allreduce_spins(r, world, s), epoch) == []
        # before any allreduce no DONE word is ready: a wait launched now would spin
        assert len(R.unready(m.f[r], R.wait_spins(r, world, 0, 1), epoch)) == world - 1
    for r in range(world):
        for s in slots:
            m.allreduce(r, s, epoch)
    for r in range(world):
        for s in slots:
            assert R.unready(m.f[r], R.wait_spins(r, world, s, 1), epoch) == []
    # exactly READY[slot][r] and DONE[slot][r] in every peer's array, nothing else
    want = np.zeros((world, R.FLAG_WORDS), dtype=np.uint32)
    for p in range(world):
        for r in range(world):
            if r != p:
                for s in slots:
                    want[p, R.ready_word(s, r)] = want[p, R.done_word(s, r)] = epoch
    assert R.flag_diff(m.f, want) == []
    # defects: a READY or DONE word at the wrong [slot][rank], a counter left non-zero
    one = R.FlagModel(world)
    one.signal(1, 5, epoch)
    one.allreduce(3, 255, epoch)
    for p, i, j in ((0, R.ready_word(5, 1), R.ready_word(5, 2)), (2, R.ready_word(5, 1), R.ready_word(6, 1)),
                    (0, R.done_word(255, 3), R.done_word(255, 0)), (1, R.done_word(255, 3), R.done_word(254, 3))):
        bad = one.f.copy()
        bad[p, i], bad[p, j] = 0, epoch
        errs = R.flag_diff(bad, one.f)
        assert any(f"rank {p}: {R.word_name(i)}" in e for e in errs) and any(f"rank {p}: {R.word_name(j)}" in e for e in errs)
    bad = m.f.copy()
    bad[2, R.counter_word(5)] = 1
    assert any("rank 2: counter[5]" in e for e in R.flag_diff(bad, want))
    # the host-side readiness rule catches a missing DONE store before a wait is launched
    bad = m.f.copy()
    bad[1, R.done_word(5, 3)] = epoch - 1
    assert R.unready(bad[1], R.wait_spins(1, world, 5, 1), epoch) == [f"DONE[5][3] = {epoch - 1:#x}"]


def test_flag_model_across_the_epoch_wrap():
    world = 3
    m = R.FlagModel(world, fill=0xFFFFFFFE)
    for epoch in (0xFFFFFFFF, 0):
        for r in range(world):
            assert R.unready(m.f[r], R.allreduce_spins(r, world, 9), epoch)       # the previous round is not ready
        for r in range(world):
            m.signal(r, 9, epoch)
        for r in range(world):
            assert R.unready(m.f[r], R.allreduce_spins(r, world, 9), epoch) == []
            m.allreduce(r, 9, epoch)
        for r in range(world):
            assert R.unready(m.f[r], R.wait_spins(r, world, 9, 1), epoch) == []
