"""Plain-numpy model of the peer-memory all-reduce of csrc/p2p_comm.cu, for the data-parallel conformance tests.

What the kernels claim, restated without a GPU:
  * data: rank r owns the 16-byte chunks [nchunks*r//W, nchunks*(r+1)//W) of the range; for each element it adds the W
    copies in fp32 in rank order, ((g0 + g1) + g2) + ..., rounds once to bf16 (round to nearest even) and stores the
    result into all W buffers.  Nothing outside [off, off + n) is touched.
  * flags: the flag array of one rank is uint32 READY[256][8] | DONE[256][8] | counters[256].
      signal(r, slot, e)     READY[slot][r] = e in the array of every peer p != r
      allreduce(r, slot, e)  spins on READY[slot][p] (p != r) of its own array; then DONE[slot][r] = e in the array of
                             every peer p != r, and its own counter[slot] is back to 0
      wait(r, lo, k, e)      spins on DONE[slot][p] (p != r, slot in [lo, lo + k)) of its own array; writes nothing
  * a flag word is ready for epoch e when (int32)(word - e) >= 0: epochs only grow and may wrap around 2^32.

Buffers are uint16 arrays of bf16 bit patterns; the checkers return lists of readable mismatches (empty = conforming).
"""
from __future__ import annotations

from typing import Callable, Iterable, List, Optional, Sequence, Tuple

import numpy as np

MAX_WORLD = 8
SLOTS = 256
FLAG_WORDS = 2 * SLOTS * MAX_WORLD + SLOTS
CHUNK = 8                      # bf16 elements per 16-byte chunk


# ---------------------------------------------------------------------------------------------------- flag layout
def ready_word(slot: int, rank: int) -> int:
    return slot * MAX_WORLD + rank


def done_word(slot: int, rank: int) -> int:
    return (SLOTS + slot) * MAX_WORLD + rank


def counter_word(slot: int) -> int:
    return 2 * SLOTS * MAX_WORLD + slot


def word_name(i: int) -> str:
    if i < SLOTS * MAX_WORLD:
        return f"READY[{i // MAX_WORLD}][{i % MAX_WORLD}]"
    if i < 2 * SLOTS * MAX_WORLD:
        j = i - SLOTS * MAX_WORLD
        return f"DONE[{j // MAX_WORLD}][{j % MAX_WORLD}]"
    return f"counter[{i - 2 * SLOTS * MAX_WORLD}]"


def ready(flag: int, epoch: int) -> bool:
    """The kernels' wrap-safe spin predicate: (int32)(flag - epoch) >= 0."""
    d = (int(flag) - int(epoch)) & 0xFFFFFFFF
    return d < 0x80000000


def allreduce_spins(rank: int, world: int, slot: int) -> List[int]:
    """The words of rank `rank`'s own flag array that its allreduce launch spins on."""
    return [ready_word(slot, p) for p in range(world) if p != rank]


def wait_spins(rank: int, world: int, slot_lo: int, n_slots: int) -> List[int]:
    """The words of rank `rank`'s own flag array that its wait launch spins on."""
    return [done_word(s, p) for s in range(slot_lo, slot_lo + n_slots) for p in range(world) if p != rank]


def unready(own_flags: np.ndarray, words: Iterable[int], epoch: int) -> List[str]:
    """Names of the words among `words` that are not ready for `epoch` (a launch spinning on them would wait)."""
    return [f"{word_name(i)} = {int(own_flags[i]):#x}" for i in words if not ready(own_flags[i], epoch)]


class FlagModel:
    """The flag arrays of `world` ranks as the protocol must leave them (uint32 [world, FLAG_WORDS])."""

    def __init__(self, world: int, fill: int = 0):
        """`fill`: the READY and DONE words left by earlier rounds (the counters are 0 between launches)"""
        self.world = world
        self.f = np.zeros((world, FLAG_WORDS), dtype=np.uint32)
        self.f[:, :counter_word(0)] = fill

    def signal(self, rank: int, slot: int, epoch: int) -> None:
        for p in range(self.world):
            if p != rank:
                self.f[p, ready_word(slot, rank)] = epoch

    def allreduce(self, rank: int, slot: int, epoch: int) -> None:
        for p in range(self.world):
            if p != rank:
                self.f[p, done_word(slot, rank)] = epoch
        self.f[rank, counter_word(slot)] = 0

    def wait(self, rank: int, slot_lo: int, n_slots: int, epoch: int) -> None:
        pass


def flag_diff(got: np.ndarray, want: np.ndarray, limit: int = 8) -> List[str]:
    """Mismatching words of [world, FLAG_WORDS] flag arrays, named."""
    got, want = np.asarray(got, dtype=np.uint32), np.asarray(want, dtype=np.uint32)
    bad = np.argwhere(got != want)
    return [f"rank {r}: {word_name(int(i))} = {int(got[r, i]):#x}, want {int(want[r, i]):#x}" for r, i in bad[:limit]] + \
        ([f"... {len(bad)} words differ"] if len(bad) > limit else [])


# ---------------------------------------------------------------------------------------------------- data
def bf16_to_f32(bits: np.ndarray) -> np.ndarray:
    return (np.asarray(bits, dtype=np.uint16).astype(np.uint32) << 16).view(np.float32)


def f32_to_bf16(x: np.ndarray) -> np.ndarray:
    """Round fp32 to bf16 bit patterns, to nearest even (subnormals kept, overflow to inf; NaN -> quiet NaN)."""
    u = np.asarray(x, dtype=np.float32).view(np.uint32)
    r = ((u + np.uint32(0x7FFF) + ((u >> 16) & np.uint32(1))) >> 16).astype(np.uint16)
    nan = np.isnan(np.asarray(x, dtype=np.float32))
    r[nan] = ((u[nan] >> 16) | np.uint32(0x40)).astype(np.uint16)
    return r


def shares(nchunks: int, world: int) -> List[Tuple[int, int]]:
    """Chunk range [lo, hi) that rank r reduces: [nchunks*r//W, nchunks*(r+1)//W)."""
    return [(nchunks * r // world, nchunks * (r + 1) // world) for r in range(world)]


def allreduce_ref(copies: Sequence[np.ndarray], off: int, n: int, order: Optional[Sequence[int]] = None) -> np.ndarray:
    """bf16 bits of the reduced range [off, off + n): fp32 sum of the W copies in rank order, rounded once."""
    order = list(range(len(copies))) if order is None else list(order)
    acc = bf16_to_f32(copies[order[0]][off:off + n])
    with np.errstate(over="ignore", invalid="ignore"):            # inf and NaN sums are part of the contract
        for p in order[1:]:
            acc = acc + bf16_to_f32(copies[p][off:off + n])    # float32 + float32: one IEEE round to nearest even
    return f32_to_bf16(acc)


def check_allreduce(outs: Sequence[np.ndarray], ins: Sequence[np.ndarray], off: int, n: int,
                    want: Optional[np.ndarray] = None, limit: int = 4) -> List[str]:
    """Every output buffer holds `allreduce_ref` in [off, off + n) bit for bit (any NaN where the reference is NaN), all
    W buffers are identical there, and every element outside the range (the guard bands) is that buffer's input."""
    return check_ranges(outs, ins, [(off, n)], None if want is None else [want], limit)


def check_ranges(outs: Sequence[np.ndarray], ins: Sequence[np.ndarray], ranges: Sequence[Tuple[int, int]],
                 wants: Optional[Sequence[np.ndarray]] = None, limit: int = 4) -> List[str]:
    """`check_allreduce` for several disjoint ranges (off, n) reduced in one round: each holds its reference, and
    everything outside all of them is unchanged."""
    errs: List[str] = []
    outside = np.ones(len(ins[0]), dtype=bool)
    for k, (off, n) in enumerate(ranges):
        outside[off:off + n] = False
        want = allreduce_ref(ins, off, n) if wants is None else wants[k]
        want_nan = np.isnan(bf16_to_f32(want))
        for r, o in enumerate(outs):
            got = o[off:off + n]
            bad = np.flatnonzero(np.where(want_nan, ~np.isnan(bf16_to_f32(got)), got != want))
            for i in bad[:limit]:
                terms = " + ".join(f"{float(bf16_to_f32(c[off + i:off + i + 1])[0]):.9g}" for c in ins)
                errs.append(f"rank {r}: element {off + i} = {int(got[i]):#06x}, want {int(want[i]):#06x} ({terms})")
            if len(bad) > limit:
                errs.append(f"rank {r}: {len(bad)} elements of [{off}, {off + n}) differ")
            if r and not np.array_equal(got, outs[0][off:off + n]):
                errs.append(f"rank {r}'s range [{off}, {off + n}) differs from rank 0's")
    for r, (o, i) in enumerate(zip(outs, ins)):
        guard = np.flatnonzero(outside & (o != i))
        if len(guard):
            errs.append(f"rank {r}: {len(guard)} elements outside the reduced ranges changed, first {int(guard[0])}")
    return errs


def simulate_allreduce(bufs: List[np.ndarray], rank: int, off: int, n: int,
                       share: Callable[[int, int], List[Tuple[int, int]]] = shares,
                       order: Optional[Sequence[int]] = None) -> None:
    """One rank's reduce kernel on host arrays, in place: its share of the chunks, summed over the CURRENT contents of
    all W buffers (as the emulated ranks on one device run one after the other), stored into all W buffers."""
    lo, hi = share(n // CHUNK, len(bufs))[rank]
    a, b = off + lo * CHUNK, off + hi * CHUNK
    if b > a:
        v = allreduce_ref([x[a:b] for x in bufs], 0, b - a, order)
        for x in bufs:
            x[a:b] = v


def bucket_plan_slots(buckets: Sequence[Tuple[int, int, int]], tail: Tuple[int, int]) -> List[Tuple[int, int]]:
    """The ranges GradSync reduces in one step, in order (slot k = k-th range): buckets, then the tail."""
    return [(lo, hi) for _, lo, hi in buckets] + [tuple(tail)]


def gradient_like(rng: np.random.Generator, n: int, scale: float = 1e-3) -> np.ndarray:
    """bf16 bits of normally distributed values of gradient scale."""
    return f32_to_bf16(rng.standard_normal(n, dtype=np.float32) * np.float32(scale))


def special_columns(world: int, n: int, rng: np.random.Generator) -> List[np.ndarray]:
    """W copies of n elements (n a multiple of 16) whose sums exercise the rounding and IEEE edges, in blocks:
    rank-order cancellations, signed zeros, infinities and inf - inf, NaN, bf16 subnormals and sums that round up to inf
    at the top of the bf16 range; the rest gradient-scale normals."""
    f = [rng.standard_normal(n, dtype=np.float32) * np.float32(1e-3) for _ in range(world)]
    kinds = np.arange(n) % 16
    big = np.float32(2.0 ** 24)
    bmax = bf16_to_f32(np.array([0x7F7F], dtype=np.uint16))[0]
    for e in range(n):
        k = int(kinds[e])
        col = [np.float32(0.0)] * world
        if k in (0, 1, 2) and world >= 3:           # in rank order (2^24 + 1) - 2^24 = 0 and (2^24 + 3) - 2^24 = 4
            i, j, l = sorted(rng.choice(world, 3, replace=False))     # (ties to even); other orders give 1 and 3
            s = np.float32(1.0 if rng.random() < 0.5 else -1.0)
            col[i], col[j], col[l] = s * big, s * np.float32(1.0 if k == 0 else 3.0), -s * big
            if k == 2:                               # the same three terms with the small one first: 4 again
                col[i], col[j], col[l] = s * np.float32(3.0), s * big, -s * big
        elif k == 3:                                 # all -0: -0
            col = [np.float32(-0.0)] * world
        elif k == 4:                                 # +0 and -0 mixed: +0
            col = [np.float32(-0.0)] * world
            col[int(rng.integers(world))] = np.float32(0.0)
        elif k == 5:                                 # x and -x: +0
            x = np.float32(rng.standard_normal())
            col[0], col[world - 1] = x, -x
        elif k == 6:                                 # +inf
            col = [np.float32(rng.standard_normal()) for _ in range(world)]
            col[int(rng.integers(world))] = np.float32(np.inf)
        elif k == 7:                                 # +inf + -inf = NaN
            i, j = rng.choice(world, 2, replace=False)
            col[i], col[j] = np.float32(np.inf), np.float32(-np.inf)
        elif k == 8:                                 # NaN
            col = [np.float32(rng.standard_normal()) for _ in range(world)]
            col[int(rng.integers(world))] = np.float32(np.nan)
        elif k in (9, 10):                           # bf16 subnormals (their fp32 sums are exact, then rounded)
            col = [bf16_to_f32(np.array([int(rng.integers(1, 0x80)) | (0x8000 if rng.random() < 0.3 else 0)],
                                        dtype=np.uint16))[0] for _ in range(world)]
        elif k == 11:                                # bf16 max + 2^119: exactly halfway, rounds (to even) up to inf
            col[0], col[world - 1] = bmax, np.float32(2.0 ** 119)
        elif k == 12:                                # bf16 max + bf16 max: fp32 overflow
            col[0], col[1] = -bmax, -bmax
        elif k == 13:                                # just below the halfway point: stays bf16 max
            col[0], col[world - 1] = bmax, np.float32(2.0 ** 118)
        else:
            continue
        for p in range(world):
            f[p][e] = col[p]
    return [f32_to_bf16(x) for x in f]
