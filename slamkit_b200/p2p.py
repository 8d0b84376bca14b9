"""Peer-memory all-reduce of the flat bf16 gradient buffer for ranks that share one NVSwitch node (csrc/p2p_comm.cu).

Takes the place of the NCCL all-reduce accelerate's DDP wrapper issues for the reference (`SLAMTrainer` under `torchrun`,
HF:trainer.py:1867-2014): every rank maps every peer's gradient buffer and a flag array with CUDA IPC (handles travel
through `torch.distributed.all_gather_object`, once, at construction) and a kernel of 128-thread CTAs with at most 32
registers per thread and no shared memory reduces a bucket in one pass while the backward pass keeps all SMs busy.
Sums are taken in rank order in fp32 and rounded once, so every rank ends up with bit-identical gradients.
"""
from __future__ import annotations

import ctypes as C
import os
import socket
from typing import Dict, List, Optional, Tuple

import torch

from . import _lib as L

MAX_WORLD = 8
MAX_SLOTS = 256

# IPC mappings are kept for the life of the process: the caching allocator reuses the same cudaMalloc block for the
# next model's gradient buffer, and a handle that is already mapped must not be opened twice
_OPENED: Dict[bytes, int] = {}
# One flag array per process (never freed: peers keep it mapped) and one epoch counter shared by all instances -- flag
# values only grow, and every rank constructs / uses its instances in the same (collective) order
_FLAGS: Dict[int, int] = {}        # device index -> device pointer
_EPOCH = [0]


def _open_cached(lib, handle: bytes) -> int:
    if handle not in _OPENED:
        base = C.c_void_p()
        L.check(lib.sk_p2p_open(C.c_char_p(handle), C.byref(base)))
        _OPENED[handle] = int(base.value)
    return _OPENED[handle]


class PeerAllReduce:
    """All ranks of `group` construct this collectively, each with its own flat CUDA bf16 buffer of the same length."""

    def __init__(self, buf: torch.Tensor, group=None):
        import torch.distributed as dist
        assert buf.is_cuda and buf.dtype == torch.bfloat16 and buf.is_contiguous()
        self.dist, self.group = dist, group
        self.rank, self.world = dist.get_rank(group), dist.get_world_size(group)
        if not 2 <= self.world <= MAX_WORLD:
            raise L.SkError(f"peer all-reduce supports 2..{MAX_WORLD} ranks on one node (world = {self.world})")
        self.lib = L.require_cuda()
        self.lib.sk_p2p_flag_bytes.restype = C.c_int64
        self.buf = buf
        self.device = buf.device
        self.epoch = 0
        with torch.cuda.device(self.device):
            # a rank that cannot export its memory still takes part in the exchange (with the reason), so that every rank
            # reaches the same verdict instead of waiting for it in a collective
            try:
                if self.device.index not in _FLAGS:
                    own = C.c_void_p()
                    L.check(self.lib.sk_p2p_alloc(C.c_int64(int(self.lib.sk_p2p_flag_bytes())), C.byref(own)))
                    _FLAGS[self.device.index] = int(own.value)
                self._flags_own = C.c_void_p(_FLAGS[self.device.index])
                mine = {"host": socket.gethostname(), "pid": os.getpid(), "dev": self.device.index, "n": buf.numel(),
                        "buf": self._export(buf.data_ptr()), "flags": self._export(self._flags_own.value)}
            except L.SkError as e:
                mine = {"error": f"rank {self.rank}: {e}"}
            infos: List[Optional[dict]] = [None] * self.world
            dist.all_gather_object(infos, mine, group=group)
            failed = [i["error"] for i in infos if "error" in i]
            if failed:
                raise L.SkError("peer all-reduce: " + "; ".join(failed))
            if len({i["host"] for i in infos}) != 1:
                raise L.SkError("peer all-reduce: ranks span several hosts")
            if len({i["n"] for i in infos}) != 1:
                raise L.SkError("peer all-reduce: gradient buffers differ in length across ranks")
            if len({(i["pid"], i["dev"]) for i in infos}) != self.world:
                raise L.SkError("peer all-reduce: one process per GPU expected")
            bufs, flags = [], []
            for r, info in enumerate(infos):
                if r == self.rank:
                    bufs.append(buf.data_ptr())
                    flags.append(int(self._flags_own.value))
                    continue
                if not torch.cuda.can_device_access_peer(self.device.index, info["dev"]):
                    raise L.SkError(f"peer all-reduce: cuda:{self.device.index} cannot access cuda:{info['dev']}")
                bufs.append(_open_cached(self.lib, info["buf"][0]) + info["buf"][1])
                flags.append(_open_cached(self.lib, info["flags"][0]) + info["flags"][1])
        self._bufs = (C.c_void_p * self.world)(*[C.c_void_p(p) for p in bufs])
        self._flags = (C.c_void_p * self.world)(*[C.c_void_p(p) for p in flags])
        self._err = torch.zeros(1, dtype=torch.int32).pin_memory()
        self._err_ptr = C.c_void_p(self._err.data_ptr())

    def _export(self, ptr: int) -> Tuple[bytes, int]:
        handle = C.create_string_buffer(64)
        off = C.c_int64()
        L.check(self.lib.sk_p2p_export(C.c_void_p(ptr), handle, C.byref(off)))
        return bytes(handle.raw), int(off.value)

    @staticmethod
    def supports(lo: int, hi: int) -> bool:
        return lo % 8 == 0 and (hi - lo) % 8 == 0 and hi > lo

    def begin(self) -> None:
        """Start a new reduction (one per optimiser step): all flag values of this round are `epoch`."""
        self.check()
        _EPOCH[0] += 1
        self.epoch = _EPOCH[0]
        self._slots = 0

    def all_reduce(self, lo: int, hi: int, ctas: int) -> None:
        """Enqueue, on the current stream, the reduction of elements [lo, hi) of the buffer: READY signal + reduce kernel.
        The result is complete on this rank only after `finish()`."""
        assert self._slots < MAX_SLOTS
        s = C.c_void_p(torch.cuda.current_stream().cuda_stream)
        L.check(self.lib.sk_p2p_signal(self._flags, self.rank, self.world, self._slots, C.c_uint32(self.epoch), s))
        L.check(self.lib.sk_p2p_allreduce_bf16(self._bufs, self._flags, self.rank, self.world, C.c_int64(lo), C.c_int64(hi - lo),
                                               self._slots, C.c_uint32(self.epoch), int(ctas), self._err_ptr, s))
        self._slots += 1

    def finish(self) -> None:
        """Enqueue the wait for every peer's share of all ranges reduced since `begin()`."""
        if self._slots:
            s = C.c_void_p(torch.cuda.current_stream().cuda_stream)
            L.check(self.lib.sk_p2p_wait(self._flags, self.rank, self.world, 0, self._slots, C.c_uint32(self.epoch), self._err_ptr, s))

    def check(self) -> None:
        """Raise if a kernel of an earlier reduction gave up waiting for a peer (pinned host flag, no device sync)."""
        if int(self._err[0]) != 0:
            raise L.SkError(f"peer all-reduce: rank {self.rank} timed out waiting for a peer (code {int(self._err[0])}: "
                            "1 = gradients never became ready, 2 = a peer never delivered its share)")

