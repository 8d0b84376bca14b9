"""Data-parallel gradient synchronisation and the train-step driver for hot path (ii).

Replaces what HF Trainer + accelerate's DDP wrapper do around `training_step` (HF:trainer.py:1867-2014;
config/training_args/default.yaml:18 `ddp_find_unused_parameters: false`) and `SLAMTrainer.training_step`
(slamkit/trainer/slam_trainer.py:59-71): one process per GPU, each rank computes gradients normalised by the GLOBAL
number of label tokens, then a SUM all-reduce of the flat bf16 gradient buffer over NVLink and the optimiser step.  The
buffer is reduced in buckets; bucket k's reduction is enqueued on a side stream as soon as the backward pass has finished
the layers it covers (CUDA events recorded inside `sk_lm_forward_backward`), so communication overlaps the rest of the
backward pass.  Ranks that share a node reduce with our own kernel over CUDA-IPC peer memory (`p2p.PeerAllReduce`,
csrc/p2p_comm.cu: small-footprint CTAs that co-reside with the backward kernels, rank-order fp32 sums, bit-identical on
every rank); across nodes, or when a peer cannot be mapped, the same buckets go through `torch.distributed.all_reduce`.

Host-side scalars (token counts) never touch the GPU: labels are counted where the collator produced them (host memory)
and summed over ranks through a gloo group, so no step of the loop waits for the device.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Dict, List, Optional, Sequence, Tuple

import torch

from . import _lib as L
from .lm import B200AdamW, B200UnitLM, cosine_with_min_lr


def plan_buckets(layer_start: Sequence[int], n_params: int, layers_per_bucket: int = 4) -> Tuple[List[Tuple[int, int, int]], Tuple[int, int]]:
    """Bucket plan of the flat gradient buffer.  `layer_start[l]` = first element of layer l, `layer_start[n_layers]` =
    first element after the last layer (final norm, then the embedding / lm_head).  Returns (buckets, tail):
    buckets = [(event index, start, end)] from the LAST layers to the first -- the order in which the backward pass
    completes them; bucket (lo..hi) may be reduced once event `lo` (layer lo's gradients final) has fired -- and tail =
    the range that is only complete when the whole backward pass is (final norm + tied embedding).  Every element of
    [0, n_params) is covered exactly once."""
    nl = len(layer_start) - 1
    buckets: List[Tuple[int, int, int]] = []
    hi = nl
    while hi > 0:
        lo = max(0, hi - layers_per_bucket)
        buckets.append((lo, layer_start[lo], layer_start[hi]))
        hi = lo
    return buckets, (layer_start[nl], n_params)


class GradSync:
    """Sum the flat gradient buffer over the data-parallel ranks (bucketed; overlapped with backward on CUDA)."""

    def __init__(self, model, layers_per_bucket: Optional[int] = None, overlap: bool = True, group=None,
                 comm: Optional[str] = None):
        import torch.distributed as dist
        self.dist = dist
        self.model = model
        self.group = group
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        if getattr(model, "master", False) and self.world > 1:
            raise NotImplementedError("data-parallel training of a model with fp32 master weights is not implemented (the "
                                      "gradient all-reduce sums bf16 buffers); train it on one GPU")
        nl = model.config.n_layers
        t = model.tensors
        # the last bucket (lm_head / tables) starts at the final norm, or at the token table of a post-LN OPT, which has none
        self.layer_start = [t[f"layers.{l}.ln1"][0] for l in range(nl)] + [t["final_norm" if "final_norm" in t else "embed"][0]]
        # backend: "p2p" = own kernels over CUDA-IPC peer memory (ranks on one NVSwitch node; p2p.PeerAllReduce), "nccl" =
        # torch.distributed all_reduce.  All ranks must agree, so a rank that cannot map its peers makes everyone use NCCL.
        want = (comm or os.environ.get("SK_DP_COMM", "p2p")).lower()
        assert want in ("p2p", "nccl"), want
        self.p2p = None
        self.backend = "nccl" if self.world > 1 else "none"
        if want == "p2p" and self.world > 1 and model.grads is not None and model.grads.is_cuda:
            why = ""
            try:
                from .p2p import PeerAllReduce
                self.p2p = PeerAllReduce(model.grads, group)
            except (L.SkError, RuntimeError, AssertionError) as e:   # noqa: PERF203
                why = f"{type(e).__name__}: {e}"
            ok = torch.tensor([1 if self.p2p is not None else 0], device=model.device, dtype=torch.int32)
            dist.all_reduce(ok, op=dist.ReduceOp.MIN, group=group)
            if int(ok) == 1:
                self.backend = "p2p"
            else:
                self.p2p = None
                if dist.get_rank(group) == 0 or why:
                    print(f"[slamkit_b200] peer-memory all-reduce unavailable ({why or 'a peer could not map this rank'}); using NCCL", flush=True)
        if layers_per_bucket is None:
            layers_per_bucket = 2 if self.backend == "p2p" else 4
        self.buckets, self.tail = plan_buckets(self.layer_start, model.n_params, layers_per_bucket)
        # CTAs of the reduce kernel: few while the backward pass still owns the SMs, many for the ranges that complete last
        self.ctas_overlap = int(os.environ.get("SK_P2P_CTAS", "148"))
        self.ctas_tail = int(os.environ.get("SK_P2P_TAIL_CTAS", "1184"))
        self.overlap = bool(overlap) and self.world > 1 and model.grads is not None and model.grads.is_cuda
        self.events: List[torch.cuda.Event] = []
        if self.overlap:
            # high priority: the reduce kernel's small CTAs are placed as soon as an SM has room for them
            prio = -1 if os.environ.get("SK_COMM_PRIO", "1") != "0" else 0
            self.comm = torch.cuda.Stream(device=model.device, priority=prio)
            self.events = [torch.cuda.Event() for _ in range(nl + 1)]
            for e in self.events:
                e.record()                      # forces creation of the underlying cudaEvent_t
            arr = (C.c_void_p * (nl + 1))(*[C.c_void_p(e.cuda_event) for e in self.events])
            L.check(model.lib.sk_lm_set_backward_events(model._h, arr, nl + 1))

    def _one(self, lo: int, hi: int, last: bool) -> None:
        """All-reduce elements [lo, hi) of the flat gradient buffer on the current stream."""
        if hi <= lo:
            return
        if self.p2p is not None and self.p2p.supports(lo, hi):
            self.p2p.all_reduce(lo, hi, self.ctas_tail if last else self.ctas_overlap)
        else:
            self.dist.all_reduce(self.model.grads[lo:hi], group=self.group)

    def reduce(self) -> None:
        """Call right after `forward_backward` of the LAST micro-batch of the accumulation window has been enqueued."""
        if self.world == 1:
            return
        if self.p2p is not None:
            self.p2p.begin()
        nb = len(self.buckets)
        if not self.overlap:
            for k, (_, lo, hi) in enumerate(self.buckets):
                self._one(lo, hi, True)
            self._one(self.tail[0], self.tail[1], True)
            if self.p2p is not None:
                self.p2p.finish()
            return
        cur = torch.cuda.current_stream()
        with torch.cuda.stream(self.comm):
            for k, (ev_idx, lo, hi) in enumerate(self.buckets):
                self.comm.wait_event(self.events[ev_idx])
                self._one(lo, hi, k == nb - 1)
            self.comm.wait_stream(cur)
            self._one(self.tail[0], self.tail[1], True)
            if self.p2p is not None:
                self.p2p.finish()
        cur.wait_stream(self.comm)

    def check(self) -> None:
        """Raise if a peer-memory reduction of an earlier step timed out (host flag; no device synchronisation)."""
        if self.p2p is not None:
            self.p2p.check()


class HostReducer:
    """SUM of small host-side vectors over the ranks (token counts).  Uses a gloo group so that no GPU stream -- and
    therefore no pending GPU work -- is involved: the accelerate `gather(...).sum().item()` of the reference
    (slam_trainer.py:70) blocks on the device every micro-step; this one never does."""

    def __init__(self):
        import torch.distributed as dist
        self.dist = dist
        self.world = dist.get_world_size() if dist.is_initialized() else 1
        self.group = None
        if self.world > 1:
            self.group = dist.new_group(backend="gloo") if dist.get_backend() != "gloo" else dist.group.WORLD

    def sum(self, values: Sequence[float]) -> List[float]:
        if self.world == 1:
            return [float(v) for v in values]
        t = torch.tensor(list(values), dtype=torch.float64)
        self.dist.all_reduce(t, group=self.group)
        return t.tolist()


def count_tokens(labels: torch.Tensor, min_token_id_count: Optional[int] = None, max_token_id_count: Optional[int] = None) -> int:
    """`SLAMTrainer.get_num_tokens` (slamkit/trainer/slam_trainer.py:59-66): labels != -100 (UN-shifted), optionally
    restricted to an id range."""
    valid = labels != -100
    if min_token_id_count is not None:
        valid = torch.logical_and(valid, labels >= min_token_id_count)
    if max_token_id_count is not None:
        valid = torch.logical_and(valid, labels <= max_token_id_count)
    return int(valid.sum())


class B200Trainer:
    """Equivalent of `SLAMTrainer.train()`'s inner loop for the unit-LM recipe: gradient accumulation with HF
    `num_items_in_batch` semantics, clip 0.5, AdamW, `cosine_with_min_lr` schedule, and the reference's token counting
    (`num_input_tokens_seen`: global, un-shifted labels, optional id range; slam_trainer.py:59-71)."""

    def __init__(self, model: B200UnitLM, lr: float = 1e-3, min_lr: float = 5e-5, warmup_steps: int = 100,
                 total_steps: int = 17625, max_grad_norm: float = 0.5, weight_decay: float = 0.0,
                 grad_accum: int = 1, overlap_comm: bool = True, min_token_id_count: Optional[int] = None,
                 max_token_id_count: Optional[int] = None, dp_comm: Optional[str] = None):
        self.model = model
        self.opt = B200AdamW(model, lr=lr, weight_decay=weight_decay, max_grad_norm=max_grad_norm)
        self.sync = GradSync(model, overlap=overlap_comm, comm=dp_comm)
        self.host = HostReducer()
        self.lr, self.min_lr, self.warmup, self.total = lr, min_lr, warmup_steps, total_steps
        self.grad_accum = grad_accum
        self.min_token_id_count, self.max_token_id_count = min_token_id_count, max_token_id_count
        self.step_idx = 0
        self.num_input_tokens_seen = 0          # global (all ranks), as TrainerState.num_input_tokens_seen
        self._loss_sum = torch.zeros((), device=model.device, dtype=torch.float32)   # local, since the last reduced_loss()
        self._loss_steps = 0
        self._loss_host = torch.zeros((), dtype=torch.float32).pin_memory() if model.device.type == "cuda" else torch.zeros(())
        self._loss_ready = torch.cuda.Event()

    def last_loss(self) -> float:
        """This rank's share of the most recent step's loss, read from pinned host memory (see train_step)."""
        self._loss_ready.synchronize()
        return float(self._loss_host)

    def train_step(self, micro_batches) -> torch.Tensor:
        """micro_batches: list of dicts with input_ids / labels (/ position_ids), normally host tensors straight from the
        collator.  Returns this rank's share of the step loss (device scalar): sum_local(nll) / global label count --
        the SUM over ranks is the loss (`reduced_loss`)."""
        assert len(micro_batches) == self.grad_accum
        # HF `_get_num_items_in_batch` (HF:trainer.py:2109-2149): labels != -100 (un-shifted, as HF counts them) over the
        # whole accumulation window, summed over ranks (average_tokens_across_devices)
        # (a collator may attach the two counts as "n_items" / "n_tokens"; labels already on the device would otherwise
        #  have to be counted there and read back)
        n_items = sum(int(mb["n_items"]) if "n_items" in mb else int((mb["labels"] != -100).sum()) for mb in micro_batches)
        n_tok = sum(int(mb["n_tokens"]) if "n_tokens" in mb else
                    count_tokens(mb["labels"], self.min_token_id_count, self.max_token_id_count) for mb in micro_batches)
        if "n_items_global" in micro_batches[0]:     # counts already summed over ranks by the caller (fixed-shape synthetic runs)
            n_items, n_tok = float(micro_batches[0]["n_items_global"]), float(micro_batches[0]["n_tokens_global"])
        else:
            n_items, n_tok = self.host.sum([n_items, n_tok])
        self.num_input_tokens_seen += int(n_tok)
        loss = torch.zeros((), device=self.model.device)
        for i, mb in enumerate(micro_batches):
            out = self.model.forward_backward(mb["input_ids"], mb["labels"], mb.get("position_ids"),
                                              num_items_in_batch=max(n_items, 1.0), accumulate=i > 0)
            loss = loss + out.stats[0]
        # this step's loss leaves for pinned host memory as soon as the last backward pass is done (before the all-reduce
        # tail and the optimiser): `last_loss()` waits for that copy only, never for the whole step
        self._loss_host.copy_(loss, non_blocking=True)
        self._loss_ready.record()
        self.sync.reduce()
        lr = cosine_with_min_lr(self.step_idx, base_lr=self.lr, min_lr=self.min_lr, warmup_steps=self.warmup,
                                total_steps=self.total)
        self.opt.step(lr=lr)
        self.step_idx += 1
        self._loss_sum += loss
        self._loss_steps += 1
        return loss

    def reduced_loss(self) -> float:
        """Mean training loss since the previous call, summed over ranks (what HF Trainer logs as `loss`).  The only
        place the loop reads a device value; call it at logging steps."""
        t = self._loss_sum / max(self._loss_steps, 1)
        if self.sync.world > 1:
            t = t.clone()
            self.sync.dist.all_reduce(t)
        self._loss_sum.zero_()
        self._loss_steps = 0
        return float(t)

    # ---- checkpoint state (cli/train.py `cont_training`) --------------------------------------------------------------
    def state_dict(self) -> Dict:
        return {"step_idx": self.step_idx, "num_input_tokens_seen": self.num_input_tokens_seen,
                "opt_step_count": self.opt.step_count, "exp_avg": self.opt.exp_avg, "exp_avg_sq": self.opt.exp_avg_sq}

    def load_state_dict(self, sd: Dict) -> None:
        self.step_idx = int(sd["step_idx"])
        self.num_input_tokens_seen = int(sd["num_input_tokens_seen"])
        self.opt.step_count = int(sd["opt_step_count"])
        self.opt.exp_avg.copy_(sd["exp_avg"])
        self.opt.exp_avg_sq.copy_(sd["exp_avg_sq"])
