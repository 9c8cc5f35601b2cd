"""Data-parallel plumbing: impressions shard by batch across ranks (one process per GPU); the only
collective on the path is the NCCL all-reduce of a flat fp32 gradient buffer per step (SURVEY.md 8e).

`FlatGradients` makes every parameter's `.grad` a view into one contiguous buffer, so the all-reduce
needs no packing copies and autograd accumulates straight into the communication buffer.  The largest
parameter (the word-embedding table: 97 % of the buffer) sits FIRST in the buffer: its gradient is
complete as soon as the news encoder's scatter GEMM has run, which the backward reports through a CUDA
event attached to that gradient view (ops.GRAD_READY_ATTR), and its all-reduce is issued from a side stream that waits for that event --
it runs under the weight-gradient GEMM that follows.  The rest of the buffer (a few hundred kB) is reduced
after the backward.  The 1/world of the mean is folded into the reduction (ReduceOp.AVG): no extra pass
over the 88 MB buffer.
"""
from __future__ import annotations

import datetime
import os

import torch
import torch.distributed as dist


def init_from_env(backend: str | None = None):
    """torchrun-style rendezvous (RANK / LOCAL_RANK / WORLD_SIZE / MASTER_ADDR / MASTER_PORT).
    Returns (rank, world_size, local_rank).  Single-process runs need no process group."""
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    if world > 1 and not dist.is_initialized():
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        os.environ.setdefault("MASTER_PORT", "29511")
        if backend is None:
            backend = "nccl" if torch.cuda.is_available() else "gloo"
        if backend == "nccl":
            torch.cuda.set_device(local)
        # generous timeout: rank 0 may spend a long validation pass (the reference's evaluate(): a Python loop over up to
        # 200k impressions) between two collectives while the other ranks already wait in the next one
        dist.init_process_group(backend=backend, rank=rank, world_size=world, timeout=datetime.timedelta(hours=6))
    return rank, world, local


def shard_range(n_items: int, rank: int, world: int):
    """Contiguous shard [lo, hi) of `n_items` impressions for `rank` (sizes differ by at most one)."""
    base, rem = divmod(n_items, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


class FlatGradients:
    def __init__(self, params, world: int = 1):
        self.params = [p for p in params if p.requires_grad]
        seen, uniq = set(), []
        for p in self.params:  # tied parameters (NAML's shared embeddings) appear once
            if id(p) not in seen:
                seen.add(id(p))
                uniq.append(p)
        # the largest parameter first: its slice of the buffer is the early all-reduce
        big = max(range(len(uniq)), key=lambda i: uniq[i].numel())
        self.params = [uniq[big]] + uniq[:big] + uniq[big + 1:]
        self.world = world
        pad4 = lambda n: (n + 3) // 4 * 4  # every view starts on a 16-byte boundary (the kernels reduce with 16-byte vectors)
        total = sum(pad4(p.numel()) for p in self.params)
        dev = self.params[0].device
        self.flat = torch.zeros(total, dtype=torch.float32, device=dev)
        off = 0
        for p in self.params:
            n = p.numel()
            p.grad = self.flat[off:off + n].view_as(p)
            setattr(p.grad, "_newsrec_direct_grad", True)  # opt-in: the kernels accumulate straight into this view (ops.grad_sink)
            off += pad4(n)
        self.big_numel = pad4(self.params[0].numel())
        self._side = None
        self._hook = None
        if world > 1 and dev.type == "cuda" and dist.is_initialized() and dist.get_backend() == "nccl":
            from . import ops
            self._side = torch.cuda.Stream(device=dev)
            event = torch.cuda.Event()
            event.record()  # materialises the cudaEvent_t handle the backward records into
            # on this buffer's own view: the backward that writes it records THIS event, whichever other FlatGradients exist
            self._hook = {"event": event, "recorded": False}
            setattr(self.params[0].grad, ops.GRAD_READY_ATTR, self._hook)
            # NCCL's channel CTAs need SMs while the weight-gradient GEMM runs (it would otherwise hold all of them)
            from . import load_library
            load_library().nr_reserve_sms_for_comm(int(os.environ.get("NEWSREC_COMM_SMS", "32")))
        # opt-in (NEWSREC_COMM_BF16=1): the embedding-gradient slice crosses the wire as bf16 (half the all-reduce time; every
        # rank's contribution is rounded to bf16 before the average -- not bit-compatible with the fp32 reduction, hence off by default)
        self._wire = None
        if self._side is not None and os.environ.get("NEWSREC_COMM_BF16") == "1":
            self._wire = torch.empty(self.big_numel, dtype=torch.bfloat16, device=dev)

    def zero(self):
        self.flat.zero_()

    def all_reduce_mean(self):
        """Mean over ranks: rank-local losses are batch means, so this equals the gradient of the mean loss over the
        global batch (reference semantics of a single process on the whole batch)."""
        if self.world <= 1:
            return
        if self._side is None:  # gloo / CPU: one reduction, explicit scaling (gloo has no AVG)
            dist.all_reduce(self.flat, op=dist.ReduceOp.SUM)
            self.flat.mul_(1.0 / self.world)
            return
        main = torch.cuda.current_stream()
        if self._hook["recorded"]:
            # early slice: starts when the event the backward recorded behind the scatter GEMM fires
            self._side.wait_event(self._hook["event"])
            with torch.cuda.stream(self._side):
                if self._wire is not None:
                    self._wire.copy_(self.flat[:self.big_numel])
                    dist.all_reduce(self._wire, op=dist.ReduceOp.AVG)
                    self.flat[:self.big_numel].copy_(self._wire)
                else:
                    dist.all_reduce(self.flat[:self.big_numel], op=dist.ReduceOp.AVG)
            if self.big_numel < self.flat.numel():
                dist.all_reduce(self.flat[self.big_numel:], op=dist.ReduceOp.AVG)
            main.wait_stream(self._side)
            self._hook["recorded"] = False
        else:
            dist.all_reduce(self.flat, op=dist.ReduceOp.AVG)
