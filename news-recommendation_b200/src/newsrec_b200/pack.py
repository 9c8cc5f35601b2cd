"""Host-side batch packing: the reference hands the model slot-major lists of per-slot CPU tensors
(default_collate output, SURVEY.md 8b).  They are stacked once into a reusable pinned buffer, copied to
the device in ONE async H2D transfer and re-ordered there into impression-major blocks."""
from __future__ import annotations

import ctypes as C

import torch


class PackedBatch:
    """Device-resident, impression-major ids of one batch, produced ahead of time on a copy stream
    (`NRMS.prefetch`): `ids` (B*H + B*C, ...), the event that marks the end of its H2D copy and re-ordering."""

    def __init__(self, ids, B, H, C, event):
        self.ids, self.B, self.H, self.C, self.event = ids, B, H, C, event

    def wait(self):
        """Make the current stream wait for the copy and keep the allocator from recycling `ids` under it."""
        cur = torch.cuda.current_stream()
        cur.wait_event(self.event)
        self.ids.record_stream(cur)
        return self.ids


class SlotPacker:
    """Two pinned staging buffers per shape, each guarded by a CUDA event so that a buffer is never
    rewritten by the host while its previous H2D copy is still in flight."""

    def __init__(self):
        self._bufs = {}
        self._inflight = []  # (event, slot tensors): page-locked inputs a pack kernel may still be reading

    def _pack_direct(self, clicked, candidates, dev):
        """One launch that reads every (B, ...) int64 slot tensor straight from page-locked host memory (or device memory)
        and writes the impression-major block -- no host staging copy, no per-slot H2D copies, no device-side stack /
        transpose / cat (nr_pack_slots, csrc/aux.cu).  None when the inputs do not qualify."""
        from . import check, load_library
        tensors = list(clicked) + list(candidates)
        t0 = tensors[0]
        if torch.device(dev).type != "cuda" or t0.dtype != torch.int64 or t0.dim() < 1:
            return None
        for t in tensors:
            if t.dtype != torch.int64 or t.shape != t0.shape or not t.is_contiguous():
                return None  # (page-locked or not is decided by nr_slots_device_readable below: Tensor.is_pinned() costs ~10 us per slot)
        lib = load_library()
        n = len(tensors)
        table = (C.c_void_p * n)(*[t.data_ptr() for t in tensors])
        if not lib.nr_slots_device_readable(table, n):
            return None
        B = t0.shape[0]
        L = 1
        for x in t0.shape[1:]:
            L *= int(x)
        out = torch.empty((B * n,) + tuple(t0.shape[1:]), dtype=torch.int64, device=dev)
        if out.numel():
            stream = torch.cuda.current_stream()
            check(lib.nr_pack_slots(table, len(clicked), len(candidates), B, L, C.c_void_p(out.data_ptr()), C.c_void_p(stream.cuda_stream)),
                  "nr_pack_slots")
            ev = torch.cuda.Event()
            ev.record(stream)
            self._inflight = [(e, ts) for e, ts in self._inflight if not e.query()]
            self._inflight.append((ev, tensors))  # keep the host tensors alive (and out of the pinned pool) until the kernel has read them
        return out, B

    def _stack(self, tensors, dev):
        t0 = tensors[0]
        dev = torch.device(dev)
        if t0.is_cuda or dev.type != "cuda":
            return torch.stack(tensors, dim=0).to(dev)
        if t0.is_pinned() and tensors[-1].is_pinned():
            # the reference's DataLoader runs with pin_memory=True (src/train.py:165-171): every slot tensor is already page
            # locked, so each goes to the device with its own asynchronous copy and is stacked THERE -- the host never touches
            # the payload (the staging copy below is ~0.4 ms of host memcpy per 512-impression batch, serialised with the
            # step by the loss.item() of the training loop)
            return torch.stack([t.to(dev, non_blocking=True) for t in tensors], dim=0)
        shape = (len(tensors),) + tuple(t0.shape)
        key = (shape, t0.dtype)
        slot = self._bufs.get(key)
        if slot is None:
            slot = {"i": 0, "buf": [torch.empty(shape, dtype=t0.dtype).pin_memory() for _ in range(2)],
                    "ev": [None, None]}
            self._bufs[key] = slot
        i = slot["i"]
        slot["i"] = 1 - i
        if slot["ev"][i] is not None:
            slot["ev"][i].synchronize()
        buf = slot["buf"][i]
        torch.stack(tensors, dim=0, out=buf)
        out = buf.to(dev, non_blocking=True)
        ev = torch.cuda.Event()
        ev.record()
        slot["ev"][i] = ev
        return out

    def pack(self, clicked, candidates, field, dev):
        """-> (ids (B*H + B*C, ...), B): rows [0, B*H) are the browsed news impression-major, then the candidates.
        A batch of the device feed (newsrec_b200.feed) already holds that block: it is returned, nothing is launched."""
        from .feed import FeedSlots
        if isinstance(clicked, FeedSlots) and isinstance(candidates, FeedSlots) and clicked.blocks is candidates.blocks:
            return clicked.blocks[field], clicked.B
        H = len(clicked)
        direct = self._pack_direct([x[field] for x in clicked], [x[field] for x in candidates], dev)
        if direct is not None:
            return direct
        slots = self._stack([x[field] for x in clicked] + [x[field] for x in candidates], dev)  # (H+C, B, ...)
        B = slots.shape[1]
        tail = slots.shape[2:]
        a = slots[:H].transpose(0, 1).reshape(B * H, *tail)
        b = slots[H:].transpose(0, 1).reshape(B * (slots.shape[0] - H), *tail)
        return torch.cat((a, b), dim=0), B

    def pack_on_stream(self, clicked, candidates, field, dev, stream):
        """`pack` issued on `stream` (a copy stream): the host-side stacking, the H2D transfer and the device-side
        re-ordering of the NEXT batch overlap the kernels of the current step.  Returns a PackedBatch."""
        with torch.cuda.stream(stream):
            ids, B = self.pack(clicked, candidates, field, dev)
            ev = torch.cuda.Event()
            ev.record(stream)
        return PackedBatch(ids, B, len(clicked), len(candidates), ev)
