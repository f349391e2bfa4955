"""Cross-partition exchange (SURVEY.md §8e): records shard by Kafka partition across the GPUs of a
box, and each batch forwards the keyed payloads whose partition (murmur2(correlation_id) % num_partitions,
computed by ck_route_kernel) is owned by another rank.  Reference analogue: the record would simply be produced
to a topic-partition that a different worker process consumes (calfkit/nodes/base.py:82-87 key=correlation_id).

`PeerExchange`: every rank maps its peers' receive buffers (CUDA IPC over NVSwitch) and `ck_exchange_send` plans,
packs and transfers in one pass on the device — a warp per forwarded payload stores it straight into the owner's
region — with no host synchronisation and no library collective (the two barriers of a step are flag words in peer
memory); torch.distributed is used once, for the handle exchange.  `plan_exchange` below is the device-agnostic
tensor statement of the same selection (tested on CPU tensors); `plan_exchange_device` runs the library's plan
kernels, which are pinned to it on the GPU."""
from __future__ import annotations

from dataclasses import dataclass

import torch
import torch.distributed as dist


@dataclass
class ExchangePlan:
    sel: torch.Tensor        # indices into the publish table, ordered by destination rank
    src_off: torch.Tensor    # int64 payload start in the output buffer
    lens: torch.Tensor       # int64 payload length
    dst_off: torch.Tensor    # int64 offset in the send buffer
    counts: torch.Tensor     # int64 [world] payloads per destination
    nbytes: torch.Tensor     # int64 [world] bytes per destination


def plan_exchange(pubs: torch.Tensor, out_off: torch.Tensor, out_len: torch.Tensor, rank: int, world: int) -> ExchangePlan:
    """pubs: int32 [npubs, 8] view of the ck_publish table (payload, topic_id, topic_off, topic_len,
    record, has_key, partition, pad); out_off: int64 [npayloads + 1] (16-byte aligned starts);
    out_len: payload lengths."""
    keyed = (pubs[:, 5] == 1) & (pubs[:, 0] != -1)
    dest = (pubs[:, 6] % world).to(torch.int64)
    sel = torch.nonzero(keyed & (dest != rank)).squeeze(1)
    d_sel = dest[sel]
    order = torch.argsort(d_sel, stable=True)
    sel, d_sel = sel[order], d_sel[order]
    pay = pubs[sel, 0].to(torch.int64)
    src_off = out_off[pay]
    lens = out_len[pay].to(torch.int64)
    dst_off = torch.cumsum(lens, 0) - lens
    counts = torch.bincount(d_sel, minlength=world)
    nbytes = torch.zeros(world, dtype=torch.int64, device=pubs.device).scatter_add_(0, d_sel, lens)
    return ExchangePlan(sel, src_off, lens, dst_off, counts, nbytes)


class _DevArray:
    """raw device pointer -> torch.as_tensor via __cuda_array_interface__ (no copy)"""
    def __init__(self, ptr: int, n: int, typestr: str):
        self.__cuda_array_interface__ = {"data": (ptr, False), "shape": (n,), "typestr": typestr, "version": 3}


def plan_exchange_device(engine, rank: int, world: int, device) -> ExchangePlan:
    """The same plan as plan_exchange(), computed by the library's own kernels (ck_exchange_plan: histogram ->
    scan -> stable scatter -> scan) instead of a dozen tensor ops over the whole publish table; one host
    synchronisation instead of three.  `counts` / `nbytes` are host tensors (payloads / bytes per destination)."""
    import ctypes as C
    src, ln, dst, pub = C.c_void_p(), C.c_void_p(), C.c_void_p(), C.c_void_p()
    counts = torch.zeros(world, dtype=torch.int64)
    nbytes = torch.zeros(world, dtype=torch.int64)
    nsel = C.c_uint32(0)
    engine._check(engine.lib.ck_exchange_plan(engine.h, rank, world, C.byref(src), C.byref(ln), C.byref(dst), C.byref(pub),
                                              counts.data_ptr(), nbytes.data_ptr(), C.byref(nsel)))
    n = nsel.value
    if n == 0:
        z = torch.zeros(0, dtype=torch.int64, device=device)
        return ExchangePlan(z, z, z, z, counts, nbytes)
    as_t = lambda p, ts: torch.as_tensor(_DevArray(p.value, n, ts), device=device)   # noqa: E731
    return ExchangePlan(as_t(pub, "<u4"), as_t(src, "<i8"), as_t(ln, "<i8"), as_t(dst, "<i8"), counts, nbytes)


META_DTYPE = None


def _meta_dtype():
    global META_DTYPE
    if META_DTYPE is None:
        import numpy as np
        META_DTYPE = np.dtype([("len", "<u4"), ("topic_id", "<i4"), ("partition", "<i4"), ("src_pub", "<u4")])
    return META_DTYPE


class PeerExchange:
    """One per engine (lane).  create -> all-gather the 64-byte IPC handles -> connect; then per step `send(step)` after
    the plan.  The receive regions stay in HBM for the next hop; `received()` copies them out for a host-side consumer."""

    def __init__(self, engine, rank: int, world: int, max_fwd: int, data_cap: int, group=None):
        import ctypes as C
        import numpy as np
        self.engine, self.rank, self.world, self.group = engine, rank, world, group
        # every rank addresses its region inside a PEER's buffer with its own geometry: the geometry must be the same
        # everywhere, so the ranks agree on the largest request before anything is allocated
        geo = torch.tensor([max_fwd, data_cap], dtype=torch.int64, device=torch.device("cuda", torch.cuda.current_device()))
        dist.all_reduce(geo, op=dist.ReduceOp.MAX, group=group)
        max_fwd, data_cap = int(geo[0].item()), int(geo[1].item())
        self.max_fwd, self.data_cap = max_fwd, data_cap
        handle = np.zeros(64, dtype=np.uint8)
        engine._check(engine.lib.ck_comm_create(engine.h, rank, world, max_fwd, data_cap, handle.ctypes.data))
        mine = torch.from_numpy(handle).to(torch.device("cuda", torch.cuda.current_device()))
        allh = [torch.empty_like(mine) for _ in range(world)]
        dist.all_gather(allh, mine, group=group)
        handles = np.ascontiguousarray(torch.stack(allh).cpu().numpy())
        engine._check(engine.lib.ck_comm_connect(engine.h, handles.ctypes.data))
        dist.barrier(group=group)
        _ = C

    def send(self, step: int) -> None:
        """forward the foreign-partition payloads of the engine's current plan.  Stream-ordered, asynchronous, no library
        collective: plan -> flag barrier (peers have consumed last step's regions) -> P2P stores -> flag barrier (landed).
        `step` must increase by one on every call of this exchange, on every rank."""
        self.engine._check(self.engine.lib.ck_exchange_send(self.engine.h, step))

    def received(self, step: int | None = None):
        """[(source rank, meta records, payload bytes)] for every other rank; raises if a sender overflowed a region"""
        import numpy as np
        out = []
        for src in range(self.world):
            if src == self.rank:
                continue
            hdr = np.zeros(4, dtype=np.uint64)
            meta = np.zeros(self.max_fwd, dtype=_meta_dtype())
            data = np.empty(self.data_cap, dtype=np.uint8)
            self.engine._check(self.engine.lib.ck_fetch_received(self.engine.h, src, hdr.ctypes.data, meta.ctypes.data, data.ctypes.data, data.nbytes))
            if hdr[2]:
                raise RuntimeError(f"rank {src} could not fit {int(hdr[2])} payloads into its region here: raise max_fwd / data_cap")
            if step is not None and int(hdr[0]) != step:
                raise RuntimeError(f"region of rank {src} holds step {int(hdr[0])}, expected {step}")
            out.append((src, meta[:int(hdr[1])], data[:int(hdr[3])]))
        return out

    def peek(self):
        """[world, 4] uint64 region headers (step, count, overflow, nbytes) — one stream synchronisation"""
        import numpy as np
        hdr = np.zeros((self.world, 4), dtype=np.uint64)
        self.engine._check(self.engine.lib.ck_peek_received(self.engine.h, hdr.ctypes.data))
        return hdr

    def fetch_async(self, src: int, count: int, nbytes: int, meta, data) -> None:
        """queue the copy of region `src` (count meta records, nbytes of payloads) into page-locked arrays; complete after
        the engine's next sync"""
        self.engine._check(self.engine.lib.ck_fetch_received_async(self.engine.h, src, count, nbytes, meta.ctypes.data, data.ctypes.data))

    @staticmethod
    def payloads(meta, data) -> list[bytes]:
        """split a region's data into payloads (16-byte aligned starts)"""
        res, pos = [], 0
        for ln in meta["len"]:
            ln = int(ln)
            res.append(data[pos:pos + ln].tobytes())
            pos += (ln + 15) & ~15
        return res
