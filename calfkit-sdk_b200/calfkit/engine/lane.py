"""Batch arenas and engine lanes: the host side of the Worker's consume -> GPU -> produce pipeline.

Reference seam: FastStream hands `node.handler` ONE decoded record at a time (calfkit/worker/worker.py:45-53).  Here the
unit is a *batch arena* — polled records landed back to back in one page-locked host buffer with an offsets table — that
goes to HBM with one cudaMemcpyAsync; results come back the same way (payload arena + offsets + lengths + the publish
table).  No Python object is created per record anywhere on this path.

  Arena          inbound batch: pinned uint8 bytes + int64 offsets[n+1]
  FetchArena     inbound batch as a Kafka fetch response carries it: the record set (RecordBatch v2 frames) in one pinned
                 buffer; CRC check, gzip / snappy / LZ4 / zstd decode, record split and field decode run on the device (ck_submit_recordbatch)
  PublishBatch   outbound batch: pinned payload arena + the ck_publish table; resolves topic names / keys lazily,
                 per topic, vectorised
  PinnedPool     recycles page-locked buffers (cudaHostAlloc costs milliseconds; the steady state allocates nothing)
  Lane           one BatchEngine (one CUDA stream + its HBM buffers) with its landing buffers
  LanePipeline   K lanes round-robin: step k's H2D + kernels run while step k-(K-1)'s results are copied back, so both
                 PCIe directions and the SMs stay busy (K = 3: the D2H never waits for kernels)
"""
from __future__ import annotations

import ctypes as C
import json
import time
from typing import Callable, Iterator

import numpy as np

from calfkit.engine import _lib
from calfkit.engine._lib import COL, FRAME_DTYPE, PUB_DTYPE, ptr
from calfkit.engine.batch import BatchEngine, FetchBytes, Frames, ToolTemplate, _SpanOffsets, fetch_positions, fetch_txn_mask, txn_partitions
from calfkit.exceptions import EngineError

NO_PAYLOAD = 0xFFFFFFFF


class PinnedBuffer:
    """page-locked host memory as a numpy uint8 array (ck_host_alloc / ck_host_free)"""
    def __init__(self, nbytes: int):
        lib = _lib.load()
        p = C.c_void_p()
        if lib.ck_host_alloc(nbytes, C.byref(p)):
            raise EngineError(lib.ck_last_error(None).decode())
        self._lib, self._ptr, self.nbytes = lib, p, nbytes
        self.array = np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_uint8)), shape=(max(nbytes, 1),))

    def view(self, dtype, count: int, offset: int = 0) -> np.ndarray:
        return self.array[offset:offset + count * np.dtype(dtype).itemsize].view(dtype)

    def free(self) -> None:
        if self._ptr:
            self.array = None
            self._lib.ck_host_free(self._ptr)
            self._ptr = None

    def __del__(self):
        try:
            self.free()
        except Exception:  # noqa: BLE001  (interpreter teardown)
            pass


class PinnedPool:
    def __init__(self):
        self._free: dict[int, list[PinnedBuffer]] = {}
        self.allocated = 0

    def take(self, nbytes: int) -> PinnedBuffer:
        size = 1 << max(12, (nbytes - 1).bit_length())           # power-of-two classes
        lst = self._free.get(size)
        if lst:
            return lst.pop()
        self.allocated += size
        return PinnedBuffer(size)

    def give(self, buf: PinnedBuffer) -> None:
        self._free.setdefault(buf.nbytes, []).append(buf)

    def close(self) -> None:
        for lst in self._free.values():
            for b in lst:
                b.free()
        self._free.clear()


class Arena:
    """a batch of wire records, contiguous: data[offsets[i]:offsets[i+1]] is record i"""
    def __init__(self, data: np.ndarray, offsets: np.ndarray, on_release: Callable[[], None] | None = None):
        assert data.dtype == np.uint8 and offsets.dtype == np.int64
        self.data, self.offsets, self._on_release = data, offsets, on_release

    @property
    def n(self) -> int:
        return len(self.offsets) - 1

    @property
    def nbytes(self) -> int:
        return int(self.offsets[-1] - self.offsets[0]) if len(self.offsets) else 0

    def record(self, i: int) -> bytes:
        return self.data[self.offsets[i]:self.offsets[i + 1]].tobytes()

    def slice(self, a: int, b: int) -> "Arena":
        """records [a, b) as a zero-copy view (offsets rebased to 0)"""
        o = self.offsets[a:b + 1]
        return Arena(self.data[int(o[0]):int(o[-1])], o - o[0])

    def release(self) -> None:
        if self._on_release is not None:
            cb, self._on_release = self._on_release, None
            cb()

    @classmethod
    def pack(cls, records: list[bytes], pool: PinnedPool | None = None) -> "Arena":
        """land a list of record values in one buffer (the low-rate edge: client publishes, host-side hops)"""
        lens = np.fromiter((len(r) for r in records), dtype=np.int64, count=len(records))
        offsets = np.zeros(len(records) + 1, dtype=np.int64)
        np.cumsum(lens, out=offsets[1:])
        total = int(offsets[-1])
        if pool is None:
            return cls(np.frombuffer(b"".join(records), dtype=np.uint8) if total else np.zeros(0, np.uint8), offsets)
        buf = pool.take(total + 64)
        mv = memoryview(buf.array)
        pos = 0
        for r in records:
            mv[pos:pos + len(r)] = r
            pos += len(r)
        return cls(buf.array[:total], offsets, on_release=lambda: pool.give(buf))


class FetchArena:
    """the record set of one fetch response — concatenated RecordBatch v2 frames as they came off the socket — in one
    buffer.  The host only chains through the 12-byte frame prefixes (baseOffset, batchLength) to count frames and records;
    a truncated trailing frame (legal in a fetch response) is carried along and ignored by the device.
    `partitions` (engine.batch.txn_partitions): where each partition's batches start, its AbortedTransactions, from
    which hidden() gives the read_committed mask, and its partition id, from which positions() gives the offsets a
    consumer resumes from; a slice carries its part of the mask and its partitions rebased to its own bytes.  `topic`:
    the topic the broker queued it on (None: not queued)"""
    def __init__(self, data: np.ndarray, on_release: Callable[[], None] | None = None, partitions=None,
                 hidden: np.ndarray | None = None, topic: str | None = None):
        assert data.dtype == np.uint8
        self.data, self._on_release, self._index = data, on_release, None
        self.partitions, self._hidden, self.topic = partitions, hidden, topic
        self._positions = None

    @classmethod
    def of(cls, buf, pool: PinnedPool | None = None, aborted_transactions=None, partitions=None) -> "FetchArena":
        """land a fetch response (bytes / uint8 array) in a page-locked buffer; aborted_transactions [(producer id, first
        offset), ...] of its one partition (partition 0), or partitions [(byte start, [(producer id, first offset), ...],
        partition id), ...] (without the id: the entry's place in the list)"""
        parts = txn_partitions(aborted_transactions, partitions)
        src = np.frombuffer(bytes(buf), dtype=np.uint8) if not isinstance(buf, np.ndarray) else buf
        if pool is None:
            return cls(src, partitions=parts)
        b = pool.take(src.nbytes + 64)
        b.array[:src.nbytes] = src
        return cls(b.array[:src.nbytes], on_release=lambda: pool.give(b), partitions=parts)

    def hidden(self) -> np.ndarray | None:
        """per complete frame, 1 where a read_committed consumer skips it; computed once over the whole fetch, since the
        aborted producers carry from batch to batch across any split.  None: the fetch names no aborted transaction"""
        if self._hidden is None and self.partitions and any(e[1] for e in self.partitions):
            self._hidden = fetch_txn_mask(self.data, self.partitions)
        return self._hidden

    def positions(self) -> dict[int, int]:
        """{partition id: the offset after its last complete batch here} (engine.batch.fetch_positions): what a consumer
        that has handed out this arena's results commits.  {} without a partition model"""
        return self._batch_positions()[0]

    def _batch_positions(self) -> tuple[dict[int, int], np.ndarray, np.ndarray]:
        """(positions(), per complete frame its partition id and the offset after it)"""
        if self._positions is None:
            starts = self.frames()[0][:-1]
            if not self.partitions:
                self._positions = ({}, np.full(len(starts), -1, np.int64), np.full(len(starts), -1, np.int64))
            else:
                pos, nxt = fetch_positions(self.data, self.partitions)
                run = np.searchsorted(np.asarray([e[0] for e in self.partitions], dtype=np.int64), starts, side="right") - 1
                ids = np.asarray([e[2] for e in self.partitions] + [-1], dtype=np.int64)[run]   # run -1: before the first start
                self._positions = (pos, ids, nxt)
        return self._positions

    def without_consumed(self, committed: dict[int, int]) -> "FetchArena | None":
        """this arena without its frames that offsets `committed` ({partition id: committed offset}) already cover, the
        read_committed mask and the topic kept: a zero-copy slice when what stays is one run of frames, else a copy.  None
        when nothing stays.  The release stays with this arena"""
        _pos, ids, nxt = self._batch_positions()
        keep = np.asarray([nx < 0 or nx > committed.get(int(p), -1) for p, nx in zip(ids.tolist(), nxt.tolist())], dtype=bool)
        if not keep.any():
            return None
        k = np.nonzero(keep)[0]
        a, b = int(k[0]), int(k[-1]) + 1
        if b - a == len(k):
            return self.slice_frames(a, b if b < len(keep) else None)
        starts, hidden = self.frames()[0], self.hidden()
        pieces = [self.data[int(starts[i]):int(starts[i + 1])] for i in k]
        parts, at = [], 0
        for i, piece in zip(k.tolist(), pieces):
            if not parts or parts[-1][2] != int(ids[i]):
                parts.append((at, [], int(ids[i])))
            at += piece.nbytes
        return FetchArena(np.concatenate(pieces), partitions=parts, hidden=None if hidden is None else hidden[k], topic=self.topic)

    def frames(self) -> tuple[np.ndarray, np.ndarray]:
        """(starts[k + 1], records[k]) of the k complete frames; starts[k] is where the truncated tail (if any) begins"""
        if self._index is None:
            d, pos, starts, counts = self.data, 0, [0], []
            while pos + 12 <= d.nbytes:
                blen = int.from_bytes(d[pos + 8:pos + 12].tobytes(), "big", signed=True)
                end = pos + 12 + blen
                if blen < 49 or end > d.nbytes:
                    break
                counts.append(int.from_bytes(d[pos + 57:pos + 61].tobytes(), "big"))
                pos = end
                starts.append(pos)
            self._index = (np.asarray(starts, dtype=np.int64), np.asarray(counts, dtype=np.int64))
        return self._index

    @property
    def n(self) -> int:
        return int(self.frames()[1].sum())

    @property
    def nbytes(self) -> int:
        return int(self.data.nbytes)

    def slice_frames(self, a: int, b: int | None) -> "FetchArena":
        """frames [a, b) as a zero-copy view; b None: to the end of the buffer (the truncated tail included)"""
        starts, hidden = self.frames()[0], self.hidden()
        lo, hi = int(starts[a]), (int(starts[b]) if b is not None else self.data.nbytes)
        parts = None
        if self.partitions:                 # rebased to the slice: the partition it starts in at 0, those after it shifted
            first = max((r for r, e in enumerate(self.partitions) if e[0] <= lo), default=0)
            parts = [(max(e[0] - lo, 0), [], e[2]) for e in self.partitions[first:] if e[0] < hi]
        return FetchArena(self.data[lo:hi], hidden=None if hidden is None else hidden[a:b], partitions=parts, topic=self.topic)

    def release(self) -> None:
        if self._on_release is not None:
            cb, self._on_release = self._on_release, None
            cb()


class FetchRecords:
    """the records of a submitted FetchArena as the device split them: record i = its value, where it lies in the frame —
    in the arena, or for a gzip, snappy, LZ4 or zstd batch in its decoded records section (`decoded` = (value offset of decoded[0], decoded))"""
    def __init__(self, arena: FetchArena, val_off: np.ndarray, val_len: np.ndarray, bad: np.ndarray,
                 decoded: tuple[int, np.ndarray] | None = None):
        data = arena.data if decoded is None else FetchBytes(arena.data, decoded[0], decoded[1])
        self.arena, self.data, self.offsets, self.bad = arena, data, _SpanOffsets(val_off, val_len), bad

    @property
    def n(self) -> int:
        return len(self.bad)

    def record(self, i: int) -> bytes:
        return self.data[int(self.offsets[i]):self.offsets.end(i)].tobytes()

    def release(self) -> None:
        self.arena.release()


class PublishBatch:
    """What one plan + encode produced: unique payloads (16-byte aligned starts in `out`) and the publish table that
    references them (ck_publish: payload index, topic id or topic span, key flag, partition).  Everything is a numpy
    view of the lane's landing buffers; nothing per record is materialised until a consumer asks for one topic."""
    def __init__(self, out: np.ndarray, out_off: np.ndarray, out_len: np.ndarray, pubs: np.ndarray, topic_names: dict[int, str],
                 source: Arena | None, key_spans: np.ndarray | None, status: np.ndarray | None, action: np.ndarray | None,
                 on_release: Callable[[], None] | None = None, overlay=None, order: np.ndarray | None = None,
                 key_counts: np.ndarray | None = None, frames: Frames | None = None, frame_topic_ids: frozenset = frozenset()):
        self.out, self.out_off, self.out_len, self.pubs, self.topic_names = out, out_off, out_len, pubs, topic_names
        self.source, self.key_spans, self.status, self.action = source, key_spans, status, action
        self.overlay = overlay          # (bytes, off[n], len[n]) canonical re-emissions: column / topic spans of those records refer to them
        # device-side grouping (ck_group_publishes): `order` = publish indices grouped by key (0 = topic without a registered
        # id, 1 + id = registered topic, 4095 = unused slot), send order kept inside a group; key_counts[4096]
        self.order, self.key_counts = order, key_counts
        self._starts = None if key_counts is None else np.concatenate(([0], np.cumsum(key_counts, dtype=np.int64)))
        # the frame pass (ck_encode_frames): the publishes to the topics frame_topic_ids as produce-ready frames
        self.frames, self.frame_topic_ids = frames, frame_topic_ids
        self._on_release = on_release
        self._refs = 1
        self._live = None

    # -- lifetime: the landing buffers go back to the pool when the last holder lets go
    def retain(self) -> "PublishBatch":
        self._refs += 1
        return self

    def release(self) -> None:
        self._refs -= 1
        if self._refs == 0 and self._on_release is not None:
            cb, self._on_release = self._on_release, None
            cb()

    # -- vectorised views
    @property
    def n_publishes(self) -> int:
        if self.key_counts is not None:
            return int(self.key_counts[:-1].sum())
        return int(self.live_mask().sum())

    def live_mask(self) -> np.ndarray:
        if self._live is None:
            self._live = self.pubs["payload"] != NO_PAYLOAD
        return self._live

    def topic_counts(self) -> dict[int, int]:
        """registered topic id -> publishes (id -1 = topic named by a span of the source record, e.g. a client reply topic)"""
        if self.key_counts is not None:                      # grouped on the device: no scan of the table
            nz = np.nonzero(self.key_counts[:-1])[0]
            return {int(k) - 1: int(self.key_counts[k]) for k in nz}
        ids = np.ascontiguousarray(self.pubs["topic_id"][self.live_mask()])
        if ids.size == 0:
            return {}
        cnt = np.bincount(ids + 1)
        return {int(i) - 1: int(c) for i, c in enumerate(cnt) if c}

    def select(self, topic_id: int) -> np.ndarray:
        """indices into the publish table of the live publishes to `topic_id`, in order"""
        if self.order is not None and -1 <= topic_id < 4093:
            return self.order[int(self._starts[topic_id + 1]):int(self._starts[topic_id + 2])]
        return np.nonzero(self.live_mask() & (self.pubs["topic_id"] == topic_id))[0]

    def payload(self, pub_index: int) -> bytes:
        p = int(self.pubs["payload"][pub_index])
        o = int(self.out_off[p])
        return self.out[o:o + int(self.out_len[p])].tobytes()

    def record_bytes(self, r: int) -> np.ndarray:
        if self.overlay is not None and self.overlay[1][r] >= 0:
            o = int(self.overlay[1][r])
            return self.overlay[0][o:o + int(self.overlay[2][r])]
        o = self.source.offsets
        if isinstance(o, _SpanOffsets):
            return self.source.data[int(o[r]):o.end(r)]
        return self.source.data[int(o[r]):int(o[r + 1])]

    def key(self, pub_index: int) -> bytes | None:
        """key = correlation_id.encode() for keyed publishes (nodes/base.py:86,103,117,134)"""
        if not self.pubs["has_key"][pub_index] or self.key_spans is None or self.source is None:
            return None
        r = int(self.pubs["record"][pub_index])
        o, n = int(self.key_spans[0, r]), int(self.key_spans[1, r])
        raw = self.record_bytes(r)[o:o + n].tobytes()
        return json.loads(b'"' + raw + b'"').encode() if b"\\" in raw else raw

    def topic_name(self, pub_index: int) -> str:
        tid = int(self.pubs["topic_id"][pub_index])
        if tid >= 0:
            return self.topic_names[tid]
        r = int(self.pubs["record"][pub_index])
        o = int(self.pubs["topic_off"][pub_index])
        raw = self.record_bytes(r)[o:o + int(self.pubs["topic_len"][pub_index])].tobytes()
        return json.loads(b'"' + raw + b'"')

    def gather(self, idx: np.ndarray, pool: PinnedPool | None = None) -> Arena:
        """the payloads of publishes `idx` as an inbound Arena (an in-process hop to another node of the same worker)"""
        if len(idx) == 0:
            return Arena(np.zeros(0, np.uint8), np.zeros(1, np.int64))
        pay = self.pubs["payload"][idx]
        starts, lens = self.out_off[pay], self.out_len[pay].astype(np.int64)
        # zero-copy when the payloads lie back to back (consecutive slots, no alignment gaps between them)
        if (np.diff(pay.astype(np.int64)) == 1).all() and (lens[:-1] % 16 == 0).all():
            self.retain()                                   # the view keeps the landing buffers alive
            return Arena(self.out[int(starts[0]):int(starts[-1] + lens[-1])], np.concatenate(([0], np.cumsum(lens))).astype(np.int64),
                         on_release=self.release)
        return Arena.pack([self.out[int(s):int(s + n)].tobytes() for s, n in zip(starts, lens)], pool)

    def iter_records(self, idx: np.ndarray | None = None) -> Iterator[tuple[str, bytes | None, bytes, int]]:
        """(topic, key, payload, pub_index) — the per-record view, for low-rate consumers and tests"""
        if idx is None:
            idx = np.nonzero(self.live_mask())[0]
        for j in idx:
            j = int(j)
            yield self.topic_name(j), self.key(j), self.payload(j), j


_FAST_COLS = np.asarray([COL["STATUS"], COL["ACTION"], COL["CORR_OFF"], COL["CORR_LEN"]], dtype=np.uint32)


def received_batch(meta: np.ndarray, data: np.ndarray, topic_names: dict[int, str], on_release=None) -> "PublishBatch":
    """a region another rank wrote into this rank's receive buffer, as a PublishBatch (payload i = forwarded payload i; its
    topic id and partition travelled with it; the key — the correlation id — is inside the payload and not needed to route)"""
    n = len(meta)
    lens = meta["len"].astype(np.int64)
    off = np.zeros(n + 1, dtype=np.int64)
    np.cumsum((lens + 15) & ~15, out=off[1:])
    pubs = np.zeros(n, dtype=PUB_DTYPE)
    pubs["payload"] = np.arange(n, dtype=np.uint32)
    pubs["topic_id"], pubs["partition"], pubs["record"], pubs["has_key"] = meta["topic_id"], meta["partition"], np.arange(n, dtype=np.uint32), 0
    return PublishBatch(data, off, meta["len"].astype(np.uint32), pubs, topic_names, None, None, None, None, on_release=on_release)


class Lane:
    """one engine + its pinned landing buffers; `submit` is asynchronous (H2D + all kernels queued on the engine's
    stream), `collect` copies the results back and hands them out as a PublishBatch that owns its buffers"""
    def __init__(self, device: int, configure: Callable[[BatchEngine], None], pool: PinnedPool, *, max_records: int,
                 max_in_bytes: int, max_out_bytes: int | None = None, exchange: tuple[int, int] | None = None):
        self.eng = BatchEngine(device, max_records=max_records, max_in_bytes=max_in_bytes, max_out_bytes=max_out_bytes)
        configure(self.eng)
        self.pool, self.max_records, self.max_in = pool, max_records, max_in_bytes
        self.arena: Arena | None = None
        self.busy = self.collecting = False
        self.d2h_bytes = 0
        # one process per GPU, records sharded by Kafka partition: keyed publishes whose partition another rank owns are
        # stored straight into that rank's receive buffer (engine/exchange.py); what arrives here is produced here
        self.px, self.step_no = None, 0
        if exchange is not None and exchange[1] > 1:
            from calfkit.engine.exchange import PeerExchange
            rank, world = exchange
            self.px = PeerExchange(self.eng, rank, world, max_fwd=max_records, data_cap=max_in_bytes + 64 * max_records)

    def submit(self, arena: "Arena | FetchArena", timestamp_ms: int | None = None, sticky: dict[str, int] | None = None) -> None:
        """device-template tool node: decode + plan + encode + route (+ frame pass, + forward to the owning ranks), all
        asynchronous.  A FetchArena goes to the device as it is (ck_submit_recordbatch), with its read_committed mask when
        the engine's isolation level is read_committed.  With frame topics set on the engine,
        their publishes are framed with baseTimestamp timestamp_ms (default: now), and, given `sticky` (topic -> partition),
        the unkeyed ones join that partition of their topic (BatchEngine.set_sticky_partitions)"""
        self.arena, self.busy = arena, True
        eng = self.eng
        if isinstance(arena, FetchArena):
            if eng.read_committed and arena.hidden() is not None:
                eng.set_fetch_hidden(arena.hidden())
            n = C.c_uint32(0)
            eng._check(eng.lib.ck_submit_recordbatch(eng.h, ptr(arena.data), arena.data.nbytes, C.byref(n)))
            eng.n = n.value
        else:
            eng.submit(arena.data, arena.offsets)
        eng.tool_plan()
        if eng.frame_topics:
            if sticky is not None:
                eng.set_sticky_partitions(sticky)
            eng.encode_frames(int(time.time() * 1000) if timestamp_ms is None else timestamp_ms)
        if self.px is not None:
            self.step_no += 1
            self.px.send(self.step_no)

    def start_collect(self) -> None:
        """queue the D2H of this lane's results into fresh landing buffers (waits only for the lane's own kernels to know
        the sizes); the copies run while the caller does host work — finish_collect() waits for them"""
        eng, pool, n = self.eng, self.pool, self.arena.n
        nb, npay, npub = eng.out_size()
        self._b_out = b_out = pool.take(nb + 64)
        self._b_meta = b_meta = pool.take(8 * (npay + 1) + 4 * npay + PUB_DTYPE.itemsize * npub + 16 * n + 4 * npub + 4 * 4096 + 512)
        off = b_meta.view(np.int64, npay + 1)
        ln = b_meta.view(np.uint32, npay, 8 * (npay + 1))
        p0 = (8 * (npay + 1) + 4 * npay + 31) & ~31
        pubs = b_meta.view(PUB_DTYPE, npub, p0)
        r0 = p0 + PUB_DTYPE.itemsize * npub
        rows = b_meta.view(np.uint32, 4 * n, r0).reshape(4, n)
        g0 = (r0 + 16 * n + 31) & ~31
        order = b_meta.view(np.uint32, npub, g0)
        key_counts = b_meta.view(np.uint32, 4096, (g0 + 4 * npub + 31) & ~31)
        eng._check(eng.lib.ck_group_publishes(eng.h))       # per-topic split on the device, before the copies are queued
        eng._check(eng.lib.ck_fetch_output_async(eng.h, ptr(b_out.array), b_out.array.nbytes, ptr(off) if npay else None,
                                                 ptr(ln) if npay else None, ptr(pubs) if npub else None))
        if n:
            eng._check(eng.lib.ck_fetch_cols_async(eng.h, ptr(_FAST_COLS), 4, ptr(rows)))
        eng._check(eng.lib.ck_fetch_groups(eng.h, ptr(order), ptr(key_counts), 0))
        self._views = (b_out.array[:nb], off, ln, pubs, rows, order, key_counts)
        # a fetch response: where every record's value lies in it, and whether its frame failed the check
        # (and, when it held gzip, snappy, LZ4 or zstd batches, their decoded records sections, which those offsets point into)
        self._b_rb = self._rb = self._b_dec = self._dec = None
        if isinstance(self.arena, FetchArena):
            self._b_rb = b_rb = pool.take(16 * n + 64)
            val_off, val_len, bad = b_rb.view(np.int64, n), b_rb.view(np.uint32, n, 8 * n), b_rb.view(np.uint32, n, 12 * n)
            if n:
                eng._check(eng.lib.ck_fetch_rb_index_async(eng.h, ptr(val_off), ptr(val_len), None, None, None, None, ptr(bad)))
            self._rb = (val_off, val_len, bad)
            base, nbytes = C.c_uint64(0), C.c_uint64(0)
            eng._check(eng.lib.ck_fetch_rb_decoded_async(eng.h, None, 0, C.byref(base), C.byref(nbytes)))
            if nbytes.value:
                self._b_dec = b_dec = pool.take(nbytes.value + 64)
                eng._check(eng.lib.ck_fetch_rb_decoded_async(eng.h, ptr(b_dec.array), b_dec.nbytes, None, None))
                self._dec = (base.value, b_dec.array[:nbytes.value])
        # the frame pass's frames and table (the stream was just synchronised for the sizes above)
        self._b_fr = self._fr = None
        if eng.frame_topics:
            nf, fb = eng.frames_size()
            self._b_fr = (pool.take(fb + 64), pool.take(FRAME_DTYPE.itemsize * nf + 64))
            data, table = self._b_fr[0].array[:fb], self._b_fr[1].view(FRAME_DTYPE, nf)
            eng._check(eng.lib.ck_fetch_frames_async(eng.h, ptr(self._b_fr[1].array), nf, ptr(self._b_fr[0].array), self._b_fr[0].nbytes))
            self._fr = Frames(table, data, eng.topic_names)
        # what the other ranks forwarded to this one during this step: the regions are complete (the stream was just
        # synchronised for the sizes, the exchange's second barrier is behind it); their copies ride along with the results
        self._recv = []
        if self.px is not None:
            from calfkit.engine.exchange import _meta_dtype
            hdr = self.px.peek()
            for src in range(self.px.world):
                step, count, overflow, rbytes = (int(x) for x in hdr[src])
                if src == self.px.rank:
                    continue
                if overflow:
                    raise EngineError(f"rank {src} could not fit {overflow} payloads into its region here: raise max_fwd / data_cap")
                if step != self.step_no:
                    raise EngineError(f"region of rank {src} holds step {step}, expected {self.step_no}")
                if count == 0:
                    continue
                b_m, b_d = pool.take(16 * count), pool.take(rbytes + 64)
                meta, data = b_m.view(_meta_dtype(), count), b_d.array[:rbytes]
                self.px.fetch_async(src, count, rbytes, meta, data)
                self._recv.append((meta, data, b_m, b_d))
        self.collecting = True

    def finish_collect(self) -> PublishBatch:
        eng, pool = self.eng, self.pool
        eng.sync()
        out, off, ln, pubs, rows, order, key_counts = self._views
        b_out, b_meta = self._b_out, self._b_meta
        self.d2h_bytes = int(out.nbytes + off.nbytes + ln.nbytes + pubs.nbytes + rows.nbytes + order.nbytes + key_counts.nbytes)
        frames, b_fr, b_rb = self._fr, self._b_fr, self._b_rb
        if frames is not None:
            self.d2h_bytes += int(frames.data.nbytes + frames.table.nbytes)
        if self._rb is not None:
            self.d2h_bytes += int(sum(a.nbytes for a in self._rb))
        if self._dec is not None:
            self.d2h_bytes += int(self._dec[1].nbytes)
        listed = C.c_uint32(0)
        eng._check(eng.lib.ck_canon_stats(eng.h, C.byref(listed), None))
        overlay = eng.overlay() if listed.value else None       # rare: some records arrived in a non-canonical spelling
        arena, self.arena, self.busy, self.collecting = self.arena, None, False, False
        source = FetchRecords(arena, *self._rb, decoded=self._dec) if self._rb is not None else arena
        b_rb = (b_rb,) if b_rb is not None else ()
        if self._b_dec is not None:
            b_rb += (self._b_dec,)
        self._views = self._b_out = self._b_meta = self._b_fr = self._fr = self._b_rb = self._rb = self._b_dec = self._dec = None
        self.received = []
        for meta, data, b_m, b_d in self._recv:
            self.received.append(received_batch(meta, data, eng.topic_names, on_release=lambda b_m=b_m, b_d=b_d: (pool.give(b_m), pool.give(b_d))))
        self._recv = []

        def done():
            pool.give(b_out)
            pool.give(b_meta)
            for b in (b_fr or ()) + b_rb:
                pool.give(b)
            arena.release()
        return PublishBatch(out, off, ln, pubs, eng.topic_names, source, rows[2:4], rows[0], rows[1], on_release=done, overlay=overlay,
                            order=order, key_counts=key_counts, frames=frames,
                            frame_topic_ids=frozenset(eng.topic_ids[t] for t in eng.frame_topics))

    def collect(self) -> PublishBatch:
        if not self.collecting:
            self.start_collect()
        return self.finish_collect()

    def close(self) -> None:
        self.eng.close()


class LanePipeline:
    """K lanes round-robin.  push(arena) queues step k and returns the results of step k-(K-1) once the pipe is full;
    drain() flushes.  With K = 3 a lane's D2H starts a full step after its kernels were queued: both PCIe directions and
    the SMs overlap (measured: bench.py e2e)."""
    def __init__(self, device: int, configure: Callable[[BatchEngine], None], *, lanes: int = 3, max_records: int, max_in_bytes: int,
                 max_out_bytes: int | None = None, pool: PinnedPool | None = None, exchange: tuple[int, int] | None = None):
        self.pool = pool or PinnedPool()
        self.lanes = [Lane(device, configure, self.pool, max_records=max_records, max_in_bytes=max_in_bytes, max_out_bytes=max_out_bytes,
                           exchange=exchange) for _ in range(lanes)]
        self.received: list[PublishBatch] = []           # batches other ranks forwarded here, collected with the last results
        self._k = 0
        self._inflight: list[Lane] = []

    def push(self, arena: "Arena | FetchArena", timestamp_ms: int | None = None, sticky: dict[str, int] | None = None) -> PublishBatch | None:
        """queue one step; returns the results of an older step once the pipe is full.  Order of work per call:
        (1) H2D + kernels of the new step are queued, (2) the copy-back that was started by the previous call is
        awaited and handed out, (3) the copy-back of the next-oldest step is started — it runs while the caller
        produces the batch just returned and while the new step computes."""
        lane = next(l for l in self.lanes if not l.busy)    # invariant: at most K-1 lanes busy between calls
        lane.submit(arena, timestamp_ms, sticky)
        self._inflight.append(lane)
        ready = None
        if self._inflight[0].collecting:
            lane0 = self._inflight.pop(0)
            ready = lane0.finish_collect()
            self.received += lane0.received
        if len(self._inflight) >= len(self.lanes) - 1 and not self._inflight[0].collecting:
            self._inflight[0].start_collect()
        return ready

    def drain(self) -> Iterator[PublishBatch]:
        while self._inflight:
            lane0 = self._inflight.pop(0)
            batch = lane0.collect()
            self.received += lane0.received
            yield batch

    def take_received(self) -> list[PublishBatch]:
        out, self.received = self.received, []
        return out

    @property
    def pending(self) -> int:
        return len(self._inflight)

    @property
    def pending_records(self) -> int:
        """records of the steps still in flight (lockstep ticks of an idle rank carry empty batches)"""
        return sum(l.arena.n for l in self._inflight if l.arena is not None)

    def launch_count(self) -> int:
        return sum(l.eng.launch_count() for l in self.lanes)

    def close(self) -> None:
        for l in self.lanes:
            l.px = None
        for l in self.lanes:
            l.close()
        self.pool.close()


__all__ = ["Arena", "FetchArena", "FetchRecords", "PublishBatch", "PinnedPool", "PinnedBuffer", "Lane", "LanePipeline", "ToolTemplate"]
