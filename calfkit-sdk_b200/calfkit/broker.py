"""In-process broker with the surface calfkit calls on FastStream's KafkaBroker
(SURVEY.md §8b "downward" face): subscriber(*topics, group_id=, max_workers=, **kw),
publisher(topic, **kw)(handler), await publish(msg, topic=, correlation_id=, key=), start/stop and a
truthy `_connection` once started (reference calfkit/worker/worker.py:45-53, calfkit/nodes/base.py:82-87,
calfkit/client/base.py:137-147,164).

Kafka itself is out of scope (SURVEY.md §2: third-party transport; no client library or broker in
the image), so topics are in-memory queues of wire records; a real Kafka source/sink would implement
the same methods the Worker uses.  Records are bytes end to end: nothing here parses JSON.

Two granularities share the topics:
  * per-record (`Record`): the client's publishes, host-side nodes (LLM boundary, Python tools), tests;
  * per-batch: `produce_arena(topic, arena)` enqueues a whole page-locked batch (what a Kafka fetch lands, what a load
    generator pre-builds) and `produce_publishes(batch)` takes the payload arena + publish table a GPU lane produced and
    splits it per topic with vectorised index selections — no Python object per record.  `poll_arena` hands a consumer the
    next batch for its topics, bounded by records AND bytes (a batch never exceeds what an engine was sized for), zero-copy
    when the entry is contiguous.
Kafka's own granularity — record batches — at both ends:
  * `produce_fetch(topic, buf)` enqueues a fetch response's record set (engine.lane.FetchArena); `poll_arena` (device-template
    nodes) and `poll_fetch` (Agent nodes, Python-tool nodes, the client's replies) split such entries only at frame boundaries,
    and the device checks, splits and decodes them.  Transactions (KIP-98): a record set
    holds the batches of one or more partitions back to back, `partitions=[(byte start, aborted, partition id), ...]` in
    byte order, where `aborted` is that partition's AbortedTransactions from the fetch response, [(producer id, first
    offset), ...] (without an id, an entry is the partition of its place in the list); `aborted_transactions=aborted`
    alone is the one-partition case, partition 0.  Control batches are skipped at every isolation level;
    a consumer at isolation_level="read_committed" also skips the aborted transactions' batches.  The mask of those is
    computed once over the whole entry (an aborted producer stays aborted across a split) and sliced with it;
  * `frame_sink(topic, fn)`: `fn(topic, partition_or_None, frame, n_records)` once per produce-ready RecordBatch v2 frame.
    A lane's frames are handed out as they are; per-record Records produced to such a topic are collected and framed by
    the engine's record form at `flush_frames` (the Worker calls it once per step and installs the `framer`).  There is no
    CPU encoder: without a framer, flushing them fails loudly.  `MemoryBroker(compression_type="lz4")` (the keyword a
    FastStream KafkaBroker takes) makes every frame an LZ4-compressed batch, compressed on the device; other codecs are
    refused by the Worker when frame sinks are registered.  `compression_level=` (Kafka's compression.lz4.level, 1 .. 17)
    trades compressor time for smaller LZ4 frames: 1 and 2 build the default frames, 3 and up search deeper per level.
Idempotent and transactional produce (KIP-98), as aiokafka and the Java producer apply `enable_idempotence=True` and
`transactional_id="..."` (which implies idempotence): `init_producer_id` hands out producer ids and epochs; every frame
carries its producer's id and epoch, and the broker writes its baseSequence when it hands the frame to its sink, from one
counter per (producer id, topic, partition): contiguous per partition in the order frames reach the sinks, whichever
engine built them.  A topic's unkeyed publishes go to one sticky partition per frame pass (`next_sticky`), advanced round
robin, so every frame has a partition.  With a transactional id, each Worker.run tick is one transaction: data frames
carry attributes bit 4, and when the tick ends every (topic, partition) that received frames in it gets a COMMIT marker
(a control batch) through the same sink, or an ABORT marker when the tick raised.
Exactly-once consume-transform-produce (KIP-447, Kafka Streams' processing.guarantee="exactly_once_v2"): committed
offsets are kept per (consumer group, topic, partition).  `send_offsets_to_transaction(offsets, group_id)` adds a group's
consumed positions to the open transaction; they become `committed(...)` at commit_transaction and are dropped at
abort_transaction.  A fetch slice that `poll_fetch` / `poll_arena` hand out with a `group_id` (only inside an open
transaction) is kept, its buffer not released, until a commit covers every partition it holds (FetchArena.positions);
an abort puts the slices no commit covers back at the head of their topic's queue, in poll order, without the batches
already covered, and with their read_committed mask, so that the next poll delivers them again.  Fetches are the only
input with offsets: a poll with a group_id refuses Records and arenas, before it takes any.
Publishes to topics nobody subscribes to are counted and dropped when they arrive batch-wise (a long-running worker must
not grow without bound); per-record publishes are kept (tests read such topics afterwards).
Limitation (documented, not hidden): one shared queue per topic — consumer GROUPS are not modelled (two subscriptions to
one topic in different groups split the records instead of each seeing all of them, unlike Kafka).
"""
from __future__ import annotations

import asyncio
from collections import defaultdict, deque
from dataclasses import dataclass
from typing import Any, Awaitable, Callable

import numpy as np


@dataclass
class Record:
    """One Kafka record as calfkit sees it: value bytes, optional key, the two headers FastStream sets."""
    topic: str
    value: bytes
    key: bytes | None = None
    correlation_id: str | None = None
    content_type: str = "application/json"


class Subscription:
    def __init__(self, topics: tuple[str, ...], group_id: str | None, max_workers: int, kwargs: dict[str, Any]):
        self.topics, self.group_id, self.max_workers, self.kwargs = topics, group_id, max_workers, kwargs
        self.handler: Callable[..., Awaitable[Any]] | None = None
        self.node = None                     # set by Worker for node subscriptions (batch path)
        self.publish_topic: str | None = None

    def __call__(self, handler):
        self.handler = handler
        self.node = getattr(handler, "__self__", None)
        return _HandlerRef(self, handler)


class _HandlerRef:
    """what `subscriber(handler)` returns; `publisher(topic)(ref)` attaches the return-value topic"""
    def __init__(self, sub: Subscription, handler):
        self.sub, self.handler = sub, handler

    def __call__(self, *a, **k):
        return self.handler(*a, **k)


class MemoryBroker:
    def __init__(self, *servers: Any, middlewares: list | None = None, num_partitions: int = 8, **kwargs: Any):
        self.servers, self.kwargs = servers, kwargs
        # the codec of the frames handed to frame sinks, as KafkaBroker(compression_type=...) takes it: None or "lz4"
        # (compressed on the device); the Worker refuses any other codec when frame sinks are registered
        self.compression_type: str | None = kwargs.get("compression_type")
        # compression.lz4.level (KIP-390) as KafkaBroker(compression_level=...) would take it: 1 .. 17, None the default;
        # the Worker checks it and applies it to LZ4 frames only, as Kafka ignores it for other codecs
        self.compression_level: int | None = kwargs.get("compression_level")
        self.num_partitions = num_partitions       # partitions per topic (Kafka's default partitioner: murmur2(key) % partitions)
        # idempotent / transactional produce (frame sinks): KafkaBroker(enable_idempotence=True) / (transactional_id="...")
        self.transactional_id: str | None = kwargs.get("transactional_id")
        self.enable_idempotence: bool = bool(kwargs.get("enable_idempotence")) or self.transactional_id is not None
        self._next_pid = 0
        self._txn_producers: dict[str, tuple[int, int]] = {}          # transactional id -> (producer id, epoch)
        self._seq: dict[tuple[int, str, int], int] = {}               # (producer id, topic, partition) -> next baseSequence
        self._sticky: dict[str, int] = {}                             # topic -> sticky partition of the next pass
        self._txn: dict[tuple[str, int], tuple[int, int]] | None = None   # open transaction: (topic, partition) -> (pid, epoch)
        self._committed: dict[tuple[str, str, int], int] = {}          # (group, topic, partition) -> committed offset
        self._txn_offsets: dict[tuple[str, str, int], int] = {}        # the offsets sent to the open transaction
        self._kept: dict[str, list] = defaultdict(list)               # topic -> [(group, FetchArena, release)] in poll order
        self._connection: Any = None
        self.queues: dict[str, deque[Record]] = defaultdict(deque)
        self.arenas: dict[str, deque] = defaultdict(deque)            # topic -> deque[Arena]
        self.frags: dict[str, deque] = defaultdict(deque)             # topic -> deque[(PublishBatch, pub indices)]
        self.sinks: dict[str, Any] = {}                               # topic -> callable(PublishBatch, pub indices)
        self.frame_sinks: dict[str, Any] = {}                         # topic -> callable(topic, partition | None, frame, n_records)
        self.framer: Callable[[str, list[Record]], Any] | None = None  # records -> engine Frames (the Worker installs it)
        self._frame_pending: dict[str, list[Record]] = defaultdict(list)
        self.subscriptions: list[Subscription] = []
        self.subscribed: set[str] = set()
        self.produced: int = 0
        self.dropped_unsubscribed: int = 0

    # --- FastStream-shaped registration ---------------------------------------------------------
    def subscriber(self, *topics: str, group_id: str | None = None, max_workers: int = 1, **kwargs: Any) -> Subscription:
        sub = Subscription(tuple(topics), group_id, max_workers, kwargs)
        self.subscriptions.append(sub)
        self.subscribed.update(topics)
        return sub

    def sink(self, topic: str, fn) -> None:
        """bulk consumer of one topic: fn(batch, pub_indices) is called from produce_publishes with the lane's batch (a
        Kafka producer would encode record batches from it; benchmarks count bytes).  The batch is valid during the call."""
        self.sinks[topic] = fn

    def frame_sink(self, topic: str, fn) -> None:
        """Kafka-shaped consumer of one topic: fn(topic, partition or None, frame, n_records) is called once per
        RecordBatch v2 frame built on the device (partition None: unkeyed records, the producer client picks one).  The
        frame (uint8 array) is valid during the call, like `sink`'s batch.  With compression_type="lz4" every frame is an
        LZ4-compressed batch (attributes 3) as Kafka clients decode it; the table's records count stays the uncompressed
        one.  With enable_idempotence or a transactional_id the partition is always an int (unkeyed records went to their
        topic's sticky partition), the frame carries producerId, producerEpoch and its baseSequence, and under a
        transactional_id fn also receives each partition's COMMIT / ABORT marker: a control batch (attributes 0x30) of one
        record, n_records 1."""
        self.frame_sinks[topic] = fn

    def publisher(self, topic: str, **kwargs: Any):
        def attach(ref: _HandlerRef):
            ref.sub.publish_topic = topic
            return ref
        return attach

    async def start(self) -> None:
        self._connection = object()

    async def stop(self) -> None:
        self._connection = None

    # --- produce side ------------------------------------------------------------------------------
    async def publish(self, msg: Any, topic: str, correlation_id: str | None = None, key: bytes | None = None, **kw: Any) -> None:
        if isinstance(msg, (bytes, bytearray, memoryview)):
            value = bytes(msg)
        elif hasattr(msg, "model_dump_json"):
            value = msg.model_dump_json().encode()       # object -> wire bytes at the user-API edge only
        else:
            raise TypeError(f"cannot publish {type(msg)!r}")
        self.produce(Record(topic, value, key, correlation_id))

    def produce(self, rec: Record) -> None:
        if rec.topic in self.frame_sinks:                 # framed with the others of this step (flush_frames), never queued
            self._frame_pending[rec.topic].append(rec)
        else:
            self.queues[rec.topic].append(rec)
        self.produced += 1

    def discard_frames(self) -> None:
        """drop the Records collected for frame-sink topics and not framed yet (the outputs of a step being undone)"""
        self._frame_pending.clear()

    def flush_frames(self) -> None:
        """frame the per-record Records collected for frame-sink topics (engine record form) and hand the frames out"""
        for topic in list(self._frame_pending):
            recs = self._frame_pending.pop(topic)
            if not recs:
                continue
            if self.framer is None:
                from calfkit.exceptions import EngineError
                raise EngineError(f"{len(recs)} records for frame-sink topic {topic!r} and no engine to frame them (Worker installs one)")
            for frames in self.framer(topic, recs):
                try:
                    self._hand_frames(frames)
                finally:
                    frames.release()

    def _hand_frames(self, frames) -> None:
        if not self.enable_idempotence:
            for topic, part, frame, n in frames:
                self.frame_sinks[topic](topic, part, frame, n)
            return
        from calfkit.engine.batch import patch_base_sequence
        from calfkit.exceptions import EngineError
        for topic, part, frame, n in frames:
            pid, epoch = int.from_bytes(frame[43:51].tobytes(), "big", signed=True), int.from_bytes(frame[51:53].tobytes(), "big", signed=True)
            if pid < 0 or part is None:
                raise EngineError(f"frame for {topic!r} without a producer id or a partition: the engine that built it was not set up for idempotence")
            key = (pid, topic, part)
            seq = self._seq.get(key, 0)
            patch_base_sequence(frame, seq)
            self._seq[key] = (seq + n) & 0x7FFFFFFF               # DefaultRecordBatch.incrementSequence: wraps to 0
            if frame[22] & 0x10:
                if self._txn is None:
                    raise EngineError(f"transactional frame for {topic!r} outside a transaction (begin_transaction first)")
                self._txn.setdefault((topic, part), (pid, epoch))
            self.frame_sinks[topic](topic, part, frame, n)

    # --- idempotent / transactional produce -------------------------------------------------------------
    def init_producer_id(self, transactional_id: str | None = None) -> tuple[int, int]:
        """(producer id, epoch) of a new producer (Kafka's InitProducerId): a fresh id for an idempotent producer; a
        transactional id keeps its producer id and each call bumps its epoch, fencing the previous holder.  The sequences
        of a re-initialised producer start again at 0"""
        if transactional_id is not None and transactional_id in self._txn_producers:
            pid, epoch = self._txn_producers[transactional_id]
            epoch += 1
            if epoch > 0x7FFF:                                # the epoch is an i16: exhausted, a fresh id as Kafka gives one
                pid, epoch = self._next_pid, 0
                self._next_pid += 1
            self._seq = {k: v for k, v in self._seq.items() if k[0] != pid}
        else:
            pid, epoch = self._next_pid, 0
            self._next_pid += 1
        if transactional_id is not None:
            self._txn_producers[transactional_id] = (pid, epoch)
        return pid, epoch

    def next_sticky(self, topics) -> dict[str, int]:
        """the sticky partition of each topic's unkeyed publishes for one frame pass; each call moves every one of these
        topics to its next partition, round robin (Kafka's uniform sticky partitioner, switching per pass)"""
        out = {}
        for t in topics:
            p = self._sticky.get(t, 0)
            out[t] = p
            self._sticky[t] = (p + 1) % max(self.num_partitions, 1)
        return out

    def begin_transaction(self) -> None:
        from calfkit.exceptions import EngineError
        if self._txn is not None:
            raise EngineError("a transaction is already open")
        self._txn = {}

    def commit_transaction(self) -> None:
        """end the open transaction: a COMMIT marker to every (topic, partition) that received its frames"""
        self._end_transaction(True)

    def abort_transaction(self) -> None:
        """end the open transaction: an ABORT marker to every (topic, partition) that received its frames"""
        self._end_transaction(False)

    def _end_transaction(self, commit: bool) -> None:
        import time
        from calfkit.engine.batch import control_batch
        from calfkit.exceptions import EngineError
        if self._txn is None:
            raise EngineError("no transaction is open")
        touched, self._txn = self._txn, None
        offsets, self._txn_offsets = self._txn_offsets, {}
        ts = int(time.time() * 1000)
        for (topic, part), (pid, epoch) in touched.items():
            self.frame_sinks[topic](topic, part, control_batch(pid, epoch, commit, ts), 1)
        if commit:
            self._committed.update(offsets)
            self._release_covered()
        else:
            self._rewind()

    # --- exactly-once: consumed offsets in the transaction ----------------------------------------------
    def send_offsets_to_transaction(self, offsets: dict[tuple[str, int], int], group_id: str) -> None:
        """consumer group `group_id`'s next offsets {(topic, partition): offset} (Kafka's sendOffsetsToTransaction): they
        are committed with the open transaction, or dropped when it aborts"""
        from calfkit.exceptions import EngineError
        if self._txn is None:
            raise EngineError("send_offsets_to_transaction outside a transaction (begin_transaction first)")
        for (topic, part), off in offsets.items():
            self._txn_offsets[(group_id, topic, int(part))] = int(off)

    def committed(self, group_id: str, topic: str, partition: int) -> int | None:
        """the offset consumer group `group_id` resumes (topic, partition) from, None when it never committed one"""
        return self._committed.get((group_id, topic, int(partition)))

    def _check_keep(self, group_id: str | None, topics) -> None:
        """a poll for a group's offsets is refused, before anything is taken, outside a transaction"""
        if group_id is not None and self._txn is None:
            from calfkit.exceptions import EngineError
            raise EngineError(f"a poll of {tuple(topics)} for group {group_id!r}'s offsets outside a transaction (begin_transaction first)")

    def _keep(self, topic: str, group_id: str, fetch):
        """hold `fetch`, polled for `group_id`, until a commit covers it; its consumer's release no longer frees the buffer"""
        self._kept[topic].append((group_id, fetch, fetch._on_release))
        fetch._on_release = None
        return fetch

    def _covered(self, group_id: str, topic: str, fetch) -> bool:
        return all(self._committed.get((group_id, topic, p), -1) >= nxt for p, nxt in fetch.positions().items())

    def _release_covered(self) -> None:
        """release the kept slices the committed offsets cover, from the oldest on: a fetch's buffer is released by its last
        slice, so none is released before a slice polled earlier"""
        for topic, kept in self._kept.items():
            while kept and self._covered(kept[0][0], topic, kept[0][1]):
                _g, _f, release = kept.pop(0)
                if release is not None:
                    release()

    def _rewind(self) -> None:
        """after an abort: the kept slices back at the head of their topics' queues, in poll order, less what is committed"""
        for topic, kept in self._kept.items():
            back, releases = [], []
            for group, fetch, release in kept:
                rest = fetch.without_consumed({p: o for (g, t, p), o in self._committed.items() if g == group and t == topic})
                if rest is None:
                    releases.append(release)
                else:
                    rest._on_release = release
                    back.append(rest)
            if back:                                        # a dropped slice's buffer may hold a later slice: freed with the last one
                releases.append(back[-1]._on_release)
                back[-1]._on_release = _chain(releases)
            else:
                _chain(releases)()
            self.arenas[topic].extendleft(reversed(back))
        self._kept.clear()

    def produce_batch(self, records: list[Record]) -> None:
        for r in records:
            self.produce(r)

    def produce_fetch(self, topic: str, buf, aborted_transactions=None, partitions=None) -> None:
        """a fetch response's record set for one topic (bytes, a uint8 array or an engine.lane.FetchArena), with the
        AbortedTransactions of its one partition, [(producer id, first offset), ...], or its partitions (see above)"""
        from calfkit.engine.lane import FetchArena
        if isinstance(buf, FetchArena) and (aborted_transactions is not None or partitions is not None):
            from calfkit.exceptions import EngineError
            raise EngineError("a FetchArena carries its own partitions: give them to FetchArena.of")
        fa = buf if isinstance(buf, FetchArena) else FetchArena.of(buf, aborted_transactions=aborted_transactions, partitions=partitions)
        fa.topic = topic
        self.arenas[topic].append(fa)
        self.produced += fa.n

    def produce_arena(self, topic: str, arena) -> None:
        """a whole batch of records for one topic (engine.lane.Arena)"""
        self.arenas[topic].append(arena)
        self.produced += arena.n

    def produce_publishes(self, batch) -> None:
        """split what a GPU lane produced (engine.lane.PublishBatch) over the topics, by index selection; the topics the lane
        framed go to their frame sinks as frames"""
        framed = set()
        if batch.frames is not None:
            framed = {batch.topic_names[i] for i in batch.frame_topic_ids}
            self._hand_frames(batch.frames)
        for tid, cnt in batch.topic_counts().items():
            self.produced += cnt
            if tid >= 0 and batch.topic_names.get(tid) in framed:
                continue
            if tid < 0 and batch.source is None:
                # forwarded by another rank without a registered topic id: the name stayed with the source record there.
                # Workers of one deployment register each other's topics (Worker(route_topics=...)): loud, not silent
                import logging
                logging.getLogger(__name__).error("%d forwarded publishes to a topic this worker has no id for: register it via route_topics", cnt)
                self.dropped_unsubscribed += cnt
                continue
            if tid < 0:
                # topics the engine has no id for (another worker's node, a client's private reply topic): the kernel left
                # the FNV-1a of the name in `pad`, so they are grouped vectorised and the name is decoded once per group
                idx = batch.select(-1)
                hashes = np.ascontiguousarray(batch.pubs["pad"][idx])
                for hv in np.unique(hashes):
                    sub = idx[hashes == hv]
                    tl = batch.pubs["topic_len"][sub]
                    if (tl != tl[0]).any():                     # hash collision between two names: per record
                        for topic, key, payload, _j in batch.iter_records(sub):
                            self.queues[topic].append(Record(topic, payload, key, key.decode() if key is not None else None))
                        continue
                    self._route(batch, batch.topic_name(int(sub[0])), sub)
                continue
            self._route(batch, batch.topic_names[tid], batch.select(tid))
        batch.release()

    def _route(self, batch, name: str, idx) -> None:
        if name in self.frame_sinks:                       # publishes the lane did not frame: the record form frames them
            for topic, key, payload, _j in batch.iter_records(idx):
                self._frame_pending[topic].append(Record(topic, payload, key, key.decode() if key is not None else None))
        elif name in self.sinks:
            self.sinks[name](batch, idx)
        elif name in self.subscribed:
            self.frags[name].append((batch.retain(), idx))
        else:
            self.dropped_unsubscribed += len(idx)

    # --- consume side -------------------------------------------------------------------------------
    def poll_batch(self, topics: tuple[str, ...], max_records: int, max_bytes: int | None = None,
                   group_id: str | None = None) -> list[Record]:
        """per-record consume, bounded by records and (optionally) bytes; batch-wise entries are materialised as Records.
        With a group_id (a consumer that commits offsets) any such input is refused: records have no offsets"""
        if group_id is not None:
            for t in topics:
                if self.queues.get(t) or self.arenas.get(t) or self.frags.get(t):
                    _no_offsets(t)
        out: list[Record] = []
        nbytes = 0
        for t in topics:
            q = self.queues.get(t)
            while q and len(out) < max_records:
                if max_bytes is not None and out and nbytes + len(q[0].value) > max_bytes:
                    return out
                nbytes += len(q[0].value)
                out.append(q.popleft())
            if self.arenas.get(t) and type(self.arenas[t][0]).__name__ == "FetchArena":
                from calfkit.exceptions import EngineError
                raise EngineError(f"topic {t!r} holds fetch responses: they are decoded on the device, take them with poll_fetch")
            if len(out) < max_records and (self.arenas.get(t) or self.frags.get(t)):
                arena = self.poll_arena((t,), max_records - len(out), None if max_bytes is None else max(max_bytes - nbytes, 1),
                                        records_too=False)
                if arena is not None:
                    for i in range(arena.n):
                        out.append(Record(t, arena.record(i)))
                    nbytes += arena.nbytes
                    arena.release()
        return out

    def poll_fetch(self, topics: tuple[str, ...], max_records: int, max_bytes: int | None = None, group_id: str | None = None):
        """the next fetch response (engine.lane.FetchArena) of the first of these topics whose next entry is one, split
        at frame boundaries under the same bounds as poll_arena (None when none is): what a consumer that decodes fetches
        on the device (a node's engine, the client's replies) takes before it asks poll_batch for Records.  With a
        group_id (inside a transaction only) the slice is kept until a commit of that group's offsets covers it"""
        self._check_keep(group_id, topics)
        for t in topics:
            head = _take_fetch(self.arenas.get(t), max_records, max_bytes)
            if head is not None:
                return head if group_id is None else self._keep(t, group_id, head)
        return None

    def poll_arena(self, topics: tuple[str, ...], max_records: int, max_bytes: int | None = None, records_too: bool = True,
                   group_id: str | None = None):
        """the next batch for these topics as one contiguous Arena (None when idle).  Never returns more than max_records
        records or max_bytes bytes (one oversized record is still returned alone: the engine reports it per record).  A
        fetch slice polled with a group_id is kept as poll_fetch keeps it"""
        from calfkit.engine.lane import Arena
        self._check_keep(group_id, topics)
        for t in topics:
            q = self.arenas.get(t)
            head = _take_fetch(q, max_records, max_bytes)
            if head is not None:
                return head if group_id is None else self._keep(t, group_id, head)
            if group_id is not None and (q or self.frags.get(t) or (records_too and self.queues.get(t))):
                _no_offsets(t)
            if q:
                a = q[0]
                k = _fit(a.offsets, max_records, max_bytes)
                if k >= a.n:
                    return q.popleft()
                head = a.slice(0, k)
                rest = a.slice(k, a.n)
                rest._on_release, a._on_release = a._on_release, None       # the tail keeps the buffer alive
                q[0] = rest
                return head
            f = self.frags.get(t)
            if f:
                batch, idx = f[0]
                lens = batch.out_len[batch.pubs["payload"][idx]].astype("int64")
                k = _fit(np.concatenate(([0], np.cumsum(lens))), max_records, max_bytes)
                arena = batch.gather(idx[:k])        # a zero-copy view retains the batch until the arena is released
                if k >= len(idx):
                    f.popleft()
                    batch.release()
                else:
                    f[0] = (batch, idx[k:])
                return arena
            if records_too and self.queues.get(t):
                recs = self.poll_batch((t,), max_records, max_bytes)
                return Arena.pack([r.value for r in recs])
        return None

    def pending(self) -> int:
        return (sum(len(q) for q in self.queues.values()) + sum(len(r) for r in self._frame_pending.values()) + sum(a.n for q in self.arenas.values() for a in q)
                + sum(len(i) for q in self.frags.values() for _b, i in q))


def _take_fetch(q: deque | None, max_records: int, max_bytes: int | None):
    """the head of q when it is a fetch response, split only at frame boundaries: its leading frames that fit max_records
    records and max_bytes bytes, at least one (an oversized frame alone: the engine reports it); the rest stays at the
    head, and the truncated tail (if any) travels with the last piece.  The read_committed mask is sliced along
    (FetchArena.slice_frames).  None when q's head is not a fetch"""
    from calfkit.engine.lane import FetchArena
    while q and isinstance(q[0], FetchArena) and len(q[0].frames()[1]) == 0:
        q.popleft().release()                       # nothing but a truncated frame: no record in it
    if not (q and isinstance(q[0], FetchArena)):
        return None
    a = q[0]
    starts, counts = a.frames()
    cum_rec, cum_bytes = np.cumsum(counts), starts[1:] - starts[0]
    fits = cum_rec <= max_records
    if max_bytes is not None:
        fits &= cum_bytes <= max_bytes
    k = max(int(np.argmin(fits)) if not fits.all() else len(counts), 1)
    if k >= len(counts):
        return q.popleft()                          # the truncated tail (if any) goes along and is ignored
    head, rest = a.slice_frames(0, k), a.slice_frames(k, None)
    rest._on_release, a._on_release = a._on_release, None
    q[0] = rest
    return head


def _no_offsets(topic: str) -> None:
    from calfkit.exceptions import EngineError
    raise EngineError(f"topic {topic!r} holds records without offsets (Records or arenas): a consumer that commits its "
                      "offsets (exactly-once) consumes fetch responses only")


def _chain(fns):
    """one callable that calls the non-None callables of fns in order"""
    fns = [f for f in fns if f is not None]

    def call() -> None:
        for f in fns:
            f()
    return call


def _fit(offsets, max_records: int, max_bytes: int | None) -> int:
    """how many leading records of a batch fit the limits (at least one)"""
    n = len(offsets) - 1
    k = min(n, max_records)
    if n and (max_bytes is None or int(offsets[k] - offsets[0]) <= max_bytes):
        return k                                            # the common case: no array work at all
    if max_bytes is not None and n:
        k = min(k, int(np.searchsorted(offsets - offsets[0], max_bytes, side="right")) - 1)
    return max(k, 1) if n else 0


# the names calfkit code imports from faststream.kafka
KafkaBroker = MemoryBroker


class TestKafkaBroker:
    """async context manager mirroring faststream's TestKafkaBroker: starts the in-memory broker"""
    def __init__(self, broker: MemoryBroker):
        self.broker = broker

    async def __aenter__(self) -> MemoryBroker:
        await self.broker.start()
        return self.broker

    async def __aexit__(self, *exc: object) -> None:
        await self.broker.stop()


async def _maybe_await(x):
    if asyncio.iscoroutine(x):
        return await x
    return x
