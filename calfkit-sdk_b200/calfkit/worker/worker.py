"""Worker (mirrors reference calfkit/worker/worker.py:12-61).

Same constructor, add_nodes, register_handlers (idempotence guard -> RuntimeError) and async run().
The reference's run() hands control to FastStream, which then delivers ONE record at a time to
node.handler.  Here run() is the batch loop itself.  Two paths per node:

  * device-template tool nodes (the data-parallel hot path): `broker.poll_arena` -> one pinned batch arena ->
    `LanePipeline.push` (H2D + decode + plan + encode + route on one of K lanes while an older step's results come
    back) -> `broker.produce_publishes(PublishBatch)`.  No Python object per record.
  * nodes with a host half (Python tools, the Agent's LLM boundary): `broker.poll_fetch`, else `broker.poll_batch` ->
    `node.process_batch` (engine for decode / plan / encode, Python only for the user callable; a fetch response is
    decoded there on the device, as on the lanes) -> `broker.produce_batch`.

A poll is bounded by records AND bytes, an engine-level failure splits the batch and retries (dequeued records are never
lost), and records the device declines as CK_UNSUPPORTED are re-run through the host-tool path.  Records of a fetch
response that a consumer does not deliver (control batches; under the subscriber's isolation_level="read_committed" the
aborted transactions' batches) come out CK_SKIPPED: counted in stats["skipped"], neither logged nor re-run.

A broker with enable_idempotence or a transactional_id (frame sinks only) gives the Worker one producer id and epoch
(MemoryBroker.init_producer_id) when it builds its first engine that frames; every lane engine and the framer engine write
them into their frames, and each frame pass takes the broker's next sticky partitions for the unkeyed publishes.  With a
transactional_id, each tick of run() is one transaction: committed when the tick ends, aborted when it raises.

Worker(..., processing_guarantee="exactly_once_v2") makes a transactional Worker exactly-once for the fetches it consumes
(Kafka Streams' guarantee of that name): every fetch slice is polled for its subscription's consumer group and kept by
the broker; when a step's results are handed out (a lane's results come back, a host node returns) the slice's
positions (FetchArena.positions) become the group's handed-out offsets, and at the end of the tick they are sent to the
tick's transaction (send_offsets_to_transaction) before it commits.  Input still in flight on a lane stays uncommitted:
its outputs and its offsets go into the later transaction that hands them out.  When a tick raises, the results in
flight are dropped, the transaction aborts, the broker puts the uncommitted slices back, and run() re-raises; a later
run() consumes them again.  Only fetches carry offsets: under this guarantee a subscribed topic that holds Records or
arenas makes the poll raise EngineError before anything is taken.
"""
from __future__ import annotations

import asyncio
import contextlib
import logging
import os
import time
from typing import Any

import numpy as np

from calfkit.broker import Record
from calfkit.client import Client
from calfkit.engine import BatchEngine
from calfkit.engine.batch import FRAME_CODECS, ISOLATION_LEVELS, check_compression_level
from calfkit.engine._lib import CK_ACT_RAISES, CK_OK, CK_SKIPPED, CK_UNSUPPORTED, STATUS_NAMES
from calfkit.exceptions import EngineError
from calfkit.engine.lane import FetchArena, FetchRecords, LanePipeline, PublishBatch
from calfkit.nodes import BaseNodeDef

logger = logging.getLogger(__name__)


def _EMPTY_ARENA():
    from calfkit.engine.lane import Arena
    return Arena(np.zeros(0, dtype=np.uint8), np.zeros(1, dtype=np.int64))


def engine_for(node: BaseNodeDef, *, device: int = 0, max_records: int = 1 << 14, max_in_bytes: int = 64 << 20,
               extra_topics: list[str] | None = None, isolation_level: str | None = None) -> BatchEngine:
    """lazily created, per-node engine (also used by the object-level BaseNodeDef.handler); isolation_level: what the
    fetches the node submits from now on deliver (BatchEngine.set_isolation_level), None: as it is"""
    eng = getattr(node, "_ck_engine", None)     # the engine lives (and dies) with its node: no id()-keyed registry
    if eng is None:
        eng = BatchEngine(device, max_records=max_records, max_in_bytes=max_in_bytes,
                          max_out_bytes=8 * max_in_bytes, max_payloads=8 * max_records)
        topics = list(node.subscribe_topics) + ([node.publish_topic] if node.publish_topic else [])
        for t in getattr(node, "tools", []) or []:
            topics += list(t.subscribe_topics)
        eng.register_topics(topics + (extra_topics or []), num_partitions=0)
        node.configure_engine(eng)
        node._ck_engine = eng
    if isolation_level is not None:
        eng.set_isolation_level(isolation_level)
    return eng


PROCESSING_GUARANTEES = ("at_least_once", "exactly_once_v2")


class Worker:
    def __init__(self, client: Client, nodes: list[BaseNodeDef] | None = None, max_workers: int = 1,
                 group_id: str | None = None, extra_publish_kwargs: dict[str, Any] | None = None,
                 extra_subscribe_kwargs: dict[str, Any] | None = None, *, device: int | None = None,
                 batch_records: int = 1 << 14, batch_bytes: int = 64 << 20, lanes: int = 3,
                 route_topics: list[str] | None = None, rank: int | None = None, world: int | None = None,
                 processing_guarantee: str = "at_least_once"):
        """Reference signature (worker/worker.py:13-31) plus keyword-only engine knobs: `device` (default: LOCAL_RANK of a
        one-process-per-GPU launch, else 0), the batch bounds a poll honours (records AND bytes: a batch never exceeds what
        the engines were sized for), the number of pipelined lanes per device-template node, and `route_topics`: names of
        topics owned by OTHER workers that this worker's outputs go to (agents' input topics ...) so that the device resolves
        them to ids too; names it does not know are still routed, grouped by hash on the host.
        `rank` / `world` (default: torch.distributed's, when initialised): one worker process per GPU, records sharded by Kafka
        partition (reference: consumer-group sharding, worker/worker.py:38,47, with every hop keyed by correlation_id,
        nodes/base.py:86,103,117,134).  A keyed publish whose partition (murmur2(key) % partitions) is owned by another rank
        (partition % world) is stored straight into that rank's receive buffer over NVLink and produced THERE; all ranks
        tick in lockstep (an idle rank submits an empty batch) so that the per-step barriers of the exchange match.
        `processing_guarantee`: "at_least_once" (the default) or "exactly_once_v2", which needs a broker with a
        transactional_id: each tick commits the consumed offsets of the results it hands out with the frames they made."""
        if processing_guarantee not in PROCESSING_GUARANTEES:
            raise EngineError(f"processing_guarantee {processing_guarantee!r}: expected one of {PROCESSING_GUARANTEES}")
        if processing_guarantee == "exactly_once_v2" and getattr(client._connection, "transactional_id", None) is None:
            raise EngineError("processing_guarantee='exactly_once_v2' needs a broker with a transactional_id")
        self._exactly_once = processing_guarantee == "exactly_once_v2"
        self._handed: dict[str, dict[tuple[str, int], int]] = {}   # group -> {(topic, partition): next offset} handed out this tick
        self._client = client
        self._nodes = nodes or list()
        self._max_workers = max_workers
        self._group_id = group_id
        self._extra_publish_kwargs = extra_publish_kwargs or {}
        self._extra_subscribe_kwargs = extra_subscribe_kwargs or {}
        self._prepared = False
        self._device = device if device is not None else int(os.environ.get("LOCAL_RANK", 0))
        self._batch_records = batch_records
        self._batch_bytes = batch_bytes
        self._lanes = lanes
        self._route_topics = list(route_topics or [])
        if rank is None or world is None:
            try:
                import torch.distributed as dist
                if dist.is_available() and dist.is_initialized():
                    rank, world = dist.get_rank(), dist.get_world_size()
            except ImportError:
                pass
        self._rank, self._world = (rank or 0), (world or 1)
        self._subs: list[tuple[BaseNodeDef, Any]] = []
        self._pipes: dict[int, LanePipeline] = {}
        self._framer_eng: BatchEngine | None = None
        self._frame_pool = None
        self._levels: dict[int, str] = {}          # node -> its subscription's isolation_level
        self._groups: dict[int, str] = {}          # node -> its subscription's consumer group
        self._producer: tuple[int, int] | None = None   # (producer id, epoch) of an idempotent broker, taken once
        self.stats = {"records": 0, "publishes": 0, "rejected": 0, "skipped": 0, "raises": 0, "host_fallback": 0, "steps": 0}

    def add_nodes(self, *nodes: BaseNodeDef) -> None:
        self._nodes.extend(nodes)

    def register_handlers(self) -> None:
        if self._prepared:
            raise RuntimeError("register_handlers() already called")
        for node in self._nodes:
            group_id = self._group_id or node.name
            logger.info("registering node=%s subscribe=%s publish=%s", node.name, node.subscribe_topics, node.publish_topic)
            subscriber = self._client._connection.subscriber(*node.subscribe_topics, group_id=group_id,
                                                             max_workers=self._max_workers, **self._extra_subscribe_kwargs)
            # a FastStream KafkaBroker.subscriber takes isolation_level among its kwargs; here it goes to the node's lanes
            level = subscriber.kwargs.get("isolation_level", "read_uncommitted")
            if level not in ISOLATION_LEVELS:
                raise EngineError(f"node {node.name}: isolation_level {level!r}, expected one of {ISOLATION_LEVELS}")
            self._levels[id(node)] = level
            self._groups[id(node)] = group_id
            handler = subscriber(node.handler)
            if node.publish_topic:
                self._client._connection.publisher(node.publish_topic, **self._extra_publish_kwargs)(handler)
            self._subs.append((node, subscriber))
        self._prepared = True

    # ---- device-template tool nodes: arena in -> pipelined lanes -> publish batch out, no Python per record ----------
    def _pipeline(self, node: BaseNodeDef) -> LanePipeline:
        pipe = self._pipes.get(id(node))
        if pipe is None:
            # frame-sink topics get ids like route_topics, so that their publishes can be framed on the device
            frame_topics = list(self._client._connection.frame_sinks)
            topics = list(node.subscribe_topics) + ([node.publish_topic] if node.publish_topic else []) + self._route_topics + frame_topics
            codec = self._frame_codec() if frame_topics else None
            clevel = self._frame_level(codec) if frame_topics else None
            level = self._levels.get(id(node), "read_uncommitted")
            producer = self._producer_of(self._client._connection) if frame_topics else None

            def configure(eng: BatchEngine) -> None:
                eng.register_topics(topics, num_partitions=getattr(self._client._connection, "num_partitions", 0))
                node.configure_engine(eng)
                eng.set_isolation_level(level)
                if frame_topics:
                    eng.set_frame_topics(frame_topics)
                    eng.set_frame_compression(codec, clevel)
                    if producer is not None:
                        eng.set_producer(*producer)
            pipe = LanePipeline(self._device, configure, lanes=self._lanes, max_records=self._batch_records,
                                max_in_bytes=self._batch_bytes, exchange=(self._rank, self._world) if self._world > 1 else None)
            self._pipes[id(node)] = pipe
        return pipe

    def _produce_fast(self, node: BaseNodeDef, batch: PublishBatch) -> None:
        broker = self._client._connection
        self._hand_out(node, batch.source)
        n = batch.source.n
        if n == 0:
            batch.release()
            return
        self.stats["records"] += n
        skipped = batch.status == CK_SKIPPED
        self.stats["skipped"] += int(np.count_nonzero(skipped))
        bad = (batch.status != CK_OK) & ~skipped
        nbad = int(np.count_nonzero(bad))
        if nbad:
            self.stats["rejected"] += nbad
            for i in np.nonzero(bad & (batch.status != CK_UNSUPPORTED))[0][:8]:
                logger.error("record %d rejected: %s", int(i), STATUS_NAMES[int(batch.status[i])])
            # the device declined these (a construct the template / fast path does not cover, e.g. `args` given as a JSON
            # string or a non-string template argument): the host-tool path handles them, nothing is dropped silently
            redo = np.nonzero((batch.status == CK_UNSUPPORTED) & (batch.action == CK_ACT_RAISES))[0]
            if len(redo):
                self.stats["host_fallback"] += len(redo)
                recs = [Record(node.subscribe_topics[0], batch.source.record(int(i))) for i in redo]
                self._run_host(node, recs, force_host=True)
        self.stats["raises"] += int(np.count_nonzero((batch.action == CK_ACT_RAISES) & (batch.status == CK_OK)))
        self.stats["publishes"] += batch.n_publishes
        broker.produce_publishes(batch)

    # ---- host-side nodes (Python tools, the Agent's LLM boundary): per-record objects are inherent there -----------
    def _run_host(self, node: BaseNodeDef, records: list[Record] | FetchArena, **kw: Any) -> None:
        """never loses a dequeued record: an engine-level failure (a batch the buffers cannot hold) splits the batch and
        retries, a fetch response at frame boundaries; a single record, or a single frame, that still fails is logged and
        dropped alone"""
        broker = self._client._connection
        engine = engine_for(node, device=self._device, max_records=self._batch_records, max_in_bytes=self._batch_bytes,
                            isolation_level=self._levels.get(id(node), "read_uncommitted"))
        fetch = isinstance(records, FetchArena)
        skipped = engine.skipped if fetch else 0
        try:
            broker.produce_batch(node.process_batch(engine, records, **kw) if kw else node.process_batch(engine, records))
            self.stats["records"] += 0 if kw else (records.n if fetch else len(records))
            if fetch:
                self.stats["skipped"] += engine.skipped - skipped
        except Exception:  # noqa: BLE001  (EngineError: capacity; user code outside the per-record guards)
            pieces = len(records.frames()[1]) if fetch else len(records)
            if pieces <= 1:
                if fetch:
                    logger.exception("node %s: frame of %d records dropped after failing alone", node.name, records.n)
                else:
                    logger.exception("node %s: record dropped after failing alone", node.name)
                return
            mid = pieces // 2
            logger.warning("node %s: batch of %d %s failed, retrying in halves", node.name, pieces, "frames" if fetch else "records")
            if fetch:
                self._run_host(node, records.slice_frames(0, mid), **kw)
                self._run_host(node, records.slice_frames(mid, None), **kw)
            else:
                self._run_host(node, records[:mid], **kw)
                self._run_host(node, records[mid:], **kw)

    def _hand_out(self, node: BaseNodeDef, source) -> None:
        """exactly-once: the positions of a fetch slice whose results are being handed out become its group's offsets of
        this tick"""
        if not self._exactly_once:
            return
        arena = source.arena if isinstance(source, FetchRecords) else source
        if isinstance(arena, FetchArena) and arena.topic is not None:
            handed = self._handed.setdefault(self._groups[id(node)], {})
            for part, nxt in arena.positions().items():
                handed[(arena.topic, part)] = nxt

    def _drop_in_flight(self, broker) -> None:
        """exactly-once, a tick that raised: the results still on the lanes and the Records not yet framed belong to input
        the abort gives back, so they are dropped, not produced"""
        for pipe in self._pipes.values():
            try:
                for done in pipe.drain():
                    done.release()
                for rb in pipe.take_received():
                    rb.release()
            except Exception:  # noqa: BLE001  (the tick's own failure is what run() re-raises)
                logger.exception("dropping the results in flight after a failed tick")
        broker.discard_frames()
        self._handed.clear()

    def _producer_of(self, broker) -> tuple[int, int, bool] | None:
        """(producer id, epoch, transactional) the engines that frame write into their frames; None: not idempotent"""
        if not getattr(broker, "enable_idempotence", False):
            return None
        if self._producer is None:
            self._producer = broker.init_producer_id(broker.transactional_id)
        return self._producer + (broker.transactional_id is not None,)

    @contextlib.contextmanager
    def _transaction(self, broker):
        """one tick of run() under a transactional broker: committed when it ends, aborted (then re-raised) when it raises"""
        if getattr(broker, "transactional_id", None) is None:
            yield
            return
        broker.begin_transaction()
        try:
            yield
            for group, offsets in self._handed.items():
                broker.send_offsets_to_transaction(offsets, group)
            self._handed.clear()
        except BaseException:
            if self._exactly_once:
                self._drop_in_flight(broker)
            broker.abort_transaction()
            raise
        broker.commit_transaction()

    def _frame_codec(self) -> str | None:
        """the broker's compression_type for the frames built on the device: None or "lz4"; any other codec is refused"""
        codec = getattr(self._client._connection, "compression_type", None)
        if codec not in FRAME_CODECS:
            raise EngineError(f"frame sinks: compression_type {codec!r} is not built on the device (None or 'lz4')")
        return codec

    def _frame_level(self, codec: str | None) -> int | None:
        """the broker's compression_level for the frames of `codec`: checked whatever the codec, applied to LZ4 frames
        only (Kafka ignores compression.lz4.level for other codecs)"""
        level = check_compression_level(getattr(self._client._connection, "compression_level", None))
        return level if codec == "lz4" else None

    def _frame_records(self, topic: str, records: list[Record]):
        """the engine's record form over Records produced to a frame-sink topic by host paths, in engine-sized chunks"""
        broker = self._client._connection
        if self._framer_eng is None:
            from calfkit.engine.lane import PinnedPool
            self._framer_eng = BatchEngine(self._device, max_records=self._batch_records, max_in_bytes=self._batch_bytes)
            self._framer_eng.register_topics(list(broker.frame_sinks), num_partitions=getattr(broker, "num_partitions", 0))
            codec = self._frame_codec()
            self._framer_eng.set_frame_compression(codec, self._frame_level(codec))
            producer = self._producer_of(broker)
            if producer is not None:
                self._framer_eng.set_producer(*producer)
            self._frame_pool = PinnedPool()
        eng, ts = self._framer_eng, int(time.time() * 1000)
        if topic not in eng.topic_ids:
            eng.register_topics(list(eng.topic_ids) + [topic], num_partitions=eng.num_partitions)
        limit = min(2 * eng.max_payloads, eng.max_records)
        a = 0
        while a < len(records):
            b, nbytes = a, 0
            while b < len(records) and b - a < limit:
                r = records[b]
                size = len(r.value) + 2 * len(r.key or b"") + 2 * len((r.correlation_id or "").encode())
                if b > a and nbytes + size > eng.max_in:
                    break
                nbytes += size
                b += 1
            if getattr(broker, "enable_idempotence", False):
                eng.set_sticky_partitions(broker.next_sticky([topic]))
            eng.encode_frames_records(topic, [(r.value, r.key, r.correlation_id) for r in records[a:b]], ts)
            yield eng.fetch_frames(self._frame_pool)
            a = b

    def step(self) -> int:
        """one pass over all nodes: poll -> CUDA batch -> produce.  Returns the number of records consumed."""
        broker = self._client._connection
        consumed = 0
        self.stats["steps"] += 1
        if broker.frame_sinks:
            if self._world > 1:
                raise EngineError("frame sinks need world == 1: publishes forwarded by other ranks are not framed yet")
            broker.framer = self._frame_records
        for node, sub in self._subs:
            group = {"group_id": sub.group_id} if self._exactly_once else {}   # exactly-once: the broker keeps the slice
            if getattr(node, "_template", None) is not None:
                pipe = self._pipeline(node)
                arena = broker.poll_arena(sub.topics, self._batch_records, self._batch_bytes, **group)
                if arena is None and self._world > 1:
                    arena = _EMPTY_ARENA()                     # lockstep: every rank runs the exchange on every tick
                if arena is not None:
                    consumed += arena.n
                    # the step's timestamp is the frames' baseTimestamp (only framing lanes use it)
                    if not broker.frame_sinks:
                        done = pipe.push(arena)
                    elif getattr(broker, "enable_idempotence", False):
                        done = pipe.push(arena, int(time.time() * 1000), broker.next_sticky(broker.frame_sinks))
                    else:
                        done = pipe.push(arena, int(time.time() * 1000))
                    if done is not None:
                        self._produce_fast(node, done)
                elif pipe.pending:                             # input idle (single rank): flush what is in flight
                    for done in pipe.drain():
                        consumed += 1                          # keeps run(until_idle) going: what was just produced may feed a node
                        self._produce_fast(node, done)
                for rb in pipe.take_received():                # forwarded here by the owners of other partitions' inputs
                    self.stats["received"] = self.stats.get("received", 0) + rb.n_publishes
                    broker.produce_publishes(rb)
                continue
            fetch = broker.poll_fetch(sub.topics, self._batch_records, self._batch_bytes, **group)
            if fetch is not None:
                consumed += fetch.n
                try:
                    self._run_host(node, fetch)
                    self._hand_out(node, fetch)
                finally:
                    fetch.release()
                continue
            records: list[Record] = broker.poll_batch(sub.topics, self._batch_records, self._batch_bytes, **group)
            if not records:
                continue
            consumed += len(records)
            self._run_host(node, records)
        broker.flush_frames()
        return consumed

    def close(self) -> None:
        for pipe in self._pipes.values():
            pipe.close()
        self._pipes.clear()
        if self._framer_eng is not None:
            self._framer_eng.close()
            self._frame_pool.close()
            self._framer_eng = self._frame_pool = None

    def _all_idle(self, n: int) -> bool:
        """N > 1: the ranks stop together — a rank with nothing to do still has to run the exchange for the others"""
        if self._world == 1:
            return n == 0
        import torch
        import torch.distributed as dist
        t = torch.tensor([n], dtype=torch.int64, device=torch.device("cuda", self._device))
        dist.all_reduce(t)
        return int(t.item()) == 0

    async def run(self, *, until_idle: bool = False, idle_sleep: float = 0.001, **extra_run_args: Any) -> None:
        """Run the worker as a service (reference: blocks in FastStream(...).run()); `until_idle=True`
        returns once every subscribed topic is drained — used by tests and the config-1 example."""
        logger.info("worker starting with %d node(s)", len(self._nodes))
        if not self._prepared:
            self.register_handlers()
        broker = self._client._connection
        if not broker._connection:
            await broker.start()
        while True:
            finished = False
            with self._transaction(broker):                # a transactional broker: one transaction per tick
                n = self.step()
                n += await self._client._dispatcher.drain(broker) if hasattr(self._client, "_dispatcher") else 0
                idle = self._all_idle(n + sum(p.pending_records for p in self._pipes.values()))
                if idle and until_idle:
                    flushed = 0
                    for node, _sub in self._subs:          # nothing in flight on any rank: flush (no exchange involved)
                        pipe = self._pipes.get(id(node))
                        if pipe is not None:
                            for done in pipe.drain():
                                flushed += done.source.n
                                self._produce_fast(node, done)
                            for rb in pipe.take_received():
                                flushed += rb.n_publishes
                                broker.produce_publishes(rb)
                    broker.flush_frames()
                    finished = self._all_idle(flushed)     # nothing came out that a subscribed node still has to consume
            if finished:
                return
            if idle and not until_idle:
                await asyncio.sleep(idle_sleep)
            elif not idle:
                await asyncio.sleep(0)
