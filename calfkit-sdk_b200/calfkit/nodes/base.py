"""Base node definition (mirrors reference calfkit/nodes/base.py:27-176).

The reference's `handler` processes ONE pydantic Envelope per call on the asyncio loop.  Here the
unit of work is a batch of wire records: `process_batch` hands the bytes to the CUDA engine, which
does decode / prepare_context / run-dispatch / _publish_action / encode for the whole batch
(csrc/ck_kernels.cuh).  `handler(envelope, correlation_id, broker)` is kept with the reference's
signature for object-level callers; it serialises the envelope and goes through the SAME engine
path as a batch of one — there is no Python re-implementation of the hot path in the product.
"""
from __future__ import annotations

import inspect
import logging
from abc import abstractmethod
from typing import Any

import numpy as np

from calfkit.broker import Record
from calfkit.engine.batch import FetchBytes, _SpanOffsets
from calfkit.engine.lane import Arena, FetchArena, FetchRecords
from calfkit.models import NodeResult, State
from calfkit.models.envelope import Envelope
from calfkit.models.node_schema import BaseNodeSchema
from calfkit.models.session_context import SessionRunContext

logger = logging.getLogger(__name__)


class BaseNodeDef(BaseNodeSchema):
    _run_accepts_input: bool

    def __init_subclass__(cls, **kwargs: Any) -> None:
        super().__init_subclass__(**kwargs)
        sig = inspect.signature(cls.run)
        cls._run_accepts_input = len(sig.parameters) > 2     # self + ctx (+ input) — base.py:34-39

    @abstractmethod
    async def run(self, ctx: SessionRunContext, *args: Any, **kwargs: Any) -> NodeResult[State]:
        raise NotImplementedError()

    # ---- batch path (what Worker.run drives) -----------------------------------------------------
    def configure_engine(self, engine) -> None:
        """load this node's routing/tool configuration into a BatchEngine"""
        raise NotImplementedError(f"{type(self).__name__} has no batch plan: the GPU worker accelerates the node kinds "
                                  "the reference ships (@agent_tool nodes, Agent); custom run() bodies are out of scope")

    def process_batch(self, engine, records: list[Record] | FetchArena) -> list[Record]:
        raise NotImplementedError

    # ---- object-level compatibility ----------------------------------------------------------------
    async def handler(self, envelope: Envelope, correlation_id: str, broker: Any) -> Envelope:
        from calfkit.worker.worker import engine_for
        engine = engine_for(self)
        rec = Record(self.subscribe_topics[0], envelope.model_dump_json().encode(), correlation_id.encode(), correlation_id)
        outs = self.process_batch(engine, [rec])
        ret = envelope
        for o in outs:
            if o.topic == self.publish_topic and o.key is None:
                ret = Envelope.model_validate_json(o.value)      # the handler's return value
            else:
                await broker.publish(o.value, topic=o.topic, correlation_id=o.correlation_id, key=o.key)
        return ret

    @property
    def id(self) -> str:
        return self.node_id

    @property
    def name(self) -> str:
        return self.node_id

    @property
    def _return_topic(self) -> str:
        return f"{self.node_id}.private.return"


def pack_records(records: list[Record]):
    lens = np.fromiter((len(r.value) for r in records), dtype=np.int64, count=len(records))
    offsets = np.zeros(len(records) + 1, dtype=np.int64)
    np.cumsum(lens, out=offsets[1:])
    data = np.frombuffer(b"".join(r.value for r in records) or b"\0", dtype=np.uint8)
    return data, offsets


class Inbound:
    """what a node reads of each record of the batch it submitted (submit_inbound): value(i), the record's value bytes —
    for a fetch, where the device found them: in the response or in a compressed batch's decoded records section —, and
    keys[i] and correlation_ids[i] (Record fields, or a fetch record's key and `correlation_id` header; None: absent)"""
    def __init__(self, values: Arena | FetchRecords, keys: list[bytes | None], correlation_ids: list[str | None]):
        self.values, self.keys, self.correlation_ids = values, keys, correlation_ids

    @property
    def n(self) -> int:
        return len(self.keys)

    def value(self, i: int) -> memoryview:
        o = self.values.offsets
        return memoryview(self.values.data[int(o[i]):(o.end(i) if isinstance(o, _SpanOffsets) else int(o[i + 1]))])


def submit_inbound(engine, batch: list[Record] | FetchArena) -> Inbound:
    """submit an inbound batch to the engine, either form: Records through engine.submit, a fetch response through
    engine.submit_recordbatch with the subscription's read_committed mask (set when the engine is at read_committed).
    The column spans of record i then lie in inbound.value(i)"""
    if not isinstance(batch, FetchArena):
        data, offsets = pack_records(batch)
        engine.submit(data, offsets)
        return Inbound(Arena(data, offsets), [r.key for r in batch], [r.correlation_id for r in batch])
    if engine.read_committed and batch.hidden() is not None:
        engine.set_fetch_hidden(batch.hidden())
    engine.submit_recordbatch(batch.data)
    ix = engine.fetch_index
    data = ix["data"]
    values = FetchRecords(batch, ix["val_off"], ix["val_len"], ix["bad"],
                          decoded=(data.base, data.decoded) if isinstance(data, FetchBytes) else None)

    def spans(off, ln):
        return [None if n < 0 else data[int(o):int(o) + int(n)].tobytes() for o, n in zip(off, ln)]
    return Inbound(values, spans(ix["key_off"], ix["key_len"]),
                   [None if c is None else c.decode() for c in spans(ix["corr_off"], ix["corr_len"])])
