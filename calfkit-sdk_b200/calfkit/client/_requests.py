"""Largely a TRANSCRIPTION of the reference's client package (same names, arguments, error behaviour: the API surface);
only `_ReplyDispatcher.drain` (the batch worker's stand-in for FastStream's consume task) is new.

Client-side request / reply machinery in ONE module, in dependency order: NodeResult -> reply projection ->
InvocationHandle -> correlation-id future table -> BaseClient.  Same names, arguments and error behaviour as the
reference's calfkit/client/{node_result,deserialize,invocation_handle,reply_dispatcher,base}.py (those module paths
re-export from here).  This is the per-request user-API edge of the path (SURVEY.md section 8 row a11): objects in,
objects out; the batched, device-side form of the reply projection is calfkit/client/batch_reply.py."""
from __future__ import annotations

import asyncio
import logging
import os
from collections.abc import Iterable, Sequence
from dataclasses import dataclass, field
from typing import Any, Generic

from pydantic import TypeAdapter
from typing_extensions import Self

from calfkit._ids import uuid7_hex
from calfkit._types import OutputT
from calfkit.broker import KafkaBroker
from calfkit.client.middleware import ContextInjectionMiddleware
from calfkit.exceptions import DeserializationError
from calfkit.models import ContentPart, DataPart, State, TextPart
from calfkit.models.messages import ModelMessage
from calfkit.nodes.base import submit_inbound
from calfkit.models.wire import CallFrame, CallFrameStack, Deps, Envelope, OverridesState, SessionRunContext, WorkflowState

logger = logging.getLogger(__name__)


# ----------------------------------------------------------------------------------------------------
# NodeResult  (reference client/node_result.py:11-32)
# ----------------------------------------------------------------------------------------------------
@dataclass(frozen=True)
class NodeResult(Generic[OutputT]):
    """Client-facing projection of a reply envelope (reference calfkit/client/node_result.py:11-32)."""
    output: OutputT
    output_parts: list[ContentPart]
    message_history: list[ModelMessage]
    metadata: Any
    correlation_id: str


# ----------------------------------------------------------------------------------------------------
# reply envelope -> NodeResult  (reference client/deserialize.py:15-89)
# ----------------------------------------------------------------------------------------------------
_UNSET: Any = object()


def deserialize_to_node_result(envelope: Envelope, output_type: type[Any] = _UNSET) -> NodeResult[Any]:
    state = envelope.context.state
    return NodeResult(output=_extract_output(state.final_output_parts, output_type), output_parts=state.final_output_parts,
                      message_history=state.message_history, metadata=state.metadata,
                      correlation_id=envelope.context.deps.correlation_id)


def _extract_output(parts: list[Any], output_type: type[Any]) -> Any:
    if output_type is _UNSET:
        for part in parts:
            if isinstance(part, DataPart):
                return part.data
        for part in parts:
            if isinstance(part, TextPart):
                return part.text
        raise DeserializationError("No DataPart or TextPart found in final_output_parts; cannot auto-detect output.")
    if output_type is str:
        for part in parts:
            if isinstance(part, TextPart):
                return part.text
        raise DeserializationError("No TextPart found in final_output_parts; expected output_type=str.")
    for part in parts:
        if isinstance(part, DataPart):
            return TypeAdapter(output_type).validate_python(part.data)
    raise DeserializationError("No DataPart found in final_output_parts; expected output_type="
                               f"{getattr(output_type, '__name__', str(output_type))}.")


# ----------------------------------------------------------------------------------------------------
# InvocationHandle  (reference client/invocation_handle.py:13-41)
# ----------------------------------------------------------------------------------------------------
@dataclass
class InvocationHandle(Generic[OutputT]):
    """reference calfkit/client/invocation_handle.py:13-41"""
    correlation_id: str
    topic: str
    reply_topic: str
    _future: asyncio.Future[Envelope] = field(repr=False, compare=False)
    _output_type: type[Any] = field(default=_UNSET, repr=False, compare=False)

    async def result(self, timeout: float | None = None) -> NodeResult[OutputT]:
        if self._future is None:
            raise RuntimeError("This handle has no associated future — was the client's reply dispatcher configured?")
        envelope = await (asyncio.wait_for(self._future, timeout=timeout) if timeout is not None else self._future)
        return deserialize_to_node_result(envelope, self._output_type)


# ----------------------------------------------------------------------------------------------------
# correlation_id -> Future table  (reference client/reply_dispatcher.py:15-53)
# ----------------------------------------------------------------------------------------------------
class _ReplyDispatcher:
    def __init__(self) -> None:
        self._pending: dict[str, asyncio.Future[Envelope]] = {}
        self._topic: str | None = None
        self._engine = None             # decodes fetch responses on the reply topic; created on the first one

    # a reply fetch is taken in pieces an engine of this size holds (replies carry the whole message history)
    FETCH_RECORDS, FETCH_BYTES = 1 << 12, 32 << 20

    def register(self, broker, reply_topic: str, group_id: str) -> None:
        self._topic = reply_topic
        self._sub = broker.subscriber(reply_topic, group_id=group_id, auto_offset_reset="latest")
        self._sub(self._handle_reply)

    async def _handle_reply(self, envelope: Envelope, correlation_id: str) -> None:
        future = self._pending.pop(correlation_id, None)
        if future is None:
            logger.warning("[%s] reply received but no pending future", correlation_id[:8])
            return
        if future.cancelled():
            return
        future.set_result(envelope)

    async def drain(self, broker) -> int:
        """deliver every queued reply record (the batch worker's stand-in for FastStream's consume task); fetch responses
        on the reply topic are checked, decompressed and split on the device (control and bad-frame records are not
        delivered; the latter are logged)"""
        if not self._topic:
            return 0
        n = 0
        while (fetch := broker.poll_fetch((self._topic,), self.FETCH_RECORDS, self.FETCH_BYTES)) is not None:
            try:
                n += fetch.n
                inb = submit_inbound(self._fetch_engine(), fetch)
                for i in range(inb.n):
                    if inb.values.bad[i] == 1:
                        logger.error("reply record %d rejected: its record batch failed the check", i)
                    elif inb.values.bad[i] == 0:
                        await self._deliver(inb.value(i).tobytes(), inb.correlation_ids[i])
            finally:
                fetch.release()
        recs = broker.poll_batch((self._topic,), 1 << 16)
        for r in recs:
            await self._deliver(r.value, r.correlation_id)
        return n + len(recs)

    async def _deliver(self, value, correlation_id: str | None) -> None:
        envelope = Envelope.model_validate_json(value)     # reply -> Python objects at the user-API edge
        await self._handle_reply(envelope, correlation_id or envelope.context.deps.correlation_id)

    def _fetch_engine(self):
        if self._engine is None:
            from calfkit.engine import BatchEngine
            self._engine = BatchEngine(int(os.environ.get("LOCAL_RANK", 0)), max_records=self.FETCH_RECORDS, max_in_bytes=self.FETCH_BYTES)
        return self._engine

    def expect(self, correlation_id: str) -> asyncio.Future[Envelope]:
        if correlation_id in self._pending:
            raise RuntimeError(f"Duplicate correlation_id: {correlation_id}")
        future: asyncio.Future[Envelope] = asyncio.get_running_loop().create_future()
        self._pending[correlation_id] = future
        future.add_done_callback(lambda _: self._pending.pop(correlation_id, None))
        return future

    def close(self) -> None:
        for future in self._pending.values():
            if not future.done():
                future.cancel()
        self._pending.clear()
        if self._engine is not None:
            self._engine.close()
            self._engine = None


# ----------------------------------------------------------------------------------------------------
# BaseClient  (reference client/base.py:27-172)
# ----------------------------------------------------------------------------------------------------
class BaseClient:
    def __init__(self, connection: KafkaBroker, reply_topic: str, dispatcher: _ReplyDispatcher) -> None:
        self._connection = connection
        self._reply_topic = reply_topic
        self._dispatcher = dispatcher

    @classmethod
    def connect(cls, server_urls: str | Iterable[str] | None = None, reply_topic: str | None = None,
                **broker_kwargs: Any) -> Self:
        if server_urls is None:
            server_urls = os.getenv("CALF_HOST_URL") or "localhost"
        client_id = uuid7_hex()
        if reply_topic is None:
            reply_topic = f"calf-client-reply-{client_id}"
        group_id = f"calf-client-reply-{client_id}"
        broker_connection = KafkaBroker(server_urls, middlewares=[ContextInjectionMiddleware], **broker_kwargs)
        dispatcher = _ReplyDispatcher()
        dispatcher.register(broker_connection, reply_topic, group_id)
        return cls(broker_connection, reply_topic, dispatcher)

    @property
    def broker(self) -> KafkaBroker:
        return self._connection

    @property
    def reply_topic(self) -> str:
        return self._reply_topic

    async def _invoke(self, topic: str, reply_topic: str, correlation_id: str, state: State,
                      overrides: OverridesState | None = None, run_args: Sequence[Any] | None = None,
                      deps: dict[str, Any] | None = None, output_type: type[Any] = _UNSET) -> InvocationHandle:
        future = self._dispatcher.expect(correlation_id)
        logger.debug("[%s] invoke topic=%s reply=%s", correlation_id[:8], topic, reply_topic)
        if not self._connection._connection:
            await self._connection.start()
        call_stack = CallFrameStack()
        call_stack.push(CallFrame(target_topic=topic, callback_topic=reply_topic, input_args=run_args, overrides=overrides))
        envelope = Envelope(internal_workflow_state=WorkflowState(call_stack=call_stack),
                            context=SessionRunContext(state=state, deps=Deps(correlation_id=correlation_id,
                                                                             provided_deps=deps or dict())))
        # the first hop is unkeyed, exactly like the reference (client/base.py:147)
        await self._connection.publish(envelope, topic=topic, correlation_id=correlation_id)
        return InvocationHandle(correlation_id=correlation_id, topic=topic, reply_topic=reply_topic, _future=future,
                                _output_type=output_type)

    async def close(self) -> None:
        self._dispatcher.close()
        await self._connection.stop()

    async def __aenter__(self) -> Self:
        return self

    async def __aexit__(self, *exc: object) -> None:
        await self.close()

