"""Agent node (mirrors reference calfkit/nodes/agent.py:26-230).

What is on the hot path here (SURVEY.md §8 a9, a10): the aggregation gate, the routing decision, the
fan-out of N Call envelopes and their encoding.  What is NOT: the LLM step (`_agent_loop.run`,
reference agent.py:124-130 — a remote HTTP call through the vendored pydantic-ai agent graph, SURVEY
§2 row 9).  `model_client` is therefore reduced to the one call the node makes at that boundary:

    model_client(messages, instructions, tools, deps) -> ModelResponse

(tests use FunctionModelClient, the analogue of the reference's FunctionModel fakes,
tests/providers.py:96-127).  Around that call the node works on wire bytes: inbound records are
validated and indexed by the CUDA walker; only the `state` span is materialised as a pydantic State
for the LLM boundary; the post-LLM envelope is re-validated on the device and the fan-out
(F envelopes per event, each a full copy of the state plus one frame), the frame pop of the final
ReturnCall, the topic routing and the partitioning all run in the engine.
"""
from __future__ import annotations

import logging
import time
from collections.abc import Callable
from typing import Any, Generic

import numpy as np
import pydantic_core

from calfkit._types import AgentOutputT
from calfkit.broker import Record
from calfkit.engine._lib import CK_ACT_FANOUT, CK_ACT_GATE_COMPLETE, CK_ACT_SILENT, CK_OK, COL, STATUS_NAMES
from calfkit.models import State
from calfkit.models.messages import (ModelMessage, ModelRequest, ModelResponse, RetryPromptPart, ToolCallPart,
                                     ToolDefinition, ToolReturnPart)
from calfkit.models.node_schema import BaseToolNodeSchema
from calfkit.models.payload import DataPart, TextPart
from calfkit.models.state import OverridesState, PendingToolBatch
from calfkit.nodes.base import BaseNodeDef, pack_records
from calfkit.nodes.tool import ToolNodeDef

logger = logging.getLogger(__name__)
ModelClient = Callable[[list[ModelMessage], str | None, list[ToolDefinition], dict[str, Any]], ModelResponse]


class FunctionModelClient:
    """Deterministic stand-in for an LLM: fn(messages, tools) -> ModelResponse."""
    def __init__(self, fn: Callable[[list[ModelMessage], list[ToolDefinition]], ModelResponse]):
        self.fn = fn

    def __call__(self, messages, instructions, tools, deps) -> ModelResponse:
        return self.fn(messages, tools)


class BaseAgentNodeDef(Generic[AgentOutputT], BaseNodeDef):
    def __init__(self, node_id: str, *, system_prompt: str = "You are a helpful AI assistant.",
                 subscribe_topics: str | list[str], publish_topic: str | None = None,
                 tools: list[ToolNodeDef] | None = None, model_client: ModelClient,
                 final_output_type: Any = str, sequential_only_mode: bool = False):
        self.final_output_type = final_output_type
        self.system_prompt = system_prompt
        self.tools = tools or list()
        self.sequential_only_mode = sequential_only_mode
        self.model_client = model_client
        self._pending_batches: dict[str, PendingToolBatch] = dict()     # host mirror of the gate (object-level callers, CPU tests)
        self._gate_stamp = 0                                            # records this node consumed so far: arrival order for the device gate
        self._instruction_fns: list[Callable[..., str | None]] = []
        if not isinstance(subscribe_topics, (list, tuple)):
            subscribe_topics = [subscribe_topics]
        super().__init__(node_id=node_id, subscribe_topics=subscribe_topics, publish_topic=publish_topic)

    async def run(self, ctx, *a, **k):
        raise RuntimeError("Agent.run is split between the host LLM boundary and the CUDA engine; use process_batch")

    def add_tools(self, *tools: ToolNodeDef) -> None:
        self.tools.extend(tools)

    def instructions(self, func: Callable[..., str | None]) -> Callable[..., str | None]:
        self._instruction_fns.append(func)
        return func

    # ---- host half: the reference's Agent.run around the LLM call (agent.py:70-220) -----------------
    def _registry(self, state: State) -> dict[str, BaseToolNodeSchema]:
        if state.overrides is not None and state.overrides.override_agent_tools is not None:
            return {t.tool_schema.name: t for t in state.overrides.override_agent_tools}
        return {t.tool_schema.name: t for t in self.tools}

    def _aggregate(self, corr: str, state: State) -> State | None:
        """_parallel_state_aggregation (agent.py:57-68): None while the batch is incomplete."""
        batch = self._pending_batches.get(corr)
        if batch is None:
            return state
        for cid in batch.expected_tool_call_ids:
            if cid not in batch.collected_results and cid in state.tool_results:
                batch.collected_results[cid] = state.tool_results[cid]
        if not batch.is_complete:
            return None
        for cid, res in batch.collected_results.items():
            batch.base_state.add_tool_result(cid, res)
        del self._pending_batches[corr]
        return batch.base_state

    def _llm_step(self, corr: str, state: State, deps: dict[str, Any], gated: bool = False) -> tuple[str, State]:
        """-> (action, new state) with action in {"silent", "fanout", "return", "tailcall"}.  gated: the aggregation gate
        already ran on the device (ck_gate_arrive): `state` is the merged base state or a pass-through."""
        registry = self._registry(state)
        if not self.sequential_only_mode and not gated:
            merged = self._aggregate(corr, state)
            if merged is None:
                return "silent", state
            state = merged
        latest = state.latest_tool_calls()
        if latest and not state.all_call_ids_complete(*[tc.tool_call_id for tc in latest]):
            if self.sequential_only_mode:
                return "fanout", state                       # next pending call goes out as a single Call
            remaining = [tc.tool_call_id for tc in latest if tc.tool_call_id not in state.tool_results]
            raise RuntimeError(f"[{corr[:8]}] Parallel mode reached incomplete tool calls outside aggregation gate. "
                               f"node={self.name} remaining_ids={remaining}. This indicates lost PendingToolBatch state "
                               "(e.g. partition rebalance or process restart).")
        if state.uncommitted_message is not None:
            state.commit_message_to_history()
        # instructions as the reference's agent loop composes them (_vendor/pydantic_ai/agent/__init__.py:1465-1487,
        # 638-650): the literals — Agent(instructions=system_prompt) and run(instructions=state.temp_instructions),
        # nodes/agent.py:54,126 — joined by "\n", then that and the outputs of the @agent.instructions functions joined by
        # "\n\n"; the ModelRequest that carries the tool returns records the same string
        literal = "\n".join(x for x in (self.system_prompt, state.temp_instructions) if isinstance(x, str)).strip() or None
        inst_parts = [x for x in [literal, *[fn() for fn in self._instruction_fns]] if x]
        instructions = "\n\n".join(inst_parts).strip() if inst_parts else None
        messages = list(state.message_history)
        if latest:                                           # tool returns go back to the model as a request
            parts = []
            for tc in latest:
                res = state.get_tool_result(tc.tool_call_id)
                if isinstance(res, RetryPromptPart):
                    parts.append(res)
                else:
                    value = getattr(res, "return_value", res)
                    parts.append(ToolReturnPart(tool_name=tc.tool_name, content=value, tool_call_id=tc.tool_call_id))
            request = ModelRequest(parts=parts, instructions=instructions)
            messages.append(request)
            state.message_history.append(request)
        response = self.model_client(messages, instructions, [t.tool_schema for t in registry.values()], deps)
        state.message_history.append(response)
        calls = [p for p in response.parts if isinstance(p, ToolCallPart)]
        if calls:
            for tc in calls:
                state.add_tool_call(tc)
                if tc.tool_name not in registry:
                    state.add_tool_result(tc.tool_call_id, RetryPromptPart(
                        content=f"There is no tool named {tc.tool_name}, it does not exist. Please ensure you are only "
                                "calling tools you are provided.", tool_name=tc.tool_name, tool_call_id=tc.tool_call_id))
            if state.all_call_ids_complete(*[tc.tool_call_id for tc in state.latest_tool_calls()]):
                return "tailcall", state
            pending = [tc for tc in state.latest_tool_calls() if tc.tool_call_id not in state.tool_results]
            if not self.sequential_only_mode and len(pending) > 1 and not gated:
                self._pending_batches[corr] = PendingToolBatch(
                    expected_tool_call_ids=frozenset(tc.tool_call_id for tc in pending), base_state=state.model_copy(deep=True))
            return "fanout", state
        text = "\n\n".join(p.content for p in response.parts if hasattr(p, "content") and isinstance(p.content, str))
        state.final_output_parts = [TextPart(text=text)] if self.final_output_type is str else [DataPart(data=text)]
        return "return", state

    # ---- batch path ----------------------------------------------------------------------------------
    def configure_engine(self, engine) -> None:
        registry = {t.tool_schema.name: t.subscribe_topics[0] for t in self.tools}
        engine.set_tool_node(self.publish_topic, None)        # publish-topic id for the ReturnCall plan
        engine.set_agent_node(self.name, self.subscribe_topics[0], self.publish_topic, registry)
        if not self.sequential_only_mode and not getattr(engine, "_gate_ready", False):
            engine.gate_create(max_entries=getattr(engine, "max_records", 1 << 14))      # pending fan-outs live in HBM
            engine._gate_ready = True

    # ---- per-request tool registries (overrides.override_agent_tools, reference agent.py:71-75) ------------------------
    def _use_registry(self, engine, registry: dict[str, str]) -> list[str]:
        """point the device fan-out plan at a request's own tool registry; returns the topic list to restore afterwards"""
        topics = [engine.topic_names[i] for i in sorted(engine.topic_names)]
        extra = [t for t in dict.fromkeys(registry.values()) if t not in engine.topic_ids]
        if extra:
            engine.register_topics(topics + extra, num_partitions=engine.num_partitions)    # same order first: ids stay put
        engine.set_agent_node(self.name, self.subscribe_topics[0], self.publish_topic, registry)
        return topics

    def _restore_registry(self, engine, topics: list[str]) -> None:
        engine.register_topics(topics, num_partitions=engine.num_partitions)
        self.configure_engine(engine)

    def process_batch(self, engine, records: list[Record]) -> list[Record]:
        data, offsets = pack_records(records)
        engine.submit(data, offsets)
        gated = not self.sequential_only_mode and getattr(engine, "_gate_ready", False)
        merged_env = None
        if gated:
            # the aggregation gate runs on the device: of the N tool returns of a fan-out N-1 end here as Silent without ever
            # becoming Python objects; the completing one comes back as the envelope carrying base_state + collected results
            engine.gate_arrive(self._gate_stamp)
            self._gate_stamp += len(records)
            merged_env = engine.fetch()
            st = engine.gate_stats()
            if st["live"] == 0 and st["arena_used"] > engine.gate_arena_bytes // 2:
                engine.gate_reset()
        cols = merged_env.cols if merged_env is not None else engine.columns()
        mv = memoryview(data)
        ovl = engine.overlay()          # records that arrived in another spelling: their canonical re-emission (the columns refer to it)
        post: dict[Any, list[tuple[int, bytes]]] = {"fanout": [], "return": []}
        canonical_in: dict[int, Any] = {}
        silent_returns: list[Record] = []
        for i in range(len(records)):
            if cols[COL["STATUS"], i] != CK_OK:
                logger.error("record %d rejected: %s", i, STATUS_NAMES[int(cols[COL["STATUS"], i])])
                continue
            if gated and cols[COL["ACTION"], i] == CK_ACT_SILENT:
                if self.publish_topic:          # handler return of a Silent: the inbound envelope (nodes/base.py:137-145, worker.py:52-53)
                    corr_raw = merged_env.record_bytes(i)[int(cols[COL["CORR_OFF"], i]):][:int(cols[COL["CORR_LEN"], i])].tobytes()
                    silent_returns.append(Record(self.publish_topic, merged_env.payload(i), None,
                                                 records[i].correlation_id or pydantic_core.from_json(b'"' + corr_raw + b'"')))
                continue
            if ovl is not None and ovl[1][i] >= 0:
                rec = memoryview(ovl[0])[int(ovl[1][i]):int(ovl[1][i]) + int(ovl[2][i])]
            else:
                rec = mv[offsets[i]:offsets[i + 1]]
            canonical_in[i] = rec
            s0, s1 = 20, int(cols[COL["SOV_OFF"], i] + cols[COL["SOV_LEN"], i]) + 1       # the `state` object span
            state_json = bytes(rec[s0:s1])
            if gated and cols[COL["ACTION"], i] == CK_ACT_GATE_COMPLETE:
                merged = merged_env.payload(i)          # inbound[:20] + merged state + inbound[s1:]
                state_json = merged[s0:len(merged) - (len(rec) - s1)]
            state = State.model_validate_json(state_json)                                    # LLM boundary
            fo, fl = int(cols[COL["FOV_OFF"], i]), int(cols[COL["FOV_LEN"], i])
            if fl and rec[fo] != ord("n"):
                state.overrides = OverridesState.model_validate_json(bytes(rec[fo:fo + fl]))
            corr = pydantic_core.from_json(b'"' + bytes(rec[int(cols[COL["CORR_OFF"], i]):][:int(cols[COL["CORR_LEN"], i])]) + b'"')
            deps = pydantic_core.from_json(bytes(rec[int(cols[COL["PD_OFF"], i]):][:int(cols[COL["PD_LEN"], i])]))
            try:
                action, new_state = self._llm_step(corr, state, deps, gated=gated)
            except Exception:  # noqa: BLE001  (model client / lost-batch RuntimeError: this record only, as one failing handler call in the reference)
                logger.exception("[%s] agent step failed for record %d; nothing is published for it", corr[:8], i)
                continue
            if action == "silent":
                # Silent (aggregation still incomplete): nothing is routed, but the handler returns the inbound envelope and
                # the worker publishes that return value to publish_topic (reference nodes/base.py:137-145, worker/worker.py:52-53)
                if self.publish_topic:
                    silent_returns.append(Record(self.publish_topic, bytes(rec), None, records[i].correlation_id or corr))
                continue
            new_bytes = bytes(rec[:s0]) + new_state.model_dump_json().encode() + bytes(rec[s1:])
            group: Any = action                                   # "tailcall": all requested tools invalid (agent.py:171-175)
            if action == "fanout" and new_state.overrides is not None and new_state.overrides.override_agent_tools is not None:
                # this request brought its own tool set: its calls are routed with that registry, in a group of their own
                reg = {t.tool_schema.name: t.subscribe_topics[0] for t in new_state.overrides.override_agent_tools}
                if reg != {t.tool_schema.name: t.subscribe_topics[0] for t in self.tools}:
                    group = ("fanout", tuple(sorted(reg.items())))
            post.setdefault(group, []).append((i, new_bytes))
        produced: list[Record] = list(silent_returns)
        now_ms = time.time_ns() // 1_000_000
        for group, items in post.items():
            if not items:
                continue
            kind, override_registry = (group[0], dict(group[1])) if isinstance(group, tuple) else (group, None)
            recs2 = [Record(records[i].topic, b, records[i].key, records[i].correlation_id) for i, b in items]
            d2, o2 = pack_records(recs2)
            saved_topics = self._use_registry(engine, override_registry) if override_registry is not None else None
            try:
                engine.submit(d2, o2)                                                        # re-validated on the device
                seed = int(np.random.SeedSequence().entropy) & ((1 << 63) - 1)
                if kind == "fanout":
                    engine.fanout_plan(now_ms, seed, max_fanout=256, sequential=self.sequential_only_mode)
                    if gated:
                        engine.gate_register()          # list[Call] records become pending entries of the device gate
                elif kind == "return":
                    engine.return_plan()
                else:
                    engine.tailcall_plan(now_ms, seed)
                out = engine.fetch()
                publishes = list(out.publishes())                 # topic ids are resolved against the registry in force
            finally:
                if saved_topics is not None:
                    self._restore_registry(engine, saved_topics)
            for r in np.flatnonzero(out.cols[COL["STATUS"]] != CK_OK):
                # e.g. more tool calls than the engine indexes per record (DESIGN.md §8): the conversation stops here
                logger.error("record %d declined after the agent step: %s; nothing is published for it",
                             items[r][0], STATUS_NAMES[int(out.cols[COL["STATUS"], r])])
            for p in publishes:
                src = recs2[p.record]
                corr = src.correlation_id or (p.key.decode() if p.key else None)
                payload = p.payload
                if kind == "fanout" and p.key is None and out.cols[COL["ACTION"], p.record] == CK_ACT_FANOUT:
                    # list[Call]: the handler's return value — what goes to publish_topic — is the INBOUND envelope, untouched:
                    # run() worked on prepare_context's deep copy (reference nodes/base.py:64-68,88; tests/golden/agent_run.json)
                    payload = bytes(canonical_in[items[p.record][0]])
                produced.append(Record(p.topic, payload, p.key, corr))
        return produced


Agent = BaseAgentNodeDef
