"""@agent_tool nodes (mirrors reference calfkit/nodes/tool.py:19-95).

Two kinds of tool are distinguished at decoration time:
  * device tools  — `@agent_tool(device_template="It's sunny in {location}")`: the return value is a
    pure string template of string arguments; ToolNodeDef.run happens entirely in
    ck_plan_tool_kernel, no host round trip.
  * host tools    — any Python callable: the engine gathers each record's `args` JSON on the device
    (the same kernel, mode 0), the callable runs on the host (the one thing a GPU cannot do: user
    Python), and its JSON result is spliced in on the device.  Argument decoding / result encoding of the *user's values* happens here
    with pydantic_core, exactly as reference nodes/tool.py:64 + messages.py:1229-1240 do.
"""
from __future__ import annotations

import inspect
import logging
from collections.abc import Awaitable, Callable
from dataclasses import dataclass, field
from typing import Any

import numpy as np
import pydantic
import pydantic_core
from typing_extensions import Self

from calfkit.broker import Record
from calfkit.engine._lib import CK_ACT_HOST_TOOL, CK_ACT_RAISES, CK_OK, CK_SKIPPED, CK_UNSUPPORTED, COL, STATUS_NAMES
from calfkit.engine.batch import ToolTemplate
from calfkit.models import SessionRunContext, State, ToolContext
from calfkit.models.actions import NodeResult
from calfkit.models.messages import ModelMessagesTypeAdapter, ToolDefinition
from calfkit.models.node_schema import BaseToolNodeSchema
from calfkit.engine.lane import FetchArena
from calfkit.nodes.base import BaseNodeDef, submit_inbound

logger = logging.getLogger(__name__)


_SECTION_TITLES = {"args", "arguments", "params", "parameters", "keyword args", "keyword arguments", "other args", "other arguments",
                   "other params", "other parameters", "raises", "exceptions", "returns", "yields", "receives", "examples", "example",
                   "attributes", "functions", "methods", "classes", "modules", "warns", "warnings", "note", "notes", "see also"}
_PARAM_TITLES = {"args", "arguments", "params", "parameters"}


def _parse_docstring(doc: str | None, names: list[str]) -> tuple[str | None, dict[str, str]]:
    """(description, {parameter: description}) of a Google / NumPy / Sphinx style docstring — what the reference obtains from
    griffe (calfkit/_vendor/pydantic_ai/_griffe.py): the text before the first section (wrapped as <summary>…</summary> plus a
    <returns> block when the docstring documents its return value), and the per-parameter texts, which go into the JSON
    schema as `description`s.  Pinned by tests/golden/tool_schemas.json for the three styles; exotic layouts may differ."""
    if not doc:
        return None, {}
    lines = inspect.cleandoc(doc).splitlines()
    params: dict[str, str] = {}
    main: list[str] = []
    ret_type: str | None = None
    ret_desc: str | None = None
    i, n = 0, len(lines)
    in_main = True

    def indented(s: str) -> bool:
        return s.startswith((" ", "\t"))

    while i < n:
        line = lines[i]
        stripped = line.strip()
        # ---- Sphinx field list
        if stripped.startswith(":") and not indented(line) and ":" in stripped[1:]:
            head, _, desc = stripped[1:].partition(":")
            words = head.split()
            kind = words[0] if words else ""
            if kind in ("param", "parameter", "arg", "argument", "key", "keyword", "return", "returns", "rtype", "raises", "raise", "type", "var", "ivar", "cvar"):
                in_main = False
                body = [desc.strip()]
                j = i + 1
                while j < n and indented(lines[j]):
                    body.append(lines[j].strip())
                    j += 1
                text = "\n".join(x for x in body if x)
                if kind in ("param", "parameter", "arg", "argument", "key", "keyword") and words[-1] in names:
                    params[words[-1]] = text
                elif kind in ("return", "returns"):
                    ret_desc = text
                elif kind == "rtype":
                    ret_type = text
                i = j
                continue
        # ---- NumPy section: a title underlined with dashes
        if i + 1 < n and stripped and lines[i + 1].strip() and set(lines[i + 1].strip()) == {"-"} and stripped.lower() in _SECTION_TITLES:
            in_main = False
            title = stripped.lower()
            j = i + 2
            entries: list[tuple[str, list[str]]] = []
            while j < n and not (j + 1 < n and lines[j].strip() and lines[j + 1].strip() and set(lines[j + 1].strip()) == {"-"}):
                raw = lines[j]
                if raw.strip():
                    if not indented(raw):
                        entries.append((raw.strip(), []))
                    elif entries:
                        entries[-1][1].append(raw.strip())
                j += 1
            if title in _PARAM_TITLES:
                for head, body in entries:
                    name = head.split(":")[0].strip()
                    if name in names:
                        params[name] = "\n".join(body)
            elif title == "returns" and entries:
                head, body = entries[0]
                ret_type = head.split(":")[-1].strip() or None
                ret_desc = "\n".join(body)
            i = j
            continue
        # ---- Google section: "Title:" on its own line, body indented
        if stripped.endswith(":") and stripped[:-1].lower() in _SECTION_TITLES and not indented(line):
            in_main = False
            title = stripped[:-1].lower()
            j = i + 1
            entries = []
            base_indent = None
            while j < n and (not lines[j].strip() or indented(lines[j])):
                raw = lines[j]
                if raw.strip():
                    indent = len(raw) - len(raw.lstrip())
                    if base_indent is None:
                        base_indent = indent
                    if indent <= base_indent:
                        entries.append((raw.strip(), []))
                    elif entries:
                        entries[-1][1].append(raw.strip())
                j += 1
            if title in _PARAM_TITLES:
                for head, body in entries:
                    if ":" not in head:
                        continue
                    h, _, desc = head.partition(":")
                    name = h.split("(")[0].strip().lstrip("*")
                    if name in names:
                        params[name] = "\n".join([desc.strip()] + body).strip()
            elif title == "returns" and entries:
                head, body = entries[0]
                if ":" in head and " " not in head.split(":")[0].strip():
                    ret_type, _, first = head.partition(":")
                    ret_type = ret_type.strip()
                else:
                    first = head
                ret_desc = "\n".join([first.strip()] + body + [h for h, _ in entries[1:]]).strip()
            i = j
            continue
        if in_main:
            main.append(line)
        i += 1
    text = "\n".join(main).strip()
    if ret_desc is not None:
        type_tag = f"<type>{ret_type}</type>\n" if ret_type else ""
        ret_xml = f"<returns>\n{type_tag}<description>{ret_desc}</description>\n</returns>"
        text = f"<summary>{text}</summary>\n{ret_xml}" if text else ret_xml
    return (text or None), params


def _sorted_schema(value: Any, parent_key: str | None = None) -> Any:
    """key order of pydantic's GenerateJsonSchema.sort: alphabetical, except the members of `properties` (declaration
    order) and whatever sits under `default`; the schema travels inside OverridesState, so its byte order is part of the wire"""
    if isinstance(value, dict):
        keys = list(value) if parent_key in ("properties", "default") else sorted(value)
        return {k: _sorted_schema(value[k], None if parent_key == "default" and False else k) for k in keys}
    if isinstance(value, list):
        return [_sorted_schema(v, parent_key) for v in value]
    return value


def _is_context_annotation(ann: Any) -> bool:
    if isinstance(ann, str):
        return ann.split("[")[0].split(".")[-1] in ("ToolContext", "RunContext")
    origin = getattr(ann, "__origin__", None) or ann
    return isinstance(origin, type) and issubclass(origin, ToolContext)


@dataclass
class Tool:
    """Minimal stand-in for pydantic_ai.Tool: the callable + its ToolDefinition (name, description, JSON schema of the
    parameters the model supplies).  reference: calfkit/_vendor/pydantic_ai/tools.py Tool + _function_schema.py — a first
    parameter ANNOTATED with the context type is injected and hidden from the schema (_takes_ctx, :236-270); parameter
    descriptions come from the docstring."""
    function: Callable[..., Any]
    takes_ctx: bool = False
    tool_def: ToolDefinition = field(init=False)

    def __post_init__(self) -> None:
        sig = inspect.signature(self.function)
        params = list(sig.parameters.values())
        try:
            import typing
            hints = typing.get_type_hints(self.function)
        except Exception:  # noqa: BLE001  (unresolvable forward references: fall back to the raw annotations)
            hints = {}
        if params and _is_context_annotation(hints.get(params[0].name, params[0].annotation)):
            self.takes_ctx = True
            params = params[1:]
        main, pdesc = _parse_docstring(inspect.getdoc(self.function), [p.name for p in params])
        fields = {}
        for p in params:
            ann = hints.get(p.name, p.annotation if p.annotation is not inspect.Parameter.empty else Any)
            default = ... if p.default is inspect.Parameter.empty else p.default
            fields[p.name] = (ann, pydantic.Field(default, description=pdesc[p.name]) if p.name in pdesc else default)
        model = pydantic.create_model(f"{self.function.__name__}_args", **fields)      # type: ignore[call-overload]
        schema = model.model_json_schema()
        schema.pop("title", None)
        for prop in schema.get("properties", {}).values():
            prop.pop("title", None)
        schema.setdefault("additionalProperties", False)
        schema.setdefault("properties", {})
        self.tool_def = ToolDefinition(name=self.function.__name__, parameters_json_schema=_sorted_schema(schema), description=main)


@dataclass
class BaseToolNodeDef(BaseToolNodeSchema, BaseNodeDef):
    _tool: Tool
    _template: ToolTemplate | None = None


class ToolNodeDef(BaseToolNodeDef):
    @classmethod
    def create_tool_node(cls, func: Callable[..., Any], subscribe_topics: str | list[str], publish_topic: str,
                         device_template: str | None = None) -> Self:
        if not isinstance(subscribe_topics, (list, tuple)):
            subscribe_topics = [subscribe_topics]
        tool = Tool(func)
        return cls(node_id=f"tool_{func.__name__}", tool_schema=tool.tool_def, subscribe_topics=subscribe_topics,
                   publish_topic=publish_topic, _tool=tool,
                   _template=ToolTemplate.from_format(device_template) if device_template else None)

    async def run(self, ctx: SessionRunContext, tool_call_id: str, source_node_name: str) -> NodeResult[State]:
        raise RuntimeError("ToolNodeDef.run is executed by the CUDA engine (ck_plan_tool_kernel); use process_batch")

    # ---- batch path ---------------------------------------------------------------------------------
    def configure_engine(self, engine) -> None:
        engine.set_tool_node(self.publish_topic, self._template)

    def _call_host(self, args_json: bytes, rec_bytes: memoryview, cols: np.ndarray, i: int) -> bytes:
        v = pydantic_core.from_json(args_json)
        if isinstance(v, str):
            v = pydantic_core.from_json(v)               # args_as_dict: JSON string -> dict
        kwargs = v or {}
        if self._tool.takes_ctx:
            def span(name: str) -> bytes:
                o, n = int(cols[COL[name + "_OFF"], i]), int(cols[COL[name + "_LEN"], i])
                return bytes(rec_bytes[o:o + n])
            deps = {"correlation_id": pydantic_core.from_json(b'"' + span("CORR") + b'"'),
                    "provided_deps": pydantic_core.from_json(span("PD"))}
            from calfkit.models import Deps
            hist = span("HIST")
            ctx = ToolContext(deps=Deps(**deps), agent_name=_jstr(span("ARG1")) if cols[COL["ARGKINDS"], i] & 2 else None,
                              tool_call_id=_jstr(span("ARG0")), tool_name=_jstr(span("TNAME")), run_id=deps["correlation_id"],
                              _messages_loader=lambda: ModelMessagesTypeAdapter.validate_json(hist))
            result = self._tool.function(ctx, **kwargs)
        else:
            result = self._tool.function(**kwargs)
        if inspect.isawaitable(result):
            result = _run_awaitable(result)      # `async def` tools (the reference awaits them, nodes/tool.py:64)
        return pydantic_core.to_json(result)

    def _host_results(self, n: int, args_of, record_of, cols: np.ndarray) -> tuple[list[bytes], set[int]]:
        """run the Python callable for every record that reached the tool; a tool that raises fails ITS record only (the
        reference handler would raise for that one message and FastStream would go on with the next): it is logged, gets a
        placeholder result and its publishes are dropped after the plan"""
        results: list[bytes] = []
        failed: set[int] = set()
        for i in range(n):
            if cols[COL["ACTION"], i] != CK_ACT_HOST_TOOL:
                results.append(b"")
                continue
            try:
                results.append(self._call_host(args_of(i), record_of(i), cols, i))
            except Exception:  # noqa: BLE001  (user code)
                logger.exception("record %d: tool %s raised; nothing is published for this record", i, self.name)
                failed.add(i)
                results.append(b"null")
        return results, failed

    def process_batch(self, engine, records: list[Record] | FetchArena, force_host: bool = False) -> list[Record]:
        """force_host: evaluate the Python callable even though the node has a device template — used for the records the
        template declined (`args` given as a JSON string, a non-string argument ...: the reference's args_as_dict / the
        callable itself handle those, nodes/tool.py:53-64), so nothing is dropped on the template path"""
        failed: set[int] = set()
        inb = submit_inbound(engine, records)
        if self._template is not None and not force_host:
            engine.tool_plan()
        else:
            blob, off, ln = engine.tool_args()
            cols = engine.columns()
            ovl = engine.overlay() if self._tool.takes_ctx else None     # the column spans refer to the canonical spelling of a record
            results, failed = self._host_results(inb.n, lambda i: blob[off[i]:off[i] + ln[i]].tobytes(),
                                                 lambda i: (memoryview(ovl[0])[int(ovl[1][i]):int(ovl[1][i]) + int(ovl[2][i])]
                                                            if ovl is not None and ovl[1][i] >= 0 else inb.value(i)), cols)
            aux_off = np.zeros(inb.n + 1, dtype=np.int64)
            np.cumsum([len(r) for r in results], out=aux_off[1:])
            engine.tool_plan(np.frombuffer(b"".join(results) or b"\0", dtype=np.uint8), aux_off)
        out = engine.fetch()
        declined = []
        for i in np.nonzero(out.cols[COL["STATUS"]] != CK_OK)[0]:
            if out.cols[COL["STATUS"], i] == CK_SKIPPED:        # not delivered to a consumer (a control / aborted batch)
                continue
            if out.cols[COL["STATUS"], i] == CK_UNSUPPORTED and out.cols[COL["ACTION"], i] == CK_ACT_RAISES and not force_host \
                    and self._template is not None:
                declined.append(int(i))                      # the template declined it: the host-tool path below takes over
                continue
            logger.error("record %d rejected: %s at byte %d", i, STATUS_NAMES[int(out.cols[COL["STATUS"], i])],
                         int(out.cols[COL["ERR"], i]))
        for i in np.nonzero((out.cols[COL["ACTION"]] == CK_ACT_RAISES) & (out.cols[COL["STATUS"]] == CK_OK))[0]:
            logger.error("record %d: the reference handler would raise here (bad input_args / empty call stack)", i)
        produced = []
        for p in out.publishes():
            if p.record in failed:
                continue
            corr = inb.correlation_ids[p.record]
            if corr is None and p.key is not None:
                corr = p.key.decode()
            produced.append(Record(p.topic, p.payload, p.key, corr))
        if declined:
            produced += self.process_batch(engine, [Record(self.subscribe_topics[0], inb.value(i).tobytes(), inb.keys[i], inb.correlation_ids[i])
                                                    for i in declined], force_host=True)
        return produced


def _run_awaitable(aw: Any) -> Any:
    """Drive an async tool to completion from the (synchronous) batch step: directly when no event loop is running in
    this thread, else on a short-lived worker thread with its own loop (Worker.run calls the batch step from inside its
    loop, where asyncio.run() is not allowed)."""
    import asyncio

    async def _wrap():
        return await aw
    try:
        asyncio.get_running_loop()
    except RuntimeError:
        return asyncio.run(_wrap())
    from concurrent.futures import ThreadPoolExecutor
    with ThreadPoolExecutor(max_workers=1) as ex:
        return ex.submit(asyncio.run, _wrap()).result()


def _jstr(raw: bytes) -> str:
    return pydantic_core.from_json(b'"' + raw + b'"')


def agent_tool(func: Callable[..., Any] | Callable[..., Awaitable[Any]] | None = None, *,
               device_template: str | None = None):
    """Decorator turning a function into a deployable tool node (reference nodes/tool.py:89-95):
    subscribes `tool.<name>.input`, publishes `tool.<name>.output`, node_id `tool_<name>`."""
    def make(f):
        return ToolNodeDef.create_tool_node(func=f, subscribe_topics=f"tool.{f.__name__}.input",
                                            publish_topic=f"tool.{f.__name__}.output", device_template=device_template)
    return make(func) if func is not None else make
