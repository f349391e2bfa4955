"""Fetch responses consumed by every host-path subscriber: an Agent node, a Python-tool node and the client's replies read
Kafka record batches decoded on the device exactly as they read the same records as Records.  The fetches are built by
the engine's record form (uncompressed and LZ4) and recompressed with gzip, zstd and snappy by the test helpers; every case
compares the fetch path with the Record path over the same records, in the same order.  Also: read_committed over
transactions, a corrupt batch and a truncated tail, and the conversations of a fan-out agent run end to end with every
topic a frame sink whose frames come back as fetches."""
import asyncio
import logging
import random
import re
import types

import pytest

import gzip_cases as gz
import kafka_snappy as ks
import kafka_txn as kt
from make_golden_lz4_batches import with_section

pytestmark = pytest.mark.gpu
TS = 1767225600123
CODECS = [None, "lz4", "gzip", "zstd", "snappy"]


@pytest.fixture(autouse=True)
def _cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def recompress(frame: bytes, codec: str) -> bytes:
    sec = frame[61:]
    if codec == "gzip":
        return with_section(frame, gz.gzip_bytes(sec), codec=1)
    if codec == "snappy":
        return with_section(frame, ks.xerial(sec, 4 << 10), codec=2)
    import zstd_ref as zr
    zr.need()
    return with_section(frame, zr.compress(sec, level=3), codec=4)


def frames_of(records, codec=None, per_frame=None) -> list[bytes]:
    """the records (value, key, correlation id) as RecordBatch v2 frames built by the engine's record form, `per_frame`
    records a frame (default: all in one); gzip, zstd and snappy frames are the uncompressed ones recompressed"""
    from calfkit.engine import BatchEngine
    eng = BatchEngine(0, max_records=1 << 12, max_in_bytes=16 << 20)
    try:
        eng.register_topics(["t"], num_partitions=0)
        if codec == "lz4":
            eng.set_frame_compression("lz4")
        out = []
        step = per_frame or max(len(records), 1)
        for a in range(0, len(records), step):
            eng.encode_frames_records("t", [(r.value, r.key, r.correlation_id) for r in records[a:a + step]], TS)
            fr = eng.fetch_frames()
            out += [fr.frame(i).tobytes() for i in range(len(fr))]
    finally:
        eng.close()
    return [recompress(f, codec) for f in out] if codec in ("gzip", "zstd", "snappy") else out


def fetch_of(records, codec=None, per_frame=None):
    from calfkit.engine.lane import FetchArena
    return FetchArena.of(b"".join(frames_of(records, codec, per_frame)))


_TS_RE = re.compile(rb'"timestamp":"[^"]*"')


def norm(recs):
    """produced records without the wall-clock timestamps the host stamps on model messages"""
    return [(r.topic, r.key, r.correlation_id, _TS_RE.sub(b'"timestamp":"T"', r.value)) for r in recs]


@pytest.fixture()
def frozen(monkeypatch):
    """the same frame ids on both paths: the agent step's clock and seed fixed"""
    import calfkit.nodes.agent as A
    monkeypatch.setattr(A, "time", types.SimpleNamespace(time_ns=lambda: TS * 1_000_000))
    monkeypatch.setattr(A.np.random, "SeedSequence", lambda: types.SimpleNamespace(entropy=987654321))


def make_tools(n=8, ctx_every=3):
    from calfkit import agent_tool
    from calfkit.models import ToolContext

    def plain(j):
        def f(x: str) -> str:
            return f"T{j}<{x}>"
        return f

    def contextual(j):
        def f(ctx: ToolContext, x: str) -> str:
            return f"T{j}<{x}:{ctx.deps.provided_deps['tenant']}:{ctx.tool_call_id}>"
        return f
    tools = []
    for j in range(n):
        f = contextual(j) if j % ctx_every == 2 else plain(j)
        f.__name__ = f.__qualname__ = f"tool_{j}"
        f.__doc__ = f"tool {j}"
        tools.append(agent_tool(f))
    return tools


def scripted(seen: list):
    """first turn "i:k" -> k tool calls (ids c<i>-<j>); a turn carrying tool returns -> their contents as text"""
    from calfkit.models.messages import ModelMessagesTypeAdapter, ModelResponse, TextPart, ToolCallPart, ToolReturnPart
    from calfkit.nodes import FunctionModelClient

    def llm(messages, tools):
        seen.append(_TS_RE.sub(b'"timestamp":"T"', ModelMessagesTypeAdapter.dump_json(messages)))
        rets = [p for p in getattr(messages[-1], "parts", []) if isinstance(p, ToolReturnPart)]
        if rets:
            return ModelResponse(parts=[TextPart(content=" | ".join(str(r.content) for r in rets))])
        i, k = (int(x) for x in messages[0].parts[0].content.split(":"))
        if k == 0:
            return ModelResponse(parts=[TextPart(content=f"direct {i}")])
        return ModelResponse(parts=[ToolCallPart(tool_name=tools[j].name, args={"x": f"v{i}"}, tool_call_id=f"c{i}-{j}") for j in range(k)])
    return FunctionModelClient(llm)


def first_turns(n, calls, reply_topic=None):
    """n client envelopes for planner.input, conversation i asking for calls(i) tool calls, as the client publishes them"""
    from calfkit import Client

    async def go():
        client = Client.connect(reply_topic=reply_topic)
        for i in range(n):
            await client.invoke_node(f"{i}:{calls(i)}", "planner.input", deps={"tenant": f"t{i}"}, correlation_id=f"corr-{i:03d}")
        recs = client.broker.poll_batch(("planner.input",), 10000)
        client._dispatcher.close()
        return recs
    return asyncio.run(go())


def agent(seen, tools, **kw):
    from calfkit import Agent
    return Agent("planner", subscribe_topics="planner.input", publish_topic="planner.output", model_client=scripted(seen),
                 tools=tools, **kw)


@pytest.mark.parametrize("codec", CODECS)
def test_agent_first_turns_and_tool_returns(codec, frozen):
    """first turns and the tool returns of fan-outs of 1 to 8 calls: the same produced records, gate stats and model
    histories from a fetch as from Records"""
    from calfkit.worker.worker import engine_for
    tools = make_tools()
    seen_a, seen_b = [], []
    a, b = agent(seen_a, tools), agent(seen_b, tools)
    ea, eb = engine_for(a), engine_for(b)
    turns = first_turns(24, lambda i: 1 + i % 8)
    out_a = a.process_batch(ea, turns)
    out_b = b.process_batch(eb, fetch_of(turns, codec, per_frame=5))
    assert norm(out_a) == norm(out_b) and len(out_a) > 24
    assert ea.gate_stats() == eb.gate_stats()
    returns = []
    for t in tools:
        calls = [r for r in out_a if r.topic == t.subscribe_topics[0]]
        returns += [r for r in t.process_batch(engine_for(t), calls) if r.topic == "planner.input"]
    assert len(returns) == sum(1 + i % 8 for i in range(24))
    random.Random(7).shuffle(returns)
    for lo, hi in ((0, 30), (30, 31), (31, len(returns))):
        got_a = a.process_batch(ea, returns[lo:hi])
        got_b = b.process_batch(eb, fetch_of(returns[lo:hi], codec, per_frame=7))
        assert norm(got_a) == norm(got_b)
        assert ea.gate_stats() == eb.gate_stats()
    assert seen_a == seen_b and len(seen_a) == 48
    assert a._gate_stamp == b._gate_stamp and ea.gate_stats()["live"] == 0


@pytest.mark.parametrize("codec", [None, "lz4", "zstd"])
def test_python_tool_node(codec, frozen):
    """a plain and a contextual Python tool: the same produced records from a fetch as from Records"""
    from calfkit.worker.worker import engine_for
    tools = make_tools(3)                      # tool_2 takes a ToolContext
    a = agent([], tools)
    calls = [r for r in a.process_batch(engine_for(a), first_turns(12, lambda i: 3)) if r.topic.startswith("tool.")]
    for t in tools:
        mine = [r for r in calls if r.topic == t.subscribe_topics[0]]
        assert len(mine) == 12
        want = t.process_batch(engine_for(t), mine)
        got = t.process_batch(engine_for(t), fetch_of(mine, codec, per_frame=4))
        assert norm(want) == norm(got) and len(got) == 24


def _replies(frozen_reply_topic):
    """replies to the client: conversations that the model answers directly, half of them as DataParts"""
    from calfkit.worker.worker import engine_for
    turns = first_turns(16, lambda i: 0, reply_topic=frozen_reply_topic)
    out = []
    for kind in (str, dict):
        a = agent([], [], final_output_type=kind)
        part = turns[:8] if kind is str else turns[8:]
        out += [r for r in a.process_batch(engine_for(a), part) if r.topic == frozen_reply_topic]
    assert len(out) == 16
    return out


@pytest.mark.parametrize("codec", [None, "lz4", "snappy"])
def test_client_replies_from_a_fetch(codec, frozen):
    from calfkit import Client
    from calfkit.broker import Record
    from calfkit.client.batch_reply import BatchReplyDecoder
    from calfkit.client.deserialize import _UNSET
    from calfkit.engine import BatchEngine
    replies = _replies("replies.c")
    eng = BatchEngine(0, max_records=1 << 10, max_in_bytes=8 << 20)
    try:
        dec = BatchReplyDecoder(eng)
        for mode in (_UNSET, str, int):
            def flat(res):
                return [(r.correlation_id, r.output, type(r.error).__name__, str(r.error)) for r in res]
            want, got = flat(dec.decode(replies, mode)), flat(dec.decode(fetch_of(replies, codec, per_frame=3), mode))
            assert want == got and len(got) == 16
    finally:
        eng.close()

    async def go():
        client = Client.connect(reply_topic="replies.c")
        futs = {f"corr-{i:03d}": client._dispatcher.expect(f"corr-{i:03d}") for i in range(16)}
        client.broker.produce_fetch("replies.c", b"".join(frames_of(replies, codec, per_frame=3)))
        n = await client._dispatcher.drain(client.broker)
        got = {c: f.result().context.state.final_output_parts[0] for c, f in futs.items() if f.done()}
        had_engine = client._dispatcher._engine is not None
        await client.close()
        plain = Client.connect(reply_topic="replies.p")               # only Records: no engine is ever created
        plain.broker.produce_batch([Record("replies.p", r.value, r.key, r.correlation_id) for r in replies])
        assert await plain._dispatcher.drain(plain.broker) == 16 and plain._dispatcher._engine is None
        await plain.close()
        return n, got, had_engine
    n, got, had_engine = asyncio.run(go())
    assert n == 16 and had_engine and len(got) == 16
    assert [getattr(got[f"corr-{i:03d}"], "text", None) or got[f"corr-{i:03d}"].data for i in range(16)] == [f"direct {i}" for i in range(16)]


def _worker_agent_over(fetch_bytes, entries, level, caplog):
    from calfkit import Client, Worker
    seen = []
    client = Client.connect()
    a = agent(seen, [])
    client.broker.produce_fetch("planner.input", fetch_bytes, aborted_transactions=entries)
    worker = Worker(client, nodes=[a], extra_subscribe_kwargs={"isolation_level": level})
    with caplog.at_level(logging.ERROR):
        asyncio.run(worker.run(until_idle=True))
    stats = dict(worker.stats)
    worker.close()
    prompts = sorted(int(re.search(rb'"content":"(\d+):0"', s).group(1)) for s in seen)
    return prompts, stats


def test_agent_read_committed_over_transactions(caplog):
    turns = first_turns(30, lambda i: 0)
    frames = frames_of(turns, per_frame=3)
    fetch, entries, aborted = kt.transactional_fetch(frames, 0.4, seed=17)
    assert any(aborted) and not all(aborted)
    markers = sum(1 for s, _e in kt.batches(fetch) if fetch[s + 22] & kt.CONTROL)
    committed = [i for f, ab in enumerate(aborted) if not ab for i in range(3 * f, 3 * f + 3)]
    prompts, stats = _worker_agent_over(fetch, entries, "read_committed", caplog)
    assert prompts == committed                                   # the model never sees an aborted record
    assert stats["skipped"] == 3 * sum(aborted) + markers and stats["records"] == 30 + markers
    prompts, stats = _worker_agent_over(fetch, entries, "read_uncommitted", caplog)
    assert prompts == list(range(30)) and stats["skipped"] == markers
    assert "rejected" not in caplog.text


def test_agent_fetch_with_a_corrupt_batch_and_a_truncated_tail(caplog):
    turns = first_turns(20, lambda i: 0)
    frames = frames_of(turns, codec="lz4", per_frame=4)
    bad = bytearray(frames[2])
    bad[-3] ^= 0x5A                                               # the CRC32C no longer matches
    fetch = b"".join(frames[:2]) + bytes(bad) + b"".join(frames[3:]) + frames[0][:40]
    prompts, stats = _worker_agent_over(fetch, None, "read_uncommitted", caplog)
    assert prompts == [i for i in range(20) if not 8 <= i < 12]
    assert caplog.text.count("rejected") == 4 and stats["records"] == 20 and stats["skipped"] == 0


def _conversations(frame_topics: bool, compression=None, n=20):
    from calfkit import Agent, Client, Worker, agent_tool
    from calfkit.models import ToolContext
    from calfkit.models.messages import ModelResponse, TextPart, ToolCallPart, ToolReturnPart
    from calfkit.nodes import FunctionModelClient

    @agent_tool
    def tool_a(x: str) -> str:
        """a"""
        return f"A<{x}>"

    @agent_tool(device_template="B<{x}>")
    def tool_b(x: str) -> str:
        """b"""
        return f"B<{x}>"

    @agent_tool
    def tool_c(ctx: ToolContext, x: str) -> str:
        """c: contextual tool reading provided deps"""
        return f"C<{x}:{ctx.deps.provided_deps['tenant']}>"

    def llm(messages, tools):
        rets = [p for p in getattr(messages[-1], "parts", []) if isinstance(p, ToolReturnPart)]
        if rets:
            return ModelResponse(parts=[TextPart(content=" | ".join(str(r.content) for r in rets))])
        return ModelResponse(parts=[ToolCallPart(tool_name=t.name, args={"x": "v"}) for t in tools])

    async def go():
        client = Client.connect(**({"compression_type": compression} if compression else {}))
        broker = client.broker
        agent_node = Agent("planner", subscribe_topics="planner.input", publish_topic="planner.output",
                           model_client=FunctionModelClient(llm), tools=[tool_a, tool_b, tool_c])
        nframes = [0]
        if frame_topics:
            def back(topic, part, frame, n_records):
                nframes[0] += 1
                broker.produce_fetch(topic, frame.tobytes())
            for t in ("planner.input", "planner.output", client.reply_topic) + tuple(
                    x for tool in (tool_a, tool_b, tool_c) for x in (tool.subscribe_topics[0], tool.publish_topic)):
                broker.frame_sink(t, back)
        worker = Worker(client, nodes=[agent_node, tool_a, tool_b, tool_c])
        hs = [await client.invoke_node("go", "planner.input", deps={"tenant": f"t{i}"}) for i in range(n)]
        await worker.run(until_idle=True)
        # the frames a step hands its sinks come back as fetches after it, the way a Kafka consumer's next poll sees them
        for _ in range(100):
            if not any(broker.arenas.get(t) for t in broker.subscribed):
                break
            await worker.run(until_idle=True)
        res = [await h.result(timeout=5) for h in hs]
        stats = dict(worker.stats)
        live = agent_node._ck_engine.gate_stats()["live"]
        worker.close()
        await client.close()
        return [(r.output, len(r.message_history)) for r in res], stats, live, nframes[0]
    return asyncio.run(go())


@pytest.mark.parametrize("compression", [None, "lz4"])
def test_fanout_conversations_end_to_end_over_frames(compression, caplog):
    """every topic, the client's reply topic included, is a frame sink whose frames come back as fetches: each
    conversation completes as it does over plain queues, nothing is rejected and the gate ends empty"""
    plain, _s, _l, _n = _conversations(False)
    with caplog.at_level(logging.WARNING):
        got, stats, live, nframes = _conversations(True, compression)
    assert got == plain and [o for o, _h in got] == [f"A<v> | B<v> | C<v:t{i}>" for i in range(20)]
    assert nframes > 0 and stats["rejected"] == 0 and live == 0
    bad = [r.getMessage() for r in caplog.records if r.levelno >= logging.WARNING and r.name.startswith("calfkit")]
    assert not bad, bad[:5]
