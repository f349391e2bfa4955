"""Config 1 (BASELINE.json configs[0]) end to end on the GPU worker: quickstart weather agent +
get_weather tool, 100 events through Client -> Worker.run -> Agent/ToolNode batch plans -> reply."""
import asyncio
import importlib.util
import os

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _skip_without_cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def test_quickstart_100_events():
    _skip_without_cuda()
    spec = importlib.util.spec_from_file_location("quickstart", os.path.join(ROOT, "examples", "quickstart", "run_quickstart.py"))
    qs = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(qs)
    outs = asyncio.run(qs.main(100))
    cities = ["Tokyo", "Paris", "São Paulo", "Kraków", "北京"]
    assert outs == [f"It's sunny in {cities[i % 5]}" for i in range(100)]


def test_parallel_fanout_three_tools_and_aggregation():
    """reference tests/test_concurrent_tool_calls.py:12-36: one model turn asks for 3 tools at once; every
    tool's value must reach the final answer and the last tool-call message carries 3 calls."""
    _skip_without_cuda()
    from calfkit import Agent, Client, Worker, agent_tool
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

    from calfkit.models import ToolContext

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
        client = Client.connect()
        agent = Agent("planner", subscribe_topics="planner.input", publish_topic="planner.output",
                      model_client=FunctionModelClient(llm), tools=[tool_a, tool_b, tool_c])
        worker = Worker(client, nodes=[agent, tool_a, tool_b, tool_c])
        hs = [await client.invoke_node("go", "planner.input", deps={"tenant": f"t{i}"}) for i in range(20)]
        await worker.run(until_idle=True)
        res = [await h.result(timeout=5) for h in hs]
        # publish_topic carries every handler return value (worker/worker.py:52-53): per conversation the inbound envelope
        # of the fan-out turn (list[Call] returns the envelope it was given, nodes/base.py:88), two Silent returns while the
        # aggregation is incomplete, and the final ReturnCall envelope
        outs = client.broker.poll_batch(("planner.output",), 1000)
        await client.close()
        return res, outs

    res, outs = asyncio.run(go())
    import json as _json
    by_corr: dict = {}
    for rec in outs:
        e = _json.loads(rec.value)
        by_corr.setdefault(e["context"]["deps"]["correlation_id"], []).append(e)
    assert len(by_corr) == 20 and all(len(v) == 4 for v in by_corr.values()), {k: len(v) for k, v in by_corr.items()}
    for envs in by_corr.values():
        first = [e for e in envs if not e["context"]["state"]["tool_calls"]]
        assert len(first) == 1 and first[0]["context"]["state"]["uncommitted_message"] is not None      # the untouched inbound envelope
        assert sum(1 for e in envs if e["context"]["state"]["final_output_parts"]) == 1
    for i, r in enumerate(res):
        assert r.output == f"A<v> | B<v> | C<v:t{i}>"
        calls = [m for m in r.message_history if getattr(m, "kind", "") == "response" and m.tool_calls]
        assert len(calls[-1].tool_calls) == 3


def _three_tools():
    from calfkit import agent_tool

    @agent_tool
    def tool_a(x: str) -> str:
        """a"""
        return f"A<{x}>"

    @agent_tool(device_template="B<{x}>")
    def tool_b(x: str) -> str:
        """b"""
        return f"B<{x}>"

    return tool_a, tool_b


def test_sequential_only_mode_routes_one_call_at_a_time():
    """Agent(sequential_only_mode=True) (reference nodes/agent.py:94-108,179-192): the pending calls of one
    model turn go out one by one as single Calls; no aggregation batch exists; same final answer."""
    _skip_without_cuda()
    from calfkit import Agent, Client, Worker
    from calfkit.models.messages import ModelResponse, TextPart, ToolCallPart, ToolReturnPart
    from calfkit.nodes import FunctionModelClient
    tool_a, tool_b = _three_tools()
    turns = []

    def llm(messages, tools):
        rets = [p for p in getattr(messages[-1], "parts", []) if isinstance(p, ToolReturnPart)]
        turns.append(len(rets))
        if rets:
            return ModelResponse(parts=[TextPart(content=" | ".join(str(r.content) for r in rets))])
        return ModelResponse(parts=[ToolCallPart(tool_name=t.name, args={"x": "v"}) for t in tools])

    async def go():
        client = Client.connect()
        agent = Agent("planner", subscribe_topics="planner.input", publish_topic="planner.output",
                      model_client=FunctionModelClient(llm), tools=[tool_a, tool_b], sequential_only_mode=True)
        worker = Worker(client, nodes=[agent, tool_a, tool_b])
        hs = [await client.invoke_node("go", "planner.input") for i in range(8)]
        await worker.run(until_idle=True)
        res = [await h.result(timeout=5) for h in hs]
        assert not agent._pending_batches
        await client.close()
        return res

    res = asyncio.run(go())
    for r in res:
        assert r.output == "A<v> | B<v>"
    assert turns.count(0) == 8 and turns.count(2) == 8          # the model ran twice per event, never on a partial batch


def test_all_tools_invalid_tailcall_retry():
    """The model asks only for tools that do not exist -> every call gets a RetryPromptPart and the agent
    TailCalls itself (reference nodes/agent.py:140-175); the next turn sees the retry prompts."""
    _skip_without_cuda()
    from calfkit import Agent, Client, Worker
    from calfkit.models.messages import ModelResponse, RetryPromptPart, TextPart, ToolCallPart
    from calfkit.nodes import FunctionModelClient
    tool_a, tool_b = _three_tools()

    def llm(messages, tools):
        retries = [p for p in getattr(messages[-1], "parts", []) if isinstance(p, RetryPromptPart)]
        if retries:
            return ModelResponse(parts=[TextPart(content=f"gave up after {len(retries)} retry prompts: {retries[0].tool_name}")])
        return ModelResponse(parts=[ToolCallPart(tool_name="nope", args={}), ToolCallPart(tool_name="nada", args={})])

    async def go():
        client = Client.connect()
        agent = Agent("planner", subscribe_topics="planner.input", publish_topic="planner.output",
                      model_client=FunctionModelClient(llm), tools=[tool_a, tool_b])
        worker = Worker(client, nodes=[agent, tool_a, tool_b])
        hs = [await client.invoke_node("go", "planner.input") for i in range(5)]
        await worker.run(until_idle=True)
        res = [await h.result(timeout=5) for h in hs]
        await client.close()
        return res

    for r in asyncio.run(go()):
        assert r.output == "gave up after 2 retry prompts: nope"


def test_worker_fast_path_arenas_match_oracle():
    """Row g: polled batches land as pinned arenas, run through the pipelined lanes of a device-template tool node and come
    out as publish batches — byte-exact against the oracle, bounded polls (records AND bytes), the records the template
    declines (args as a JSON string / non-string argument) re-run through the host tool, nothing lost."""
    _skip_without_cuda()
    import numpy as np
    import tools_def
    from calfkit import Client, Worker, agent_tool, synth
    from calfkit.engine.lane import Arena, PinnedPool
    from oracle import port

    recs = synth.tool_events(3000, seed=31) + synth.tool_events(300, seed=32, size=None, full_history=True)
    # OpenAI-style args (a JSON string) and a numeric argument: the device template declines both
    recs[7] = recs[7].replace(b'"args":{"location":"', b'"args":"{\\"location\\":\\"').replace(b'"},"tool_call_id"', b'\\"}","tool_call_id"', 1)
    recs[11] = recs[11][:recs[11].index(b'"args":{"location":')] + b'"args":{"location":42}' + recs[11][recs[11].index(b',"tool_call_id"'):]
    recs[13] = b"{ " + recs[13][1:]                       # non-canonical spelling: canonicalised on the device
    recs[17] = recs[17][:200]                              # truncated: json_invalid, reported, nothing published
    node_def = agent_tool(tools_def.get_weather, device_template="It's sunny in {location}")
    client = Client.connect("localhost")
    pool = PinnedPool()
    client.broker.produce_arena("tool.get_weather.input", Arena.pack(recs, pool))
    got: dict[str, list] = {"weather_agent.input": [], "tool.get_weather.output": []}
    for t in got:
        client.broker.sink(t, lambda b, idx, t=t: got[t].extend((k, p) for (_t, k, p, _j) in b.iter_records(idx)))
    worker = Worker(client, nodes=[node_def], batch_records=512, batch_bytes=400_000, lanes=3, route_topics=["weather_agent.input"])
    asyncio.run(worker.run(until_idle=True))
    # host fallbacks are produced per record
    for t in got:
        got[t] += [(r.key, r.value) for r in client.broker.poll_batch((t,), 100)]
    node = port.ToolNode.of(tools_def.get_weather)
    want: dict[str, list] = {t: [] for t in got}
    for r in recs:
        try:
            for (tp, k, _c, pl) in port.tool_node_event(node, r):
                want[tp].append((k, pl))
        except Exception:  # noqa: BLE001  (the invalid record)
            pass
    for t in got:
        assert sorted(got[t], key=lambda x: x[1]) == sorted(want[t], key=lambda x: x[1]), t
    assert worker.stats["records"] == len(recs) and worker.stats["host_fallback"] == 2 and worker.stats["rejected"] == 3
    assert worker.stats["steps"] >= 7                     # 3300 records in polls of <= 512 records / 400 kB
    worker.close()


def test_quickstart_with_device_template_goes_through_the_fast_path():
    _skip_without_cuda()
    spec = importlib.util.spec_from_file_location("quickstart2", os.path.join(ROOT, "examples", "quickstart", "run_quickstart.py"))
    qs = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(qs)
    from calfkit import agent_tool
    qs.get_weather = agent_tool(qs.get_weather._tool.function, device_template="It's sunny in {location}")
    outs = asyncio.run(qs.main(60))
    cities = ["Tokyo", "Paris", "São Paulo", "Kraków", "北京"]
    assert outs == [f"It's sunny in {cities[i % 5]}" for i in range(60)]
