"""Cost of one Agent step over tool returns as Records and as fetch responses (uncompressed and LZ4).

An Agent with 8 Python tools fans each of N conversations out to 4 of them (a scripted model, no network); the tool
nodes' returns for `planner.input` are collected once.  They are then consumed in three forms, one Agent and engine per
leg, the legs alternating:
  records    the returns as Records: pack + engine.submit (what poll_batch hands a host node)
  fetch      the same records as one fetch response of uncompressed RecordBatch v2 frames of about 64 KB built by the
             engine's record form (what a frame-sink producer writes): engine.submit_recordbatch, values read in place
  fetch_lz4  the same with LZ4 frames, decoded on the device (a warp per batch)
Before every timed step the leg's Agent processes the first turns again (untimed), so the step's returns complete real
fan-outs: the device gate merges them and the model is called once per conversation.  The timed region is
Agent.process_batch, which ends in a device synchronise (its results are copied back).  This path is bound by the host
LLM boundary (one model call and one State validation per completed conversation).  Prints one JSON line with the card
name and power limit read in the same run.

    python scripts/quick_agent_fetch.py [conversations] [reps]
"""
import asyncio
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "calfkit-sdk_b200"))
TS = 1767225600123


def main(n: int = 512, reps: int = 15) -> None:
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("quick_agent_fetch: no CUDA device")
    from calfkit import Agent, Client, agent_tool
    from calfkit.engine import BatchEngine
    from calfkit.engine.lane import FetchArena
    from calfkit.models.messages import ModelResponse, TextPart, ToolCallPart, ToolReturnPart
    from calfkit.nodes import FunctionModelClient
    from calfkit.worker.worker import engine_for

    def make(j):
        def f(x: str) -> str:
            return f"T{j}<{x}>"
        f.__name__ = f.__qualname__ = f"tool_{j}"
        f.__doc__ = f"tool {j}"
        return agent_tool(f)
    tools = [make(j) for j in range(8)]

    def llm(messages, tools_):
        rets = [p for p in getattr(messages[-1], "parts", []) if isinstance(p, ToolReturnPart)]
        if rets:
            return ModelResponse(parts=[TextPart(content=" | ".join(str(r.content) for r in rets))])
        i = int(messages[0].parts[0].content)
        return ModelResponse(parts=[ToolCallPart(tool_name=tools_[(i + j) % 8].name, args={"x": f"v{i}"}, tool_call_id=f"c{i}-{j}")
                                    for j in range(4)])

    def agent():
        return Agent("planner", subscribe_topics="planner.input", publish_topic="planner.output",
                     model_client=FunctionModelClient(llm), tools=tools)

    async def turns():
        client = Client.connect()
        for i in range(n):
            await client.invoke_node(str(i), "planner.input", correlation_id=f"corr-{i:05d}")
        recs = client.broker.poll_batch(("planner.input",), 1 << 20)
        client._dispatcher.close()
        return recs
    first = asyncio.run(turns())
    src = agent()
    out = src.process_batch(engine_for(src), first)
    returns = []
    for t in tools:
        calls = [r for r in out if r.topic == t.subscribe_topics[0]]
        returns += [r for r in t.process_batch(engine_for(t), calls) if r.topic == "planner.input"]
    assert len(returns) == 4 * n

    def framed(codec):
        eng = BatchEngine(0, max_records=1 << 14, max_in_bytes=64 << 20)
        try:
            eng.register_topics(["planner.input"], num_partitions=0)
            eng.set_frame_compression(codec)
            eng.set_frame_bytes(64 << 10)
            eng.encode_frames_records("planner.input", [(r.value, r.key, r.correlation_id) for r in returns], TS)
            fr = eng.fetch_frames()
            return b"".join(fr.frame(i).tobytes() for i in range(len(fr)))
        finally:
            eng.close()
    forms = {"records": lambda: returns, "fetch": (lambda b=framed(None): FetchArena.of(b)),
             "fetch_lz4": (lambda b=framed("lz4"): FetchArena.of(b))}
    legs = {k: agent() for k in forms}
    times = {k: [] for k in forms}
    outputs = {}
    for rep in range(reps + 1):                      # rep 0 warms every leg up
        for k, node in legs.items():
            eng = engine_for(node)
            node.process_batch(eng, first)
            batch = forms[k]()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            produced = node.process_batch(eng, batch)
            dt = (time.perf_counter() - t0) * 1e3
            if rep:
                times[k].append(dt)
            outputs[k] = len(produced)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    res = {"conversations": n, "tool_returns": len(returns), "reps": reps, "gpu": q.stdout.strip(),
           "produced": outputs,
           "ms_per_step": {k: {"median": round(statistics.median(v), 3), "min": round(min(v), 3), "max": round(max(v), 3)}
                           for k, v in times.items()}}
    print(json.dumps(res))


if __name__ == "__main__":
    main(*(int(a) for a in sys.argv[1:3]))
