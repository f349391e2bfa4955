"""BASELINE.json configs[0]: the reference's quickstart (examples/quickstart/{weather_tool,agent_service,
invoke}.py) — weather_agent + get_weather tool, 100 events — on the GPU worker.

Differences from the reference scripts, all outside the hot path: the three processes share one
in-memory broker (no Kafka broker in the image) and the LLM is a deterministic function model
(no network): it asks for `get_weather(location=<city in the prompt>)` and then repeats the tool's answer.
"""
import asyncio
import os
import re
import sys
import time

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "..", "calfkit-sdk_b200"))

from calfkit import Agent, Client, Worker, agent_tool  # noqa: E402
from calfkit.models.messages import ModelResponse, TextPart, ToolCallPart, ToolReturnPart  # noqa: E402
from calfkit.nodes import FunctionModelClient  # noqa: E402


@agent_tool                      # host tool: arbitrary Python (add device_template=... to run it on the GPU)
def get_weather(location: str) -> str:
    """Get the current weather at a location"""
    return f"It's sunny in {location}"


def fake_llm(messages, tools):
    last = messages[-1]
    returns = [p for p in getattr(last, "parts", []) if isinstance(p, ToolReturnPart)]
    if returns:
        return ModelResponse(parts=[TextPart(content=str(returns[0].content))], model_name="function:fake_llm")
    prompt = next(p.content for m in messages for p in m.parts if getattr(p, "part_kind", "") == "user-prompt")
    city = re.search(r"in (.+?)\?", prompt).group(1)
    return ModelResponse(parts=[ToolCallPart(tool_name="get_weather", args={"location": city})], model_name="function:fake_llm")


async def main(n_events: int = 100) -> list[str]:
    client = Client.connect("localhost")
    agent = Agent("weather_agent", system_prompt="You are a helpful assistant.", subscribe_topics="weather_agent.input",
                  model_client=FunctionModelClient(fake_llm), tools=[get_weather])
    worker = Worker(client, nodes=[agent, get_weather])
    cities = ["Tokyo", "Paris", "São Paulo", "Kraków", "北京"]
    t0 = time.perf_counter()
    handles = [await client.invoke_node(f"What's the weather in {cities[i % len(cities)]}?", "weather_agent.input")
               for i in range(n_events)]
    await worker.run(until_idle=True)
    results = [await h.result(timeout=5) for h in handles]
    dt = time.perf_counter() - t0
    outs = [r.output for r in results]
    print(f"{n_events} events in {dt * 1e3:.1f} ms; first: {outs[0]!r}; history of first: {len(results[0].message_history)} messages")
    await client.close()
    return outs


if __name__ == "__main__":
    asyncio.run(main(int(sys.argv[1]) if len(sys.argv) > 1 else 100))
