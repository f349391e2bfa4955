"""Tool plans whose pieces fall at any byte of the payload: call ids and template arguments shorter than a 16-byte
vector (an empty argument included), 1-byte template literals, frame overrides and existing results, so that many
output vectors overlap three or more segments of the splice.  Every publish is compared with the oracle.  The last
case needs more segments than a descriptor holds and goes, record by record, to the global-memory planner."""
import json
import random
import string

import pytest

pytestmark = pytest.mark.gpu

TOPICS = ["tool.get_weather.input", "tool.get_weather.output", "weather_agent.input"]
IDS = ["a", "b7", "c_1", "call", "id_12", "x" * 7, "call_12", "q" * 9, "call_0123", "k" * 11, "z" * 13, "call_abcdef01",
       "y" * 15, "w" * 16, "call_1273d27b0476"]                  # 1 .. 17 bytes; today's configs use 17
VALUES = ["", "P", "Ab", "Rome", "Paris", "Zürich", 'say "hi"', "a\\b", "Reykjavík, Iceland", "x" * 37]


@pytest.fixture(scope="module")
def engine():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from calfkit.engine import BatchEngine
    e = BatchEngine(device=0, max_records=1 << 12, max_in_bytes=16 << 20)
    e.register_topics(TOPICS, num_partitions=8)
    yield e
    e.close()


def _respell(rec: bytes, call_id: str, args: dict, *, overrides: bool, existing: bool) -> bytes:
    """The tool-stage record `rec` with its pending call renamed to `call_id` and given `args`; optionally frame
    overrides on the current frame and a result already present for the call; canonical again through the oracle."""
    from oracle import port
    obj = json.loads(rec)
    st = obj["context"]["state"]
    (old, part), = st["tool_calls"].items()
    part["tool_call_id"] = call_id
    part["args"] = args
    st["tool_calls"] = {call_id: part}
    if existing:
        st["tool_results"] = {call_id: {"return_value": "stale", "content": None, "metadata": {"tool_call_id": call_id},
                                        "kind": "tool-return"}}
    top = obj["internal_workflow_state"]["call_stack"]["_internal_list"][-1]
    top["input_args"][0] = call_id
    if overrides:
        top["overrides"] = {"override_agent_tools": None}
    return port.encode(port.decode(json.dumps(obj, ensure_ascii=False).encode()))


def _records(n: int, seed: int, make_args) -> list[bytes]:
    from calfkit import synth
    rng = random.Random(seed)
    base = synth.tool_events(n // 2, seed=seed, size=None) + synth.tool_events(n - n // 2, seed=seed + 1)
    out = []
    for k, r in enumerate(base):
        cid = IDS[k % len(IDS)] if k < 4 * len(IDS) else "".join(rng.choices(string.ascii_lowercase + "_", k=rng.randrange(1, 18)))
        out.append(_respell(r, cid, make_args(rng, k), overrides=k % 3 == 1, existing=k % 5 == 2))
    return out


def _check(engine, recs, node):
    from oracle import port
    from calfkit import synth
    b = synth.pack(recs)
    out = engine.run_tool_batch(b.data, b.offsets)
    assert (out.cols[0] == 0).all()
    got = [(p.topic, p.key, p.payload) for p in out.publishes()]
    want = [(t, k, pl) for r in recs for (t, k, _c, pl) in port.tool_node_event(node, r)]
    assert len(got) == len(want) == 2 * len(recs)
    for i in range(len(recs)):
        assert got[2 * i:2 * i + 2] == want[2 * i:2 * i + 2], (i, recs[i][:120])


@pytest.mark.parametrize("fmt", ["It's sunny in {location}", "{location}"])
def test_short_ids_and_arguments_match_oracle(engine, fmt):
    from oracle import port
    from calfkit.engine import ToolTemplate

    def get_weather(location: str) -> str:
        return fmt.format(location=location)
    engine.set_tool_node("tool.get_weather.output", ToolTemplate.from_format(fmt))
    recs = _records(600, 71, lambda rng, k: {"location": VALUES[k % len(VALUES)] if k < 300 else rng.choice(VALUES)})
    _check(engine, recs, port.ToolNode(get_weather, "tool_get_weather", [TOPICS[0]], TOPICS[1]))


def test_more_pieces_than_a_descriptor_holds_match_oracle(engine):
    """A template of six parts (four adjacent arguments): with frame overrides the splice has 17 pieces, one more than a
    descriptor holds, so those records take the global-memory planner; without overrides they stay on the staged path."""
    from oracle import port
    from calfkit.engine import ToolTemplate

    def concat(a: str, b: str, c: str, d: str) -> str:
        return a + b + c + d
    engine.set_tool_node("tool.get_weather.output", ToolTemplate([0, 1, 1, 1, 1, 0], [b'"', b"a", b"b", b"c", b"d", b'"']))
    recs = _records(200, 73, lambda rng, k: {key: rng.choice(VALUES) for key in ("d", "b", "a", "c")})

    def pieces(r: bytes) -> int:           # non-empty pieces of the splice (ck_plan_tool2_one)
        obj = json.loads(r)
        st, top = obj["context"]["state"], obj["internal_workflow_state"]["call_stack"]["_internal_list"][-1]
        (part,) = st["tool_calls"].values()
        return (2 if st["tool_results"] else 4) + 2 + sum(1 for v in part["args"].values() if v) + 3 + \
            (2 if top["overrides"] is not None else 0) + 2
    n = [pieces(r) for r in recs]
    assert sum(k > 16 for k in n) >= 10 and sum(k <= 16 for k in n) >= 10
    _check(engine, recs, port.ToolNode(concat, "tool_get_weather", [TOPICS[0]], TOPICS[1]))
