"""Tool plans whose pieces fall at any byte of the payload: call ids and template arguments shorter than a 16-byte
vector (an empty argument included), 1-byte template literals, frame overrides and existing results, so that many
output vectors overlap three or more segments of the splice.  Every publish is compared with the oracle.  A splice
never needs more segments than a descriptor holds: templates of more than five parts are refused.  Correlation ids of
every length and host results of every length put the key hash and the host's piece at every alignment; the engine has
2^31 - 1 partitions, so a publish's partition is 31 bits of its key's hash."""
import json
import random
import string

import pytest
from test_gpu_parity import ALL_BITS, _host_tool, _murmur2, _with_corr_ids, corr_ids_of_every_length

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
    e.register_topics(TOPICS, num_partitions=ALL_BITS)
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


def _check(engine, recs, node, host_tool=None):
    from oracle import port
    from calfkit import synth
    b = synth.pack(recs)
    out = engine.run_tool_batch(b.data, b.offsets, host_tool)
    assert (out.cols[0] == 0).all()
    got = [(p.topic, p.key, p.payload, p.partition) for p in out.publishes()]
    want = [(t, k, pl, -1 if k is None else (_murmur2(k) & 0x7FFFFFFF) % ALL_BITS)
            for r in recs for (t, k, _c, pl) in port.tool_node_event(node, r)]
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
    ids = corr_ids_of_every_length()            # the key hash through the plan's shared-memory window
    recs += _with_corr_ids(_records(len(ids), 72, lambda rng, k: {"location": rng.choice(VALUES)}), ids)
    _check(engine, recs, port.ToolNode(get_weather, "tool_get_weather", [TOPICS[0]], TOPICS[1]))


def _text(rng, n: int) -> str:
    """n characters of ASCII, multi-byte UTF-8 and characters JSON escapes"""
    return "".join(rng.choice(string.ascii_letters + ' "\\\n\t\x01\x1féü東😀') for _ in range(n))


def test_host_results_of_every_length_match_oracle(engine):
    """A host tool that returns its string argument: results of 0-300 characters with escapes and multi-byte UTF-8, so
    that the host's piece of the splice starts and ends at every alignment of the payload."""
    from oracle import port

    def get_weather(location: str) -> str:
        return location
    engine.set_tool_node("tool.get_weather.output", None)
    recs = _records(700, 81, lambda rng, k: {"location": _text(rng, k % 301 if k < 602 else rng.randrange(301))})
    _check(engine, recs, port.ToolNode(get_weather, "tool_get_weather", [TOPICS[0]], TOPICS[1]), _host_tool(get_weather))


def _pieces(r: bytes) -> int:
    """non-empty pieces of the splice (ck_plan_tool_one) under the five-part template "<{a}|{b}>" """
    obj = json.loads(r)
    st, top = obj["context"]["state"], obj["internal_workflow_state"]["call_stack"]["_internal_list"][-1]
    (cid, part), = st["tool_calls"].items()
    return (2 if cid in st["tool_results"] else 4) + 3 + sum(1 for v in part["args"].values() if v) + 3 + \
        (2 if top["overrides"] is not None else 0) + 2


def _concat_node():
    from oracle import port

    def concat(a: str, b: str) -> str:
        return f"<{a}|{b}>"
    return port.ToolNode(concat, "tool_get_weather", [TOPICS[0]], TOPICS[1])


def test_worst_case_splice_fills_a_descriptor_and_matches_oracle(engine):
    """A five-part template with three non-empty literals and non-empty arguments: records with frame overrides and no
    existing result have 16 pieces, as many as a descriptor holds (CK_TOOL_FIXED_PIECES + CK_TPL_MAX_PARTS)."""
    from calfkit.engine import ToolTemplate
    engine.set_tool_node("tool.get_weather.output", ToolTemplate.from_format("<{a}|{b}>"))
    recs = _records(200, 73, lambda rng, k: {key: rng.choice(VALUES[1:]) for key in ("b", "a")})
    n = [_pieces(r) for r in recs]
    assert max(n) == 16 and sum(k == 16 for k in n) >= 10 and sum(k < 16 for k in n) >= 10
    _check(engine, recs, _concat_node())


def test_six_part_template_is_refused(engine):
    """A descriptor has no room for a six-part template's splice: set_tool_node refuses it, and the node's template
    stays usable afterwards."""
    from calfkit.engine import ToolTemplate
    from calfkit.exceptions import EngineError
    with pytest.raises(EngineError, match="too many template parts"):
        engine.set_tool_node("tool.get_weather.output", ToolTemplate([0, 1, 1, 1, 1, 0], [b'"', b"a", b"b", b"c", b"d", b'"']))
    engine.set_tool_node("tool.get_weather.output", ToolTemplate.from_format("<{a}|{b}>"))
    _check(engine, _records(60, 79, lambda rng, k: {"a": rng.choice(VALUES), "b": rng.choice(VALUES)}), _concat_node())
