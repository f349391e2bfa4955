"""The agent's fan-out, the tool node and the aggregation gate chained on the device, hop by hop, on multi-call envelopes.

Each hop's device output is the next hop's input, and every hop is compared byte for byte with the oracle before the
next one runs, so a divergence is reported at the hop that caused it.  The conversations are post-LLM agent envelopes
with 1 to 128 tool calls in one batch, so the thread walker, the element-list walker and the warp walker (records of
CK_LONG_MIN = 16 KB and more) all resolve tool_calls[input_args[0]] / tool_results[input_args[0]] at every index:
call ids of 1-40 bytes with escapes and non-ASCII, several tools with their argument not the first key, frame and
state overrides, and "second round" conversations whose tool_results already hold answers of mixed kinds.

Envelopes with more than 128 tool calls are declined by the walker (its per-dict key tables, ck_walk.cuh CK_DICT_KEYS):
they get CK_UNSUPPORTED at the first hop and publish nothing, and nothing else in the batch may be declined."""
import asyncio
import json
import logging
import random
from collections import defaultdict

import pytest

from test_gpu_parity import _host_tool, _murmur2

pytestmark = pytest.mark.gpu

AGENT, AGENT_IN, AGENT_OUT = "planner", "planner.input", "planner.output"
FS = [1, 2, 3, 4, 5, 31, 32, 33, 40, 64, 65, 100, 128]
BAND = [129, 200]                           # more tool calls than the walker's dict tables hold (CK_DICT_KEYS = 128)
SEQ_FS = [3, 33, 64, 128]
NPART = 8
MS = 1767225600000
LONG = 16384                                # CK_LONG_MIN: records this long are walked one per warp
LX_MIN = 4                                  # CK_LX_MIN: the warp walker indexes dicts of this many entries in parallel
VALUES = ["", "P", "Rome", "Zürich", "北京", 'say "hi"', "a\\b", "tab\there\n", "\u0001ctl", "Reykjavík, Iceland", "x" * 37]
SPECIAL = ['"', "\\", "\u0001", "é", "北"]
OVERRIDES = '{"override_agent_tools":null}'


def get_weather(unit: str, location: str) -> str:
    return f"It's sunny in {location}"


def convert(note: str, to: str, amount: str) -> str:
    return f"{amount} → {to}"


def lookup(query: str) -> str:
    return f"user:{query}!"


def echo(text: str) -> str:
    return text


TOOLS = {"get_weather": (get_weather, "It's sunny in {location}"), "convert": (convert, "{amount} → {to}"),
         "lookup": (lookup, "user:{query}!"), "echo": (echo, "{text}")}
REGISTRY = {name: f"tool.{name}.input" for name in TOOLS}
TOPICS = list(REGISTRY.values()) + [f"tool.{name}.output" for name in TOOLS] + [AGENT_IN, AGENT_OUT]

# conversations the device declines at the first hop, by name; nothing else may be declined
DECLARED_UNSUPPORTED = [f"calls_{f}_{v}" for v in range(3) for f in BAND]


def _args(name: str, rng: random.Random) -> dict:
    v = lambda: rng.choice(VALUES)       # noqa: E731
    if name == "get_weather":
        return {"unit": rng.choice(["C", "°F"]), "location": v()}
    if name == "convert":
        return {"note": v(), "to": v(), "amount": v()}
    if name == "lookup":
        return {"query": v()}
    return {"text": v()}


def _call_ids(n: int, rng: random.Random) -> list[str]:
    """unique ids of 1-40 UTF-8 bytes; about a third start with a quote, a backslash, a control character or non-ASCII"""
    ids: list[str] = []
    seen = set()
    while len(ids) < n:
        head = (rng.choice(SPECIAL) if rng.random() < 0.3 else "") + format(len(ids), "x")
        want = rng.randrange(len(head.encode()), 41)
        cid = head + "".join(rng.choices("ghijkmnopqrstuvwxyz_-", k=want - len(head.encode())))
        if cid not in seen:
            seen.add(cid)
            ids.append(cid)
    return ids


def _result(kind: int, j: int, cid: str, tool: str) -> str:
    if kind == 0:
        return ('{"return_value":%s,"content":null,"metadata":{"tool_call_id":%s},"kind":"tool-return"}'
                % (json.dumps(f"done {j} — é\n"), json.dumps(cid)))
    if kind == 1:
        return ('{"content":"bad arguments","tool_name":%s,"tool_call_id":%s,"timestamp":"2026-01-01T00:00:00Z",'
                '"part_kind":"retry-prompt"}' % (json.dumps(tool), json.dumps(cid)))
    return '{"raw":[%d,1.5,null],"note":"an untagged value"}' % j


def conversation(n_calls: int, variant: int) -> bytes:
    """A post-LLM agent envelope (the state Agent.run holds after the model turn) with `n_calls` tool calls.
    variant 1: overrides on the agent frame, and so on the state (the agent step copies them there);
    variant 2: a second round, tool_results already holds answers for every third call (mixed kinds)."""
    from calfkit import synth
    from oracle import port
    rng = random.Random(1000 * variant + n_calls)
    ids = _call_ids(n_calls, rng)
    names = [rng.choice(list(TOOLS)) for _ in ids]
    parts = [synth.tool_call_part(t, json.dumps(_args(t, rng), ensure_ascii=False, separators=(",", ":")), c)
             for t, c in zip(names, ids)]
    results = {}
    if variant == 2:
        answered = [j for j in range(n_calls) if j % 3 == 1]
        rng.shuffle(answered)
        results = {ids[j]: _result(j // 3 % 3, j, ids[j], names[j]) for j in answered}
    hexid = lambda: "".join(rng.choices("0123456789abcdef", k=32))    # noqa: E731
    frames = [synth.frame(AGENT_IN, "calf-client-reply-" + hexid()[:16], None, hexid(), OVERRIDES if variant == 1 else "null")]
    state_ovr = OVERRIDES if variant == 1 or (variant == 0 and n_calls % 2) else "null"
    env = synth.envelope(tool_calls=dict(zip(ids, parts)), tool_results=results, uncommitted="null",
                         history=[synth.user_request(f"Compare {n_calls} things, please — «now»."), synth.model_response(parts)],
                         final_parts=[], temp_instructions=None, state_metadata="null", state_overrides=state_ovr,
                         correlation_id=hexid(), provided_deps='{"tenant":"t-%d"}' % n_calls, frames=frames)
    return port.encode(port.decode(env.encode()))


def conversations() -> list[tuple[str, int, bytes]]:
    """(name, calls, envelope): every size in one batch, the declined band between accepted neighbours"""
    sizes = FS[:11] + [BAND[0]] + FS[11:] + [BAND[1]]
    return [(f"calls_{f}_{v}", f, conversation(f, v)) for v in range(3) for f in sizes]


def oracle_tool_hop_inputs() -> list[bytes]:
    """Call envelopes of the round trip's conversations as the oracle writes them (frame ids from the device's generator),
    those that look up the call at index 0, 1, 2, the middle and the last of each fan-out.  CPU only: also fuzz seeds."""
    from oracle import port
    from calfkit import _ids
    from calfkit.engine.batch import device_uuid7_hex
    out = []
    slot = iter(range(1 << 30))
    _ids.set_id_source(lambda: device_uuid7_hex(MS, 1, next(slot)))
    try:
        for _name, f, rec in conversations():
            if f > 128:
                continue
            calls = [pl for (t, _k, _c, pl) in port.agent_fanout(AGENT, AGENT_IN, AGENT_OUT, REGISTRY, rec) if t != AGENT_OUT]
            out += [calls[j] for j in sorted({0, 1, 2, len(calls) // 2, len(calls) - 1} & set(range(len(calls))))]
    finally:
        _ids.set_id_source(None)
    return out


# ---- helpers ------------------------------------------------------------------------------------------------------------
def _part(key: bytes | None) -> int:
    return -1 if key is None else (_murmur2(key) & 0x7FFFFFFF) % NPART


def _want(pubs) -> list[tuple]:
    return [(t, k, pl, _part(k)) for (t, k, _c, pl) in pubs]


def _by_record(out) -> dict[int, list[tuple]]:
    got = defaultdict(list)
    for p in out.publishes():
        got[p.record].append((p.topic, p.key, p.payload, p.partition))
    return got


def _node(name: str):
    from oracle import port
    return port.ToolNode(TOOLS[name][0], f"tool_{name}", [REGISTRY[name]], f"tool.{name}.output")


def _pending(rec: bytes) -> list[str]:
    from oracle import port
    st = port.decode(rec).context.state
    return [tc.tool_call_id for tc in st.latest_tool_calls() if tc.tool_call_id not in st.tool_results]


def _tool_hop(eng, calls: list[tuple[str, bytes]], host: bool) -> list[tuple[int, int, list]]:
    """every (tool, Call envelope) through the tool node of that tool: -> [(status, action, publishes)] in input order"""
    from calfkit import synth
    from calfkit.engine import ToolTemplate
    from calfkit.engine._lib import COL
    groups = defaultdict(list)
    for j, (tool, _c) in enumerate(calls):
        groups[tool].append(j)
    res: list = [None] * len(calls)
    for tool, idx in groups.items():
        fn, fmt = TOOLS[tool]
        eng.set_tool_node(f"tool.{tool}.output", None if host else ToolTemplate.from_format(fmt))
        b = synth.pack([calls[j][1] for j in idx])
        out = eng.run_tool_batch(b.data, b.offsets, _host_tool(fn) if host else None)
        got = _by_record(out)
        for r, j in enumerate(idx):
            res[j] = (int(out.cols[COL["STATUS"], r]), int(out.cols[COL["ACTION"], r]), got[r])
    return res


def _lookup(call: bytes) -> tuple[int, int, list[str], str]:
    """(bytes, index of the looked-up call in tool_calls, tool_results keys, the looked-up id) of a tool-hop input"""
    obj = json.loads(call)
    st = obj["context"]["state"]
    cid = obj["internal_workflow_state"]["call_stack"]["_internal_list"][-1]["input_args"][0]
    return len(call), list(st["tool_calls"]).index(cid), list(st["tool_results"]), cid


def _redelivered(call: bytes) -> bytes:
    """the Call with a stale answer for its own id placed in the middle of tool_results: the tool hop overwrites it there"""
    from oracle import port
    obj = json.loads(call)
    st = obj["context"]["state"]
    cid = obj["internal_workflow_state"]["call_stack"]["_internal_list"][-1]["input_args"][0]
    items = list(st["tool_results"].items())
    items.insert(len(items) // 2, (cid, {"return_value": "stale", "content": None, "metadata": {"tool_call_id": cid},
                                         "kind": "tool-return"}))
    st["tool_results"] = dict(items)
    return port.encode(port.decode(json.dumps(obj, ensure_ascii=False).encode()))


@pytest.fixture(scope="module")
def engines():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from calfkit.engine import BatchEngine
    agent = BatchEngine(0, max_records=4096, max_in_bytes=128 << 20, max_out_bytes=256 << 20, max_payloads=8192)
    tool = BatchEngine(0, max_records=4096, max_in_bytes=96 << 20)
    for e in (agent, tool):
        e.register_topics(TOPICS, num_partitions=NPART)
    agent.set_tool_node(AGENT_OUT, None)
    agent.set_agent_node(AGENT, AGENT_IN, AGENT_OUT, REGISTRY)
    agent.gate_create(max_entries=1024, arena_bytes=128 << 20)
    yield agent, tool
    agent.close()
    tool.close()


def _hop_a(agent, convs, seed: int):
    """fan-out + gate registration of the whole batch: -> BatchOutput"""
    from calfkit import synth
    b = synth.pack([rec for _n, _f, rec in convs])
    agent.gate_reset()
    agent.submit(b.data, b.offsets)
    agent.fanout_plan(MS, seed, max_fanout=256)
    agent.gate_register()
    return agent.fetch()


# ---- the parallel flow ----------------------------------------------------------------------------------------------------
def test_parallel_round_trip_hop_by_hop(engines):
    from oracle import port
    from calfkit import _ids
    from calfkit.engine._lib import (CK_ACT_CALL, CK_ACT_FANOUT, CK_ACT_GATE_COMPLETE, CK_ACT_GATE_PASS, CK_ACT_RETURN,
                                     CK_ACT_SILENT, CK_UNSUPPORTED, COL)
    from calfkit.engine.batch import device_uuid7_hex
    from calfkit.models.state import PendingToolBatch
    agent, tool = engines
    convs = conversations()
    seed = 4242

    # hop A: every pending call of every conversation -> one Call; list[Call] records become pending gate entries
    out = _hop_a(agent, convs, seed)
    got = _by_record(out)
    st, act = out.cols[COL["STATUS"]], out.cols[COL["ACTION"]]
    declined = [convs[i][0] for i in range(len(convs)) if st[i] != 0]
    assert declined == DECLARED_UNSUPPORTED
    calls: list[tuple[int, str, bytes]] = []           # (conversation, tool, Call envelope)
    slot = n_pubs = 0
    for i, (name, _f, rec) in enumerate(convs):
        if name in DECLARED_UNSUPPORTED:
            assert st[i] == CK_UNSUPPORTED and i not in got, name
            continue
        npend = len(_pending(rec))
        assert act[i] == (CK_ACT_FANOUT if npend > 1 else CK_ACT_CALL), name
        it = iter([device_uuid7_hex(MS, seed, slot + j) for j in range(npend)])
        _ids.set_id_source(lambda: next(it))
        try:
            want = _want(port.agent_fanout(AGENT, AGENT_IN, AGENT_OUT, REGISTRY, rec))
        finally:
            _ids.set_id_source(None)
        assert len(want) == npend + 1 and got[i] == want, name
        n_pubs += len(want)
        slot += npend + (1 if npend > 1 else 0)
        calls += [(i, t.split(".")[1], pl) for (t, _k, pl, _p) in want if t != AGENT_OUT]
    assert n_pubs == len(out.live())

    # hop B inputs: the Calls, plus some re-delivered with a stale answer for their own id in the middle of tool_results
    extra = [(t, _redelivered(c)) for (i, t, c) in calls if convs[i][1] >= 31 and convs[i][0].endswith("_2")][::7]
    hop_b = [(t, c) for (_i, t, c) in calls] + extra
    looks = [_lookup(c) for _t, c in hop_b]
    assert any(n < 2048 for n, *_ in looks) and any(2048 <= n < LONG for n, *_ in looks)
    ncalls = [len(json.loads(c)["context"]["state"]["tool_calls"]) for _t, c in hop_b]
    for warp in (False, True):       # thread walker / warp walker: the looked-up call at 0, 1, 2, the middle and the last
        sel = [(k, nc) for (n, k, _r, _c), nc in zip(looks, ncalls) if (n >= LONG) == warp and nc >= LX_MIN]
        assert {0, 1, 2} <= {k for k, _nc in sel} and any(k == nc // 2 for k, nc in sel) and any(k == nc - 1 for k, nc in sel)
    assert any(n >= LONG and nc >= LX_MIN for (n, *_), nc in zip(looks, ncalls))
    assert any(res and cid not in res for _n, _k, res, cid in looks)                          # inserts after other ids
    assert any(cid in res and 0 < res.index(cid) < len(res) - 1 for _n, _k, res, cid in looks)  # overwrites in the middle
    assert any(cid in res and 0 < res.index(cid) < len(res) - 1 for (n, _k, res, cid) in looks if n >= LONG)

    # hop B: each Call through its tool's node, with the device template and with the host tool
    want_b = [_want(port.tool_node_event(_node(t), c)) for t, c in hop_b]
    for host in (False, True):
        res = _tool_hop(tool, hop_b, host)
        for j, ((t, c), (s, a, g)) in enumerate(zip(hop_b, res)):
            assert (s, a) == (0, CK_ACT_RETURN) and g == want_b[j], (j, t, host, looks[j][:2])
    arrivals = [(convs[i][2], want_b[j][0][2]) for j, (i, _t, _c) in enumerate(calls)]     # (conversation, ReturnCall)
    assert all(w[0][0] == AGENT_IN for w in want_b)

    # hop C: the ReturnCalls back at the agent through the device gate, shuffled, in chunks, with duplicates
    rng = random.Random(7)
    from calfkit import synth
    for chunk in (1, 7, len(arrivals) + 3):
        out = _hop_a(agent, convs, seed)
        batches = {}
        for (name, _f, rec), a in zip(convs, out.cols[COL["ACTION"]]):
            if a == CK_ACT_FANOUT:
                env = port.decode(rec)
                batches[env.context.deps.correlation_id] = PendingToolBatch(
                    expected_tool_call_ids=frozenset(_pending(rec)), base_state=env.context.state)
        order = [r for _conv, r in arrivals]
        rng.shuffle(order)
        order[5:5] = [order[0], order[-1]]                                  # at-least-once delivery: duplicates
        got_c = []
        for a0 in range(0, len(order), chunk):
            b = synth.pack(order[a0:a0 + chunk])
            agent.submit(b.data, b.offsets)
            agent.gate_arrive(100000 * chunk + a0)
            o = agent.fetch()
            got_c += [(int(o.cols[COL["STATUS"], k]), int(o.cols[COL["ACTION"], k]), o.payload(k)) for k in range(b.n)]
        completes = 0
        for k, (r, (s, a, payload)) in enumerate(zip(order, got_c)):
            env = port.decode(r)
            corr = env.context.deps.correlation_id
            pending_before = corr in batches
            merged = port.aggregate(batches, env.context.state, corr)
            assert s == 0, (chunk, k)
            if not pending_before:
                assert a == CK_ACT_GATE_PASS, (chunk, k)
            elif merged is None:
                assert a == CK_ACT_SILENT and payload == r, (chunk, k)
            else:
                completes += 1
                env.context.state = merged
                assert a == CK_ACT_GATE_COMPLETE and payload == port.encode(env), (chunk, k)
        assert completes == sum(1 for a in out.cols[COL["ACTION"]] if a == CK_ACT_FANOUT) and not batches
        assert agent.gate_stats()["live"] == 0


# ---- the sequential flow --------------------------------------------------------------------------------------------------
def test_sequential_round_trip_until_nothing_is_pending(engines):
    """fanout_plan(sequential=True) -> tool node -> the ReturnCall back into fanout_plan(sequential=True), round after
    round, so that tool_results grows on the device through every size up to 128; then one TailCall"""
    from oracle import port
    from calfkit import _ids, synth
    from calfkit.engine._lib import CK_ACT_CALL, CK_ACT_RETURN, COL
    from calfkit.engine.batch import device_uuid7_hex
    agent, tool = engines
    cur = [conversation(f, v) for f in SEQ_FS for v in (0, 2)]
    done, sizes, rnd = [], set(), 0
    while cur:
        seed = 900 + rnd
        b = synth.pack(cur)
        agent.submit(b.data, b.offsets)
        agent.fanout_plan(MS, seed, max_fanout=256, sequential=True)
        out = agent.fetch()
        got = _by_record(out)
        calls = []
        for i, rec in enumerate(cur):
            _ids.set_id_source(lambda: device_uuid7_hex(MS, seed, i))
            try:
                want = _want(port.agent_fanout(AGENT, AGENT_IN, AGENT_OUT, REGISTRY, rec, sequential=True))
            finally:
                _ids.set_id_source(None)
            assert out.cols[COL["STATUS"], i] == 0 and out.cols[COL["ACTION"], i] == CK_ACT_CALL, (rnd, i)
            assert got[i] == want, (rnd, i)
            calls.append((want[0][0].split(".")[1], want[0][2]))
        res = _tool_hop(tool, calls, host=False)
        nxt = []
        for (t, c), (s, a, g) in zip(calls, res):
            want = _want(port.tool_node_event(_node(t), c))
            assert (s, a) == (0, CK_ACT_RETURN) and g == want, (rnd, t)
            back = g[0][2]
            sizes.add(len(port.decode(back).context.state.tool_results))
            (nxt if _pending(back) else done).append(back)
        cur, rnd = nxt, rnd + 1
    assert rnd == 128 and sizes >= set(range(1, 129))
    b = synth.pack(done)
    agent.submit(b.data, b.offsets)
    agent.tailcall_plan(MS, 31)
    out = agent.fetch()
    got = _by_record(out)
    for i, rec in enumerate(done):
        env = port.decode(rec)
        _ids.set_id_source(lambda: device_uuid7_hex(MS, 31, i))
        try:
            corr = env.context.deps.correlation_id
            pubs, returned = port.publish_action(AGENT_IN, port.TailCall(AGENT_IN, port.prepare_context(env).state), env, corr)
        finally:
            _ids.set_id_source(None)
        want = [(t, k, port.encode(e), _part(k)) for (t, k, _c, e) in pubs] + [(AGENT_OUT, None, port.encode(returned), -1)]
        assert out.cols[COL["STATUS"], i] == 0 and got[i] == want, i


# ---- the declined band through the Worker -------------------------------------------------------------------------------
def test_worker_logs_a_declined_fanout_and_completes_the_others(caplog):
    """A model turn that asks for 129 tool calls gives an envelope the engine declines after the agent step: the Worker logs
    it, publishes nothing for that conversation, and the other conversations of the batch complete."""
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from calfkit import Agent, Client, Worker, agent_tool
    from calfkit.models.messages import ModelResponse, TextPart, ToolCallPart, ToolReturnPart
    from calfkit.nodes import FunctionModelClient

    @agent_tool(device_template="T<{x}>")
    def tool_t(x: str) -> str:
        """t"""
        return f"T<{x}>"

    def llm(messages, tools):
        rets = [p for p in getattr(messages[-1], "parts", []) if isinstance(p, ToolReturnPart)]
        if rets:
            return ModelResponse(parts=[TextPart(content=f"{len(rets)} results")])
        n = int(messages[0].parts[0].content)
        return ModelResponse(parts=[ToolCallPart(tool_name="tool_t", args={"x": str(j)}) for j in range(n)])

    async def go():
        client = Client.connect()
        agent = Agent("planner", subscribe_topics="planner.input", publish_topic="planner.output",
                      model_client=FunctionModelClient(llm), tools=[tool_t])
        worker = Worker(client, nodes=[agent, tool_t])
        sizes = [3, 129, 5, 2]
        hs = [await client.invoke_node(str(n), "planner.input") for n in sizes]
        with caplog.at_level(logging.ERROR, logger="calfkit.nodes.agent"):
            await worker.run(until_idle=True)
        res = {}
        for n, h in zip(sizes, hs):
            try:
                res[n] = (await h.result(timeout=0.5)).output
            except asyncio.TimeoutError:
                res[n] = None
        outs = client.broker.poll_batch(("planner.output",), 100000)
        await client.close()
        return hs, res, outs

    hs, res, outs = asyncio.run(go())
    assert res == {3: "3 results", 129: None, 5: "5 results", 2: "2 results"}
    declined = [r for r in caplog.records if "declined" in r.getMessage()]
    assert len(declined) == 1 and "unsupported" in declined[0].getMessage()
    corrs = [json.loads(r.value)["context"]["deps"]["correlation_id"] for r in outs]
    assert hs[1].correlation_id not in corrs
    # the others: the handler return of the fan-out turn, n - 1 Silent returns of the gate and the final ReturnCall
    assert [corrs.count(hs[k].correlation_id) for k in (0, 2, 3)] == [3 + 1, 5 + 1, 2 + 1]
