"""GPU parity: the CUDA path (through the C-ABI) against the oracle and the reference's golden
vectors.  Bit-exact: byte equality of every payload, equality of (topic, key) of every publish."""
import json
import random

import numpy as np
import pytest
from conftest import as_bytes, golden

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def engine():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from calfkit.engine import BatchEngine
    e = BatchEngine(device=0, max_records=1 << 16, max_in_bytes=256 << 20)
    yield e
    e.close()


def _host_tool(fn):
    import pydantic_core

    def call(args_json: bytes) -> bytes:
        v = pydantic_core.from_json(args_json)
        if isinstance(v, str):            # args_as_dict: JSON string -> parsed (messages.py:1229-1240)
            v = pydantic_core.from_json(v)
        kwargs = v or {}
        return pydantic_core.to_json(fn(**kwargs))
    return call


def _pubs(out):
    return [(p.topic, p.key, p.payload) for p in out.publishes()]


def _setup(engine, tool_name, template=None):
    from calfkit import synth  # noqa: F401
    topics = [f"tool.{tool_name}.input", f"tool.{tool_name}.output", "weather_agent.input"]
    engine.register_topics(topics, num_partitions=8)
    engine.set_tool_node(f"tool.{tool_name}.output", template)


@pytest.mark.parametrize("use_template", [False, True])
def test_tool_node_goldens(engine, use_template):
    import tools_def
    from calfkit import synth
    from calfkit.engine import ToolTemplate
    from calfkit.engine._lib import CK_ACT_RAISES, COL
    for case in golden("tool_node.json"):
        if use_template and case["tool"] != "get_weather":
            continue
        if case["name"] == "header_corr_differs":
            continue   # header != deps.correlation_id never happens on the reference's own flows (client sets both)
        _setup(engine, case["tool"], ToolTemplate.from_format("It's sunny in {location}") if use_template else None)
        b = synth.pack([as_bytes(case["input"])])
        engine.submit(b.data, b.offsets)
        st0 = int(engine.columns()[COL["STATUS"], 0])
        if st0 != 0:
            # the only golden inputs the device declines are the ones whose canonical form needs a shortest-digits
            # float printer (exponent floats with > 15 digits etc.): declared UNSUPPORTED, never wrong
            assert st0 == 4 and case["name"] in ("any_values",), (case["name"], st0)
            continue
        out = engine.run_tool_batch(b.data, b.offsets, None if use_template else _host_tool(tools_def.TOOLS[case["tool"]]))
        if "raises" in case:
            assert out.cols[COL["ACTION"], 0] == CK_ACT_RAISES and len(out.live()) == 0, case["name"]
            continue
        if use_template and case["name"].startswith("args_json_string"):
            # args given as a JSON *string*: the device template does not parse nested JSON -> loud, not silent
            assert out.cols[COL["STATUS"], 0] != 0 and len(out.live()) == 0
            continue
        want = [(p["topic"], p["key"].encode() if p["key"] is not None else None, p["payload"].encode())
                for p in case["publishes"]]
        assert _pubs(out) == want, case["name"]


def test_synthetic_batch_matches_oracle(engine):
    import tools_def
    from oracle import port
    from calfkit import synth
    from calfkit.engine import ToolTemplate
    _setup(engine, "get_weather", ToolTemplate.from_format("It's sunny in {location}"))
    recs = synth.tool_events(20000, seed=5) + synth.tool_events(3000, seed=6, size=None, full_history=True)
    b = synth.pack(recs)
    out = engine.run_tool_batch(b.data, b.offsets)
    assert (out.cols[0] == 0).all()
    node = port.ToolNode.of(tools_def.get_weather)
    pubs = list(out.publishes())
    assert len(pubs) == 2 * len(recs)
    rng = random.Random(0)
    for i in rng.sample(range(len(recs)), 400):
        want = port.tool_node_event(node, recs[i])
        assert [(p.topic, p.key, p.payload) for p in pubs[2 * i:2 * i + 2]] == [(t, k, pl) for (t, k, c, pl) in want]
    # size-independent property at full batch size: every payload is again a canonical Envelope the
    # engine itself accepts, one frame shorter, with exactly one more tool result
    outs = [out.payload(i) for i in range(out.out_off.size - 1)]
    b2 = synth.pack(outs)
    engine.submit(b2.data, b2.offsets)
    cols2 = engine.columns()
    from calfkit.engine._lib import COL
    assert (cols2[COL["STATUS"]] == 0).all()
    assert (cols2[COL["NFRAMES"]] == out.cols[COL["NFRAMES"]] - 1).all()
    # murmur2 partition of the key agrees with the Kafka default partitioner formula
    live = out.live()
    keyed = live[live["has_key"] == 1]
    for p in keyed[:50]:
        key = out.key_of(p)
        assert int(p["partition"]) == (_murmur2(key) & 0x7FFFFFFF) % 8


def _murmur2(data: bytes) -> int:
    """Kafka's murmur2 (org.apache.kafka.common.utils.Utils.murmur2; aiokafka partitioner)."""
    length = len(data)
    seed = 0x9747B28C
    m = 0x5BD1E995
    r = 24
    h = (seed ^ length) & 0xFFFFFFFF
    for i in range(length // 4):
        k = int.from_bytes(data[4 * i:4 * i + 4], "little")
        k = (k * m) & 0xFFFFFFFF
        k ^= k >> r
        k = (k * m) & 0xFFFFFFFF
        h = (h * m) & 0xFFFFFFFF
        h ^= k
    extra = length % 4
    base = length & ~3
    if extra == 3:
        h ^= (data[base + 2] & 0xFF) << 16
    if extra >= 2:
        h ^= (data[base + 1] & 0xFF) << 8
    if extra >= 1:
        h ^= data[base] & 0xFF
        h = (h * m) & 0xFFFFFFFF
    h ^= h >> 13
    h = (h * m) & 0xFFFFFFFF
    h ^= h >> 15
    return h


def test_device_walker_equals_host_build_on_fuzz(engine):
    """The g++ build of the walker was fuzzed against pydantic on the CPU (tests/test_walker_hostsim.py);
    here the nvcc build must agree with it column for column on the same inputs."""
    from hostsim import walk                  # g++ build of the source the GPU kernel compiles (csrc/ck_walk.cuh)
    from calfkit import synth
    from test_gpu_round_trip import oracle_tool_hop_inputs
    rng = random.Random(1)
    calls = oracle_tool_hop_inputs()          # multi-call Call envelopes: the looked-up call at index 0, 1, 2, middle, last
    seeds = [as_bytes(c["input"]) for c in golden("codec.json")] + synth.tool_events(50, seed=2) + \
        synth.mixed_events(40, seed=3, hi=20000) + calls
    recs = list(seeds)
    for _ in range(6000):
        s = bytearray(rng.choice(seeds))
        if not s:
            continue
        for _ in range(rng.choice([1, 1, 2])):
            i = rng.randrange(len(s))
            op = rng.randrange(3)
            if op == 0:
                s[i] = rng.randrange(256)
            elif op == 1:
                del s[i]
            else:
                s[i:i] = rng.choice([b'"', b"{", b"}", b",", b":", b" ", b"\\", b"0", b"null", b"1.5", b"\xc3\xa9", b"\xff"])
            if not s:
                break
        recs.append(bytes(s))
    b = synth.pack(recs)
    engine.submit(b.data, b.offsets)
    cols = engine.columns()
    from hostsim import canon, walk_trust
    ncmp = 50   # walker-owned columns (incl. the resolved tool call / existing result spans)
    for i, r in enumerate(recs):
        if len(r) == 0:
            assert cols[0, i] == 5
            continue
        ok, hc = walk(r)
        if not ok:
            # not a fixed point: the device ran its canonicaliser; the same source built for the host must agree
            st, cbytes = canon(r)
            assert cols[0, i] == st, (i, int(cols[0, i]), st, r[:200])
            if st != 0:
                continue
            ok, hc = walk_trust(cbytes)          # the second walk of the decode pass (trusting reader, ck_walk.cuh WRdT)
            assert ok
        assert cols[0, i] == 0, (i, r[:200])
        assert (cols[2:ncmp, i] == hc[2:ncmp]).all(), i   # columns 0/1 (status/action) are owned by the kernels
    # the warp walker (records of 16 KB and more, GPU only) resolves the looked-up call from its shared-memory key tables:
    # its spans must be those of the host thread walker on the same bytes
    from calfkit.engine._lib import COL
    n_long = 0
    for i in range(len(seeds) - len(calls), len(seeds)):
        if len(recs[i]) < 16384:
            continue
        ok, hc = walk(recs[i])
        assert ok and hc[COL["CALL_VAL_LEN"]] > 0
        for name in ("CALL_VAL", "TNAME", "ARGS", "RES"):
            assert cols[COL[name + "_OFF"], i] == hc[COL[name + "_OFF"]] and cols[COL[name + "_LEN"], i] == hc[COL[name + "_LEN"]], (i, name)
        n_long += 1
    assert n_long >= 40

def test_fanout_matches_oracle(engine):
    """Agent fan-out (config 3): every pending tool call -> one Call envelope, frame ids injected into
    the oracle from the device's own uuid7 generator (seed, slot index)."""
    from oracle import port
    from calfkit import _ids, synth
    from calfkit.engine.batch import device_uuid7_hex
    from calfkit.engine import BatchEngine
    F = 16
    recs = synth.fanout_events(40, seed=9, fanout=F) + synth.fanout_events(5, seed=10, fanout=1) + \
        [as_bytes(golden("actions.json")[0]["input"])]
    registry = {f"tool_{j:02d}": f"tool.tool_{j:02d}.input" for j in range(64)}
    e = BatchEngine(0, max_records=256, max_in_bytes=8 << 20, max_out_bytes=256 << 20, max_payloads=256 * (F + 1))
    try:
        e.register_topics(list(registry.values()) + ["planner.input", "planner.output"], num_partitions=8)
        e.set_agent_node("planner", "planner.input", "planner.output", registry)
        b = synth.pack(recs)
        ms, seed = 1767225600000, 1234
        e.submit(b.data, b.offsets)
        e.fanout_plan(ms, seed, max_fanout=64)
        out = e.fetch()
        assert (out.cols[0] == 0).all()
        pubs = list(out.publishes())
        slot = 0
        k = 0
        for i, rec in enumerate(recs):
            npend = len(port.decode(rec).context.state.tool_calls)
            ids = iter([device_uuid7_hex(ms, seed, slot + j) for j in range(npend)])
            _ids.set_id_source(lambda: next(ids))
            try:
                want = port.agent_fanout("planner", "planner.input", "planner.output", registry, rec)
            finally:
                _ids.set_id_source(None)
            got = [(p.topic, p.key, p.payload) for p in pubs[k:k + len(want)]]
            assert got == [(t, kk, pl) for (t, kk, c, pl) in want], i
            k += len(want)
            slot += npend + (1 if npend > 1 else 0)
        assert k == len(pubs)
    finally:
        e.close()


def test_sequential_call_and_tailcall_match_oracle(engine):
    """Agent(sequential_only_mode=True): first pending call only, as a single Call; no pending call at
    all -> TailCall to the agent's own topic (reference nodes/agent.py:94-108,171-175; nodes/base.py:90-136)."""
    from oracle import port
    from calfkit import _ids, synth
    from calfkit.engine.batch import device_uuid7_hex
    from calfkit.engine import BatchEngine
    recs = synth.fanout_events(12, seed=3, fanout=5) + synth.fanout_events(3, seed=4, fanout=1)
    registry = {f"tool_{j:02d}": f"tool.tool_{j:02d}.input" for j in range(64)}
    e = BatchEngine(0, max_records=64, max_in_bytes=8 << 20, max_out_bytes=64 << 20, max_payloads=256)
    try:
        e.register_topics(list(registry.values()) + ["planner.input", "planner.output"], num_partitions=8)
        e.set_agent_node("planner", "planner.input", "planner.output", registry)
        b = synth.pack(recs)
        ms, seed = 1767225600000, 77
        e.submit(b.data, b.offsets)
        e.fanout_plan(ms, seed, max_fanout=64, sequential=True)
        out = e.fetch()
        assert (out.cols[0] == 0).all()
        pubs = list(out.publishes())
        assert len(pubs) == 2 * len(recs)
        for i, rec in enumerate(recs):
            _ids.set_id_source(lambda: device_uuid7_hex(ms, seed, i))
            try:
                want = port.agent_fanout("planner", "planner.input", "planner.output", registry, rec, sequential=True)
            finally:
                _ids.set_id_source(None)
            assert [(p.topic, p.key, p.payload) for p in pubs[2 * i:2 * i + 2]] == [(t, k, pl) for (t, k, c, pl) in want], i
        # TailCall: tool-stage events (a frame with input_args, overrides on some) + the golden TailCall input
        recs2 = synth.tool_events(40, seed=5) + synth.mixed_events(20, seed=6)
        b2 = synth.pack(recs2)
        e.submit(b2.data, b2.offsets)
        e.tailcall_plan(ms, seed)
        out = e.fetch()
        pubs = list(out.publishes())
        k = 0
        for i, rec in enumerate(recs2):
            env = port.decode(rec)
            if not env.internal_workflow_state.call_stack._internal_list:
                assert out.cols[1][i] == 3            # CK_ACT_RAISES: unwind_frame on an empty stack
                continue
            _ids.set_id_source(lambda: device_uuid7_hex(ms, seed, i))
            try:
                corr = env.context.deps.correlation_id
                ctx_state = port.prepare_context(env).state
                got_pubs, returned = port.publish_action("planner.input", port.TailCall("planner.input", ctx_state), env, corr)
            finally:
                _ids.set_id_source(None)
            want = [(t, kk, port.encode(en)) for (t, kk, c, en) in got_pubs] + [("planner.output", None, port.encode(returned))]
            assert [(p.topic, p.key, p.payload) for p in pubs[k:k + 2]] == want, i
            k += 2
        assert k == len(pubs)
    finally:
        e.close()


def test_mixed_sizes_and_edge_batches(engine):
    """config 5 shapes (128 B .. 64 KB, 256 topics' worth of tools, UTF-8 + escapes) and degenerate
    batches: empty batch, zero-length record, a batch of one."""
    import tools_def
    from oracle import port
    from calfkit import synth
    from calfkit.engine import ToolTemplate
    from calfkit.engine._lib import COL
    tools = [f"tool_{j:02d}" for j in range(32)]
    topics = [f"tool.{t}.input" for t in tools] + ["tool.out", "weather_agent.input"]
    engine.register_topics(topics, num_partitions=8)
    engine.set_tool_node("tool.out", ToolTemplate.from_format("It's sunny in {location}"))
    recs = synth.mixed_events(300, seed=21, lo=128, hi=65536, n_tools=32) + [b""]
    b = synth.pack(recs)
    out = engine.run_tool_batch(b.data, b.offsets)
    st = out.cols[COL["STATUS"]]
    assert (st[:-1] == 0).all() and st[-1] == 5                 # the empty record is CK_EMPTY, the batch goes on
    assert max(len(r) for r in recs) > 40000
    pubs = list(out.publishes())
    assert len(pubs) == 2 * (len(recs) - 1)

    def get_weather(location: str) -> str:
        return f"It's sunny in {location}"
    k = 0
    for i, r in enumerate(recs[:-1]):
        tname = port.decode(r).internal_workflow_state.current_frame.target_topic.split(".")[1]
        node = port.ToolNode(get_weather, f"tool_{tname}", [f"tool.{tname}.input"], "tool.out")
        want = port.tool_node_event(node, r)
        assert [(p.topic, p.key, p.payload) for p in pubs[k:k + 2]] == [(t, kk, pl) for (t, kk, c, pl) in want], i
        k += 2
    # empty batch and a batch of one
    e0 = synth.pack([])
    out0 = engine.run_tool_batch(e0.data if e0.data.size else np.zeros(1, dtype=np.uint8), e0.offsets)
    assert len(out0.live()) == 0
    one = synth.pack(recs[:1])
    assert len(list(engine.run_tool_batch(one.data, one.offsets).publishes())) == 2


def test_noncanonical_inputs_are_canonicalised_on_device(engine):
    """Valid records in a non-canonical spelling (pretty-printed, key-sorted, ASCII-escaped, missing defaults,
    unknown keys, exponent floats) go through ck_canon on the device and then produce exactly what the reference
    produces; invalid ones get the reference's error class; nothing falls back to the CPU."""
    import tools_def
    from oracle import port
    from pydantic import ValidationError
    from calfkit import synth
    from calfkit.engine import ToolTemplate
    from calfkit.engine._lib import COL
    _setup(engine, "get_weather", ToolTemplate.from_format("It's sunny in {location}"))
    canon = synth.tool_events(40, seed=41) + synth.tool_events(20, seed=42, size=None, full_history=True)
    recs, expect_ok = [], []
    for i, r in enumerate(canon):
        obj = json.loads(r)
        if i % 4 == 0:
            obj["context"]["state"].pop("final_output_parts"); obj["zzz"] = {"unknown": [1, 2.50, 1e3]}
            obj["context"]["state"]["metadata"] = {"f": [1E-7, 12.5e20, 0.10], "s": "é"}
        v = [json.dumps(obj, indent=2), json.dumps(obj, ensure_ascii=True, separators=(" , ", " : ")), r.decode(),
             json.dumps(obj, sort_keys=False)][i % 4]
        recs.append(v.encode()); expect_ok.append(True)
    bad = [b"", b"{", b'{"context":{}}', b"[1,2]", recs[0][:-1], recs[1].replace(b'"correlation_id"', b'"correlation_idx"'),
           b'{"context":{"state":{},"deps":{"correlation_id":5,"provided_deps":{}}},"internal_workflow_state":{"call_stack":{}}}']
    recs += bad
    b = synth.pack(recs)
    out = engine.run_tool_batch(b.data, b.offsets)
    st = out.cols[COL["STATUS"]]
    node = port.ToolNode.of(tools_def.get_weather)
    pubs = list(out.publishes())
    k = 0
    for i, r in enumerate(recs):
        if i < len(canon):
            assert st[i] == 0, (i, st[i], r[:200])
            want = port.tool_node_event(node, r)
            got = [(p.topic, p.key, p.payload) for p in pubs[k:k + len(want)]]
            assert got == [(t, kk, pl) for (t, kk, c, pl) in want], i
            k += len(want)
        else:
            if len(r) == 0:
                assert st[i] == 5
                continue
            try:
                port.decode(r)
                raise AssertionError("expected the reference to reject")
            except ValidationError as e:
                cls = 2 if e.errors()[0]["type"] == "json_invalid" else 3
            assert st[i] == cls, (i, st[i], cls, r[:120])
    assert k == len(pubs)
    assert out.overlay is not None and (out.overlay[1] >= 0).sum() >= 40


def test_long_records_with_bad_or_respelled_history_messages(engine):
    """Records long enough for the warp-per-record walker, whose history messages are validated one thread each from the
    batch-wide element list (ck_walk_elems_kernel): a message in the middle that is schema-invalid, not JSON, or merely
    spelled differently must give exactly what the sequential walk gives — the reference's error class, or the reference's
    output after canonicalisation — and must not disturb its neighbours in the batch."""
    import tools_def
    from oracle import port
    from pydantic import ValidationError
    from calfkit import synth
    from calfkit.engine import ToolTemplate
    from calfkit.engine._lib import COL
    _setup(engine, "get_weather", ToolTemplate.from_format("It's sunny in {location}"))
    base = [r for r in synth.mixed_events(400, seed=77, lo=20000, hi=65536, n_tools=1) if len(r) >= 20000][:24]
    assert len(base) >= 16
    marker = b'"part_kind":"text"'
    recs, kinds = [], []
    for i, r in enumerate(base):
        hits = [m for m in range(len(r)) if r.startswith(marker, m)]
        mid = hits[len(hits) // 2]
        kind = i % 6
        if kind == 0:   v = r                                                            # untouched
        elif kind == 1: v = r[:mid] + b'"part_kind":"texx"' + r[mid + len(marker):]      # unknown union tag: schema-invalid
        elif kind == 2: v = r[:mid] + b'"part_kind": "text"' + r[mid + len(marker):]     # valid, one space: canonicalised
        elif kind == 3: v = r[:mid] + b'"part_kind":"text"}' + r[mid + len(marker):]     # unbalanced: not JSON
        elif kind == 4: v = r[:mid] + b'"part_kind":"text","zz":[1,{"a":"}]"}]' + r[mid + len(marker):]   # unknown key with brackets in a string: dropped by the reference
        else:           v = r[:mid - 1] + b' ' + r[mid - 1:]                             # whitespace before a key
        recs.append(v); kinds.append(kind)
    b = synth.pack(recs)
    out = engine.run_tool_batch(b.data, b.offsets)
    st = out.cols[COL["STATUS"]]
    node = port.ToolNode.of(tools_def.get_weather)
    pubs = list(out.publishes())
    k = 0
    for i, r in enumerate(recs):
        try:
            port.decode(r)
            ok = True
        except ValidationError as e:
            ok, cls = False, (2 if e.errors()[0]["type"] == "json_invalid" else 3)
        if ok:
            assert st[i] == 0, (i, kinds[i], st[i])
            want = port.tool_node_event(node, r)
            got = [(p.topic, p.key, p.payload) for p in pubs[k:k + len(want)]]
            assert got == [(t, kk, pl) for (t, kk, c, pl) in want], (i, kinds[i])
            k += len(want)
        else:
            assert st[i] == cls, (i, kinds[i], st[i], cls)
    assert k == len(pubs)
    assert {kinds[i] for i in range(len(recs)) if st[i] == 0} >= {0, 2, 4, 5} and {kinds[i] for i in range(len(recs)) if st[i] != 0} == {1, 3}


def test_element_list_overflow_falls_back_to_the_warp_walk():
    """More history messages in a batch than the element list holds (tiny messages, an engine sized to the bytes): the
    reservations that do not fit are voided and those records are walked by their warp instead — same outputs."""
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import tools_def
    from oracle import port
    from calfkit import synth
    from calfkit.engine import BatchEngine, ToolTemplate
    base = synth.tool_events(96, seed=13)
    marker = b'"message_history":['
    recs = []
    for i, r in enumerate(base):
        turns = ",".join(synth.user_request("q%d" % k) for k in range(120 + i % 5))
        p = r.index(marker) + len(marker)
        recs.append(r[:p] + turns.encode() + b"," + r[p:])
    b = synth.pack(recs)
    n_msgs = sum(120 + i % 5 for i in range(len(recs)))
    e = BatchEngine(0, max_records=128, max_in_bytes=int(b.data.nbytes) + 4096)
    assert n_msgs > (int(b.data.nbytes) + 4096) // 256 + 1024          # more messages than list entries (ck_api.cu: elem_cap)
    try:
        e.register_topics(["tool.get_weather.input", "tool.get_weather.output", "weather_agent.input"], num_partitions=8)
        e.set_tool_node("tool.get_weather.output", ToolTemplate.from_format("It's sunny in {location}"))
        out = e.run_tool_batch(b.data, b.offsets)
        assert (out.cols[0] == 0).all()
        node = port.ToolNode.of(tools_def.get_weather)
        got = [(p.topic, p.key, p.payload) for p in out.publishes()]
        want = [(t, k, pl) for r in recs for (t, k, _c, pl) in port.tool_node_event(node, r)]
        assert got == want
    finally:
        e.close()


def test_exchange_plan_kernels_match_tensor_plan(engine):
    """ck_exchange_plan (histogram -> scan -> stable scatter -> scan) against the device-agnostic tensor plan that
    the world-size-2 gloo test covers (calfkit/engine/exchange.py), on a real publish table, for every rank of
    several world sizes."""
    import torch
    from calfkit import synth
    from calfkit.engine._lib import PUB_DTYPE
    from calfkit.engine.exchange import plan_exchange, plan_exchange_device
    recs = synth.tool_events(3000, seed=21) + synth.mixed_events(200, seed=22)
    b = synth.pack(recs)
    out = engine.run_tool_batch(b.data, b.offsets)
    dev = torch.device("cuda", 0)
    pubs = torch.from_numpy(out.pubs.view(np.int32).reshape(-1, PUB_DTYPE.itemsize // 4).copy()).to(dev)
    off = torch.from_numpy(out.out_off.astype(np.int64)).to(dev)
    ln = torch.from_numpy(out.out_len.astype(np.int32)).to(dev)
    for world in (1, 2, 3, 8):
        for rank in range(world):
            want = plan_exchange(pubs, off, ln, rank, world)
            got = plan_exchange_device(engine, rank, world, dev)
            assert got.counts.tolist() == want.counts.tolist() and got.nbytes.tolist() == want.nbytes.tolist()
            assert got.sel.to(torch.int64).tolist() == want.sel.tolist()
            assert got.src_off.tolist() == want.src_off.tolist() and got.lens.tolist() == want.lens.tolist()
            assert got.dst_off.tolist() == want.dst_off.tolist()


def test_reply_outputs_match_reference_goldens_and_oracle(engine):
    """client reply path (SURVEY §8f row 3): ck_reply_plan + emit against tests/golden/replies.json (the unmodified
    reference's deserialize_to_node_result) and against the oracle on replies produced by the tool / agent path."""
    import pydantic_core
    from oracle import port
    from calfkit import synth
    from calfkit.client.batch_reply import BatchReplyDecoder
    from calfkit.engine._lib import CK_ACT_RAISES, CK_ACT_REPLY, COL
    cases = golden("replies.json")
    recs = [c["input"].encode() for c in cases]
    b = synth.pack(recs)
    for mode, label in ((0, "auto"), (1, "str"), (2, "dict")):
        engine.submit(b.data, b.offsets)
        engine.reply_plan(mode)
        out = engine.fetch()
        assert (out.cols[COL["STATUS"]] == 0).all()
        for i, c in enumerate(cases):
            exp = c["expect"][label]
            if exp["ok"] or exp["error"] == "ValidationError":       # the typed validation is the host's step (as in the reference)
                assert out.cols[COL["ACTION"], i] == CK_ACT_REPLY, (c["name"], label)
                if exp["ok"]:
                    assert out.payload(i).decode() == exp["output_json"], (c["name"], label)
            else:
                assert out.cols[COL["ACTION"], i] == CK_ACT_RAISES and out.payload(i) == b"", (c["name"], label)
    # the host wrapper: same values / same exception classes as the reference, typed output included
    dec = BatchReplyDecoder(engine)
    for label, ot in (("auto", None), ("str", str), ("dict", dict)):
        got = dec.decode(recs) if ot is None else dec.decode(recs, ot)
        for c, g in zip(cases, got):
            exp = c["expect"][label]
            if exp["ok"]:
                assert g.error is None and pydantic_core.to_json(g.output).decode() == exp["output_json"] and g.correlation_id == exp["correlation_id"]
            else:
                assert type(g.error).__name__ == exp["error"], (c["name"], label, g)
    # replies as the path itself produces them: tool-stage events popped down to the client frame, random final parts
    rng = random.Random(5)
    recs2 = []
    for r in synth.mixed_events(200, seed=33, hi=6000):
        parts = []
        for _ in range(rng.randrange(0, 4)):
            k = rng.randrange(3)
            if k == 0:
                parts.append('{"kind":"text","text":%s,"metadata":null}' % json.dumps("t" * rng.randrange(0, 200) + "é\n", ensure_ascii=False))
            elif k == 1:
                parts.append('{"kind":"data","data":%s,"schema_":null,"metadata":null}' % json.dumps({"v": [round(rng.random(), 6) for _ in range(rng.randrange(0, 30))]}, separators=(",", ":")))
            else:
                parts.append('{"kind":"file","media_type":"text/plain","uri":null,"data":null,"metadata":null}')
        recs2.append(r.replace(b'"final_output_parts":[]', ('"final_output_parts":[' + ",".join(parts) + "]").encode()))
    b2 = synth.pack(recs2)
    engine.submit(b2.data, b2.offsets)
    engine.reply_plan(0)
    out = engine.fetch()
    n_ok = 0
    for i, r in enumerate(recs2):
        if out.cols[COL["STATUS"], i] != 0:
            continue                                                # floats with > 15 digits: declared UNSUPPORTED, never wrong
        n_ok += 1
        try:
            _corr, want = port.reply_output(r)
            assert out.cols[COL["ACTION"], i] == CK_ACT_REPLY and out.payload(i) == want, i
        except Exception as e:  # noqa: BLE001
            assert type(e).__name__ == "DeserializationError" and out.cols[COL["ACTION"], i] == CK_ACT_RAISES, (i, repr(e))
    assert n_ok > 50


def test_long_floats_on_device(engine):
    """16-17 digit floats (computed values such as 0.30000000000000004): accepted in place when they are the
    shortest round-trip spelling (csrc/ck_float.cuh), in canonical and in re-spelled records; literals of 16-19 digits that
    are NOT that spelling are replaced by it (exact search, ckf_shortest); outputs byte-exact."""
    import tools_def
    from oracle import port
    from calfkit import synth
    from calfkit.engine import ToolTemplate
    rng = random.Random(12)
    _setup(engine, "get_weather", ToolTemplate.from_format("It's sunny in {location}"))
    node = port.ToolNode.of(tools_def.get_weather)
    base = synth.tool_events(300, seed=41)
    recs = []
    for k, r in enumerate(base):
        vals = [repr(rng.choice([rng.random(), 0.1 + 0.2, rng.uniform(-1e6, 1e6), rng.random() * 1e-7, rng.random() * 1e18]))
                for _ in range(rng.randrange(1, 6))]
        if k % 5 == 0:      # literals longer than the shortest spelling (%.17e / %.18e): the device finds the reference's spelling
            vals += [("%." + str(rng.choice([16, 17, 18])) + "e") % rng.choice([rng.random(), rng.uniform(-1e9, 1e9), rng.random() * 1e-12])
                     for _ in range(2)] + ["123456789.123456789", "0.1000000000000000055"]
        i = r.index(b'"provided_deps":{') + len(b'"provided_deps":{')
        j = r.index(b"}", i)
        sep = b" , " if k % 3 == 0 else b","                       # every third record is re-spelled (canonicaliser path)
        recs.append(r[:i] + b'"v":[' + sep.join(v.encode() for v in vals) + b"]" + r[j:])
    b = synth.pack(recs)
    out = engine.run_tool_batch(b.data, b.offsets)
    assert (out.cols[0] == 0).all(), np.bincount(out.cols[0])
    want = [(tp, k, pl) for r in recs for (tp, k, _c, pl) in port.tool_node_event(node, r)]
    assert _pubs(out) == want


def test_fanout_64_matches_oracle_config3(engine):
    """BASELINE.json configs[2]: 1 Agent node -> 64 @agent_tool nodes.  Every one of the 64 Call envelopes of every event
    (and the handler-return publish) byte-exact against the oracle, ids injected from the device generator; plus records with
    some results already present (partial fan-out) and one whose tool the registry does not know."""
    from oracle import port
    from calfkit import _ids, synth
    from calfkit.engine.batch import device_uuid7_hex
    from calfkit.engine import BatchEngine
    F = 64
    recs = synth.fanout_events(24, seed=19, fanout=F)
    # partial: give record 3 results for a third of its calls (they are no longer pending)
    env = json.loads(recs[3])
    ids = list(env["context"]["state"]["tool_calls"])
    for cid in ids[::3]:
        env["context"]["state"]["tool_results"][cid] = {"return_value": "done", "content": None, "metadata": {"tool_call_id": cid}, "kind": "tool-return"}
    recs[3] = port.encode(port.decode(json.dumps(env).encode()))
    registry = {f"tool_{j:02d}": f"tool.tool_{j:02d}.input" for j in range(F)}
    e = BatchEngine(0, max_records=64, max_in_bytes=8 << 20, max_out_bytes=256 << 20, max_payloads=64 * (F + 1))
    try:
        e.register_topics(list(registry.values()) + ["planner.input", "planner.output"], num_partitions=8)
        e.set_agent_node("planner", "planner.input", "planner.output", registry)
        b = synth.pack(recs)
        ms, seed = 1767225600000, 4321
        e.submit(b.data, b.offsets)
        e.fanout_plan(ms, seed, max_fanout=64)
        out = e.fetch()
        assert (out.cols[0] == 0).all()
        pubs = list(out.publishes())
        slot = k = 0
        for i, rec in enumerate(recs):
            st = port.decode(rec).context.state
            npend = len([c for c in st.tool_calls if c not in st.tool_results])
            it = iter([device_uuid7_hex(ms, seed, slot + j) for j in range(npend)])
            _ids.set_id_source(lambda: next(it))
            try:
                want = port.agent_fanout("planner", "planner.input", "planner.output", registry, rec)
            finally:
                _ids.set_id_source(None)
            got = [(p.topic, p.key, p.payload) for p in pubs[k:k + len(want)]]
            assert len(want) == npend + 1 and got == [(t, kk, pl) for (t, kk, c, pl) in want], i
            k += len(want)
            slot += npend + 1
        assert k == len(pubs)
    finally:
        e.close()


def test_mixed_sizes_256_topics_config5(engine):
    """BASELINE.json configs[4] shape: sizes log-uniform 128 B - 64 KB (multi-turn histories with escapes and multi-byte
    UTF-8), callbacks spread over 256 registered topics: every publish (topic, key, partition, payload) against the oracle."""
    import tools_def
    from oracle import port
    from calfkit import synth
    from calfkit.engine import BatchEngine, ToolTemplate
    recs = synth.mixed_events(700, seed=41, hi=65536, n_agents=256)
    assert max(len(r) for r in recs) > 40000 and min(len(r) for r in recs) < 1500
    topics = [f"agent_{k:03d}.input" for k in range(256)] + ["tool.get_weather.input", "tool.get_weather.output"]
    e = BatchEngine(0, max_records=1024, max_in_bytes=32 << 20)
    try:
        e.register_topics(topics, num_partitions=8)
        e.set_tool_node("tool.get_weather.output", ToolTemplate.from_format("It's sunny in {location}"))
        b = synth.pack(recs)
        e.submit(b.data, b.offsets)
        e.tool_plan()
        out = e.fetch()
        assert (out.cols[0] == 0).all()
        assert (out.live()["topic_id"] >= 0).all()            # all 256 callback topics resolved on the device
        node = port.ToolNode.of(tools_def.get_weather)
        got = [(p.topic, p.key, p.payload, p.partition) for p in out.publishes()]
        want = []
        for r in recs:
            for (t, k, _c, pl) in port.tool_node_event(node, r):
                want.append((t, k, pl, -1 if k is None else (_murmur2(k) & 0x7FFFFFFF) % 8))
        assert got == want
        assert len({t for t, *_ in got}) > 200             # 700 records spread over 256 callback topics + the publish topic
    finally:
        e.close()


def _murmur2(data: bytes) -> int:
    m, h = 0x5BD1E995, (0x9747B28C ^ len(data)) & 0xFFFFFFFF
    n4 = len(data) // 4
    for i in range(n4):
        k = int.from_bytes(data[4 * i:4 * i + 4], "little")
        k = (k * m) & 0xFFFFFFFF; k ^= k >> 24; k = (k * m) & 0xFFFFFFFF
        h = (h * m) & 0xFFFFFFFF; h ^= k
    t = data[4 * n4:]
    if len(t) == 3: h ^= t[2] << 16
    if len(t) >= 2: h ^= t[1] << 8
    if len(t) >= 1: h ^= t[0]; h = (h * m) & 0xFFFFFFFF
    h ^= h >> 13; h = (h * m) & 0xFFFFFFFF; h ^= h >> 15
    return h


DECLARED_UNSUPPORTED = {"frame_missing_frame_id": "default_factory field: the reference invents a fresh id"}


def test_codec_goldens_on_device(engine):
    """All 109 reference codec vectors through decode on the device: fixed points are recognised in place, other valid
    spellings (whitespace, missing defaults, aliases, duplicate keys, lax int / bool spellings, a tagged-but-invalid tool
    result ...) come back as exactly the reference's dump, invalid ones carry the reference's error class.  The declared
    carve-outs are listed above by name — nothing else may be declined."""
    from calfkit import synth
    from calfkit.engine._lib import COL
    cases = golden("codec.json")
    recs = [as_bytes(c["input"]) for c in cases]
    b = synth.pack(recs)
    engine.submit(b.data, b.offsets)
    cols = engine.columns()
    ovl = engine.overlay()
    declined = []
    for i, c in enumerate(cases):
        st = int(cols[COL["STATUS"], i])
        if st == 4:
            declined.append(c["name"])
            continue
        if len(recs[i]) == 0:
            assert st == 5
            continue
        if c["ok"]:
            assert st == 0, (c["name"], st)
            have = recs[i] if (ovl is None or ovl[1][i] < 0) else ovl[0][int(ovl[1][i]):int(ovl[1][i]) + int(ovl[2][i])].tobytes()
            assert have == c["output"].encode(), c["name"]
        else:
            assert st == (2 if c["first_type"] == "json_invalid" and c["n_errors"] == 1 else 3), (c["name"], st)
    assert set(declined) <= set(DECLARED_UNSUPPORTED), declined


def test_length_bucketing_changes_nothing_but_the_schedule(engine):
    """CK_OPT_BUCKET: the walk takes the records in length order (a permutation built on the device); every column, payload
    and publish must be identical to the unbucketed run — on a batch that mixes sizes, shapes, invalid and empty records."""
    from calfkit import synth
    from calfkit.engine import BatchEngine, ToolTemplate
    rng = random.Random(3)
    recs = synth.mixed_events(300, seed=51, hi=30000, n_agents=16) + synth.tool_events(500, seed=52) + \
        synth.tool_events(100, seed=53, size=None, full_history=True) + [b"", b"{", b'{"context":{}}']
    recs += [bytes(r[:-3]) for r in recs[:20]] + [b"{ " + r[1:] for r in recs[300:320]]
    rng.shuffle(recs)
    b = synth.pack(recs)
    topics = [f"agent_{k:03d}.input" for k in range(16)] + ["tool.get_weather.input", "tool.get_weather.output", "weather_agent.input"]
    outs = []
    for bucket in (False, True):
        e = BatchEngine(0, max_records=2048, max_in_bytes=32 << 20)
        try:
            e.register_topics(topics, num_partitions=8)
            e.set_tool_node("tool.get_weather.output", ToolTemplate.from_format("It's sunny in {location}"))
            e.set_bucketing(bucket)
            e.submit(b.data, b.offsets)
            e.tool_plan()
            o = e.fetch()
            outs.append((o.cols.copy(), [(p.topic, p.key, p.payload, p.partition, p.record) for p in o.publishes()]))
        finally:
            e.close()
    ok_rows = outs[0][0][0] == 0
    assert (outs[0][0][0] == outs[1][0][0]).all() and (outs[0][0][:, ok_rows] == outs[1][0][:, ok_rows]).all()
    assert outs[0][1] == outs[1][1] and ok_rows.sum() > 900
