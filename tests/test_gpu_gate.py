"""SURVEY.md section 8 rows a10 / f4 — the aggregation gate on the device (csrc/ck_gate.cuh) against the reference's own gate:
tests/golden/aggregation.json was produced by the unmodified `_parallel_state_aggregation` (reference nodes/agent.py:57-68);
a 64-way fan-out with shuffled, duplicated and foreign arrivals is checked against the oracle port of the same function."""
import json
import random

import numpy as np
import pytest

from conftest import golden

pytestmark = pytest.mark.gpu

FRAME = ('{"target_topic":"planner.input","callback_topic":"calf-client-reply-1","input_args":null,'
         '"frame_id":"00000000000000000000000000000001","overrides":null}')


def envelope(state_json: str, corr: str) -> bytes:
    return ('{"context":{"state":' + state_json + ',"deps":{"correlation_id":' + json.dumps(corr) + ',"provided_deps":{}}},'
            '"internal_workflow_state":{"call_stack":{"_internal_list":[' + FRAME + ']},"metadata":null}}').encode()


def state_of(env: bytes) -> str:
    s = env.decode()
    return s[len('{"context":{"state":'):s.index(',"deps":{"correlation_id":')]


@pytest.fixture()
def engine():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from calfkit.engine import BatchEngine
    e = BatchEngine(0, max_records=4096, max_in_bytes=128 << 20, max_payloads=4096 * 70)
    tools = {f"tool_{j:02d}": f"tool.tool_{j:02d}.input" for j in range(64)}
    e.register_topics(list(tools.values()) + ["planner.input", "planner.output"], num_partitions=8)
    e.set_tool_node("planner.output", None)
    e.set_agent_node("planner", "planner.input", "planner.output", tools)
    e.gate_create(max_entries=1024, arena_bytes=64 << 20)
    yield e
    e.close()


def register(engine, base_envs):
    from calfkit import synth
    b = synth.pack(base_envs)
    engine.submit(b.data, b.offsets)
    engine.fanout_plan(1767225600000, 7, max_fanout=256)
    engine.gate_register(min_pending=1)      # the golden cases include a one-id batch (the reference's rule is > 1)
    engine.sync()
    assert engine.gate_stats()["live"] == len(base_envs)


def arrive(engine, envs, stamp_base):
    from calfkit import synth
    from calfkit.engine._lib import COL
    b = synth.pack(envs)
    engine.submit(b.data, b.offsets)
    engine.gate_arrive(stamp_base)
    out = engine.fetch()
    return out, out.cols[COL["ACTION"]]


@pytest.mark.parametrize("case", golden("aggregation.json"), ids=lambda c: c["name"])
@pytest.mark.parametrize("batched", [False, True], ids=["one_by_one", "one_batch"])
def test_gate_matches_reference_goldens(engine, case, batched):
    from calfkit.engine._lib import CK_ACT_GATE_COMPLETE, CK_ACT_GATE_PASS, CK_ACT_SILENT
    register(engine, [envelope(case["base_state"], case["correlation_id"])])
    envs = [envelope(st["incoming"], st["correlation_id"]) for st in case["steps"]]
    results = []
    if batched:
        out, act = arrive(engine, envs, 100)
        results = [(int(act[i]), out.payload(i)) for i in range(len(envs))]
    else:
        for k, e in enumerate(envs):
            out, act = arrive(engine, [e], 100 + k)
            results.append((int(act[0]), out.payload(0)))
    for st, env, (action, payload) in zip(case["steps"], envs, results):
        if st["correlation_id"] != case["correlation_id"]:
            assert action == CK_ACT_GATE_PASS                   # no pending fan-out for that id: continues with its own state
        elif st["complete"]:
            assert action == CK_ACT_GATE_COMPLETE, case["name"]
            assert state_of(payload) == st["state"], case["name"]
            assert payload == envelope(st["state"], st["correlation_id"])
        else:
            assert action == CK_ACT_SILENT, case["name"]
            assert payload == env                               # handler return of a Silent: the inbound envelope -> publish_topic
    assert engine.gate_stats()["live"] == (0 if case["steps"][-1]["complete"] else 1)


@pytest.mark.parametrize("chunk", [1, 7, 1000], ids=["one_by_one", "chunks_of_7", "one_batch"])
def test_gate_64_way_shuffled_against_oracle(engine, chunk):
    """two concurrent 64-way fan-outs; arrivals shuffled together, with duplicates, a foreign correlation id and late
    arrivals after completion; the device (batched, stamps) must agree with the oracle's one-at-a-time gate."""
    from calfkit import synth
    from calfkit.engine._lib import CK_ACT_GATE_COMPLETE, CK_ACT_GATE_PASS, CK_ACT_SILENT
    from calfkit.models import State
    from calfkit.models.state import PendingToolBatch
    from oracle import port
    rng = random.Random(5)
    bases = synth.fanout_events(2, seed=77, fanout=64)
    register(engine, bases)
    batches, arrivals = {}, []
    for b in bases:
        env = json.loads(b)
        corr = env["context"]["deps"]["correlation_id"]
        st = State.model_validate(env["context"]["state"])
        ids = list(st.tool_calls)
        batches[corr] = PendingToolBatch(expected_tool_call_ids=frozenset(ids), base_state=st.model_copy(deep=True))
        for j, cid in enumerate(ids):
            s2 = st.model_copy(deep=True)
            value = {"return_value": f"It's sunny in city {j} é\n", "content": None, "metadata": {"tool_call_id": cid}, "kind": "tool-return"}
            s2.tool_results[cid] = value if j % 5 else {"raw": [j, 1.5, None], "note": "an untagged value"}
            arrivals.append((corr, s2.model_dump_json()))
        arrivals += rng.sample(arrivals[-64:], 5)                 # duplicates (at-least-once delivery)
    rng.shuffle(arrivals)
    arrivals.insert(3, ("f" * 32, arrivals[0][1]))             # a correlation id nobody is waiting for
    arrivals += [arrivals[10], arrivals[20]]                   # late arrivals: their fan-outs are complete by then
    envs = [envelope(s, c) for c, s in arrivals]
    got = []
    for a in range(0, len(envs), chunk):
        out, act = arrive(engine, envs[a:a + chunk], 1000 + a)
        got += [(int(act[i]), out.payload(i)) for i in range(len(envs[a:a + chunk]))]
    completes = 0
    for (corr, sjson), env, (action, payload) in zip(arrivals, envs, got):
        pending_before = corr in batches
        merged = port.aggregate(batches, State.model_validate_json(sjson), corr)
        if not pending_before:
            assert action == CK_ACT_GATE_PASS
        elif merged is None:
            assert action == CK_ACT_SILENT and payload == env
        else:
            completes += 1
            assert action == CK_ACT_GATE_COMPLETE
            assert payload == envelope(merged.model_dump_json(), corr)
    assert completes == 2 and not batches and engine.gate_stats()["live"] == 0


# ---- the gate as a long-lived Worker runs it: many fan-outs, colliding ids, duplicates, capacity -------------------------
N_TOOLS = 71                                    # fan-outs of up to 70 calls, plus one call answered before the fan-out


@pytest.fixture()
def make_engine():
    """engines with a gate of the given size; closed after the test"""
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from calfkit.engine import BatchEngine
    made = []

    def make(max_entries, max_slots=None, arena_bytes=64 << 20):
        e = BatchEngine(0, max_records=4096, max_in_bytes=64 << 20, max_payloads=4096 * 8)
        tools = {f"tool_{j:02d}": f"tool.tool_{j:02d}.input" for j in range(N_TOOLS)}
        e.register_topics(list(tools.values()) + ["planner.input", "planner.output"], num_partitions=8)
        e.set_tool_node("planner.output", None)
        e.set_agent_node("planner", "planner.input", "planner.output", tools)
        e.gate_create(max_entries=max_entries, max_slots=max_slots, arena_bytes=arena_bytes)
        made.append(e)
        return e
    yield make
    for e in made:
        e.close()


def to_json(v) -> str:
    import pydantic_core
    return pydantic_core.to_json(v).decode()


def tool_value(j: int, cid: str):
    """tool results with escapes and multi-byte UTF-8, in three shapes"""
    if j % 3 == 0:
        return {"return_value": f"It's sunny in city {j} é\n\"quoted\" back\\slash\t漢字 🙂", "content": None,
                "metadata": {"tool_call_id": cid}, "kind": "tool-return"}
    if j % 3 == 1:
        return {"raw": [j, 1.5, None, "ü"], "note": "an untagged value / «»"}
    return f"plain {j}:   \"x\" 🙂"


class FanOut:
    """one agent turn that fanned out `k` tool calls (base envelope from synth, correlation id replaced); with `pre` the
    state already carries one answered call, so tool_results is not {} at fan-out"""

    def __init__(self, corr: str, k: int, seed: int, pre: bool = False):
        from calfkit import synth
        from calfkit.models import State
        raw = synth.fanout_events(1, seed=seed, fanout=k + pre)[0]
        old = json.loads(raw)["context"]["deps"]["correlation_id"].encode()
        assert raw.count(old) == 1
        raw = raw.replace(old, corr.encode())
        ids = list(json.loads(raw)["context"]["state"]["tool_calls"])
        self.pre_text = ""
        if pre:
            assert raw.count(b'"tool_results":{}') == 1
            self.pre_text = json.dumps(ids[0]) + ":" + to_json({"raw": ["answered earlier"], "note": "é"})
            raw = raw.replace(b'"tool_results":{}', ('"tool_results":{' + self.pre_text + "}").encode())
        self.corr, self.env, self.sj = corr, raw, state_of(raw)
        self.state = State.model_validate_json(self.sj)
        assert self.state.model_dump_json() == self.sj          # the expected merges are pydantic dumps of this state
        self.pending = ids[1:] if pre else ids
        self.pre_keys = list(self.state.tool_results)

    def arrival(self, cids, values=None):
        """(corr, state JSON, tool_results) of a tool return carrying the results of `cids`"""
        from types import SimpleNamespace
        vals = values or {c: tool_value(self.pending.index(c), c) for c in cids}
        pieces = ([self.pre_text] if self.pre_text else []) + [json.dumps(c) + ":" + to_json(vals[c]) for c in cids]
        old = '"tool_results":{' + self.pre_text + "}"
        assert self.sj.count(old) == 1
        sj = self.sj.replace(old, '"tool_results":{' + ",".join(pieces) + "}")
        res = dict(self.state.tool_results)
        res.update(vals)
        return self.corr, sj, SimpleNamespace(tool_results=res)


class GateSim:
    """drives the device gate and `port.aggregate` (one arrival at a time, the reference's rule) side by side and checks
    every arrival: its ACTION, and its payload byte for byte, and after every call the live count and the failures."""

    def __init__(self, engine, stamp: int = 1000):
        self.e, self.stamp = engine, stamp
        self.batches, self.fos, self.seq = {}, {}, {}
        self.n_arrivals = self.compactions = self.completes = 0

    def register(self, fos, failures: int = 0, compact: bool = True):
        from calfkit import synth
        from calfkit.models.state import PendingToolBatch
        if compact:
            self.compactions += self.e.gate_compact(room=len(fos))
        b = synth.pack([f.env for f in fos])
        self.e.submit(b.data, b.offsets)
        self.e.fanout_plan(1767225600000, 7, max_fanout=256)
        self.e.gate_register()
        self.e.sync()
        for f in fos:                                           # dict assignment in record order: the later one wins
            self.batches[f.corr] = PendingToolBatch(expected_tool_call_ids=frozenset(f.pending),
                                                    base_state=f.state.model_copy(deep=True))
            self.fos[f.corr] = f
        st = self.e.gate_stats()
        assert st["failures"] == failures, st
        if not failures:
            assert st["live"] == len(self.batches), st

    def expect(self, corr, res):
        """(action, expected payload or None) of the next arrival by the oracle"""
        from calfkit.engine._lib import CK_ACT_GATE_COMPLETE, CK_ACT_GATE_PASS, CK_ACT_SILENT
        from oracle import port
        batch = self.batches.get(corr)
        if batch is None:
            port.aggregate(self.batches, res, corr)
            return CK_ACT_GATE_PASS, None
        before = set(batch.collected_results)
        merged = port.aggregate(self.batches, res, corr)
        for c in batch.collected_results:
            if c not in before:
                self.seq[(corr, c)] = self.n_arrivals
        if merged is None:
            return CK_ACT_SILENT, None
        # collection order: arrival by arrival; the results one arrival carries are collected by the device in tool_calls
        # order, while the reference iterates a frozenset there (unspecified order): only those pieces are reordered
        f = self.fos[corr]
        got = [c for c in merged.tool_results if c not in f.pre_keys]
        got.sort(key=lambda c: (self.seq[(corr, c)], f.pending.index(c)))
        merged.tool_results = {c: merged.tool_results[c] for c in f.pre_keys + got}
        return CK_ACT_GATE_COMPLETE, envelope(merged.model_dump_json(), corr)

    def arrive(self, items, compact: bool = True):
        """items: (corr, state JSON, tool_results) in arrival order, delivered as one batch"""
        from calfkit.engine._lib import CK_ACT_GATE_COMPLETE, CK_ACT_SILENT
        if compact:
            self.compactions += self.e.gate_compact()
        envs = [envelope(sj, c) for c, sj, _ in items]
        out, act = arrive(self.e, envs, self.stamp)
        self.stamp += len(envs)
        for i, ((corr, _sj, res), env) in enumerate(zip(items, envs)):
            want, payload = self.expect(corr, res)
            self.n_arrivals += 1
            assert int(act[i]) == want, (i, corr, int(act[i]), want)
            if want == CK_ACT_SILENT:
                assert out.payload(i) == env                    # the handler return of a Silent: the inbound envelope
            elif want == CK_ACT_GATE_COMPLETE:
                self.completes += 1
                assert out.payload(i) == payload, (i, corr)
        st = self.e.gate_stats()
        assert st["failures"] == 0 and st["live"] == len(self.batches), st
        return out, act


def hexid(rng) -> str:
    return "%032x" % rng.getrandbits(128)


def soak_sizes(rng, n):
    """fan-out sizes 2..70: the merge's 32-lane loops at 31, 32, 33, 63, 64, 65 and 70, the rest mostly small"""
    edges = [31, 32, 33, 63, 64, 65, 70]
    sizes = [edges[i % len(edges)] for i in range(3 * len(edges))]
    while len(sizes) < n:
        sizes.append(rng.randint(2, 8) if rng.random() < 0.7 else rng.randint(2, 70))
    rng.shuffle(sizes)
    return sizes


def soak(sim, rng, n: int) -> dict:
    """drive `sim` through `n` fan-outs: at most 16 live and 150 expected ids pending at a time, arrivals shuffled across
    fan-outs in batches of 1..48 with redeliveries, late arrivals and a foreign id; one or two long-lived "anchor"
    fan-outs get one arrival per batch, and the next anchor is registered before the current one drains, so the live
    count never returns to 0 while fan-outs remain"""
    todo = [FanOut(hexid(rng), k, seed=10_000 + j, pre=(j % 7 == 3)) for j, k in enumerate(soak_sizes(rng, n))]
    todo.reverse()
    outstanding, late, anchors = [], [], []
    pending_ids = lambda: sum(len(b.expected_tool_call_ids) for b in sim.batches.values())   # noqa: E731
    min_live, slots_total = None, 0
    while todo or outstanding or late or anchors:
        new = []
        while todo and len(sim.batches) + len(new) < 16 and pending_ids() + sum(len(f.pending) for f in new) + len(todo[-1].pending) <= 150:
            new.append(todo.pop())
        if new:
            sim.register(new)
            slots_total += sum(len(f.pending) for f in new)
            for f in new:
                cids = list(f.pending)
                rng.shuffle(cids)
                groups, g = [], 0
                while g < len(cids):                            # most tool returns carry one result, some two or three
                    w = 1 if rng.random() < 0.75 else rng.randint(2, 3)
                    groups.append(cids[g:g + w])
                    g += w
                arr = [f.arrival(grp) for grp in groups]
                if rng.random() < 0.2:
                    arr += rng.sample(arr, min(len(arr), rng.randint(1, 3)))      # at-least-once redelivery
                if rng.random() < 0.1:
                    late.append(rng.choice(arr))                                   # delivered after the fan-out completed
                if len(arr) >= 6 and len(anchors) < 2:
                    anchors.append(arr)
                else:
                    outstanding += arr
        rng.shuffle(outstanding)
        take = rng.randint(1, 48)
        chunk, outstanding = outstanding[:take], outstanding[take:]
        if anchors:
            chunk.append(anchors[0].pop())
            if not anchors[0]:
                anchors.pop(0)
        if not (outstanding or todo or anchors):
            chunk += late
            late = []
        elif late and rng.random() < 0.3:
            chunk.append(late.pop())
        if chunk and rng.random() < 0.05:
            chunk.insert(rng.randrange(len(chunk) + 1), ("f" * 32, chunk[0][1], chunk[0][2]))   # nobody waits for this id
        rng.shuffle(chunk)
        sim.arrive(chunk)
        if todo:
            min_live = len(sim.batches) if min_live is None else min(min_live, len(sim.batches))
    return {"min_live": min_live, "slots_total": slots_total}


def test_gate_soak_against_oracle(make_engine):
    """~3,000 fan-outs of 2..70 calls through a gate of 64 entries, 384 slots and 1 MiB of arena: lifetimes overlap (the
    live count never returns to 0), arrivals are shuffled across fan-outs with duplicates, late arrivals and a foreign id,
    some arrivals carry several results, and stamps cross 2^32.  In all it registers many times the entries, slots and
    arena bytes the gate holds: only reclaiming finished fan-outs keeps it going."""
    eng = make_engine(max_entries=64, max_slots=384, arena_bytes=1 << 20)
    sim = GateSim(eng, stamp=(1 << 32) - 4000)
    r = soak(sim, random.Random(2026), 3000)
    assert sim.completes == 3000 and not sim.batches and eng.gate_stats()["live"] == 0
    assert sim.stamp > 1 << 32
    assert r["min_live"] > 0                                    # lifetimes overlap: the old reset rule never applied
    assert r["slots_total"] > 50 * 384 and sim.compactions >= 3000 // 64, (r, sim.compactions)


def fnv1a64(b: bytes) -> int:
    h = 14695981039346656037
    for x in b:
        h = ((h ^ x) * 1099511628211) & 0xFFFFFFFFFFFFFFFF
    return h + 2 if h < 2 else h


def colliding_ids(rng, bucket: int, cap: int, n: int) -> list[str]:
    """32-hex correlation ids whose FNV-1a-64 (the device's key hash, over the id as it lies in the envelope) starts
    its probe at `bucket` of a table of `cap` key slots"""
    out = []
    while len(out) < n:
        c = hexid(rng)
        if fnv1a64(c.encode()) & (cap - 1) == bucket:
            out.append(c)
    return out


def test_gate_probe_chains(make_engine):
    """ids that share a bucket: a chain starting in the last bucket wraps to bucket 0, where a second chain starts;
    lookups walk past completed (dead) keys, a live id is registered again (replaced) and a completed id is registered
    again; a compaction rebuilds the key table halfway through.  Everything is checked against the oracle."""
    eng = make_engine(max_entries=64, max_slots=512, arena_bytes=4 << 20)
    cap = 256                                                   # ck_gate_create: the power of two >= 4 * max_entries
    rng = random.Random(9)
    last = colliding_ids(rng, cap - 1, cap, 5)
    zero = colliding_ids(rng, 0, cap, 3)
    sim = GateSim(eng)
    seed = iter(range(500, 10_000))
    fos = {c: FanOut(c, rng.randint(2, 5), next(seed)) for c in last + zero}

    def all_of(f, order=None):
        items = [f.arrival([c]) for c in (order or f.pending)]
        return items

    sim.register([fos[c] for c in last + zero], compact=False)
    # complete the first ids of each chain: their keys stay behind as dead keys until the next compaction
    sim.arrive(all_of(fos[last[0]]) + all_of(fos[zero[0]]), compact=False)
    sim.arrive(all_of(fos[last[1]])[:1] + all_of(fos[zero[2]])[:1] + all_of(fos[last[4]])[1:], compact=False)
    # a live id registered again: the new fan-out replaces the old one (the old one's results no longer count)
    old = fos[last[2]]
    fos[last[2]] = FanOut(last[2], 3, next(seed))
    sim.register([fos[last[2]]], compact=False)
    sim.arrive(all_of(old) + all_of(fos[last[2]])[:2], compact=False)
    # a completed id registered again
    fos[last[0]] = FanOut(last[0], 4, next(seed))
    sim.register([fos[last[0]]], compact=False)
    sim.arrive(all_of(fos[last[0]])[:1] + all_of(fos[last[3]])[:1], compact=False)
    assert eng.gate_compact(force=True)
    assert eng.gate_stats()["entries_used"] == len(sim.batches)
    rest = []
    for c in last + zero:
        if c in sim.batches:
            rest += all_of(fos[c])
    rng.shuffle(rest)
    sim.arrive(rest, compact=False)
    assert not sim.batches and eng.gate_stats()["live"] == 0


def test_gate_duplicate_registration_in_one_batch(make_engine):
    """at-least-once redelivery: 300 correlation ids, each fanned out by 2 or 3 records of ONE register batch with
    different tool_call_ids, spread over the batch (different blocks).  The highest record index wins, as dict
    assignment in record order does in the reference; live counts distinct ids; arrivals for the losers' tool_call_ids
    stay Silent and the winners' complete."""
    eng = make_engine(max_entries=1024)
    rng = random.Random(31)
    sim = GateSim(eng)
    fos, seed = [], 20_000
    for _ in range(300):
        corr = hexid(rng)
        for _ in range(rng.randint(2, 3)):
            fos.append(FanOut(corr, rng.randint(2, 4), seed))
            seed += 1
    rng.shuffle(fos)
    sim.register(fos)
    assert eng.gate_stats()["live"] == 300
    items = [f.arrival([c]) for f in fos for c in f.pending]
    rng.shuffle(items)
    for a in range(0, len(items), 500):
        sim.arrive(items[a:a + 500])
    assert sim.completes == 300 and not sim.batches


def test_gate_capacity_entries(make_engine):
    """one batch registers more live fan-outs than the gate holds: that call reports the failures, those ids' tool
    returns pass through, every other fan-out matches the oracle, later calls neither raise nor fail, and new
    registrations succeed once the entries drain"""
    from calfkit.engine._lib import CK_ACT_GATE_PASS
    eng = make_engine(max_entries=16, max_slots=1024)
    rng = random.Random(4)
    sim = GateSim(eng)
    fos = [FanOut(hexid(rng), rng.randint(2, 6), 30_000 + n) for n in range(24)]
    sim.register(fos, failures=8, compact=False)
    assert eng.gate_stats()["live"] == 16
    # which 8 found no room is up to the device: their first tool return passes through, the other 16 are Silent
    firsts = [f.arrival(f.pending[:1]) for f in fos]
    from calfkit.engine._lib import CK_ACT_SILENT
    out, act = arrive(eng, [envelope(sj, c) for c, sj, _ in firsts], sim.stamp)
    sim.stamp += len(firsts)
    failed = {f.corr for f, a in zip(fos, act) if int(a) == CK_ACT_GATE_PASS}
    assert len(failed) == 8 and all(int(a) == CK_ACT_SILENT for f, a in zip(fos, act) if f.corr not in failed)
    assert eng.gate_stats()["failures"] == 0
    for c in failed:
        del sim.batches[c]
    for item in firsts:
        sim.expect(item[0], item[2])
        sim.n_arrivals += 1
    rest = [f.arrival([c]) for f in fos for c in f.pending[1:]]
    rng.shuffle(rest)
    sim.arrive(rest)                                            # the failed ids pass through, the others complete
    assert not sim.batches and sim.completes == 16
    more = [FanOut(hexid(rng), rng.randint(2, 6), 31_000 + n) for n in range(16)]
    sim.register(more)                                          # compacts first: the 16 finished entries come back
    assert sim.compactions >= 1
    sim.arrive([f.arrival([c]) for f in more for c in f.pending])
    assert not sim.batches and eng.gate_stats()["live"] == 0


@pytest.mark.parametrize("short", ["value", "merge"])
@pytest.mark.parametrize("chunk", [1, 3], ids=["one_by_one", "one_batch"])
def test_gate_capacity_arena(make_engine, short, chunk):
    """an arena too small for the collected values (or, with them in, for the merged pieces): the completing tool return
    is declined (STATUS CK_UNSUPPORTED, ACTION CK_ACT_RAISES) and never becomes an envelope, its fan-out is given up
    (live reaches 0), and the gate keeps working after a compaction"""
    from calfkit.engine._lib import COL, CK_ACT_GATE_COMPLETE, CK_ACT_RAISES, CK_ACT_SILENT, CK_UNSUPPORTED
    rng = random.Random(12)
    f = FanOut(hexid(rng), 3, 40_000)
    big = {c: "x" * 3000 for c in f.pending}                   # each value is 3,002 bytes of JSON: 3,008 in the arena
    reg = (len(f.sj) + 15) // 16 * 16 + 32                     # base-state blob + correlation id
    arena = reg + (3008 if short == "value" else 3 * 3008) + 16
    eng = make_engine(max_entries=8, max_slots=64, arena_bytes=arena)
    sim = GateSim(eng)
    sim.register([f], compact=False)
    assert eng.gate_stats()["arena_used"] == reg
    items = [f.arrival([c], big) for c in f.pending]
    envs = [envelope(sj, c) for c, sj, _ in items]
    acts, stats = [], []
    for a in range(0, 3, chunk):
        out, act = arrive(eng, envs[a:a + chunk], sim.stamp)
        sim.stamp += len(envs[a:a + chunk])
        for i in range(len(envs[a:a + chunk])):
            acts.append((int(act[i]), int(out.cols[COL["STATUS"], i]), out.payload(i)))
        stats.append(eng.gate_stats())
    assert [a for a, _, _ in acts[:2]] == [CK_ACT_SILENT, CK_ACT_SILENT]
    assert acts[2][:2] == (CK_ACT_RAISES, CK_UNSUPPORTED) and acts[2][2] == b""
    for a, _, p in acts[:2]:
        json.loads(p)                                           # the Silent returns are the inbound envelopes
    assert stats[-1]["failures"] >= 1 and stats[-1]["live"] == 0
    # the next call reports nothing, and after a compaction a fan-out goes through again
    assert eng.gate_compact(force=True) and eng.gate_stats()["arena_used"] == 0
    g = FanOut(hexid(rng), 2, 40_001)
    sim.batches.clear()
    sim.register([g], compact=False)
    out, act = sim.arrive([g.arrival([c]) for c in g.pending], compact=False)
    assert int(act[1]) == CK_ACT_GATE_COMPLETE and json.loads(out.payload(1))
