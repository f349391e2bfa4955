"""The frame pass on the device (csrc/ck_kafka.cuh): the publishes of a whole step, grouped by (topic, partition), become
produce-ready Kafka RecordBatch v2 frames.  Every frame is compared byte for byte with oracle/kafka_batch.py (pinned to
published known-answer vectors in tests/test_kafka_batch.py), and the frame boundaries with a Python restatement of the
split rule."""
import json

import numpy as np
import pytest

from test_gpu_parity import ESCAPED_CORR_IDS, _murmur2, _with_corr_ids, corr_ids_of_every_length

pytestmark = pytest.mark.gpu

TS = 1767225600123
TOOL_TOPICS = ["tool.get_weather.input", "tool.get_weather.output", "weather_agent.input"]
FRAME_TOPICS = ["weather_agent.input", "tool.get_weather.output"]


@pytest.fixture(autouse=True)
def _cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def tool_engine(nparts, **kw):
    from calfkit.engine import BatchEngine, ToolTemplate
    e = BatchEngine(0, max_records=kw.pop("max_records", 1 << 13), max_in_bytes=kw.pop("max_in_bytes", 64 << 20), **kw)
    e.register_topics(TOOL_TOPICS, num_partitions=nparts)
    e.set_tool_node("tool.get_weather.output", ToolTemplate.from_format("It's sunny in {location}"))
    e.set_frame_topics(FRAME_TOPICS)
    return e


def split_rule(krecs, window):
    """start index of every frame of one group: s_k = encoded size at offsetDelta = rank in the group, P_k = exclusive
    prefix of s; k starts a frame when k == 0 or P_k // W != P_{k-1} // W"""
    from oracle import kafka_batch as kb
    P = np.concatenate(([0], np.cumsum([len(kb.encode_record(r, k, 0)) for k, r in enumerate(krecs)])))
    return [k for k in range(len(krecs)) if k == 0 or P[k] // window != P[k - 1] // window]


def expected_frames(groups, window):
    """groups: ordered {(topic, partition): [KRecord...]} -> [(topic, partition, frame bytes, records)]"""
    from oracle import kafka_batch as kb
    out = []
    for (topic, part), krecs in groups.items():
        starts = split_rule(krecs, window) + [len(krecs)]
        for a, b in zip(starts, starts[1:]):
            f = kb.encode_batch(krecs[a:b], base_offset=0, base_timestamp=TS)
            # the documented bound: 61 + W + one record (its size at its rank in the group)
            assert len(f) <= 61 + window + len(kb.encode_record(krecs[b - 1], b - 1, 0))
            out.append((topic, part, f, b - a))
    return out


def groups_of(out, frame_topics, nparts):
    """the frame topics' publishes of a plan (oracle records), grouped as the device groups them: frame topic in the
    order given, partition + 1 (unkeyed = -1 first), send order inside a group"""
    from calfkit.engine._lib import COL
    from oracle import kafka_batch as kb
    groups = {}
    for p in out.live():
        topic = out.topic_of(p)
        if topic not in frame_topics:
            continue
        r = int(p["record"])
        o = int(out.cols[COL["CORR_OFF"], r])
        corr = json.loads(b'"' + out.record_bytes(r)[o:o + int(out.cols[COL["CORR_LEN"], r])].tobytes() + b'"')
        part = int(p["partition"]) if p["has_key"] else -1
        groups.setdefault((topic, part), []).append(kb.calfkit_record(out.payload(int(p["payload"])), corr, keyed=bool(p["has_key"])))
    order = sorted(groups, key=lambda g: (frame_topics.index(g[0]), g[1] + 1))
    return {g: groups[g] for g in order}


def check_frames(frames, groups, window, nparts):
    from oracle import kafka_batch as kb
    want = expected_frames(groups, window)
    got = [(t, -1 if p is None else p, f.tobytes(), n) for t, p, f, n in frames]
    assert len(got) == len(want)
    for g, w in zip(got, want):
        assert g == w
    # decoded per group: exactly that group's publishes in send order, keyed ones on murmur2(key) % P
    for (topic, part), krecs in groups.items():
        dec = kb.decode_batches(b"".join(f for t, p, f, _n in got if (t, p) == (topic, part)))
        assert [(r.value, r.key, r.headers) for r in dec] == [(r.value, r.key, r.headers) for r in krecs]
        for r in dec:
            assert (r.key is None) == (part == -1)
            if r.key is not None:
                assert part == (_murmur2(r.key) & 0x7FFFFFFF) % nparts


def tool_step(e, recs, window=None):
    from calfkit import synth
    b = synth.pack(recs)
    if window is not None:
        e.set_frame_bytes(window)
    e.submit(b.data, b.offsets)
    e.tool_plan()
    e.encode_frames(TS)
    out = e.fetch()
    return out, e.fetch_frames()


@pytest.mark.parametrize("nparts", [8, 1000, 5000])        # 5000: a group key of three radix passes
def test_tool_step_frames_match_oracle(nparts):
    """config-2-shaped steps, with full-history and mixed-size records: every (topic, partition) group and the unkeyed
    group of the handler-return topic as frames equal to the oracle's, and together exactly the frame topics' publishes"""
    from calfkit import synth
    recs = synth.tool_events(3000, seed=81) + synth.tool_events(200, seed=82, size=None, full_history=True) + \
        synth.tool_events(300, seed=83, size=4000, jitter=3000)
    e = tool_engine(nparts)
    try:
        out, frames = tool_step(e, recs)
        assert (out.cols[0] == 0).all()
        groups = groups_of(out, FRAME_TOPICS, nparts)
        assert sum(len(v) for v in groups.values()) == sum(1 for p in out.publishes() if p.topic in FRAME_TOPICS) >= len(recs)
        assert ("tool.get_weather.output", -1) in groups and len(groups) > min(nparts, 8)
        check_frames(frames, groups, 1 << 20, nparts)
        # the union of the frames: exactly the frame topics' publishes, topic, partition, key and value
        from oracle import kafka_batch as kb
        got = sorted((t, -1 if p is None else p, r.key, r.value) for t, p, f, _n in frames for r in kb.decode_batches(f.tobytes()))
        want = sorted((p.topic, p.partition if p.key is not None else -1, p.key, p.payload) for p in out.publishes() if p.topic in FRAME_TOPICS)
        assert got == want
    finally:
        e.close()


@pytest.mark.parametrize("window", [4 << 10, 64 << 10, 1 << 20])
def test_frame_split_follows_the_window_rule(window):
    """frame boundaries equal the Python restatement of the split rule, with records larger than a window"""
    from calfkit import synth
    recs = synth.tool_events(1500, seed=91) + synth.tool_events(150, seed=92, size=None, full_history=True) + \
        synth.tool_events(200, seed=93, size=9000, jitter=8000)
    e = tool_engine(8)
    try:
        out, frames = tool_step(e, recs, window)
        groups = groups_of(out, FRAME_TOPICS, 8)
        assert max(len(r.value) for g in groups.values() for r in g) > 4 << 10
        check_frames(frames, groups, window, 8)
        if window == 4 << 10:
            assert len(frames) > 2 * len(groups)
    finally:
        e.close()


def test_fanout_step_frames_match_oracle():
    """fan-out steps (64 calls per record): many publishes share a record and its correlation id"""
    from calfkit import synth
    from calfkit.engine import BatchEngine
    F = 64
    recs = synth.fanout_events(60, seed=94, fanout=F) + _with_corr_ids(synth.fanout_events(6, seed=95, fanout=3), ESCAPED_CORR_IDS)
    registry = {f"tool_{j:02d}": f"tool.tool_{j:02d}.input" for j in range(64)}
    e = BatchEngine(0, max_records=128, max_in_bytes=8 << 20, max_out_bytes=256 << 20, max_payloads=128 * (F + 1))
    try:
        topics = list(registry.values()) + ["planner.input", "planner.output"]
        e.register_topics(topics, num_partitions=16)
        e.set_agent_node("planner", "planner.input", "planner.output", registry)
        e.set_frame_topics(topics)
        b = synth.pack(recs)
        e.submit(b.data, b.offsets)
        e.fanout_plan(1767225600000, 77, max_fanout=64)
        e.encode_frames(TS)
        out = e.fetch()
        frames = e.fetch_frames()
        groups = groups_of(out, topics, 16)
        assert sum(len(v) for v in groups.values()) == sum(1 for _ in out.publishes()) > 60 * F
        check_frames(frames, groups, 1 << 20, 16)
    finally:
        e.close()


def test_escaped_correlation_ids_are_unescaped_in_key_and_header():
    """ids with \\", \\\\, é and an emoji: key and header carry the unescaped UTF-8, the partition is murmur2(key) % P"""
    from calfkit import synth
    from oracle import kafka_batch as kb
    ids = ESCAPED_CORR_IDS + ['say "hi"', "C:\\dir\\file", "café", "smile 😀", '😀"\\é'] + corr_ids_of_every_length()
    recs = _with_corr_ids(synth.tool_events(len(ids), seed=96), ids)
    e = tool_engine(1000)
    try:
        out, frames = tool_step(e, recs)
        groups = groups_of(out, FRAME_TOPICS, 1000)
        check_frames(frames, groups, 1 << 20, 1000)
        keys = set()
        for t, p, f, _n in frames:
            for r in kb.decode_batches(f.tobytes()):
                corr = dict(r.headers)["correlation_id"]
                assert corr.decode() in ids
                if r.key is not None:
                    assert r.key == corr and p == (_murmur2(r.key) & 0x7FFFFFFF) % 1000
                    keys.add(r.key.decode())
        assert keys == set(ids)
    finally:
        e.close()


def test_record_form_matches_oracle():
    """records a host path produced (with and without keys / ids) framed by the same kernels: partition = the plan's
    murmur2 rule, frames equal to the oracle's"""
    from oracle import kafka_batch as kb
    rng = np.random.default_rng(97)
    ids = ESCAPED_CORR_IDS + ["plain-id", "😀", "é\\\"", ""] + [f"{rng.integers(1 << 62):x}" for _ in range(300)]
    records = []
    for i, cid in enumerate(ids):
        value = json.dumps({"n": i, "pad": "x" * int(rng.integers(0, 3000)), "id": cid}, ensure_ascii=False).encode()
        kind = i % 4
        records.append((value, cid.encode() if kind != 0 else None, cid if kind != 1 else None))
    nparts = 64
    e = tool_engine(nparts)
    try:
        for window in (1 << 20, 8 << 10):
            e.set_frame_bytes(window)
            e.encode_frames_records("weather_agent.input", records, TS)
            frames = e.fetch_frames()
            groups = {}
            for value, key, cid in records:
                part = (_murmur2(key) & 0x7FFFFFFF) % nparts if key is not None else -1
                hdrs = [("content-type", b"application/json")] + ([("correlation_id", cid.encode())] if cid is not None else [])
                groups.setdefault(("weather_agent.input", part), []).append(kb.KRecord(value, key, hdrs))
            groups = {g: groups[g] for g in sorted(groups, key=lambda g: g[1])}
            check_frames(frames, groups, window, nparts)
    finally:
        e.close()


def test_encode_recordbatch_is_the_one_group_case():
    """ck_encode_recordbatch on the inputs of test_produce_frames_match_oracle, plus groups with escaped ids: one frame
    equal to the oracle's, built by the frame pass"""
    from calfkit import synth
    from oracle import kafka_batch as kb
    recs = synth.tool_events(4000, seed=71) + synth.tool_events(300, seed=72, size=None, full_history=True) + \
        _with_corr_ids(synth.tool_events(len(ESCAPED_CORR_IDS) * 20, seed=73), ESCAPED_CORR_IDS * 20)
    e = tool_engine(8, max_records=1 << 15)
    try:
        b = synth.pack(recs)
        e.submit(b.data, b.offsets)
        e.tool_plan()
        out = e.fetch()
        tid = e.topic_ids["weather_agent.input"]
        groups = groups_of(out, ["weather_agent.input", "tool.get_weather.output"], 8)
        live = np.nonzero(out.pubs["payload"] != 0xFFFFFFFF)[0]
        for part in (0, 3, 7):
            idx = live[(out.pubs["topic_id"][live] == tid) & (out.pubs["partition"][live] == part)]
            assert len(idx) > 100
            frame = e.encode_recordbatch(idx, base_offset=5000 + part, timestamp_ms=TS).tobytes()
            want = kb.encode_batch(groups[("weather_agent.input", part)], base_offset=5000 + part, base_timestamp=TS)
            assert frame == want
        esc = [j for j in live if out.pubs["topic_id"][j] == e.topic_ids["tool.get_weather.output"]][-len(ESCAPED_CORR_IDS) * 20:]
        frame = e.encode_recordbatch(np.asarray(esc), base_offset=9, timestamp_ms=1).tobytes()
        want = kb.encode_batch(groups[("tool.get_weather.output", -1)][-len(esc):], base_offset=9, base_timestamp=1)
        assert frame == want
        assert {dict(r.headers)["correlation_id"].decode() for r in kb.decode_batches(frame)} == set(ESCAPED_CORR_IDS)
    finally:
        e.close()


def _worker_run(buf, frame_mode):
    """one Worker over the fetch response `buf`: frame sinks (frame_mode) or the per-batch sinks on both output topics;
    returns the (topic, key, value) produced and the worker's stats"""
    import asyncio
    import tools_def
    from calfkit import Client, Worker, agent_tool
    from calfkit.engine.lane import FetchArena, PinnedPool
    from oracle import kafka_batch as kb
    node_def = agent_tool(tools_def.get_weather, device_template="It's sunny in {location}")
    client = Client.connect("localhost")
    pool = PinnedPool()
    client.broker.produce_fetch("tool.get_weather.input", FetchArena.of(buf, pool))
    got, parts = [], []
    for t in ("weather_agent.input", "tool.get_weather.output"):
        if frame_mode:
            def on_frame(topic, part, frame, n):
                recs = kb.decode_batches(frame.tobytes())
                assert len(recs) == n
                got.extend((topic, r.key, r.value) for r in recs)
                parts.extend((part, r.key) for r in recs)
            client.broker.frame_sink(t, on_frame)
        else:
            client.broker.sink(t, lambda b, idx, t=t: got.extend((t, k, p) for (_t, k, p, _j) in b.iter_records(idx)))
    worker = Worker(client, nodes=[node_def], batch_records=256, batch_bytes=8 << 20, lanes=3, route_topics=["weather_agent.input"])
    asyncio.run(worker.run(until_idle=True))
    for t in ("weather_agent.input", "tool.get_weather.output"):      # per-record host fallbacks (sink path: queued)
        got += [(t, r.key, r.value) for r in client.broker.poll_batch((t,), 1000)]
    stats = dict(worker.stats)
    worker.close()
    pool.close()
    return got, parts, stats


def test_worker_fetch_responses_to_frame_sinks():
    """fetch responses (one frame with a flipped bit, a truncated trailing frame) through Worker.run: what the frame sinks
    receive, decoded, equals what the same Worker produces through the per-batch sink path; the corrupt frame's records
    are rejected and produce nothing; template-declined records reach the frame sinks through the record form"""
    import tools_def
    from calfkit import synth
    from oracle import port
    from test_gpu_kafka import frames_of
    recs = synth.tool_events(1200, seed=101) + synth.tool_events(100, seed=102, size=None, full_history=True)
    recs[7] = recs[7].replace(b'"args":{"location":"', b'"args":"{\\"location\\":\\"').replace(b'"},"tool_call_id"', b'\\"}","tool_call_id"', 1)
    recs[11] = recs[11][:recs[11].index(b'"args":{"location":')] + b'"args":{"location":42}' + recs[11][recs[11].index(b',"tool_call_id"'):]
    sizes = [40] * 30 + [100]
    assert sum(sizes) == len(recs)
    buf, _krecs = frames_of(recs, sizes, corrupt=5, truncate_tail=True)
    lo, hi = 200, 240                                           # the records of the corrupted frame
    framed, parts, st = _worker_run(buf, True)
    sunk, _p, st2 = _worker_run(buf, False)
    assert sorted(framed) == sorted(sunk)
    node = port.ToolNode.of(tools_def.get_weather)
    want = sorted((t, k, pl) for i, r in enumerate(recs) if not lo <= i < hi for (t, k, _c, pl) in port.tool_node_event(node, r))
    assert sorted(framed) == want
    for i in (7, 11):                                           # declined on the device, framed from the host tool's records
        for (t, k, _c, pl) in port.tool_node_event(node, recs[i]):
            assert (t, k, pl) in framed
    for part, key in parts:
        assert (part is None) == (key is None) and (key is None or part == (_murmur2(key) & 0x7FFFFFFF) % 8)
    assert st["records"] == len(recs) and st["rejected"] == (hi - lo) + 2 and st["host_fallback"] == 2
    assert st["rejected"] == st2["rejected"]


def test_frame_sinks_refuse_more_than_one_rank():
    import asyncio
    import tools_def
    from calfkit import Client, Worker, agent_tool
    from calfkit.exceptions import EngineError
    client = Client.connect("localhost")
    client.broker.frame_sink("weather_agent.input", lambda *a: None)
    worker = Worker(client, nodes=[agent_tool(tools_def.get_weather, device_template="It's sunny in {location}")], rank=0, world=2)
    with pytest.raises(EngineError, match="world"):
        asyncio.run(worker.run(until_idle=True))
    worker.close()
