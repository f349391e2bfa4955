"""Idempotent and transactional frames built on the device (ck_set_producer, ck_set_sticky_partitions): every frame of a
tool step, the record form and ck_encode_recordbatch, uncompressed and LZ4, carries the producer's id and epoch (and
attributes bit 4 when transactional), groups the unkeyed publishes with their topic's sticky partition, and once the host
wrote its baseSequence equals the oracle's frame byte for byte; the grow path writes the same headers; with the options
off the frames are today's.  Through Worker.run, sequences are contiguous per partition in sink order; and a
transactional Worker's sink log, one tick of it aborted, read back at read_committed delivers exactly the committed
records."""
import asyncio
import json
import struct

import numpy as np
import pytest

import kafka_lz4 as lz
import kafka_txn as kt
from oracle import kafka_batch as kb
from test_gpu_kafka_frames import FRAME_TOPICS, TS, check_frames, groups_of, split_rule, tool_engine, tool_step
from test_gpu_parity import _murmur2

pytestmark = pytest.mark.gpu

PID, EPOCH = 4242, 7


@pytest.fixture(autouse=True)
def _cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def tool_recs():
    from calfkit import synth
    return synth.tool_events(1500, seed=191) + synth.tool_events(150, seed=192, size=None, full_history=True) + \
        synth.tool_events(200, seed=193, size=9000, jitter=8000)


def sticky_groups(out, sticky):
    """the frame topics' publishes grouped as the device groups them with sticky partitions: unkeyed publishes join
    their topic's sticky partition, send order kept inside a group"""
    from calfkit.engine._lib import COL
    groups = {}
    for p in out.live():
        topic = out.topic_of(p)
        if topic not in FRAME_TOPICS:
            continue
        r = int(p["record"])
        o = int(out.cols[COL["CORR_OFF"], r])
        corr = json.loads(b'"' + out.record_bytes(r)[o:o + int(out.cols[COL["CORR_LEN"], r])].tobytes() + b'"')
        part = int(p["partition"]) if p["has_key"] else sticky[topic]
        groups.setdefault((topic, part), []).append(kb.calfkit_record(out.payload(int(p["payload"])), corr, keyed=bool(p["has_key"])))
    return {g: groups[g] for g in sorted(groups, key=lambda g: (FRAME_TOPICS.index(g[0]), g[1]))}


def oracle_frames(groups, window, transactional):
    """[(topic, partition, frame, records)] with the producer fields, baseSequence counted per partition from 0"""
    out = []
    for (topic, part), krecs in groups.items():
        starts, seq = split_rule(krecs, window) + [len(krecs)], 0
        for a, b in zip(starts, starts[1:]):
            f = kb.encode_batch(krecs[a:b], base_offset=0, base_timestamp=TS, producer_id=PID, producer_epoch=EPOCH, base_sequence=seq)
            out.append((topic, part, kt.with_attrs(f, kt.TRANSACTIONAL) if transactional else f, b - a))
            seq += b - a
    return out


def handed(frames, lz4, transactional):
    """the device frames as the broker hands them out: headers checked, baseSequence written per partition, LZ4 frames
    decompressed; [(topic, partition, frame bytes, records)]"""
    from calfkit.engine.batch import patch_base_sequence
    seq, out = {}, []
    for t, p, f, n in frames:
        f = f.copy()
        assert p is not None
        assert kb.crc32c(f[kb.CRC_FROM:].tobytes()) == struct.unpack_from(">I", f, 17)[0]
        assert struct.unpack_from(">qhi", f, 43) == (PID, EPOCH, -1)
        assert struct.unpack_from(">h", f, 21)[0] == (3 if lz4 else 0) | (kt.TRANSACTIONAL if transactional else 0)
        patch_base_sequence(f, seq.get((t, p), 0))
        seq[(t, p)] = seq.get((t, p), 0) + n
        b = f.tobytes()
        out.append((t, p, lz.decompress_batch(b) if lz4 else b, n))
    return out


@pytest.mark.parametrize("nparts,window,codec", [(8, 4 << 10, None), (8, 1 << 20, None), (1000, 4 << 10, None), (1000, 1 << 20, None),
                                                 (8, 4 << 10, "lz4"), (8, 1 << 20, "lz4"), (1000, 4 << 10, "lz4"), (1000, 1 << 20, "lz4")])
def test_tool_step_frames_carry_the_producer(nparts, window, codec):
    """a config-2-shaped tool step: today's frames with the options off; with them on, every frame equals the oracle's
    frame of the sticky grouping with the producer fields; off again, today's frames byte for byte"""
    transactional = window == 4 << 10
    recs = tool_recs()
    e = tool_engine(nparts)
    try:
        e.set_frame_compression(codec)
        out, plain = tool_step(e, recs, window)
        plain = (plain.table.copy(), plain.data.tobytes())
        if codec is None:
            check_frames([(t, p, f, n) for t, p, f, n in _frames_of(plain, e)], groups_of(out, FRAME_TOPICS, nparts), window, nparts)
        sticky = {"weather_agent.input": 3 % nparts, "tool.get_weather.output": 5 % nparts}
        e.set_producer(PID, EPOCH, transactional)
        e.set_sticky_partitions(sticky)
        out, frames = tool_step(e, recs, window)
        groups = sticky_groups(out, sticky)
        assert ("tool.get_weather.output", sticky["tool.get_weather.output"]) in groups
        assert (frames.table["partition"] >= 0).all()
        got = handed(frames, codec == "lz4", transactional)
        want = oracle_frames(groups, window, transactional)
        assert [(t, p, n) for t, p, _f, n in got] == [(t, p, n) for t, p, _f, n in want]
        assert [f for _t, _p, f, _n in got] == [f for _t, _p, f, _n in want]
        e.set_producer(-1, -1)
        e.set_sticky_partitions(None)
        _out, back = tool_step(e, recs, window)
        assert back.data.tobytes() == plain[1] and (back.table == plain[0]).all()
    finally:
        e.close()


def _frames_of(snap, e):
    table, data = snap
    d = np.frombuffer(data, dtype=np.uint8)
    for r in table:
        p = int(r["partition"])
        yield e.topic_names[int(r["topic_id"])], (p if p >= 0 else None), d[int(r["offset"]):int(r["offset"]) + int(r["length"])], int(r["n_records"])


@pytest.mark.parametrize("codec", [None, "lz4"])
def test_record_form_and_encode_recordbatch(codec):
    """the record form with a sticky partition and the one-group ck_encode_recordbatch, both with the producer fields"""
    from calfkit import synth
    rng = np.random.default_rng(197)
    records = []
    for i in range(400):
        cid = f"{rng.integers(1 << 62):x}"
        value = json.dumps({"n": i, "pad": "x" * int(rng.integers(0, 3000))}).encode()
        records.append((value, cid.encode() if i % 3 else None, cid))
    nparts = 16
    e = tool_engine(nparts)
    try:
        e.set_frame_compression(codec)
        e.set_frame_bytes(8 << 10)
        e.set_producer(PID, EPOCH, True)
        e.set_sticky_partitions({"weather_agent.input": 11})
        e.encode_frames_records("weather_agent.input", records, TS)
        frames = e.fetch_frames()
        groups = {}
        for value, key, cid in records:
            part = (_murmur2(key) & 0x7FFFFFFF) % nparts if key is not None else 11
            hdrs = [("content-type", b"application/json"), ("correlation_id", cid.encode())]
            groups.setdefault(("weather_agent.input", part), []).append(kb.KRecord(value, key, hdrs))
        groups = {g: groups[g] for g in sorted(groups, key=lambda g: g[1])}
        assert [f for _t, _p, f, _n in handed(frames, codec == "lz4", True)] == [f for _t, _p, f, _n in oracle_frames(groups, 8 << 10, True)]
        # ck_encode_recordbatch: one group of the plan's publishes, producer fields, baseSequence -1
        e.set_frame_compression(None)
        e.set_producer(PID, EPOCH, False)
        recs = synth.tool_events(500, seed=198)
        b = synth.pack(recs)
        e.submit(b.data, b.offsets)
        e.tool_plan()
        out = e.fetch()
        tid = e.topic_ids["weather_agent.input"]
        live = np.nonzero(out.pubs["payload"] != 0xFFFFFFFF)[0]
        idx = live[(out.pubs["topic_id"][live] == tid) & (out.pubs["partition"][live] == 2)]
        frame = e.encode_recordbatch(idx, base_offset=77, timestamp_ms=TS).tobytes()
        want = groups_of(out, ["weather_agent.input"], nparts)[("weather_agent.input", 2)]
        assert frame == kb.encode_batch(want, base_offset=77, base_timestamp=TS, producer_id=PID, producer_epoch=EPOCH, base_sequence=-1)
    finally:
        e.close()


def test_grow_path_writes_the_same_headers():
    """frames larger than the first frame buffer are written again into a grown one: the producer fields and the sticky
    grouping of the pass, not anything set after it"""
    from calfkit.engine import BatchEngine
    rng = np.random.default_rng(199)
    e = BatchEngine(0, max_records=64, max_in_bytes=24 << 20, max_out_bytes=1 << 20)
    try:
        e.register_topics(["weather_agent.input"], num_partitions=8)
        cap = 2 * e.max_out + 160 * 2 * e.max_payloads + 4096
        values = [rng.integers(0, 256, 150_000, dtype=np.uint8).tobytes() for _ in range(40)]
        assert sum(map(len, values)) > 2 * cap
        records = [(v, f"k{i}".encode() if i % 2 else None, None) for i, v in enumerate(values)]
        for codec in (None, "lz4"):
            e.set_frame_compression(codec)
            e.set_producer(PID, EPOCH, True)
            e.set_sticky_partitions({"weather_agent.input": 6})
            e.encode_frames_records("weather_agent.input", records, TS)
            e.set_producer(1, 1, False)                  # after the pass: the rewrite does not take it
            e.set_sticky_partitions({"weather_agent.input": 0})
            frames = e.fetch_frames()
            groups = {}
            for value, key, _c in records:
                part = (_murmur2(key) & 0x7FFFFFFF) % 8 if key is not None else 6
                groups.setdefault(("weather_agent.input", part), []).append(kb.KRecord(value, key, [("content-type", b"application/json")]))
            groups = {g: groups[g] for g in sorted(groups, key=lambda g: g[1])}
            got = handed(frames, codec == "lz4", True)
            assert [f for _t, _p, f, _n in got] == [f for _t, _p, f, _n in oracle_frames(groups, 1 << 20, True)]
    finally:
        e.close()


def _tool_worker(client, **kw):
    import tools_def
    from calfkit import Worker, agent_tool
    node_def = agent_tool(tools_def.get_weather, device_template="It's sunny in {location}")
    return Worker(client, nodes=[node_def], batch_records=kw.pop("batch_records", 128), batch_bytes=8 << 20,
                  lanes=kw.pop("lanes", 2), route_topics=["weather_agent.input"], **kw)


def _inputs(seed, n):
    from calfkit import synth
    from calfkit.broker import Record
    recs = synth.tool_events(n, seed=seed)
    recs[7] = recs[7].replace(b'"args":{"location":"', b'"args":"{\\"location\\":\\"').replace(b'"},"tool_call_id"', b'\\"}","tool_call_id"', 1)
    return recs, [Record("tool.get_weather.input", r) for r in recs]


def test_worker_sequences_are_contiguous_in_sink_order():
    """Worker.run over many ticks with two lanes and a declined record (framed by the record form): per (topic,
    partition) the baseSequences are contiguous in the order the frames reach the sinks, every frame carries the
    producer, and the records are those of a Worker without idempotence"""
    from calfkit import Client

    def run(**broker_kw):
        client = Client.connect("localhost", **broker_kw)
        recs, inputs = _inputs(201, 1500)
        client.broker.produce_batch(inputs)
        log = []
        for t in FRAME_TOPICS:
            client.broker.frame_sink(t, lambda topic, part, f, n: log.append((topic, part, f.tobytes(), n)))
        w = _tool_worker(client)
        asyncio.run(w.run(until_idle=True))
        stats = dict(w.stats)
        w.close()
        return log, stats, client.broker
    log, stats, broker = run(enable_idempotence=True)
    plain, stats0, _b = run()
    assert stats["host_fallback"] == 1 and stats["steps"] > 10
    nxt, pids = {}, set()
    for t, p, f, n in log:
        assert isinstance(p, int) and kb.crc32c(f[kb.CRC_FROM:]) == struct.unpack_from(">I", f, 17)[0]
        pid, epoch, seq = struct.unpack_from(">qhi", f, 43)
        pids.add((pid, epoch))
        assert seq == nxt.get((t, p), 0), (t, p)
        nxt[(t, p)] = seq + n
        assert not f[22] & kt.TRANSACTIONAL
    assert len(pids) == 1 and next(iter(pids))[0] >= 0
    assert sum(nxt.values()) == sum(n for _t, _p, _f, n in plain)
    recs_of = lambda lg: sorted((t, r.key, r.value) for t, _p, f, _n in lg for r in kb.decode_batches(f))  # noqa: E731
    assert recs_of(log) == recs_of(plain)
    for t, p, f, _n in log:
        for r in kb.decode_batches(f):
            if r.key is not None:
                assert p == (_murmur2(r.key) & 0x7FFFFFFF) % broker.num_partitions
    assert stats["records"] == stats0["records"]


def _partition_logs(log):
    """the sink log as per-partition record sets (offsets assigned as the broker appends) plus, per partition, its
    AbortedTransactions from the markers, and per data frame whether its transaction committed"""
    parts = {}
    for t, p, f, n in log:
        parts.setdefault((t, p), []).append((f, n))
    out = {}
    for key, frames in parts.items():
        off, buf, aborted, open_first, committed = 0, b"", [], None, []
        pending = []
        for f, n in frames:
            pid = struct.unpack_from(">q", f, 43)[0]
            if f[22] & kt.CONTROL:
                ctype = kt.control_type(f)
                if ctype == kt.ABORT:
                    aborted.append((pid, open_first))
                committed += [(g, ctype == kt.COMMIT) for g in pending]
                pending, open_first = [], None
            else:
                open_first = off if open_first is None else open_first
                pending.append(f)
            buf += struct.pack(">q", off) + f[8:]
            off += n
        assert not pending                                  # every transaction ended
        out[key] = (buf, aborted, committed)
    return out


def test_exactly_once_loop():
    """a transactional Worker whose third tick raises: its sink log (tool outputs built by the lanes, and tool inputs the
    record form framed from published Records) carries COMMIT and ABORT markers; read back through produce_fetch with the
    AbortedTransactions the markers give, a read_committed Lane delivers exactly the committed records, and a second
    Worker at read_committed consumes exactly the committed tool inputs: it publishes the oracle's outputs of those"""
    import tools_def
    from calfkit import Client
    from calfkit.broker import Record
    from calfkit.engine.lane import FetchArena, Lane, PinnedPool
    from oracle import port
    from test_gpu_kafka_lz4_fetch import configure
    client = Client.connect("localhost", transactional_id="loop")
    broker = client.broker
    _recs, inputs = _inputs(211, 1200)
    broker.produce_batch(inputs)
    b_recs, _b = _inputs(212, 600)
    log = []
    for t in FRAME_TOPICS + ["b.input"]:
        broker.frame_sink(t, lambda topic, part, f, n: log.append((topic, part, f.tobytes(), n)))
    w = _tool_worker(client)
    real_step, ticks = w.step, {"n": 0}

    def step():
        k = ticks["n"]
        ticks["n"] += 1
        more = b_recs[40 * k:40 * (k + 1)]                          # tool inputs for the second Worker, framed this tick
        for j, r in enumerate(more):
            cid = json.loads(r)["context"]["deps"]["correlation_id"]
            broker.produce(Record("b.input", r, cid.encode() if j % 3 else None, cid))
        n = real_step()
        if k == 2:
            raise RuntimeError("tick failed")
        return n + len(more)
    w.step = step
    with pytest.raises(RuntimeError, match="tick failed"):
        asyncio.run(w.run(until_idle=True))
    asyncio.run(w.run(until_idle=True))
    w.close()
    assert ticks["n"] * 40 >= len(b_recs)
    plogs = _partition_logs(log)
    assert any(ab for _b, ab, _c in plogs.values()) and any(c for _b, _a, cs in plogs.values() for _f, c in cs)
    assert all(struct.unpack_from(">q", f, 43)[0] >= 0 and f[22] & kt.TRANSACTIONAL for _t, _p, f, _n in log)

    # the lanes' frames: a read_committed Lane delivers exactly the committed records, partition by partition
    pool = PinnedPool()
    lane = Lane(0, lambda e: (configure(e), e.set_isolation_level("read_committed")), pool, max_records=1 << 14, max_in_bytes=64 << 20)
    try:
        for (t, _p), (buf, aborted, committed) in plogs.items():
            if t == "b.input":
                continue
            markers = sum(1 for s, _e in kt.batches(buf) if buf[s + 22] & kt.CONTROL)
            assert kt.verdicts(buf, [(0, aborted)], True).count(kt.SKIP) == sum(1 for _f, c in committed if not c) + markers
            lane.submit(FetchArena.of(buf, pool, aborted_transactions=aborted))
            batch = lane.collect()
            src = batch.source
            got = [src.record(i) for i in range(src.n) if src.bad[i] == 0]
            want = [r.value for f, c in committed if c for r in kb.decode_batches(f)]
            assert got == want and (src.bad != 1).all()
            batch.release()
    finally:
        lane.close()
        pool.close()

    # the record form's frames: tool inputs for a second Worker at read_committed
    client2 = Client.connect("localhost")
    parts, buf = [], b""
    for (t, _p), (pb, aborted, _c) in plogs.items():
        if t == "b.input":
            parts.append((len(buf), aborted))
            buf += pb
    pool2 = PinnedPool()
    client2.broker.produce_fetch("tool.get_weather.input", FetchArena.of(buf, pool2, partitions=parts))
    got = []
    for t in FRAME_TOPICS:
        client2.broker.sink(t, lambda b, idx, t=t: got.extend((t, k, p) for (_t, k, p, _j) in b.iter_records(idx)))
    w2 = _tool_worker(client2, extra_subscribe_kwargs={"isolation_level": "read_committed"})
    asyncio.run(w2.run(until_idle=True))
    for t in FRAME_TOPICS:
        got += [(t, r.key, r.value) for r in client2.broker.poll_batch((t,), 100000)]
    stats = dict(w2.stats)
    w2.close()
    pool2.close()
    kept = [r.value for (t, _p), (_b, _a, committed) in plogs.items() if t == "b.input" for f, c in committed if c
            for r in kb.decode_batches(f)]
    dropped = sum(len(kb.decode_batches(f)) for (t, _p), (_b, _a, cs) in plogs.items() if t == "b.input" for f, c in cs if not c)
    markers = sum(1 for t, _p, f, _n in log if t == "b.input" and f[22] & kt.CONTROL)
    assert 0 < len(kept) < len(b_recs) and dropped > 0 and len(kept) + dropped == len(b_recs)
    node = port.ToolNode.of(tools_def.get_weather)
    want = sorted((t, kk, pl) for r in kept for (t, kk, _c, pl) in port.tool_node_event(node, r))
    assert sorted(got) == want
    assert stats["skipped"] == dropped + markers and stats["records"] == len(b_recs) + markers
