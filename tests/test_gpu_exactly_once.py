"""Exactly-once consume-transform-produce on the device (Worker(processing_guarantee="exactly_once_v2")): a transactional
Worker with frame sinks and three pipelined lanes consumes two multi-partition fetches of tool events, uncompressed,
gzip, LZ4 or zstd; one tick in the middle raises after its frames went out.  Run to idle again, its sink log holds every
input's outputs exactly once among the committed transactions: read back at read_committed, by a Lane partition by
partition and by a second Worker, it equals the oracle's outputs of the inputs, and the consumer group's committed
offsets are each partition's end."""
import asyncio
import struct

import pytest

from calfkit.nodes import BaseNodeDef
from calfkit.nodes.base import submit_inbound
from test_gpu_fetch_subscribers import frames_of
from test_gpu_kafka_frames import FRAME_TOPICS
from test_gpu_kafka_idempotent_frames import _partition_logs, _tool_worker

pytestmark = pytest.mark.gpu

IN = "tool.get_weather.input"
PARTS = (2, 5, 7)                   # partition ids of the input topic
PER_FRAME = 25


@pytest.fixture(autouse=True)
def _cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def _input(codec, n=900):
    """the tool events dealt over PARTS, framed PER_FRAME records a frame, offsets from 1000 * partition id; returned as two
    fetches (each holds part of every partition, partition by partition) with their partition models, the events, and
    each partition's end offset"""
    from calfkit import synth
    from calfkit.broker import Record
    if codec == "zstd":
        import zstd_ref as zr
        zr.need()
    recs = synth.tool_events(n, seed=301)
    per_part, ends = {}, {}
    for j, p in enumerate(PARTS):
        mine = [Record(IN, r, None, None) for r in recs[j::len(PARTS)]]
        off, frames = 1000 * p, []
        for f in frames_of(mine, codec, PER_FRAME):
            frames.append(struct.pack(">q", off) + f[8:])             # baseOffset lies outside the CRC
            off += struct.unpack_from(">i", f, 57)[0]
        per_part[p], ends[p] = frames, off
    fetches = []
    for half in (0, 1):
        buf, parts = b"", []
        for p in PARTS:
            fr = per_part[p]
            mid = len(fr) // 2 + (p % 3)                               # uneven halves
            parts.append((len(buf), [], p))
            buf += b"".join(fr[:mid] if half == 0 else fr[mid:])
        fetches.append((buf, parts))
    return fetches, recs, ends


class Collect(BaseNodeDef):
    """a host node of a second Worker that decodes the fetches of its topics on the device and keeps each delivered
    record as (topic, value)"""
    def __init__(self, topics):
        self.node_id, self.subscribe_topics, self.publish_topic = "collect", list(topics), None
        self.got = []

    async def run(self, *a, **k):
        raise NotImplementedError

    def configure_engine(self, engine):
        pass

    def process_batch(self, engine, batch, **kw):
        inb = submit_inbound(engine, batch)
        self.got += [(batch.topic, bytes(inb.value(i))) for i in range(inb.values.n) if inb.values.bad[i] == 0]
        return []


@pytest.mark.parametrize("codec", [None, "gzip", "lz4", "zstd"])
def test_exactly_once_over_a_failed_tick(codec):
    import tools_def
    from calfkit import Client, Worker
    from calfkit.engine.lane import FetchArena, Lane, PinnedPool
    from oracle import port
    from test_gpu_kafka_lz4_fetch import configure
    fetches, recs, ends = _input(codec)
    client = Client.connect("localhost", transactional_id="eos")
    broker = client.broker
    for buf, parts in fetches:
        broker.produce_fetch(IN, buf, partitions=parts)
    log = []
    for t in FRAME_TOPICS:
        broker.frame_sink(t, lambda topic, part, f, n: log.append((topic, part, f.tobytes(), n)))
    w = _tool_worker(client, lanes=3, batch_records=80, processing_guarantee="exactly_once_v2")
    real_step, ticks = w.step, {"n": 0}

    def step():
        k = ticks["n"]
        ticks["n"] += 1
        n = real_step()
        if k == 4:
            raise RuntimeError("tick failed")
        return n
    w.step = step
    with pytest.raises(RuntimeError, match="tick failed"):
        asyncio.run(w.run(until_idle=True))
    asyncio.run(w.run(until_idle=True))
    group = w._subs[0][1].group_id
    w.close()
    assert {p: broker.committed(group, IN, p) for p in PARTS} == ends
    assert broker.pending() == 0 and not any(broker._kept.values())

    node = port.ToolNode.of(tools_def.get_weather)
    want = sorted((t, pl) for r in recs for (t, _k, _c, pl) in port.tool_node_event(node, r))
    assert {t for t, _pl in want} <= set(FRAME_TOPICS)
    plogs = _partition_logs(log)
    assert any(ab for _b, ab, _c in plogs.values())            # the failed tick's frames were written, then aborted

    # a read_committed Lane, partition by partition
    pool = PinnedPool()
    lane = Lane(0, lambda e: (configure(e), e.set_isolation_level("read_committed")), pool, max_records=1 << 14, max_in_bytes=64 << 20)
    got = []
    try:
        for (t, _p), (buf, aborted, _committed) in plogs.items():
            lane.submit(FetchArena.of(buf, pool, aborted_transactions=aborted))
            batch = lane.collect()
            src = batch.source
            assert (src.bad != 1).all()
            got += [(t, src.record(i)) for i in range(src.n) if src.bad[i] == 0]
            batch.release()
    finally:
        lane.close()
        pool.close()
    assert sorted(got) == want

    # a second Worker at read_committed, one multi-partition fetch per topic
    client2 = Client.connect("localhost")
    for t in FRAME_TOPICS:
        buf, parts = b"", []
        for (tt, p), (pb, aborted, _c) in plogs.items():
            if tt == t:
                parts.append((len(buf), aborted, p))
                buf += pb
        if buf:
            client2.broker.produce_fetch(t, buf, partitions=parts)
    collect = Collect(FRAME_TOPICS)
    w2 = Worker(client2, nodes=[collect], extra_subscribe_kwargs={"isolation_level": "read_committed"})
    asyncio.run(w2.run(until_idle=True))
    w2.close()
    assert sorted(collect.got) == want
