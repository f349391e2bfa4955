"""Fetch responses for host-path subscribers, without a GPU: `MemoryBroker.poll_fetch` splits a fetch only at frame
boundaries under the record and byte bounds (the truncated tail with the last piece, the read_committed mask sliced along);
a Worker whose host node subscribes to a topic holding a fetch hands it to the node as it is; and `_run_host` splits a
fetch that fails at frame boundaries, loses no record, and drops a frame that fails alone."""
import asyncio
import logging
import types

import numpy as np
import pytest

from calfkit import Client, Worker
from calfkit.broker import MemoryBroker, Record
from calfkit.engine.lane import FetchArena
from calfkit.nodes import BaseNodeDef
from oracle import kafka_batch as kb

COUNTS = [3, 1, 4, 2, 5]


def _fetch(counts, tail):
    frames = [kb.encode_batch([kb.KRecord(b"f%d-r%d" % (f, i) * (1 + f)) for i in range(c)]) for f, c in enumerate(counts)]
    return frames, b"".join(frames) + (frames[0][:40] if tail else b"")


def _bounds():
    frames, _ = _fetch(COUNTS, False)
    sizes = np.cumsum([len(f) for f in frames])
    byte_bounds = [None] + sorted({int(s) + d for s in sizes for d in (-1, 0, 1)})
    return [(r, b) for r in range(1, sum(COUNTS) + 1) for b in byte_bounds]


@pytest.mark.parametrize("tail", [False, True])
@pytest.mark.parametrize("masked", [False, True])
def test_poll_fetch_splits_at_frame_boundaries_under_every_bound(tail, masked):
    frames, buf = _fetch(COUNTS, tail)
    mask = np.array([0, 1, 0, 1, 1], dtype=np.uint8)
    for max_records, max_bytes in _bounds():
        b = MemoryBroker()
        b.produce_fetch("t", FetchArena(np.frombuffer(buf, dtype=np.uint8), hidden=mask.copy() if masked else None))
        b.produce(Record("other", b"x"))
        got, seen, hidden, k = [], b"", [], 0
        while (a := b.poll_fetch(("other", "t"), max_records, max_bytes)) is not None:
            starts, cnt = a.frames()
            assert len(cnt) >= 1
            if len(cnt) > 1:                                  # several frames only when they all fit
                assert cnt.sum() <= max_records and (max_bytes is None or starts[-1] <= max_bytes)
            nxt = k + len(cnt)
            if nxt < len(frames):                             # and as many as fit: the next frame would not
                more = sum(COUNTS[k:nxt + 1]), sum(len(f) for f in frames[k:nxt + 1])
                assert more[0] > max_records or (max_bytes is not None and more[1] > max_bytes)
            got += [a.data[starts[j]:starts[j + 1]].tobytes() for j in range(len(cnt))]
            seen += a.data.tobytes()
            if masked:
                assert len(a.hidden()) == len(cnt)
                hidden += list(a.hidden())
            else:
                assert a.hidden() is None
            a.release()
            k = nxt
        assert got == frames, (max_records, max_bytes)        # whole frames, in order, none split or lost
        assert seen == buf                                    # the truncated tail travelled with the last piece
        assert hidden == (list(mask) if masked else [])
        assert b.pending() == 1 and b.poll_batch(("other",), 10)[0].value == b"x"     # Records stay for poll_batch


def test_poll_fetch_leaves_record_entries_and_poll_batch_still_refuses_a_fetch():
    from calfkit.exceptions import EngineError
    _frames, buf = _fetch([2], False)
    b = MemoryBroker()
    assert b.poll_fetch(("t",), 10) is None
    b.produce(Record("t", b"r"))
    assert b.poll_fetch(("t",), 10) is None and b.pending() == 1
    b.produce_fetch("t", buf)
    with pytest.raises(EngineError):
        b.poll_batch(("t",), 10)
    a = b.poll_fetch(("t",), 10)
    assert a.n == 2 and b.poll_fetch(("t",), 10) is None
    b.produce_fetch("t", buf[:30])                            # nothing but a truncated frame: dropped, never returned
    assert b.poll_fetch(("t",), 10) is None and b.pending() == 0


class FetchNode(BaseNodeDef):
    """consumes `fake.in`, publishes every record's value upper-cased to `fake.out`.  A stand-in for a node's engine step:
    it reads a fetch's records with the Kafka oracle, refuses batches above `max_batch` records (an engine whose buffers
    are too small) and any batch holding a poisoned record"""
    def __init__(self, max_batch: int):
        self.node_id = "fake"
        self.subscribe_topics = ["fake.in"]
        self.publish_topic = "fake.out"
        self.max_batch = max_batch
        self.calls: list[tuple[str, int]] = []

    async def run(self, *a, **k):
        raise NotImplementedError

    def process_batch(self, engine, batch, **kw):
        if isinstance(batch, FetchArena):
            starts, _cnt = batch.frames()
            values = [r.value for j in range(len(starts) - 1) for r in kb.decode_batches(batch.data[starts[j]:starts[j + 1]].tobytes())]
        else:
            values = [r.value for r in batch]
        self.calls.append((type(batch).__name__, len(values)))
        if len(values) > self.max_batch:
            raise RuntimeError("batch does not fit the engine")
        if b"poison" in values:
            raise ValueError("user code raised outside the per-record guard")
        return [Record("fake.out", v.upper()) for v in values]


@pytest.fixture()
def setup(monkeypatch):
    import calfkit.worker.worker as W
    levels = []

    def stub(node, isolation_level=None, **kw):
        levels.append(isolation_level)
        return types.SimpleNamespace(skipped=0)
    monkeypatch.setattr(W, "engine_for", stub)
    client = Client.connect()
    return client, client._connection, levels


def _frames(groups):
    return [kb.encode_batch([kb.KRecord(v) for v in g]) for g in groups]


def test_a_host_node_consumes_a_fetch(setup):
    client, broker, levels = setup
    node = FetchNode(max_batch=100)
    worker = Worker(client, nodes=[node], batch_records=100, batch_bytes=1 << 20,
                    extra_subscribe_kwargs={"isolation_level": "read_committed"})
    groups = [[b"a%d" % i for i in range(5)], [b"b%d" % i for i in range(3)]]
    broker.produce_fetch("fake.in", b"".join(_frames(groups)))
    broker.produce(Record("fake.in", b"plain"))
    asyncio.run(worker.run(until_idle=True))
    assert [r.value for r in broker.queues["fake.out"]] == [v.upper() for g in groups for v in g] + [b"PLAIN"]
    assert node.calls == [("FetchArena", 8), ("list", 1)]   # the fetch as it is, then the Records
    assert worker.stats["records"] == 9
    assert set(levels) == {"read_committed"}                  # the subscription's level goes to the node's engine


def test_a_fetch_that_fails_is_split_at_frame_boundaries_and_a_failing_frame_dropped_alone(setup, caplog):
    client, broker, _levels = setup
    node = FetchNode(max_batch=6)
    worker = Worker(client, nodes=[node], batch_records=64, batch_bytes=1 << 20)
    groups = [[b"x%d-%d" % (f, i) for i in range(c)] for f, c in enumerate([4, 2, 5, 1, 3, 6, 2])]
    groups[4][1] = b"poison"
    frames = _frames(groups)
    broker.produce_fetch("fake.in", b"".join(frames) + frames[0][:25])
    with caplog.at_level(logging.WARNING):
        asyncio.run(worker.run(until_idle=True))
    want = [v.upper() for f, g in enumerate(groups) if f != 4 for v in g]
    assert [r.value for r in broker.queues["fake.out"]] == want          # every other record, once, in order
    assert node.calls[0] == ("FetchArena", 23) and node.calls.count(("FetchArena", 3)) >= 1
    dropped = [r.getMessage() for r in caplog.records if "dropped" in r.getMessage()]
    assert dropped == ["node fake: frame of 3 records dropped after failing alone"]
    assert worker.stats["records"] == sum(len(g) for f, g in enumerate(groups) if f != 4)
