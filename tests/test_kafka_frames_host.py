"""Host side of Kafka framing without a GPU: fetch responses in the broker are split only at frame boundaries, and frames
(from a lane or framed from per-record produces) go to frame sinks instead of the per-record routes."""
import numpy as np
import pytest

from calfkit.broker import MemoryBroker, Record
from calfkit.engine.batch import Frames
from calfkit.engine.lane import FetchArena
from calfkit.exceptions import EngineError
from oracle import kafka_batch as kb
from test_host_batch import _batch


def _response(counts, tail=True, big=()):
    frames = [kb.encode_batch([kb.KRecord(b"v%d-%d" % (f, i) * (400 if f in big else 1)) for i in range(c)]) for f, c in enumerate(counts)]
    return frames, b"".join(frames) + (frames[0][:37] if tail else b"")


@pytest.mark.parametrize("max_records,max_bytes", [(1, None), (7, None), (10, None), (1000, 300), (12, 200), (1000, None)])
def test_poll_arena_splits_fetch_responses_at_frame_boundaries(max_records, max_bytes):
    counts = [3, 4, 1, 6, 2, 2, 5]
    frames, buf = _response(counts, big=(3,))
    b = MemoryBroker()
    b.produce_fetch("t", buf)
    assert b.pending() == sum(counts)
    got, seen = [], b""
    while (a := b.poll_arena(("t",), max_records, max_bytes)) is not None:
        assert isinstance(a, FetchArena)
        starts, cnt = a.frames()
        assert len(cnt) >= 1
        if len(cnt) > 1:                                      # more than one frame only when all of them fit
            assert cnt.sum() <= max_records and (max_bytes is None or starts[-1] <= max_bytes)
        got += [a.data[starts[k]:starts[k + 1]].tobytes() for k in range(len(cnt))]
        seen += a.data.tobytes()
        a.release()
    assert got == frames                                      # whole frames, in order, none split or lost
    assert seen == buf                                        # the truncated tail travelled with the last chunk
    assert b.pending() == 0


def test_poll_arena_drops_a_response_of_only_a_truncated_frame():
    frames, _ = _response([2])
    b = MemoryBroker()
    b.produce_fetch("t", frames[0][:30])
    assert b.poll_arena(("t",), 10) is None and b.pending() == 0


def _frames_of(groups, names):
    """stand-in for a frame pass: the oracle's frames for {(topic id, partition): [KRecord]} in one buffer + table"""
    from calfkit.engine._lib import FRAME_DTYPE
    blobs, table = [], np.zeros(len(groups), dtype=FRAME_DTYPE)
    pos = 0
    for i, ((tid, part), recs) in enumerate(groups.items()):
        f = kb.encode_batch(recs)
        table[i] = (tid, part, len(recs), 0, pos, len(f))
        blobs.append(f)
        pos += len(f)
    return Frames(table, np.frombuffer(b"".join(blobs), dtype=np.uint8), names)


def test_produce_publishes_hands_frames_to_frame_sinks():
    batch, recs, payloads, released = _batch(True)
    batch.frames = _frames_of({(1, 2): [kb.KRecord(b"x")], (1, -1): [kb.KRecord(b"y"), kb.KRecord(b"z")]}, batch.topic_names)
    batch.frame_topic_ids = frozenset({1})
    b = MemoryBroker()
    b.subscriber("alpha", "beta")
    framed, routed = [], []
    b.frame_sink("beta", lambda t, p, f, n: framed.append((t, p, [r.value for r in kb.decode_batches(f.tobytes())], n)))
    b.sink("alpha", lambda bb, idx: routed.append(list(idx)))
    b.produce_publishes(batch)
    assert framed == [("beta", 2, [b"x"], 1), ("beta", None, [b"y", b"z"], 2)]
    assert routed == [[0]]                                     # alpha: per batch, as before
    assert not b.frags.get("beta")                            # the framed topic's publishes are not routed per record
    assert released == [1]


def test_records_produced_to_a_frame_sink_are_framed_per_step():
    b = MemoryBroker()
    framed = []
    b.frame_sink("out", lambda t, p, f, n: framed.append((t, p, [(r.key, r.value) for r in kb.decode_batches(f.tobytes())])))
    b.produce(Record("out", b"v1", b"k1", "k1"))
    b.produce_batch([Record("out", b"v2", None, "k2"), Record("other", b"v3")])
    assert not b.queues.get("out") and len(b.queues["other"]) == 1     # never queued
    with pytest.raises(EngineError):
        b.flush_frames()                                      # no framer: loud, never a CPU encoder
    b.produce(Record("out", b"v1", b"k1", "k1"))
    calls = []

    def framer(topic, records):
        calls.append((topic, [(r.value, r.key, r.correlation_id) for r in records]))
        return [_frames_of({(0, 3): [kb.KRecord(r.value, r.key) for r in records]}, {0: "out"})]
    b.framer = framer
    b.flush_frames()
    assert calls == [("out", [(b"v1", b"k1", "k1")])]
    assert framed == [("out", 3, [(b"k1", b"v1")])]
    b.flush_frames()                                          # nothing pending: nothing framed
    assert len(calls) == 1
