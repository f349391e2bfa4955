"""Exactly-once consume-transform-produce without a GPU: ck_fetch_positions against a plain-Python restatement over seeded
random multi-partition logs (control batches, aborted transactions, bad CRCs, offsets that jump back, truncated tails)
and over every split of them at a frame boundary; the broker's offset commit, the drop of an aborted transaction's
offsets, and the rewind of the fetch slices no commit covers, trimmed at frame boundaries; and Worker.run with a
stand-in lane pipeline: pipelined results commit their offsets with the tick that hands them out, and a tick that
raises puts exactly the uncommitted slices back."""
import asyncio
import random
import re
import struct

import numpy as np
import pytest

import kafka_txn as kt
from oracle import kafka_batch as kb


def positions_restated(buf: bytes, parts) -> tuple[dict[int, int], list[int]]:
    """per partition id the offset after its last complete batch, and the offset after each complete batch: every batch
    counts, whatever it holds and whether or not its CRC matches"""
    starts = [p[0] for p in parts]
    out, per = {}, []
    for s, _e in kt.batches(buf):
        run = max((r for r, st in enumerate(starts) if st <= s), default=-1)
        nxt = struct.unpack_from(">q", buf, s)[0] + struct.unpack_from(">i", buf, s + 23)[0] + 1
        per.append(nxt)
        if run >= 0:
            out[parts[run][2] if len(parts[run]) > 2 else run] = nxt
    return out, per


def with_ids(parts, rng):
    ids = rng.sample(range(64), len(parts))
    return [(s, ab, i) for (s, ab), i in zip(parts, ids)]


def test_positions_match_the_restatement_over_random_logs():
    from calfkit.engine.batch import fetch_positions, txn_partitions
    kinds = {"control": 0, "bad": 0, "multi": 0}
    for seed in range(300):
        buf, parts = kt.random_log(seed)
        parts = with_ids(parts, random.Random(seed)) if seed % 2 else parts
        want, per = positions_restated(buf, parts)
        got, got_per = fetch_positions(np.frombuffer(buf, dtype=np.uint8), txn_partitions(partitions=parts))
        assert got == want and list(got_per) == per, seed
        kinds["multi"] += len(parts) > 1
        for s, e in kt.batches(buf):
            kinds["control"] += bool(buf[s + 22] & kt.CONTROL)
            kinds["bad"] += not kt._framed(buf[s:e])
    assert all(kinds.values()), kinds


def test_positions_of_every_split_at_a_frame_boundary():
    """every slice [a, b) of a fetch cut at frame boundaries: its positions are those of its own batches, each partition's
    last one"""
    from calfkit.engine.lane import FetchArena
    for seed in range(0, 300, 23):
        buf, parts = kt.random_log(seed)
        parts = with_ids(parts, random.Random(seed))
        fa = FetchArena.of(buf, partitions=parts)
        per = positions_restated(buf, parts)[1]
        owner = [next((parts[r][2] for r in reversed(range(len(parts))) if parts[r][0] <= s), None) for s, _e in kt.batches(buf)]
        nf = len(per)
        assert fa.positions() == {p: x for p, x in zip(owner, per) if p is not None}
        for a in range(nf):
            for b in range(a + 1, nf + 1):
                sl = fa.slice_frames(a, b if b < nf else None)
                want = {p: x for p, x in zip(owner[a:b], per[a:b]) if p is not None}
                assert sl.positions() == want, (seed, a, b)


def test_one_partition_form_is_partition_zero():
    from calfkit.engine.lane import FetchArena
    buf, ab = kt.random_partition(random.Random(7), "one")
    fa = FetchArena.of(buf, aborted_transactions=ab)
    assert list(fa.positions()) == [0] and fa.positions() == positions_restated(buf, [(0, ab)])[0]
    assert FetchArena.of(buf, partitions=[(0, ab, 5)]).positions() == {5: fa.positions()[0]}
    assert FetchArena(np.frombuffer(buf, dtype=np.uint8)).positions() == {}    # no partition model: nothing to commit


def test_positions_refuse_runs_out_of_order():
    from calfkit.engine.batch import fetch_positions
    buf, _ab = kt.random_partition(random.Random(8), "x")
    with pytest.raises(Exception, match="out of order"):
        fetch_positions(np.frombuffer(buf, dtype=np.uint8), [(100, [], 0), (0, [], 1)])


# ---- broker ------------------------------------------------------------------------------------------------------------
def rec(tag):
    return kb.calfkit_record(b'{"v":"%s"}' % tag.encode(), tag)


def log_of(partitions: dict[int, list[int]], base: int = 10):
    """a fetch of plain batches: per partition id, batches of the given record counts from offset `base`"""
    buf, parts = b"", []
    for pid, counts in partitions.items():
        parts.append((len(buf), [], pid))
        off = base
        for j, n in enumerate(counts):
            buf += kb.encode_batch([rec(f"p{pid}-{off + i}") for i in range(n)], base_offset=off)
            off += n
    return buf, parts


def frame_bytes(fa):
    starts = fa.frames()[0]
    return [fa.data[int(starts[i]):int(starts[i + 1])].tobytes() for i in range(len(starts) - 1)]


def test_offsets_commit_with_the_transaction_and_drop_with_an_abort():
    from calfkit.broker import MemoryBroker
    b = MemoryBroker(transactional_id="t")
    with pytest.raises(Exception, match="outside a transaction"):
        b.send_offsets_to_transaction({("in", 0): 5}, "g")
    assert b.committed("g", "in", 0) is None
    b.begin_transaction()
    b.send_offsets_to_transaction({("in", 0): 5, ("in", 3): 9}, "g")
    assert b.committed("g", "in", 0) is None                   # not before the commit
    b.commit_transaction()
    assert (b.committed("g", "in", 0), b.committed("g", "in", 3), b.committed("h", "in", 0)) == (5, 9, None)
    b.begin_transaction()
    b.send_offsets_to_transaction({("in", 0): 7}, "g")
    b.abort_transaction()
    assert b.committed("g", "in", 0) == 5
    b.begin_transaction()
    b.send_offsets_to_transaction({("in", 0): 8}, "g")
    b.send_offsets_to_transaction({("in", 0): 11}, "h")
    b.commit_transaction()
    assert (b.committed("g", "in", 0), b.committed("h", "in", 0)) == (8, 11)


def test_polls_without_a_group_are_unchanged_and_with_one_need_a_transaction():
    from calfkit.broker import MemoryBroker
    buf, parts = log_of({0: [2, 3, 1]})
    b = MemoryBroker(transactional_id="t")
    b.produce_fetch("in", buf, partitions=parts)
    with pytest.raises(Exception, match="outside a transaction"):
        b.poll_fetch(("in",), 2, group_id="g")
    a = b.poll_fetch(("in",), 5)
    assert a.n == 5 and a.topic == "in" and not b._kept
    b.begin_transaction()
    c = b.poll_arena(("in",), 5, group_id="g")
    assert c.n == 1 and b._kept["in"][0][1] is c
    b.commit_transaction()                                      # no offsets sent: the slice stays kept
    assert len(b._kept["in"]) == 1


def test_polls_for_a_group_refuse_input_without_offsets():
    from calfkit.broker import MemoryBroker, Record
    from calfkit.engine.lane import Arena
    b = MemoryBroker(transactional_id="t")
    b.produce(Record("r", b"x"))
    b.produce_arena("a", Arena.pack([b"y", b"z"]))
    b.begin_transaction()
    for poll in (b.poll_arena, b.poll_fetch, b.poll_batch):
        for t in ("r", "a"):
            if poll == b.poll_fetch:
                assert poll((t,), 10, group_id="g") is None
                continue
            with pytest.raises(Exception, match="without offsets"):
                poll((t,), 10, group_id="g")
    assert b.pending() == 3                                     # nothing was taken
    b.abort_transaction()


def test_kept_slices_are_released_when_a_commit_covers_them():
    from calfkit.broker import MemoryBroker
    from calfkit.engine.lane import FetchArena
    buf, parts = log_of({0: [2, 2], 4: [1, 3]})
    released = []
    b = MemoryBroker(transactional_id="t")
    b.produce_fetch("in", FetchArena(np.frombuffer(buf, dtype=np.uint8).copy(), on_release=lambda: released.append(1),
                                     partitions=[(s, ab, p) for s, ab, p in parts]))
    b.begin_transaction()
    s1 = b.poll_fetch(("in",), 3, group_id="g")                 # partition 0's first batch
    s2 = b.poll_fetch(("in",), 100, group_id="g")               # the rest: it owns the buffer's release
    assert s1.positions() == {0: 12} and s2.positions() == {0: 14, 4: 14}
    s2.release()
    assert released == []                                       # kept: the consumer's release does not free it
    b.send_offsets_to_transaction({("in", 0): 14}, "g")
    b.commit_transaction()
    assert [f is s2 for _g, f, _r in b._kept["in"]] == [True] and released == []
    b.begin_transaction()
    b.send_offsets_to_transaction({("in", 4): 14}, "g")
    b.commit_transaction()
    assert not b._kept["in"] and released == [1]


def test_abort_rewinds_the_uncovered_slices_in_poll_order_trimmed_at_frame_boundaries():
    from calfkit.broker import MemoryBroker
    from calfkit.engine.lane import FetchArena
    buf, parts = log_of({0: [2, 2, 1], 4: [1, 3], 6: [2]})
    fa = FetchArena.of(buf, partitions=parts)
    frames = frame_bytes(fa)                                   # p0: 0 1 2, p4: 3 4, p6: 5
    b = MemoryBroker(transactional_id="t")
    b.produce_fetch("in", buf, partitions=parts)
    b.begin_transaction()
    s1 = b.poll_fetch(("in",), 4, group_id="g")                 # frames 0, 1
    b.send_offsets_to_transaction({("in", 0): 12}, "g")         # covers frame 0 only
    b.commit_transaction()
    b.begin_transaction()
    s2 = b.poll_fetch(("in",), 4, group_id="g")                 # frames 2, 3 (p0's last, p4's first)
    s3 = b.poll_fetch(("in",), 3, group_id="g")                 # frame 4
    assert frame_bytes(s1) + frame_bytes(s2) + frame_bytes(s3) == frames[:5]
    b.send_offsets_to_transaction({("in", 0): 15, ("in", 4): 11}, "g")    # dropped by the abort
    b.abort_transaction()
    assert b.committed("g", "in", 0) == 12 and b.committed("g", "in", 4) is None
    again = []
    b.begin_transaction()
    while (a := b.poll_fetch(("in",), 100, group_id="g")) is not None:
        again += frame_bytes(a)
    assert again == frames[1:]                                  # frame 0 was committed: trimmed away
    # now commit all of p4, then abort: frames 3 and 4 are trimmed away
    b.send_offsets_to_transaction({("in", 4): 14}, "g")
    b.commit_transaction()
    b.begin_transaction()
    b.abort_transaction()
    back = []
    while (a := b.poll_fetch(("in",), 100)) is not None:
        back += frame_bytes(a)
    assert back == [frames[1], frames[2], frames[5]]
    # one slice of the whole fetch, p4 committed: what stays is cut in its middle (a copy, not a view)
    b = MemoryBroker(transactional_id="t")
    b.produce_fetch("in", buf, partitions=parts)
    b.begin_transaction()
    b.poll_fetch(("in",), 100, group_id="g")
    b.send_offsets_to_transaction({("in", 4): 14}, "g")
    b.commit_transaction()
    b.begin_transaction()
    b.abort_transaction()
    back = b.poll_fetch(("in",), 100)
    assert frame_bytes(back) == [frames[0], frames[1], frames[2], frames[5]] and back.positions() == {0: 15, 6: 12}
    assert b.poll_fetch(("in",), 100) is None


def test_rewound_slices_of_random_logs_keep_their_mask():
    """random transactional multi-partition logs polled in slices, the first partition's position committed, then an
    abort: every frame the commit does not cover comes back, in order, with its read_committed mask"""
    from calfkit.broker import MemoryBroker
    from calfkit.engine.lane import FetchArena
    for seed in (3, 17, 40, 77):
        buf, parts = kt.random_log(seed)
        parts = with_ids(parts, random.Random(seed))
        fa = FetchArena.of(buf, partitions=parts)
        frames, full = frame_bytes(fa), fa.hidden()
        mask = dict(zip(frames, full)) if full is not None else None
        b = MemoryBroker(transactional_id="t")
        b.produce_fetch("in", buf, partitions=parts)
        b.begin_transaction()
        polled = []
        while (a := b.poll_fetch(("in",), 7, group_id="g")) is not None:
            polled.append(a)
        p_first = parts[0][2]
        b.send_offsets_to_transaction({("in", p_first): fa.positions()[p_first]}, "g")
        b.commit_transaction()
        b.begin_transaction()
        b.abort_transaction()
        got, hidden = [], []
        while (a := b.poll_fetch(("in",), 5)) is not None:
            got += frame_bytes(a)
            if a.hidden() is not None:
                hidden += list(a.hidden())
        start_p1 = parts[1][0] if len(parts) > 1 else len(buf)
        per = positions_restated(buf, parts)[1]                 # offsets may jump back: a batch of p0 may stay
        want = [f for f, (s, _e), nx in zip(frames, kt.batches(buf), per) if s >= start_p1 or nx > fa.positions()[p_first]]
        assert got == want, seed
        if mask is not None and want:
            assert hidden == [mask[f] for f in want]


# ---- Worker.run with a stand-in lane pipeline -------------------------------------------------------------------------
def _stand_in(monkeypatch):
    """device-template nodes on a stand-in pipeline (K = 3: a push returns the step pushed two calls earlier) whose
    results carry each fetch slice as their source, one output per record (its value + "+out")"""
    from calfkit import Worker
    from calfkit.engine._lib import PUB_DTYPE
    from calfkit.engine.lane import PublishBatch

    class FakePipe:
        def __init__(self, node):
            self.node, self.inflight, self.pushed = node, [], 0

        def _result(self, arena):
            starts = arena.frames()[0]
            values = [r.value for i in range(len(starts) - 1) for r in kb.decode_batches(arena.data[int(starts[i]):int(starts[i + 1])].tobytes())]
            payloads = [v + b"+out" for v in values]
            n = len(payloads)
            lens = np.asarray([len(p) for p in payloads], dtype=np.uint32)
            off = np.zeros(n + 1, dtype=np.int64)
            np.cumsum((lens.astype(np.int64) + 15) & ~15, out=off[1:])
            out = np.zeros(int(off[-1]) if n else 0, dtype=np.uint8)
            for i, p in enumerate(payloads):
                out[off[i]:off[i] + len(p)] = np.frombuffer(p, dtype=np.uint8)
            pubs = np.zeros(n, dtype=PUB_DTYPE)
            pubs["payload"], pubs["record"], pubs["topic_id"], pubs["partition"] = np.arange(n), np.arange(n), 0, -1
            return PublishBatch(out, off, lens, pubs, {0: self.node.publish_topic}, arena, None, np.zeros(n, np.uint32),
                                np.zeros(n, np.uint32), on_release=arena.release)

        def push(self, arena, *a):
            self.pushed += 1
            self.inflight.append(arena)
            return self._result(self.inflight.pop(0)) if len(self.inflight) > 2 else None

        def drain(self):
            while self.inflight:
                yield self._result(self.inflight.pop(0))

        def take_received(self):
            return []

        @property
        def pending(self):
            return len(self.inflight)

        @property
        def pending_records(self):
            return sum(a.n for a in self.inflight)

        def close(self):
            pass

    pipes = {}

    def _pipeline(self, node):
        if id(node) not in self._pipes:
            self._pipes[id(node)] = pipes[node.node_id] = FakePipe(node)
        return self._pipes[id(node)]
    monkeypatch.setattr(Worker, "_pipeline", _pipeline)
    return pipes


def _node():
    from calfkit.nodes import BaseNodeDef

    class Node(BaseNodeDef):
        def __init__(self):
            self.node_id, self.subscribe_topics, self.publish_topic = "A", ["in"], "out"
            self._template = object()

        async def run(self, *a, **k):
            raise NotImplementedError
    return Node()


def _rig(monkeypatch, fail_tick=None):
    """a transactional broker with a sink on `out` whose records count only when their tick commits, a multi-partition
    fetch on `in`, and an exactly-once Worker; returns (worker, broker, committed outputs, per tick the committed offsets
    seen when it starts, the input values in offset order per partition)"""
    from calfkit import Client, Worker
    pipes = _stand_in(monkeypatch)
    client = Client.connect("localhost", transactional_id="eos")
    broker = client.broker
    buf, parts = log_of({1: [3, 2, 4, 1], 5: [2, 2, 2], 2: [5, 1]})
    broker.produce_fetch("in", buf, partitions=parts)
    tick_out, outs, seen, checks = [], [], [], []
    broker.sink("out", lambda batch, idx: tick_out.extend(batch.payload(int(j)) for j in idx))
    commit, abort = broker.commit_transaction, broker.abort_transaction

    def on_commit():
        outs.extend(tick_out)
        tick_out.clear()
        commit()
        # the committed offsets are those of exactly the committed outputs: each partition's highest + 1
        done = {}
        for o in outs:
            pid, off = (int(x) for x in re.match(rb'\{"v":"p(\d+)-(\d+)"\}', o).groups())
            done[pid] = max(done.get(pid, 0), off + 1)
        checks.append(({p: broker.committed("A", "in", p) for p in (1, 5, 2)}, {p: done.get(p) for p in (1, 5, 2)}))

    def on_abort():
        tick_out.clear()
        abort()
    broker.commit_transaction, broker.abort_transaction = on_commit, on_abort
    worker = Worker(client, nodes=[_node()], batch_records=4, batch_bytes=1 << 20, processing_guarantee="exactly_once_v2")
    real_step, ticks = worker.step, {"n": 0}

    def step():
        seen.append({p: broker.committed("A", "in", p) for p in (1, 5, 2)})
        k = ticks["n"]
        ticks["n"] += 1
        n = real_step()
        if k == fail_tick:
            raise RuntimeError("tick failed")
        return n
    worker.step = step
    values = {pid: [f"p{pid}-{10 + i}".encode() for i in range(sum(c))] for pid, c in {1: [3, 2, 4, 1], 5: [2, 2, 2], 2: [5, 1]}.items()}
    return worker, broker, outs, seen, values, pipes, checks


def test_pipelined_results_commit_with_the_tick_that_hands_them_out(monkeypatch):
    worker, broker, outs, seen, values, pipes, checks = _rig(monkeypatch)
    asyncio.run(worker.run(until_idle=True))
    assert len(checks) > 4 and all(got == want for got, want in checks)
    want = [v for pid in (1, 5, 2) for v in values[pid]]
    assert sorted(outs) == sorted(json_val(v) + b"+out" for v in want) and len(outs) == len(want)
    assert {p: broker.committed("A", "in", p) for p in (1, 5, 2)} == {1: 20, 5: 16, 2: 16}
    # the first two ticks only fill the pipe: nothing is handed out, nothing committed
    assert seen[1] == seen[2] == {1: None, 5: None, 2: None}
    assert any(o is not None for o in seen[3].values())
    assert not broker._kept["in"] and broker.pending() == 0


def json_val(tag: bytes) -> bytes:
    return b'{"v":"%s"}' % tag


def test_a_tick_that_raises_redelivers_exactly_the_uncommitted_slices(monkeypatch):
    worker, broker, outs, seen, values, pipes, checks = _rig(monkeypatch, fail_tick=4)
    with pytest.raises(RuntimeError, match="tick failed"):
        asyncio.run(worker.run(until_idle=True))
    committed = {p: broker.committed("A", "in", p) for p in (1, 5, 2)}
    assert pipes["A"].pending == 0                              # the results in flight were dropped
    # the queue's head is exactly what no commit covers: per partition, the records from its committed offset on
    again = []
    for a in list(broker.arenas["in"]):
        starts = a.frames()[0]
        again += [r.value for i in range(len(starts) - 1) for r in kb.decode_batches(a.data[int(starts[i]):int(starts[i + 1])].tobytes())]
    want_again = [json_val(v) for pid in (1, 5, 2) for i, v in enumerate(values[pid]) if committed[pid] is None or 10 + i >= committed[pid]]
    assert again == want_again
    assert len(outs) + len(again) == sum(len(v) for v in values.values())
    asyncio.run(worker.run(until_idle=True))
    assert all(got == want for got, want in checks)
    want = [json_val(v) + b"+out" for pid in (1, 5, 2) for v in values[pid]]
    assert sorted(outs) == sorted(want) and len(outs) == len(want)   # every input's output exactly once
    assert {p: broker.committed("A", "in", p) for p in (1, 5, 2)} == {1: 20, 5: 16, 2: 16}


def test_exactly_once_needs_a_transactional_broker():
    from calfkit import Client, Worker
    from calfkit.exceptions import EngineError
    with pytest.raises(EngineError, match="transactional_id"):
        Worker(Client.connect("localhost"), nodes=[], processing_guarantee="exactly_once_v2")
    with pytest.raises(EngineError, match="processing_guarantee"):
        Worker(Client.connect("localhost", transactional_id="x"), nodes=[], processing_guarantee="exactly_once")
    Worker(Client.connect("localhost", transactional_id="x"), nodes=[], processing_guarantee="exactly_once_v2")
