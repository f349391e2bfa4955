"""Idempotent and transactional produce without a GPU: ck_crc32c_patch against a full recomputation, ck_encode_control_batch
against the plain-Python control batch writer (tests/kafka_txn.py) and the g++ build of ck_txn.h's control-batch check,
and the broker's side: producer ids and fencing, baseSequence hand-off per partition (its 2^31 - 1 wrap included),
COMMIT / ABORT markers for exactly the partitions a transaction touched, the abort of a tick that raises, the sticky round
robin, and a broker with neither keyword handing frames out untouched."""
import asyncio
import ctypes as C
import random
import struct

import numpy as np
import pytest

import kafka_txn as kt
import txnmask
from oracle import kafka_batch as kb


def _lib():
    from calfkit.engine import _lib
    return _lib.load()


def crc_patch(crc, length, pos, old4, new4):
    c = C.c_uint32(crc)
    a, b = np.frombuffer(old4, dtype=np.uint8).copy(), np.frombuffer(new4, dtype=np.uint8).copy()
    assert _lib().ck_crc32c_patch(C.byref(c), length, pos, a.ctypes.data, b.ctypes.data) == 0
    return c.value


@pytest.mark.parametrize("length", [61, 62, 64, 100, 4096, 65_537, 1 << 20, 64 << 20])
def test_crc32c_patch_equals_full_recomputation(length):
    rng = np.random.default_rng(length)
    data = rng.integers(0, 256, length, dtype=np.uint8)
    crc = txnmask.crc32c(data.tobytes())
    positions = {0, length - 4, 32 if length >= 36 else 0} | {int(p) for p in rng.integers(0, length - 3, 6)}
    for pos in sorted(positions):
        new = rng.integers(0, 256, 4, dtype=np.uint8)
        old = data[pos:pos + 4].copy()
        got = crc_patch(crc, length, pos, old.tobytes(), new.tobytes())
        data[pos:pos + 4] = new
        assert got == txnmask.crc32c(data.tobytes()), (length, pos)
        crc = got


def test_crc32c_patch_refuses_bytes_outside_the_span():
    c = C.c_uint32(0)
    four = (C.c_uint8 * 4)()
    assert _lib().ck_crc32c_patch(C.byref(c), 10, 7, four, four) != 0
    assert _lib().ck_crc32c_patch(C.byref(c), 3, 0, four, four) != 0


def test_patch_base_sequence_gives_the_frame_the_oracle_writes():
    from calfkit.engine.batch import patch_base_sequence
    rng = random.Random(5)
    for n in (1, 3, 40):
        recs = [kb.calfkit_record(b'{"v":%d}' % i + b"x" * rng.randrange(0, 3000), f"id-{i}") for i in range(n)]
        frame = np.frombuffer(kb.encode_batch(recs, producer_id=77, producer_epoch=3, base_sequence=-1), dtype=np.uint8).copy()
        for seq in (0, 5, 0x7FFFFFFF, 12345678):
            patch_base_sequence(frame, seq)
            assert frame.tobytes() == kb.encode_batch(recs, producer_id=77, producer_epoch=3, base_sequence=seq)


@pytest.mark.parametrize("ctype", [kt.ABORT, kt.COMMIT])
def test_control_batch_equals_the_writer_and_passes_the_check(ctype):
    from calfkit.engine.batch import control_batch
    for pid, epoch, off in ((0, 0, 0), (7, 1, 123), ((1 << 62) + 5, 0x7FFF, (1 << 40) + 3)):
        got = control_batch(pid, epoch, ctype == kt.COMMIT, 1767225600000, base_offset=off).tobytes()
        assert got == kt.control_batch(off, pid, ctype, producer_epoch=epoch)
        assert kt.control_type(got) == ctype
        assert txnmask.verdicts(got, [(0, [])], False) == [kt.SKIP]          # ck_txn_control accepts it
    out, n = np.empty(77, dtype=np.uint8), C.c_uint64(0)
    assert _lib().ck_encode_control_batch(0, 0, 1, 0, 1, out.ctypes.data, 77, C.byref(n)) != 0


# ---- the broker ----------------------------------------------------------------------------------------------------
def frame(pid, epoch, n, transactional=False, tag="r"):
    recs = [kb.calfkit_record(b'{"n":%d}' % i, f"{tag}-{i}") for i in range(n)]
    b = kt.txn_batch(recs, 0, pid, epoch, base_sequence=-1, transactional=transactional)
    return np.frombuffer(b, dtype=np.uint8).copy()


def sink_log(broker, topics):
    log = []
    for t in topics:
        broker.frame_sink(t, lambda topic, part, f, n: log.append((topic, part, f.tobytes(), n)))
    return log


def test_init_producer_id_fences_a_transactional_id():
    from calfkit.broker import MemoryBroker
    b = MemoryBroker(enable_idempotence=True)
    assert b.enable_idempotence and b.transactional_id is None
    p1, p2 = b.init_producer_id(), b.init_producer_id()
    assert p1[0] != p2[0] and p1[1] == p2[1] == 0
    t1 = b.init_producer_id("tx")
    t2 = b.init_producer_id("tx")
    t3 = b.init_producer_id("tx")
    assert t1[0] == t2[0] == t3[0] not in (p1[0], p2[0]) and (t1[1], t2[1], t3[1]) == (0, 1, 2)
    assert b.init_producer_id("other")[0] != t1[0]
    assert MemoryBroker(transactional_id="x").enable_idempotence


def test_sequences_are_contiguous_per_partition_across_hand_offs():
    from calfkit.broker import MemoryBroker
    b = MemoryBroker(enable_idempotence=True)
    log = sink_log(b, ["a", "b"])
    pid, epoch = b.init_producer_id()
    rng = random.Random(11)
    want = {}
    for _ in range(40):                                 # many hand-offs, as lanes and the framer engine make them
        frames = []
        for _k in range(rng.randint(1, 6)):
            t, p, n = rng.choice("ab"), rng.randrange(4), rng.randint(1, 9)
            frames.append((t, p, frame(pid, epoch, n), n))
        b._hand_frames(frames)
    for topic, part, f, n in log:
        seq = struct.unpack_from(">i", f, 53)[0]
        assert seq == want.get((topic, part), 0)
        want[(topic, part)] = seq + n
        assert kb.crc32c(f[kb.CRC_FROM:]) == struct.unpack_from(">I", f, 17)[0]
        assert struct.unpack_from(">qh", f, 43) == (pid, epoch)
    assert len(want) == 8
    # a second producer counts on its own
    pid2, _e = b.init_producer_id()
    b._hand_frames([("a", 0, frame(pid2, 0, 3), 3)])
    assert struct.unpack_from(">i", log[-1][2], 53)[0] == 0


def test_sequence_wraps_from_int32_max_to_zero():
    from calfkit.broker import MemoryBroker
    b = MemoryBroker(enable_idempotence=True)
    log = sink_log(b, ["a"])
    pid, epoch = b.init_producer_id()
    b._seq[(pid, "a", 2)] = 0x7FFFFFFF - 2
    b._hand_frames([("a", 2, frame(pid, epoch, 5), 5), ("a", 2, frame(pid, epoch, 1), 1)])
    assert [struct.unpack_from(">i", f, 53)[0] for _t, _p, f, _n in log] == [0x7FFFFFFF - 2, 2]
    assert b._seq[(pid, "a", 2)] == 3


def test_reinit_restarts_the_sequences_of_the_producer():
    from calfkit.broker import MemoryBroker
    b = MemoryBroker(transactional_id="tx")
    log = sink_log(b, ["a"])
    pid, e0 = b.init_producer_id("tx")
    b.begin_transaction()
    b._hand_frames([("a", 0, frame(pid, e0, 4, True), 4)])
    b.commit_transaction()
    _pid, e1 = b.init_producer_id("tx")
    b.begin_transaction()
    b._hand_frames([("a", 0, frame(pid, e1, 2, True), 2)])
    b.commit_transaction()
    data = [f for _t, _p, f, _n in log if not f[22] & kt.CONTROL]
    assert [struct.unpack_from(">hi", f, 51) for f in data] == [(e0, 0), (e1, 0)]


def test_markers_go_to_the_partitions_a_transaction_touched():
    from calfkit.broker import MemoryBroker
    b = MemoryBroker(transactional_id="tx")
    log = sink_log(b, ["a", "b", "c"])
    pid, epoch = b.init_producer_id("tx")
    b.begin_transaction()
    b._hand_frames([("a", 1, frame(pid, epoch, 2, True), 2), ("b", 0, frame(pid, epoch, 1, True), 1),
                    ("a", 1, frame(pid, epoch, 3, True), 3)])
    b.commit_transaction()
    b.begin_transaction()
    b._hand_frames([("c", 5, frame(pid, epoch, 1, True), 1)])
    b.abort_transaction()
    b.begin_transaction()
    b.commit_transaction()                              # an empty transaction writes no marker
    markers = [(t, p, kt.control_type(f), n) for t, p, f, n in log if f[22] & kt.CONTROL]
    assert markers == [("a", 1, kt.COMMIT, 1), ("b", 0, kt.COMMIT, 1), ("c", 5, kt.ABORT, 1)]
    for _t, _p, f, _n in log:
        assert struct.unpack_from(">qh", f, 43) == (pid, epoch)
        assert txnmask.verdicts(f, [(0, [])], False) in ([kt.SKIP], [kt.DELIVER])
    with pytest.raises(Exception, match="outside a transaction"):
        b._hand_frames([("a", 0, frame(pid, epoch, 1, True), 1)])
    with pytest.raises(Exception, match="no transaction"):
        b.commit_transaction()


def test_a_tick_that_raises_aborts_its_partitions():
    """Worker.run under a transactional broker: the first tick's frames are committed; the second tick raises after its
    frames went out, so their partitions get ABORT markers and the exception propagates"""
    from calfkit import Client, Worker
    client = Client.connect("localhost", transactional_id="tx")
    broker = client.broker
    log = sink_log(broker, ["a", "b"])
    worker = Worker(client, nodes=[])
    pid, epoch = broker.init_producer_id("tx")
    ticks = {"n": 0}

    def step():
        ticks["n"] += 1
        if ticks["n"] == 1:
            broker._hand_frames([("a", 0, frame(pid, epoch, 2, True), 2), ("b", 3, frame(pid, epoch, 1, True), 1)])
            return 1
        broker._hand_frames([("b", 3, frame(pid, epoch, 4, True), 4), ("b", 4, frame(pid, epoch, 1, True), 1)])
        raise RuntimeError("tool failed")
    worker.step = step
    with pytest.raises(RuntimeError, match="tool failed"):
        asyncio.run(worker.run(until_idle=True))
    kinds = [(t, p, kt.control_type(f) if f[22] & kt.CONTROL else "data") for t, p, f, _n in log]
    assert kinds == [("a", 0, "data"), ("b", 3, "data"), ("a", 0, kt.COMMIT), ("b", 3, kt.COMMIT),
                     ("b", 3, "data"), ("b", 4, "data"), ("b", 3, kt.ABORT), ("b", 4, kt.ABORT)]
    assert broker._txn is None


def test_sticky_partitions_advance_round_robin_per_topic():
    from calfkit.broker import MemoryBroker
    b = MemoryBroker(enable_idempotence=True, num_partitions=3)
    seen = [b.next_sticky(["a", "b"]) for _ in range(4)]
    assert seen == [{"a": 0, "b": 0}, {"a": 1, "b": 1}, {"a": 2, "b": 2}, {"a": 0, "b": 0}]
    assert b.next_sticky(["c"]) == {"c": 0} and b.next_sticky(["a", "c"]) == {"a": 1, "c": 1}


def test_without_either_keyword_frames_are_handed_out_untouched():
    from calfkit.broker import MemoryBroker
    b = MemoryBroker()
    assert not b.enable_idempotence and b.transactional_id is None
    calls = []
    b.frame_sink("a", lambda *a: calls.append(a))
    frames = [("a", None, frame(-1, -1, 2), 2), ("a", 4, frame(-1, -1, 1), 1)]
    before = [f.tobytes() for _t, _p, f, _n in frames]
    b._hand_frames(frames)
    assert [(t, p, n) for t, p, _f, n in calls] == [("a", None, 2), ("a", 4, 1)]
    assert all(c[2] is f[2] for c, f in zip(calls, frames))
    assert [f.tobytes() for _t, _p, f, _n in frames] == before
    assert struct.unpack_from(">i", before[0], 53)[0] == -1 and b._seq == {}


def test_idempotent_broker_refuses_frames_it_cannot_sequence():
    from calfkit.broker import MemoryBroker
    b = MemoryBroker(enable_idempotence=True)
    sink_log(b, ["a"])
    with pytest.raises(Exception, match="producer id or a partition"):
        b._hand_frames([("a", 0, frame(-1, -1, 1), 1)])
    with pytest.raises(Exception, match="producer id or a partition"):
        b._hand_frames([("a", None, frame(3, 0, 1), 1)])
