"""Transactions on the consume side without a GPU: the rule of csrc/ck_txn.h, built with g++ on its own, gives every batch
of seeded random transactional logs the verdict the plain-Python restatement (tests/kafka_txn.py) gives it, at both
isolation levels; the library's ck_fetch_txn_mask agrees; a fetch's read_committed mask is computed once and carried by
FetchArena slices and broker polls across every split point; isolation levels are validated; the Worker takes its
isolation level from the subscriber kwargs."""
import random
import struct

import numpy as np
import pytest

import kafka_txn as kt
import txnmask
from oracle import kafka_batch as kb

SEEDS = range(600)


def rec(tag):
    return kb.calfkit_record(b'{"v":"%s"}' % tag.encode(), tag)


@pytest.mark.parametrize("read_committed", [False, True])
def test_rule_matches_restatement_over_random_logs(read_committed):
    seen = {kt.DELIVER: 0, kt.BAD: 0, kt.SKIP: 0}
    for seed in SEEDS:
        buf, parts = kt.random_log(seed)
        want = kt.verdicts(buf, parts, read_committed)
        assert txnmask.verdicts(buf, parts, read_committed) == want, seed
        for v in want:
            seen[v] += 1
    assert min(seen.values()) > 500                 # every verdict is exercised many times


def test_read_committed_hides_more_than_control_batches():
    """over the random logs read_committed skips data batches that read_uncommitted delivers, and never the reverse"""
    extra = 0
    for seed in SEEDS:
        buf, parts = kt.random_log(seed)
        ru, rc = kt.verdicts(buf, parts, False), kt.verdicts(buf, parts, True)
        assert all(a == b or (a == kt.DELIVER and b == kt.SKIP) for a, b in zip(ru, rc))
        extra += sum(a != b for a, b in zip(ru, rc))
    assert extra > 1000


def test_library_export_matches_the_host_build():
    from calfkit.engine.batch import fetch_txn_mask
    for seed in range(0, 600, 7):
        buf, parts = kt.random_log(seed)
        got = fetch_txn_mask(np.frombuffer(buf, dtype=np.uint8), parts)
        assert list(got) == list(txnmask.mask(buf, parts)), seed
        assert len(got) == len(kt.batches(buf))


def test_hand_written_cases():
    """nested transactions of two producers, an abort marker past the end of the fetch, an entry no batch reaches, an
    unknown marker type and version, and malformed control batches"""
    A, B = 7, 9
    log = [kt.txn_batch([rec("a0")], 0, A),                 # A's aborted txn starts at 0
           kt.txn_batch([rec("b0")], 1, B),                 # B's committed txn starts at 1
           kt.txn_batch([rec("a1")], 2, A),
           kt.control_batch(3, B, kt.COMMIT),
           kt.control_batch(4, A, kt.ABORT),
           kt.txn_batch([rec("a2")], 5, A),                 # A's next txn: aborted, marker past the end
           kt.txn_batch([rec("n")], 6, -1, transactional=False),
           kt.control_batch(7, A, 5),                       # unknown type: skipped, changes nothing
           kt.control_batch(8, B, kt.ABORT, key=kt.control_key(kt.ABORT, version=1)),   # unknown version: parsed
           kt.control_batch(9, A, kt.ABORT, key=b"\x00\x00\x00"),                      # short key: bad
           kt.control_batch(10, A, kt.ABORT, key=kt.control_key(kt.ABORT, version=-1)),  # negative version: bad
           kt.control_batch(11, A, kt.ABORT, extra_records=1),                          # two records: bad
           kt.txn_batch([rec("a3")], 13, A)]
    buf = b"".join(log)
    parts = [(0, [(A, 0), (A, 5), (B, 1000)])]
    D, X, S = kt.DELIVER, kt.BAD, kt.SKIP
    assert kt.verdicts(buf, parts, True) == [S, D, S, S, S, S, D, S, S, X, X, X, S]
    assert kt.verdicts(buf, parts, False) == [D, D, D, S, S, D, D, S, S, X, X, X, D]
    for rc in (False, True):
        assert txnmask.verdicts(buf, parts, rc) == kt.verdicts(buf, parts, rc)


def test_control_record_length_varint_must_fit_64_bits():
    """a control batch whose record length is a 10-byte varint with 2^64 added (a 10th byte of 2, lost by a reader that
    keeps 64 bits) is bad; the same length padded to 10 bytes (a 10th byte of 0) is a well-formed marker"""
    import kafka_record_cases as kc
    from make_golden_lz4_batches import with_section
    f = kt.control_batch(0, 7, kt.ABORT)
    n, p = kb.get_varint(f, kb.HEADER_LEN)
    assert p == kb.HEADER_LEN + 1 and n == len(f) - p
    over = with_section(f, kc.overflow(n) + f[p:], 0)
    padded = with_section(f, kc.varint(n, 10) + f[p:], 0)
    assert txnmask.verdicts(over, [(0, [])], False) == [kt.BAD]
    assert txnmask.verdicts(padded, [(0, [])], False) == [kt.SKIP]
    assert kt.control_type(padded) == kt.ABORT


def test_partitions_reset_state_and_bad_partitions_are_refused():
    """the same producer id aborted in partition 0 is not aborted in partition 1; partition starts out of order are
    refused, as is an entry naming no partition"""
    p0 = kt.txn_batch([rec("x")], 0, 5)
    p1 = kt.txn_batch([rec("y")], 0, 5)
    buf = p0 + p1
    assert list(txnmask.mask(buf, [(0, [(5, 0)]), (len(p0), [])])) == [1, 0]
    assert list(txnmask.mask(buf, [(0, []), (len(p0), [(5, 0)])])) == [0, 1]
    assert txnmask.mask(buf, [(len(p0), []), (0, [(5, 0)])]) is None
    from calfkit.engine.batch import fetch_txn_mask
    from calfkit.exceptions import EngineError
    with pytest.raises(EngineError):
        fetch_txn_mask(np.frombuffer(buf, dtype=np.uint8), [(len(p0), []), (0, [(5, 0)])])


def test_bad_crc_data_batch_changes_no_state():
    """a data batch failing its CRC32C does not move aborted transactions into the set, even where its (corrupt)
    lastOffset reaches them: the next batch of the producer is delivered"""
    bad = kt.txn_batch([rec("c")], 0, 3)
    bad = bad[:23] + struct.pack(">i", 50) + bad[27:]          # lastOffsetDelta changed after the CRC was computed
    buf = bad + kt.txn_batch([rec("d")], 1, 3)
    parts = [(0, [(3, 40)])]
    assert kt.verdicts(buf, parts, True) == [kt.BAD, kt.DELIVER]
    assert txnmask.verdicts(buf, parts, True) == [kt.BAD, kt.DELIVER]


def test_fetch_arena_slices_carry_the_mask_across_every_split():
    from calfkit.engine.lane import FetchArena
    for seed in range(0, 600, 37):
        buf, parts = kt.random_log(seed)
        fa = FetchArena.of(buf, partitions=parts)
        full = fa.hidden()
        assert list(full) == list(txnmask.mask(buf, parts))
        nf = len(fa.frames()[1])
        for k in range(1, nf):
            head, rest = fa.slice_frames(0, k), fa.slice_frames(k, None)
            assert list(head.hidden()) == list(full[:k]) and list(rest.hidden()) == list(full[k:])
            assert len(rest.hidden()) == len(rest.frames()[1])
    # without aborted transactions there is no mask to carry
    assert FetchArena.of(buf).hidden() is None and FetchArena.of(buf).slice_frames(0, 1).hidden() is None
    with pytest.raises(Exception):
        FetchArena.of(buf, aborted_transactions=[], partitions=[])


def test_one_partition_form_equals_the_general_one():
    from calfkit.engine.lane import FetchArena
    buf, parts = kt.random_partition(random.Random(5), "one")
    a = FetchArena.of(buf, aborted_transactions=parts).hidden()
    b = FetchArena.of(buf, partitions=[(0, parts)]).hidden()
    assert list(a) == list(b) and a.sum() > 0


@pytest.mark.parametrize("max_records", [1, 3, 7, 50])
def test_broker_polls_carry_the_mask(max_records):
    """the fetch enqueued by produce_fetch and polled in pieces: the pieces' masks are the fetch's mask, in order"""
    from calfkit.broker import MemoryBroker
    from calfkit.engine.lane import FetchArena
    for seed in (3, 11, 29, 41):
        buf, parts = kt.random_log(seed)
        full = list(FetchArena.of(buf, partitions=parts).hidden())
        br = MemoryBroker()
        br.produce_fetch("t", buf, partitions=parts)
        got = []
        while (a := br.poll_arena(("t",), max_records)) is not None:
            assert len(a.hidden()) == len(a.frames()[1])
            got += list(a.hidden())
        assert got == full
    with pytest.raises(Exception):
        MemoryBroker().produce_fetch("t", FetchArena.of(buf), aborted_transactions=[(1, 0)])


def test_set_isolation_level_validation():
    from calfkit.engine.batch import BatchEngine
    from calfkit.exceptions import EngineError
    e = object.__new__(BatchEngine)                 # the level is host state: no device needed to validate it
    e.read_committed = False
    e.set_isolation_level("read_committed")
    assert e.read_committed
    e.set_isolation_level("read_uncommitted")
    assert not e.read_committed
    for bad in ("READ_COMMITTED", "committed", "", None, 1):
        with pytest.raises(EngineError):
            e.set_isolation_level(bad)


def test_worker_reads_isolation_level_from_subscriber_kwargs():
    import tools_def
    from calfkit import Client, Worker, agent_tool
    from calfkit.exceptions import EngineError
    for kwargs, want in (({"isolation_level": "read_committed"}, "read_committed"), ({}, "read_uncommitted"),
                         ({"isolation_level": "read_uncommitted"}, "read_uncommitted")):
        client = Client.connect("localhost")
        node = agent_tool(tools_def.get_weather, device_template="It's sunny in {location}")
        w = Worker(client, nodes=[node], extra_subscribe_kwargs=kwargs)
        w.register_handlers()
        assert w._levels[id(node)] == want
        assert w._subs[0][1].kwargs.get("isolation_level", "read_uncommitted") == want
        assert w.stats["skipped"] == 0
    client = Client.connect("localhost")
    node = agent_tool(tools_def.get_weather, device_template="It's sunny in {location}")
    with pytest.raises(EngineError):
        Worker(client, nodes=[node], extra_subscribe_kwargs={"isolation_level": "serializable"}).register_handlers()
