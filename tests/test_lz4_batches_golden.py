"""LZ4 batches as liblz4 writes them (tests/golden/lz4_batches.json, written by make_golden_lz4_batches.py): each one's
records section decompresses (tests/kafka_lz4.decompress_batch) to the oracle's uncompressed batch of the same records,
and the golden file covers every block size and frame flag the device decoder takes.  And the host view of a fetch
response whose LZ4 batches were decoded on the device: values in the raw bytes and in the decoded slots, by offset."""
import numpy as np
import pytest

import kafka_lz4 as lz
from make_golden_lz4_batches import load, uncompressed
from oracle import kafka_batch as kb

BATCHES = load()


@pytest.mark.parametrize("name", [n for n, _s, _b in BATCHES])
def test_golden_batch_decompresses_to_the_oracle_batch(name):
    _n, spec, batch = next(c for c in BATCHES if c[0] == name)
    assert batch[22] & 7 == 3
    want = uncompressed(spec)
    assert lz.decompress_batch(batch) == want
    assert [(r.value, r.key, r.headers) for r in kb.decode_batches(want)] == \
        [(r.value, r.key, r.headers) for r in kb.decode_batches(lz.decompress_batch(batch))]


def test_golden_batches_cover_block_sizes_and_flags():
    flg = {b[61 + 4] for _n, _s, b in BATCHES}
    bd = {b[61 + 5] for _n, _s, b in BATCHES}
    assert bd == {0x40, 0x50, 0x60, 0x70}
    assert {0x60, 0x40, 0x70, 0x64, 0x68, 0x5C} <= flg
    # the incompressible section goes out as stored blocks (bit 31 of the size word)
    _n, _s, b = next(c for c in BATCHES if c[0] == "incompressible")
    pos, words = 61 + 7, []
    while (w := int.from_bytes(b[pos:pos + 4], "little")):
        words.append(w)
        pos += 4 + (w & 0x7FFFFFFF) + 4                          # + its block checksum
    assert any(w >> 31 for w in words)
    # linked frames of more than one block
    assert any(not (b[61 + 4] & 0x20) and len(lz.decompress_batch(b)) > 2 * 65536 for _n, _s, b in BATCHES)


def test_fetch_bytes_reads_raw_and_decoded_spans():
    from calfkit.engine.batch import FetchBytes
    raw = np.frombuffer(b"0123456789abcdef-raw", dtype=np.uint8)
    dec = np.frombuffer(b"DECODED-VALUES", dtype=np.uint8)
    fb = FetchBytes(raw, 32, dec)
    assert fb[3:7].tobytes() == b"3456"
    assert fb[16:20].tobytes() == b"-raw"
    assert fb[32:39].tobytes() == b"DECODED"
    assert fb[40:46].tobytes() == b"VALUES"
    assert fb.nbytes == raw.nbytes + dec.nbytes
    with pytest.raises(IndexError):
        fb[18:34]


def test_fetch_records_and_publish_batch_over_raw_and_decoded():
    """synthetic offsets: records 0 and 2 lie in the raw bytes, record 1 in the decoded slots; keys and reply-topic spans
    are read relative to each record wherever it lies"""
    from calfkit.engine._lib import PUB_DTYPE
    from calfkit.engine.lane import FetchArena, FetchRecords, PublishBatch
    raw = b"....AAAA{\"k\":\"key-a\"}....CC{\"k\":\"key-c\",\"t\":\"reply.c\"}"
    dec = b"xx{\"k\":\"key-b\",\"t\":\"reply.b\"}yy"
    base = 64
    a0, c0 = raw.index(b"{\"k\":\"key-a"), raw.index(b"{\"k\":\"key-c")
    b0 = base + dec.index(b"{")
    a_len = raw.index(b"}", a0) + 1 - a0
    c_len = raw.index(b"}", c0) + 1 - c0
    b_len = dec.index(b"}") + 1 - dec.index(b"{")
    arena = FetchArena(np.frombuffer(raw, dtype=np.uint8))
    val_off = np.array([a0, b0, c0], dtype=np.int64)
    val_len = np.array([a_len, b_len, c_len], dtype=np.uint32)
    recs = FetchRecords(arena, val_off, val_len, np.zeros(3, np.uint32), decoded=(base, np.frombuffer(dec, dtype=np.uint8)))
    assert recs.n == 3
    assert recs.record(0) == b"{\"k\":\"key-a\"}"
    assert recs.record(1) == b"{\"k\":\"key-b\",\"t\":\"reply.b\"}"
    assert recs.record(2) == b"{\"k\":\"key-c\",\"t\":\"reply.c\"}"
    # without decoded slots the view is the arena itself, as before
    assert FetchRecords(arena, val_off[[0, 2]], val_len[[0, 2]], np.zeros(2, np.uint32)).data is arena.data
    # publishes: keyed, topic named by a span of the source record (topic id -1)
    pubs = np.zeros(3, dtype=PUB_DTYPE)
    pubs["payload"], pubs["record"], pubs["has_key"], pubs["topic_id"] = [0, 1, 2], [0, 1, 2], 1, [0, -1, -1]
    key_spans = np.zeros((2, 3), dtype=np.uint32)
    for r in range(3):
        rec = recs.record(r)
        key_spans[0, r] = rec.index(b"key-")
        key_spans[1, r] = 5
        if r:
            pubs["topic_off"][r] = rec.index(b"reply.")
            pubs["topic_len"][r] = 7
    out = np.frombuffer(b"P" * 48, dtype=np.uint8)
    pb = PublishBatch(out, np.array([0, 16, 32, 48], np.int64), np.array([1, 1, 1], np.uint32), pubs, {0: "t0"}, recs, key_spans,
                      None, None)
    assert [pb.key(j) for j in range(3)] == [b"key-a", b"key-b", b"key-c"]
    assert [pb.topic_name(j) for j in range(3)] == ["t0", "reply.b", "reply.c"]
    assert pb.record_bytes(1).tobytes() == recs.record(1)
