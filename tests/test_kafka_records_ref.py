"""The strict record parser (tests/kafka_records_ref.py) without a GPU: on well-formed fetches it reads every record as
oracle.kafka_batch.decode_batches does; byte-exact hand vectors pin its varint rule, its spans, its correlation id and
its batch chain; every hand-built case (tests/kafka_record_cases.py) gets the verdict it is named for; and a records
section in each codec's simplest container parses as the same section uncompressed."""
import struct

import pytest

import kafka_record_cases as kc
import kafka_records_ref as ref
from oracle import kafka_batch as kb


def last_corr(r: kb.KRecord):
    vals = [v for k, v in r.headers if k == "correlation_id" and v is not None]
    return vals[-1] if vals else None


def well_formed_fetches():
    from calfkit import synth
    tool = [kb.calfkit_record(v, f"id-{i}", keyed=i % 3 != 0) for i, v in enumerate(synth.tool_events(40, seed=5))]
    odd = [kb.KRecord(None, None), kb.KRecord(b"", b""), kb.KRecord(b"v", None, [("correlation_id", None)]),
           kb.KRecord(b"x" * 300, b"k" * 200, [(f"h{i}", b"y" * i) for i in range(60)]),
           kb.KRecord(b"v", b"k", [("correlation_id", b"a"), ("content-type", b"json"), ("correlation_id", b"b")]),
           kb.KRecord(b"v", b"k", [("correlation_id", b"a"), ("correlation_id", None)])]
    yield "tool events", kb.encode_batch(tool[:25], base_timestamp=kc.TS) + kb.encode_batch(tool[25:], base_offset=25)
    yield "null, empty, long, many headers, repeated correlation ids", kb.encode_batch(odd, base_timestamp=kc.TS)
    for seed in range(4):
        yield f"seeded sources {seed}", b"".join(kc.sources(seed, 30))


@pytest.mark.parametrize("name,buf", list(well_formed_fetches()), ids=lambda x: x if isinstance(x, str) else "")
def test_well_formed_fetches_read_as_the_oracle_reads_them(name, buf):
    want = kb.decode_batches(buf)
    got = ref.parse_fetch(buf)
    assert len(got) == len(want) > 0
    for g, w in zip(got, want):
        assert g.bad == 0 and not g.decoded and g.data is not None
        assert (g.value(), g.key_bytes(), g.corr_bytes()) == (w.value or b"", w.key, last_corr(w))


def test_varint_vectors():
    assert ref.read_varint(b"\x80\x00", 0, 2) == (0, 2)                          # non-minimal: accepted
    assert ref.read_varint(b"\x03", 0, 1) == (-2, 1)
    assert ref.read_varint(b"\xff" * 9 + b"\x01", 0, 10) == (-2**63, 10)        # 2^64 - 1: the largest that fits
    assert ref.read_varint(b"\xfe" + b"\xff" * 8 + b"\x01", 0, 10) == (2**63 - 1, 10)
    for bad in (b"\x80" * 9 + b"\x02", b"\xff" * 9 + b"\x03", b"\x80" * 10 + b"\x00", b"\x80", b""):
        with pytest.raises(ref.Corrupt):
            ref.read_varint(bad, 0, len(bad))
    with pytest.raises(ref.Corrupt):                                              # the bound, not the buffer, ends it
        ref.read_varint(b"\x80\x00", 0, 1)
    assert kc.overflow(5) == b"\x8a" + b"\x80" * 8 + b"\x02"
    assert kc.varint(1, 3) == b"\x82\x80\x00"


def test_value_length_past_2_32_is_refused():
    """the record of value "hello" with its value length 0a rewritten as 8a 80 80 80 20 (2^32 + 5) and its record length
    raised by 4: a reader that narrows to 32 bits delivers "hello"; this one and the oracle refuse it"""
    good = kb.encode_record(kb.KRecord(b"hello", b"k", [("correlation_id", b"c1")]), 0, 0)
    assert good.hex(" ") == "3c 00 00 00 02 6b 0a 68 65 6c 6c 6f 02 1c 63 6f 72 72 65 6c 61 74 69 6f 6e 5f 69 64 04 63 31"
    bad = bytes.fromhex("44 00 00 00 02 6b 8a 80 80 80 20") + good[7:]
    assert bad == kc.rec(kc.fields(vlen=kc.varint(5 + 2**32)))
    buf = kc.batch(bad, 1)
    with pytest.raises((ValueError, IndexError)):          # the oracle reads on past the record, then past the fetch
        kb.decode_batches(buf)
    (r,) = ref.parse_fetch(buf)
    assert (r.bad, r.val, r.key, r.corr) == (1, (0, 0), None, None)
    (r,) = ref.parse_fetch(kc.batch(good, 1))
    assert (r.bad, r.value(), r.key_bytes(), r.corr_bytes()) == (0, b"hello", b"k", b"c1")


def test_spans_are_byte_exact():
    """A, the default record, B in one batch behind a 61-byte header: the spans as offsets into the fetch"""
    buf = kc.batch(kc.A + kc.rec(kc.F) + kc.B, 3)
    a, f, b = ref.parse_fetch(buf)
    at = kb.HEADER_LEN + len(kc.A)                     # the default record's length varint
    assert (f.bad, f.key, f.val, f.corr) == (0, (at + 5, 1), (at + 7, 5), (at + 29, 2))
    assert (a.key, a.val) == ((kb.HEADER_LEN + 6, 5), (kb.HEADER_LEN + 12, 7))   # A's length takes 2 bytes
    assert (b.key, b.corr, b.value()) == (None, None, b"bbb")
    two = buf + kc.batch(kc.B, 1)
    assert ref.parse_fetch(two)[3].val == (len(buf) + kb.HEADER_LEN + 6, 3)   # B: a null key, then its value


def test_correlation_id_is_the_last_non_null_one():
    c = kc.hand_cases()
    want = {"two correlation_id headers": b"second", "null correlation_id after a valid one": b"kept",
            "null correlation_id only": None, "near-miss header names": None, "forty headers": b"last"}
    for name, corr in want.items():
        r = ref.parse_fetch(c[name][0])[1]
        assert r.bad == 0 and r.corr_bytes() == corr, name


def test_batch_chain():
    """the chain stops at a batchLength below 49 and at a truncated trailing batch: nothing from there on is counted; a
    recordsCount that passes max_records refuses the fetch"""
    good = kc.batch(kc.A + kc.B, 2)
    short = struct.pack(">qi", 0, 48) + b"\0" * 48
    assert len(ref.parse_fetch(good + short + good)) == 2
    assert len(ref.parse_fetch(good + struct.pack(">qi", 0, -1) + good)) == 2
    assert len(ref.parse_fetch(good + good[:-1])) == 2
    assert len(ref.parse_fetch(good + good, max_records=4)) == 4
    with pytest.raises(ref.RecordsLimit):
        ref.parse_fetch(good + good, max_records=3)
    with pytest.raises(ref.RecordsLimit):
        ref.parse_fetch(good + kc.batch(kc.A, 0xFFFFFFFF), max_records=1 << 16)


@pytest.mark.parametrize("name", list(kc.hand_cases()))
def test_hand_case_has_its_verdict(name):
    b, verdict = kc.hand_cases()[name]
    got = [r.bad for r in ref.parse_fetch(b)]
    want = {"ok": [0, 0, 0], "record": [0, 1, 0], "batch": [1] * len(got)}[verdict]
    assert got == want and len(got) >= 2
    if verdict == "ok":
        assert [r.value() for r in ref.parse_fetch(b)][::2] == [b'{"a":1}', b"bbb"]


def test_mutants_cover_every_verdict():
    seen = {"ok": 0, "record": 0, "batch": 0}
    for _label, b in kc.mutants(kc.sources(1, 3)) + kc.mutants(kc.sources(2, 10), exhaustive=False, sample=600, seed=4):
        bad = [r.bad for r in ref.parse_fetch(b)]
        if bad:
            seen["batch" if all(bad) else "record" if any(bad) else "ok"] += 1
    assert min(seen.values()) > 100, seen


@pytest.mark.parametrize("codec", sorted(kc.CONTAINERS), ids=lambda c: kc.CODEC_NAMES[c])
def test_containers_parse_as_the_uncompressed_section(codec):
    cases = [b for n, (b, _v) in kc.hand_cases().items() if n not in kc.HEADER_CASES]
    cases += [b for _l, b in kc.mutants(kc.sources(7, 4), exhaustive=False, sample=150, seed=8)]
    for b in cases:
        plain, packed = ref.parse_fetch(b), ref.parse_fetch(kc.wrap(b, codec))
        assert len(plain) == len(packed)
        for p, q in zip(plain, packed):
            assert q.bad == p.bad and (q.decoded or q.bad)
            assert (q.value(), q.key_bytes(), q.corr_bytes()) == (p.value(), p.key_bytes(), p.corr_bytes())
