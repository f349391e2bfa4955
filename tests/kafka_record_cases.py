"""TEST INFRASTRUCTURE ONLY — record sets that reach the record split and field decode with a valid CRC32C: a writer of
varints and records field by field, a hand-built table with one named case per parse rule (tests/kafka_records_ref.py),
seeded structured mutations of well-formed batches, and each codec's simplest container around a records section.

  hand_cases()      {name: (batch, verdict)}: the case record between two good records A and B; verdict "ok" (all three
                    delivered), "record" (only the case record bad) or "batch" (the whole batch bad)
  sources(seed, n)  well-formed batches: null, empty and long keys and values, several headers, repeated correlation ids
  mutants(...)      every varint operator at every varint of the given batches, or a seeded sample of all operators:
                    value +-1, + and - 2^32, padded forms, an overflowing 10th byte, an inserted, deleted or flipped byte,
                    a cut section.  A mutation inside a record's fields may rewrite the record's length to match, so that
                    it reaches the field decode rather than the split
  wrap(batch, c)    the batch's records section in codec c's simplest container: a zlib gzip member, an LZ4 frame of
                    stored blocks, a snappy raw block of literals, a zstd frame of raw blocks
"""
from __future__ import annotations

import random
import struct

import gzip_cases as gz
import kafka_lz4 as lz
import kafka_snappy as ks
import zstd_cases as zc
from make_golden_lz4_batches import with_section
from oracle import kafka_batch as kb

TS = 1767225600000


def zigzag(n: int) -> int:
    """exact: no 64-bit wrap, so that lengths past 2^63 can be written"""
    return 2 * n if n >= 0 else -2 * n - 1


def uvarint(u: int, width: int | None = None) -> bytes:
    """u as 7-bit groups in `width` bytes (default: the fewest); u may need more than 64 bits"""
    n = max(1, (u.bit_length() + 6) // 7) if width is None else width
    assert 0 <= u < 1 << (7 * n), (u, width)
    return bytes(((u >> (7 * i)) & 0x7F) | (0x80 if i < n - 1 else 0) for i in range(n))


def varint(n: int, width: int | None = None) -> bytes:
    return uvarint(zigzag(n), width)


def overflow(n: int) -> bytes:
    """the 10-byte varint of n with 2^64 added: a 10th byte of 2 or 3, refused by a reader that keeps 64 bits exactly"""
    return uvarint(zigzag(n) + (1 << 64), 10)


def recrc(b: bytes) -> bytes:
    return b[:17] + struct.pack(">I", kb.crc32c(b[kb.CRC_FROM:])) + b[21:]


def batch(section: bytes, count: int, codec: int = 0, base_offset: int = 0, magic: int = 2) -> bytes:
    """a RecordBatch v2 frame around a records section, recordsCount `count` (written as 32 bits), CRC32C valid"""
    covered = struct.pack(">hiqqqhi", codec, min(max(count - 1, 0), 2**31 - 1), TS, TS, -1, -1, -1) + struct.pack(">I", count & 0xFFFFFFFF) + section
    return struct.pack(">qiib", base_offset, len(covered) + 9, 0, magic) + struct.pack(">I", kb.crc32c(covered)) + covered


def fields(key=b"k", value=b"hello", headers=(("correlation_id", b"c1"),), *, ts=b"\0", od=b"\0", klen=None, vlen=None,
           nh=None, extra=b"") -> bytes:
    """a record after its length varint; klen / vlen / nh: raw bytes written in place of the right varint.  A header is
    (name, value) or raw bytes"""
    out = b"\0" + ts + od
    out += (varint(-1 if key is None else len(key)) if klen is None else klen) + (key or b"")
    out += (varint(-1 if value is None else len(value)) if vlen is None else vlen) + (value or b"")
    out += varint(len(headers)) if nh is None else nh
    for h in headers:
        if isinstance(h, bytes):
            out += h
        else:
            name, v = h[0].encode(), h[1]
            out += varint(len(name)) + name + varint(-1 if v is None else len(v)) + (v or b"")
    return out + extra


def rec(body: bytes, length: bytes | None = None) -> bytes:
    return (varint(len(body)) if length is None else length) + body


def header(name: bytes, value: bytes | None, klen: bytes | None = None, vlen: bytes | None = None) -> bytes:
    return (varint(len(name)) if klen is None else klen) + name + \
        (varint(-1 if value is None else len(value)) if vlen is None else vlen) + (value or b"")


A = rec(fields(b"key-a", b'{"a":1}', [("content-type", b"application/json"), ("correlation_id", b"id-a")]))
B = rec(fields(None, b"bbb", []))
F = fields()                                           # the default case record: key k, value hello, correlation_id c1


def _around(r: bytes, count_delta: int = 0) -> bytes:
    return batch(A + r + B, 3 + count_delta)


def hand_cases() -> dict[str, tuple[bytes, str]]:
    K, V = b"k", b"hello"
    big = [2**31 - 1, 2**31]
    c: dict[str, tuple[bytes, str]] = {}

    def case(name, r, verdict, count_delta=0):
        c[name] = (_around(r, count_delta), verdict)

    # the record length (the split): a bad one fails the whole batch
    for d, nm in ((2**32, "+2^32"), (2**33, "+2^33"), (-2**32, "-2^32")):
        case(f"record length {nm}", rec(F, varint(len(F) + d)), "batch")
    case("record length 2^32 - 1 (would wrap the position)", rec(F, varint(2**32 - 1)), "batch")
    for v in big + [-1, -2]:
        case(f"record length {v}", rec(F, varint(v)), "batch")
    case("record length 10 bytes, 10th byte 0x02", rec(F, overflow(len(F))), "batch")
    case("record length 10 bytes, 10th byte 0x01", rec(F, uvarint(zigzag(len(F)) + (1 << 63), 10)), "batch")
    case("record length 11 bytes", rec(F, uvarint(zigzag(len(F)), 11)), "batch")
    case("record length padded to 2 bytes", rec(F, varint(len(F), 2)), "ok")
    case("record length padded to 10 bytes", rec(F, varint(len(F), 10)), "ok")
    # key and value lengths
    for nm, kw, n in (("key", "klen", len(K)), ("value", "vlen", len(V))):
        for d, dn in ((2**32, "+2^32"), (2**33, "+2^33"), (-2**32, "-2^32")):
            case(f"{nm} length {dn}", rec(fields(**{kw: varint(n + d)})), "record")
        for v in big:
            case(f"{nm} length {v}", rec(fields(**{kw: varint(v)})), "record")
        case(f"{nm} length 10 bytes, 10th byte 0x02", rec(fields(**{kw: overflow(n)})), "record")
        case(f"{nm} length 11 bytes", rec(fields(**{kw: uvarint(zigzag(n), 11)})), "record")
        case(f"{nm} length padded to 10 bytes", rec(fields(**{kw: varint(n, 10)})), "ok")
        case(f"{nm} length one past the record", rec(fields(**{kw: varint(n + 1)})), "record")
        for v in (-1, -2):
            case(f"{nm} length {v} (null)", rec(fields(**{nm: None, kw: varint(v)})), "ok")
    case("empty key and empty value", rec(fields(b"", b"")), "ok")
    # header lengths and count
    for d, dn in ((2**32, "+2^32"), (-2**32, "-2^32")):
        case(f"correlation_id value length {dn}", rec(fields(headers=[header(b"correlation_id", b"c1", vlen=varint(2 + d))])), "record")
        case(f"header key length {dn}", rec(fields(headers=[header(b"correlation_id", b"c1", klen=varint(14 + d))])), "record")
    for v in big:
        case(f"correlation_id value length {v}", rec(fields(headers=[header(b"correlation_id", b"c1", vlen=varint(v))])), "record")
        case(f"header key length {v}", rec(fields(headers=[header(b"correlation_id", b"c1", klen=varint(v))])), "record")
    case("correlation_id value length 10 bytes, 10th byte 0x02", rec(fields(headers=[header(b"correlation_id", b"c1", vlen=overflow(2))])), "record")
    case("header key length -1", rec(fields(headers=[header(b"", b"c1", klen=varint(-1))])), "record")
    case("header value one past the record", rec(fields(headers=[header(b"correlation_id", b"c1", vlen=varint(3))])), "record")
    for v in (-1, -2):
        case(f"header count {v}", rec(fields(headers=[], nh=varint(v))), "record")
    case("header count -1 before a header", rec(fields(nh=varint(-1))), "record")
    case("header count one more than written", rec(fields(nh=varint(2))), "record")
    case("header count 10 bytes, 10th byte 0x02", rec(fields(nh=overflow(1))), "record")
    case("header count padded to 3 bytes", rec(fields(nh=varint(1, 3))), "ok")
    # the other varints of a record
    case("timestampDelta 10 bytes, 10th byte 0x01", rec(fields(ts=uvarint(1 << 63, 10))), "ok")
    case("timestampDelta 10 bytes, 10th byte 0x02", rec(fields(ts=uvarint(1 << 64, 10))), "record")
    case("timestampDelta 11 bytes", rec(fields(ts=uvarint(5, 11))), "record")
    case("offsetDelta padded to 2 bytes (80 00)", rec(fields(od=b"\x80\x00")), "ok")
    # record boundaries
    case("zero-length record", rec(b""), "record")
    case("attributes-only record", rec(b"\0"), "record")
    case("record ends one byte early", rec(fields(extra=b"\0")), "record")
    case("record ends one byte late", rec(F, varint(len(F) - 1)), "batch")
    case("recordsCount + 1", rec(F), "batch", 1)
    case("recordsCount - 1", rec(F), "batch", -1)
    # the correlation id
    case("two correlation_id headers", rec(fields(headers=[("correlation_id", b"first"), ("correlation_id", b"second")])), "ok")
    case("null correlation_id after a valid one", rec(fields(headers=[("correlation_id", b"kept"), ("correlation_id", None)])), "ok")
    case("null correlation_id only", rec(fields(headers=[("correlation_id", None)])), "ok")
    case("near-miss header names", rec(fields(headers=[("correlation_i", b"x"), ("correlation_idx", b"y"), ("Correlation_id", b"z")])), "ok")
    case("forty headers", rec(fields(headers=[(f"h{i}", bytes([i]) * i) for i in range(39)] + [("correlation_id", b"last")])), "ok")
    # the batch header: these never reach the split
    good = _around(rec(F))
    c["magic 1"] = (recrc(good[:16] + b"\x01" + good[17:]), "batch")
    c["codec 5"] = (recrc(good[:22] + b"\x05" + good[23:]), "batch")
    c["CRC32C mismatch"] = (good[:-1] + bytes([good[-1] ^ 1]), "batch")
    return c


HEADER_CASES = ("magic 1", "codec 5", "CRC32C mismatch")


# ---- seeded well-formed batches and their mutations ----------------------------------------------------------------------
def _record(rng: random.Random, i: int) -> kb.KRecord:
    key = rng.choice([None, b"", b"k%d" % i, bytes(rng.randrange(256) for _ in range(rng.randrange(1, 200)))])
    value = rng.choice([None, b"", b'{"i":%d}' % i, b'{"pad":"%s"}' % (b"x" * rng.randrange(0, 300))])
    headers = []
    for _ in range(rng.randrange(0, 5)):
        name = rng.choice(["correlation_id", "content-type", "correlation_i", "h" * rng.randrange(0, 20)])
        headers.append((name, rng.choice([None, b"", b"id-%d" % rng.randrange(1 << 20), b"application/json"])))
    return kb.KRecord(value, key, headers, timestamp=rng.choice([0, TS + rng.randrange(1 << 40)]))


def sources(seed: int, n: int) -> list[bytes]:
    rng = random.Random(seed)
    return [kb.encode_batch([_record(rng, i) for i in range(rng.randint(1, 4))], base_offset=b * 10, base_timestamp=TS)
            for b in range(n)]


def varint_sites(section: bytes) -> list[tuple[int, int, int, tuple[int, int] | None]]:
    """(start, end, value, record) of every varint of a well-formed records section; record = (start of its length varint,
    end of it) for a varint inside a record's fields, None for a record length"""
    out, pos = [], 0
    while pos < len(section):
        n, p = kb.get_varint(section, pos)
        out.append((pos, p, n, None))
        r, end, q = (pos, p), p + n, p + 1
        for _ in range(2):                                     # timestampDelta, offsetDelta
            v, q2 = kb.get_varint(section, q)
            out.append((q, q2, v, r))
            q = q2
        for _ in range(2):                                     # key, value
            v, q2 = kb.get_varint(section, q)
            out.append((q, q2, v, r))
            q = q2 + max(v, 0)
        nh, q2 = kb.get_varint(section, q)
        out.append((q, q2, nh, r))
        q = q2
        for _ in range(nh):
            for _ in range(2):
                v, q2 = kb.get_varint(section, q)
                out.append((q, q2, v, r))
                q = q2 + max(v, 0)
        assert q == end
        pos = end
    return out


def _replace(section: bytes, start: int, end: int, new: bytes, r: tuple[int, int] | None) -> bytes:
    """section with [start, end) replaced by new; r: the enclosing record's length varint, rewritten to the new length"""
    out = section[:start] + new + section[end:]
    if r is None:
        return out
    n, _ = kb.get_varint(section, r[0])
    return out[:r[0]] + varint(n + len(new) - (end - start)) + out[r[1]:]


VARINT_OPS = {
    "+1": lambda v: varint(v + 1),
    "-1": lambda v: varint(v - 1),
    "+2^32": lambda v: varint(v + 2**32),
    "-2^32": lambda v: varint(v - 2**32),
    "padded": lambda v: varint(v, len(varint(v)) + 1),
    "padded to 10": lambda v: varint(v, 10),
    "10th byte overflow": overflow,
}


def _byte_op(rng: random.Random, section: bytes) -> tuple[str, bytes]:
    sites = [s for s in varint_sites(section) if s[3] is not None]
    op = rng.choice(["insert", "delete", "flip", "cut"])
    if op == "cut":
        return op, section[:rng.randrange(len(section))]
    at = rng.randrange(len(section))
    # the record whose fields hold `at`, when the mutation should keep the split aligned
    inner = [s[3] for s in sites if s[3][1] <= at] if rng.random() < 0.6 else []
    r = inner[-1] if inner else None
    if op == "insert":
        return op, _replace(section, at, at, bytes([rng.randrange(256)]), r)
    if op == "delete":
        return op, _replace(section, at, at + 1, b"", r)
    return op, _replace(section, at, at + 1, bytes([section[at] ^ rng.randrange(1, 256)]), None)


def mutants(srcs: list[bytes], exhaustive: bool = True, sample: int = 0, seed: int = 0) -> list[tuple[str, bytes]]:
    """[(label, batch)]: exhaustive, every VARINT_OPS operator at every varint of every source (a varint inside a record's
    fields with the record's length rewritten, and again without); then `sample` seeded operators (varint or byte) at
    random places of random sources.  recordsCount is kept and the CRC32C recomputed"""
    out = []
    for si, b in enumerate(srcs if exhaustive else []):
        sec = b[kb.HEADER_LEN:]
        for start, end, v, r in varint_sites(sec):
            for name, op in VARINT_OPS.items():
                out.append((f"src {si} @{start} {name}", with_section(b, _replace(sec, start, end, op(v), r), 0)))
                if r is not None:
                    out.append((f"src {si} @{start} {name} unaligned", with_section(b, _replace(sec, start, end, op(v), None), 0)))
    rng = random.Random(seed)
    for k in range(sample):
        si = rng.randrange(len(srcs))
        b = srcs[si]
        sec = b[kb.HEADER_LEN:]
        if rng.random() < 0.5:
            start, end, v, r = rng.choice(varint_sites(sec))
            name = rng.choice(list(VARINT_OPS))
            new = _replace(sec, start, end, VARINT_OPS[name](v), r if rng.random() < 0.7 else None)
        else:
            name, new = _byte_op(rng, sec)
            start = "-"
        out.append((f"sample {k} src {si} @{start} {name}", with_section(b, new, 0)))
    return out


# ---- containers ----------------------------------------------------------------------------------------------------------
def lz4_stored(sec: bytes) -> bytes:
    desc = bytes([0x60, 0x40])                                 # version 1, independent blocks; 64 KB blocks
    out = struct.pack("<I", lz.MAGIC) + desc + bytes([(lz.xxh32(desc) >> 8) & 0xFF])
    for i in range(0, len(sec), 64 << 10):
        blk = sec[i:i + (64 << 10)]
        out += struct.pack("<I", 0x80000000 | len(blk)) + blk
    return out + b"\0\0\0\0"


def snappy_literals(sec: bytes) -> bytes:
    return ks.block([ks.lit(sec[i:i + (64 << 10)]) for i in range(0, len(sec), 64 << 10)], content=sec)


def zstd_raw(sec: bytes) -> bytes:
    chunks = [sec[i:i + (128 << 10)] for i in range(0, len(sec), 128 << 10)] or [b""]
    return zc.frame([zc.block(i == len(chunks) - 1, 0, ch) for i, ch in enumerate(chunks)])


CONTAINERS = {1: gz.gzip_bytes, 2: snappy_literals, 3: lz4_stored, 4: zstd_raw}
CODEC_NAMES = {1: "gzip", 2: "snappy", 3: "lz4", 4: "zstd"}


def wrap(b: bytes, codec: int) -> bytes:
    return with_section(b, CONTAINERS[codec](b[kb.HEADER_LEN:]), codec)
