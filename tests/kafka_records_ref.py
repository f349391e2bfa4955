"""TEST INFRASTRUCTURE ONLY — a strict parser of a fetch response's record set (concatenated RecordBatch v2 frames), in
plain Python.  For every record it gives the verdict and the spans that BatchEngine.rb_index() reports, so the device's
record split (ck_rb_split_kernel) and field decode (ck_rb_fields_kernel) are checked record by record against it.

The rules follow kafka-python's DefaultRecordBatch, which calfkit's consumer (aiokafka) uses; lengths are exact integers
and never wrap:
  batch chain     the host's (ck_txn_frame_end): 12 + batchLength bytes from where the previous batch ended; the chain
                  stops at a truncated trailing batch or at one whose batchLength is below 49, and nothing from there on
                  is counted.  recordsCount is read as an unsigned 32-bit number; a fetch whose counted records (or
                  batches) would pass max_records is refused as a whole (RecordsLimit)
  batch failure   every record of the batch gets bad = 1 and no spans.  A batch fails on magic != 2, a codec id above 4,
                  a CRC32C mismatch, a compressed section that does not decode (only the container forms the tests build
                  are decoded here: any gzip member, an LZ4 frame, a snappy section, a zstd frame of raw and RLE blocks),
                  a record length that is not a valid varint, is negative or runs past the records section, or
                  recordsCount records that do not end exactly at the section's end
  varints         zig-zag, at most 10 bytes, and the unsigned value must fit in 64 bits: a 10th byte above 1 is refused.
                  Non-minimal encodings (80 00 for 0) are accepted, as kafka-python accepts them
  record failure  the record gets bad = 1 and no spans; the other records of its batch are unaffected.  A record fails on
                  a varint that is invalid or runs past the record's end, a key or value length >= 0 that runs past the
                  record's end, a negative header count or header key length, a header key or value that runs past the
                  record's end, or fields that do not end exactly at the record's length.  A negative key or value length
                  means null: key None, value the empty span (0, 0)
  correlation id  the value of the last header whose key is exactly `correlation_id` and whose value is not null; None
                  when there is none
Known divergence: kafka-python decodes header keys as UTF-8 and raises on invalid UTF-8; neither this parser nor the
device checks them.  Control batches (attributes bit 5) are outside this parser: it raises on them.
"""
from __future__ import annotations

import struct
from dataclasses import dataclass

import gzip_cases as gz
import kafka_lz4 as lz
import kafka_snappy as ks
import kafka_txn as kt
import zstd_cases as zc
from oracle import kafka_batch as kb

CORRELATION_ID = b"correlation_id"


class Corrupt(Exception):
    """a varint or a length the rules above refuse"""


class RecordsLimit(ValueError):
    """the fetch counts more records (or batches) than max_records"""


@dataclass(frozen=True)
class Record:
    bad: int
    data: bytes                                # the bytes the spans index: the fetch, or a compressed batch's decoded section
    decoded: bool = False                      # data is a decoded section
    val: tuple[int, int] = (0, 0)              # (offset, length); (0, 0) for a null value and for a bad record
    key: tuple[int, int] | None = None         # None: null key, or a bad record
    corr: tuple[int, int] | None = None        # None: no correlation id, or a bad record

    def _at(self, span):
        return None if span is None else bytes(self.data[span[0]:span[0] + span[1]])

    def value(self) -> bytes:
        return self._at(self.val)

    def key_bytes(self) -> bytes | None:
        return self._at(self.key)

    def corr_bytes(self) -> bytes | None:
        return self._at(self.corr)


def read_varint(data: bytes, pos: int, end: int) -> tuple[int, int]:
    """(value, position after it) of the zig-zag varint at pos, read no further than end"""
    u = 0
    for i in range(10):
        if pos >= end:
            raise Corrupt("varint runs past its bound")
        b = data[pos]
        pos += 1
        if i == 9 and b > 1:
            raise Corrupt("varint does not fit in 64 bits")
        u |= (b & 0x7F) << (7 * i)
        if not b & 0x80:
            return (u >> 1) ^ -(u & 1), pos
    raise AssertionError("unreachable: a 10th byte of at most 1 ends the varint")


def _span(length: int, pos: int, end: int) -> tuple[int, int]:
    if length > end - pos:
        raise Corrupt("length runs past the record")
    return pos, length


def record(data: bytes, pos: int, end: int, decoded: bool) -> Record:
    """the record whose fields are data[pos, end) (after its length varint)"""
    try:
        pos += 1                                               # attributes
        _ts, pos = read_varint(data, pos, end)                 # timestampDelta
        _od, pos = read_varint(data, pos, end)                 # offsetDelta
        n, pos = read_varint(data, pos, end)
        key = None
        if n >= 0:
            key = _span(n, pos, end)
            pos += n
        n, pos = read_varint(data, pos, end)
        val = (0, 0)
        if n >= 0:
            val = _span(n, pos, end)
            pos += n
        nh, pos = read_varint(data, pos, end)
        if nh < 0:
            raise Corrupt("negative header count")
        corr = None
        for _ in range(nh):                                    # every header takes at least 2 bytes: bounded by the record
            n, pos = read_varint(data, pos, end)
            if n < 0:
                raise Corrupt("negative header key length")
            k = _span(n, pos, end)
            pos += n
            n, pos = read_varint(data, pos, end)
            if n >= 0:
                v = _span(n, pos, end)
                pos += n
                if data[k[0]:k[0] + k[1]] == CORRELATION_ID:
                    corr = v
        if pos != end:
            raise Corrupt("fields do not end at the record's length")
    except Corrupt:
        return Record(1, data, decoded)
    return Record(0, data, decoded, val, key, corr)


def split(data: bytes, lo: int, hi: int, count: int) -> list[tuple[int, int]] | None:
    """[(fields start, record end)] of the `count` records of the section data[lo, hi), or None when the batch fails"""
    out, pos = [], lo
    for _ in range(count):
        try:
            n, pos = read_varint(data, pos, hi)
        except Corrupt:
            return None
        if n < 0 or n > hi - pos:
            return None
        out.append((pos, pos + n))
        pos += n
    return out if pos == hi else None


def zstd_raw_frame(z: bytes) -> bytes | None:
    """the content of a zstd frame of raw and RLE blocks, None when it is not a well-formed one; a compressed block is not
    decoded here"""
    if len(z) < 6 or z[:4] != zc.MAGIC:
        return None
    fhd = z[4]
    ss, fid, csum = (fhd >> 5) & 1, fhd >> 6, (fhd >> 2) & 1
    if fhd & 0x0B:                                             # the reserved bit, a dictionary id
        return None
    pos = 5 + (not ss)
    fcs_len = [1 if ss else 0, 2, 4, 8][fid]
    fcs = int.from_bytes(z[pos:pos + fcs_len], "little") + (256 if fid == 1 else 0) if fcs_len else None
    pos += fcs_len
    out = bytearray()
    while True:
        if pos + 3 > len(z):
            return None
        bh = int.from_bytes(z[pos:pos + 3], "little")
        btype, size, last = (bh >> 1) & 3, bh >> 3, bh & 1
        pos += 3
        if btype == 2:
            raise NotImplementedError("compressed zstd blocks are not decoded by this reference")
        if btype == 3 or size > 128 << 10 or pos + (1 if btype else size) > len(z):
            return None
        out += z[pos:pos + size] if btype == 0 else z[pos:pos + 1] * size
        pos += 1 if btype else size
        if last:
            break
    if csum:
        if pos + 4 > len(z) or struct.unpack_from("<I", z, pos)[0] != zc.xxh64(bytes(out)) & 0xFFFFFFFF:
            return None
        pos += 4
    if pos != len(z) or (fcs is not None and fcs != len(out)):
        return None
    return bytes(out)


def _lz4(z: bytes) -> bytes | None:
    try:
        return lz.decompress_frame(z)
    except ValueError:
        return None


DECODERS = {1: lambda z: gz.zlib_ref(z, 31), 2: ks.decompress_section, 3: _lz4, 4: zstd_raw_frame}


def parse_fetch(buf: bytes, max_records: int | None = None) -> list[Record]:
    """every record the fetch counts, in order, with its verdict and spans"""
    buf = bytes(buf)
    out: list[Record] = []
    for nb, (s, e) in enumerate(kt.batches(buf)):
        count = struct.unpack_from(">I", buf, s + 57)[0]
        if max_records is not None and (len(out) + count > max_records or nb >= max_records):
            raise RecordsLimit(f"more records than max_records ({max_records})")
        attrs, codec = buf[s + 22], buf[s + 22] & 7
        if attrs & kt.CONTROL:
            raise ValueError("control batches are outside this reference")
        data, lo, hi, decoded, spans = buf, s + kb.HEADER_LEN, e, False, None
        if buf[s + 16] == 2 and codec <= 4 and kb.crc32c(buf[s + kb.CRC_FROM:e]) == struct.unpack_from(">I", buf, s + 17)[0]:
            if codec:
                data = DECODERS[codec](buf[lo:hi])
                lo, hi, decoded = 0, 0 if data is None else len(data), True
            if data is not None:
                spans = split(data, lo, hi, count)
        if spans is None:
            out += [Record(1, buf)] * count
        else:
            out += [record(data, a, b, decoded) for a, b in spans]
    return out
