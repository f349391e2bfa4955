"""TEST INFRASTRUCTURE ONLY — CPU restatement of the LZ4 frame and block formats, of XXH32, and of Kafka's LZ4-compressed
RecordBatch v2 (attributes 3), against which the device's compressed frames are checked.

Restated from the published specifications (lz4 `doc/lz4_Frame_format.md` and `doc/lz4_Block_format.md`, XXH32 from the
xxHash specification); tests/golden/lz4_frames.json pins it to what liblz4 (LZ4F_compressFrame) writes, for every
frame flag and block size, and to XXH32 vectors (tests/test_lz4_oracle.py).

LZ4 frame:  magic 04 22 4D 18 | FLG | BD | [content size u64 LE] | [dict id u32 LE] | HC | blocks | 00 00 00 00 |
            [content checksum u32 LE]
  FLG: version (bits 7-6 = 01), independent blocks (5), block checksum (4), content size (3), content checksum (2),
       reserved (1) = 0, dict id (0).   BD: block max size id (bits 6-4: 4 = 64 KB, 5 = 256 KB, 6 = 1 MB, 7 = 4 MB).
  HC = (xxh32(FLG .. last descriptor byte, seed 0) >> 8) & 0xFF.
  block: size u32 LE (bit 31: stored raw) | data | [xxh32(data) u32 LE when block checksums are on].
LZ4 block: sequences of token (literal length << 4 | match length - 4), literal length bytes (when 15: 255 ... rest),
  literals, offset u16 LE (1 .. 65535), match length bytes.  The last sequence holds literals only; the last match starts
  at least 12 bytes before the end of the block and ends at least 5 bytes before it.
Kafka: attributes & 7 = 3 (LZ4); everything after recordsCount, [61, end) of the uncompressed batch, is one LZ4 frame; the
  CRC32C covers [21, end) of the compressed batch and batchLength is the compressed length - 12.
"""
from __future__ import annotations

import struct

from oracle import kafka_batch as kb

MAGIC = 0x184D2204
BLOCK_MAX = {4: 64 << 10, 5: 256 << 10, 6: 1 << 20, 7: 4 << 20}
CODEC_LZ4 = 3

_P1, _P2, _P3, _P4, _P5 = 2654435761, 2246822519, 3266489917, 668265263, 374761393
_M = 0xFFFFFFFF


def _rotl(x: int, r: int) -> int:
    return ((x << r) | (x >> (32 - r))) & _M


def xxh32(data: bytes, seed: int = 0) -> int:
    data = bytes(data)
    n, p = len(data), 0
    if n >= 16:
        v = [(seed + _P1 + _P2) & _M, (seed + _P2) & _M, seed & _M, (seed - _P1) & _M]
        stripes = n // 16
        for i, w in enumerate(struct.iter_unpack("<I", data[:16 * stripes])):
            k = i & 3
            v[k] = (_rotl((v[k] + w[0] * _P2) & _M, 13) * _P1) & _M
        p = 16 * stripes
        h = (_rotl(v[0], 1) + _rotl(v[1], 7) + _rotl(v[2], 12) + _rotl(v[3], 18)) & _M
    else:
        h = (seed + _P5) & _M
    h = (h + n) & _M
    while p + 4 <= n:
        h = (_rotl((h + struct.unpack_from("<I", data, p)[0] * _P3) & _M, 17) * _P4) & _M
        p += 4
    while p < n:
        h = (_rotl((h + data[p] * _P5) & _M, 11) * _P1) & _M
        p += 1
    h ^= h >> 15
    h = (h * _P2) & _M
    h ^= h >> 13
    h = (h * _P3) & _M
    h ^= h >> 16
    return h


def _length(src: bytes, ip: int, base: int) -> tuple[int, int]:
    n = base
    if base == 15:
        while True:
            if ip >= len(src):
                raise ValueError("block truncated inside a length")
            b = src[ip]
            ip += 1
            n += b
            if b != 255:
                break
    return n, ip


def decompress_block(src: bytes, out: bytearray, max_size: int, history: int = 0) -> None:
    """append the decoded block to `out`; matches may reach `history` bytes before the block (linked blocks, dictionary)"""
    start, ip, end = len(out), 0, len(src)
    last_match = None                                            # (start, end) of the last match, relative to the block
    while True:
        if ip >= end:
            raise ValueError("block does not end with a literals-only sequence")
        token = src[ip]
        ip += 1
        ll, ip = _length(src, ip, token >> 4)
        if ip + ll > end:
            raise ValueError("literals run past the block")
        out += src[ip:ip + ll]
        ip += ll
        if ip == end:
            break                                                # the last sequence: literals only
        if ip + 2 > end:
            raise ValueError("block truncated inside an offset")
        off = src[ip] | src[ip + 1] << 8
        ip += 2
        if off == 0:
            raise ValueError("offset 0")
        ml, ip = _length(src, ip, token & 15)
        ml += 4
        pos = len(out)
        if off > pos - start + history:
            raise ValueError("offset reaches before the block")
        m0 = pos - off
        if off >= ml:
            out += out[m0:m0 + ml]
        else:                                                    # overlapping copy: the pattern repeats
            pat = bytes(out[m0:pos])
            out += (pat * (ml // off + 1))[:ml]
        last_match = (pos - start, len(out) - start)
        if len(out) - start > max_size:
            raise ValueError("block larger than the block maximum")
    n = len(out) - start
    if n > max_size:
        raise ValueError("block larger than the block maximum")
    if last_match is not None:
        if last_match[0] > n - 12:
            raise ValueError("the last match starts less than 12 bytes before the end of the block")
        if last_match[1] > n - 5:
            raise ValueError("a match runs into the last 5 bytes of the block")


def decompress_frame(buf: bytes, dictionary: bytes = b"") -> bytes:
    """the content of one LZ4 frame that spans `buf` exactly; every FLG / BD combination, HC, block and content checksums
    checked when present"""
    buf = bytes(buf)
    if len(buf) < 7 or struct.unpack_from("<I", buf, 0)[0] != MAGIC:
        raise ValueError("not an LZ4 frame")
    flg, bd = buf[4], buf[5]
    if flg >> 6 != 1 or flg & 2 or bd & 0x8F:
        raise ValueError(f"bad frame descriptor FLG {flg:#04x} BD {bd:#04x}")
    indep, bsum, csize, csum, dictf = flg & 0x20, flg & 0x10, flg & 8, flg & 4, flg & 1
    bid = (bd >> 4) & 7
    if bid not in BLOCK_MAX:
        raise ValueError(f"block maximum id {bid}")
    pos = 6
    content_size = None
    if csize:
        content_size = struct.unpack_from("<Q", buf, pos)[0]
        pos += 8
    if dictf:
        pos += 4
    if pos >= len(buf):
        raise ValueError("frame truncated inside the descriptor")
    if buf[pos] != (xxh32(buf[4:pos]) >> 8) & 0xFF:
        raise ValueError("header checksum mismatch")
    pos += 1
    out = bytearray(dictionary)
    base = len(out)
    while True:
        if pos + 4 > len(buf):
            raise ValueError("frame truncated: no end mark")
        word = struct.unpack_from("<I", buf, pos)[0]
        pos += 4
        if word == 0:
            break
        size, stored = word & 0x7FFFFFFF, word >> 31
        if size > BLOCK_MAX[bid] or pos + size > len(buf):
            raise ValueError("block size out of range")
        data = buf[pos:pos + size]
        pos += size
        if bsum:
            if pos + 4 > len(buf) or struct.unpack_from("<I", buf, pos)[0] != xxh32(data):
                raise ValueError("block checksum mismatch")
            pos += 4
        if stored:
            out += data
        else:
            decompress_block(data, out, BLOCK_MAX[bid], 0 if indep else min(len(out), 65535))
    content = bytes(out[base:])
    if csum:
        if pos + 4 > len(buf) or struct.unpack_from("<I", buf, pos)[0] != xxh32(content):
            raise ValueError("content checksum mismatch")
        pos += 4
    if pos != len(buf):
        raise ValueError("bytes after the frame")
    if content_size is not None and content_size != len(content):
        raise ValueError("content size mismatch")
    return content


def decompress_batch(frame: bytes) -> bytes:
    """the uncompressed RecordBatch v2 equivalent of an LZ4 batch: the records section decompressed, attributes without the
    codec, batchLength and CRC32C recomputed.  The compressed batch's own length and CRC are checked first"""
    frame = bytes(frame)
    if len(frame) < kb.HEADER_LEN or frame[16] != 2:
        raise ValueError("not a v2 batch")
    if struct.unpack_from(">i", frame, 8)[0] != len(frame) - 12:
        raise ValueError("batchLength mismatch")
    if kb.crc32c(frame[kb.CRC_FROM:]) != struct.unpack_from(">I", frame, 17)[0]:
        raise ValueError("CRC32C mismatch")
    attrs = struct.unpack_from(">h", frame, 21)[0]
    if attrs & 7 != CODEC_LZ4:
        raise ValueError(f"codec {attrs & 7} is not LZ4")
    records = decompress_frame(frame[kb.HEADER_LEN:])
    covered = struct.pack(">h", attrs & ~7) + frame[23:kb.HEADER_LEN] + records
    return frame[:8] + struct.pack(">i", len(covered) + 9) + frame[12:17] + struct.pack(">I", kb.crc32c(covered)) + covered
