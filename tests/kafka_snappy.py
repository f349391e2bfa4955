"""TEST INFRASTRUCTURE ONLY — Kafka's snappy records sections (attributes codec 2) restated in plain Python: the raw-block
decoder, the section walk (snappy-java framing or one raw block), a writer of both, and malformed blocks and framings.

  raw block      varint32 decoded length (at most 5 bytes, a 5th byte below 16), then elements to the end of the input:
                   literal  tag 00: length (tag >> 2) + 1, or for tag >> 2 >= 60 a little-endian length of (tag >> 2) - 59
                            bytes, plus 1 (32-bit, as snappy computes it: 0xffffffff + 1 is an empty literal)
                   copy-1   tag 01: length 4 + ((tag >> 2) & 7), offset (tag >> 5) << 8 | next byte
                   copy-2   tag 10: length (tag >> 2) + 1, offset LE16
                   copy-4   tag 11: length (tag >> 2) + 1, offset LE32
                 refused on an element cut off, offset 0 or before the block's start, output past or short of the length
  framed         (snappy-java, "xerial") a section longer than 16 bytes starting with 82 'SNAPPY' 00: two big-endian
                 version words, stepped over; then chunks, a big-endian u32 length c (1 <= c <= bytes left) and one raw
                 block of c bytes each, tiling the rest of the section exactly
  the walk       also refuses a block that declares more than RATIO times its own size (snappy cannot produce it)

The writer takes hand-written element lists, so it writes what Google's compressor never does (copy-4, wide literal
lengths).  pyarrow knows only raw blocks: every malformed block here is asserted refused by it (tests/snappy_ref.py); the
malformed framings hold valid blocks, and the rule above decides them.
"""
from __future__ import annotations

import struct

MAGIC = b"\x82SNAPPY\x00"
FRAME_HDR = 16
RATIO = 22


# ---- decoding ---------------------------------------------------------------------------------------------------------
def varint(z: bytes):
    """(decoded length, first element) of the raw block z, or None"""
    v = 0
    for k in range(5):
        if k >= len(z) or (k == 4 and z[k] >= 16):
            return None
        v |= (z[k] & 0x7F) << (7 * k)
        if z[k] < 0x80:
            return v, k + 1
    return None


def decompress_block(z: bytes):
    """the raw block z decoded, or None when snappy refuses it"""
    h = varint(z)
    if h is None:
        return None
    n, ip = h
    out = bytearray()
    while ip < len(z):
        tag = z[ip]
        ip += 1
        kind = tag & 3
        if kind == 0:
            ln = (tag >> 2) + 1
            if ln > 60:
                k = ln - 60
                if ip + k > len(z):
                    return None
                ln = (int.from_bytes(z[ip:ip + k], "little") + 1) & 0xFFFFFFFF
                ip += k
            if ip + ln > len(z) or len(out) + ln > n:
                return None
            out += z[ip:ip + ln]
            ip += ln
            continue
        if kind == 1:
            if ip >= len(z):
                return None
            ln, off = 4 + ((tag >> 2) & 7), ((tag >> 5) << 8) | z[ip]
            ip += 1
        else:
            w = 2 if kind == 2 else 4
            if ip + w > len(z):
                return None
            ln, off = (tag >> 2) + 1, int.from_bytes(z[ip:ip + w], "little")
            ip += w
        if off == 0 or off > len(out) or len(out) + ln > n:
            return None
        for _ in range(ln):
            out.append(out[-off])
    return bytes(out) if len(out) == n else None


def framed(sec: bytes) -> bool:
    return len(sec) > FRAME_HDR and sec[:8] == MAGIC


def walk(sec: bytes):
    """[(input offset, input length, declared length)] of the section's raw blocks, or None when it cannot be walked"""
    def blk(off, ln):
        h = varint(sec[off:off + ln])
        return None if h is None or h[0] > RATIO * ln else (off, ln, h[0])
    if not framed(sec):
        b = blk(0, len(sec))
        return None if b is None else [b]
    out, pos = [], FRAME_HDR
    while pos < len(sec):
        if len(sec) - pos < 4:
            return None
        c = struct.unpack(">I", sec[pos:pos + 4])[0]
        pos += 4
        if c == 0 or c > len(sec) - pos:
            return None
        b = blk(pos, c)
        if b is None:
            return None
        out.append(b)
        pos += c
    return out


def decompress_section(sec: bytes):
    """a snappy batch's records section decoded, or None"""
    w = walk(sec)
    if w is None:
        return None
    out = bytearray()
    for off, ln, _d in w:
        d = decompress_block(sec[off:off + ln])
        if d is None:
            return None
        out += d
    return bytes(out)


def decompress_batch(batch: bytes) -> bytes:
    """a snappy batch as the same batch uncompressed (attributes codec 0, CRC32C recomputed)"""
    from oracle import kafka_batch as kb
    sec = decompress_section(batch[kb.HEADER_LEN:])
    assert sec is not None
    b = bytearray(batch[:kb.HEADER_LEN] + sec)
    struct.pack_into(">I", b, 8, len(b) - 12)
    b[22] &= ~7 & 0xFF
    struct.pack_into(">I", b, 17, kb.crc32c(bytes(b[kb.CRC_FROM:])))
    return bytes(b)


# ---- writing ----------------------------------------------------------------------------------------------------------
def put_varint(n: int) -> bytes:
    out = bytearray()
    while n >= 0x80:
        out.append((n & 0x7F) | 0x80)
        n >>= 7
    out.append(n)
    return bytes(out)


def lit(data: bytes, width: int | None = None) -> bytes:
    """a literal element; width: bytes of its length field (0: in the tag, 1-4: behind it), default the smallest"""
    n = len(data) - 1
    if width is None:
        width = 0 if n < 60 else (n.bit_length() + 7) // 8
    if width == 0:
        assert 0 <= n < 60
        return bytes([n << 2]) + data
    return bytes([(59 + width) << 2]) + n.to_bytes(width, "little") + data


def copy(off: int, ln: int, kind: int = 2) -> bytes:
    """a copy element of kind 1 (copy-1), 2 (copy-2) or 4 (copy-4)"""
    if kind == 1:
        assert 4 <= ln <= 11 and off < 2048
        return bytes([1 | ((ln - 4) << 2) | ((off >> 8) << 5), off & 0xFF])
    assert 1 <= ln <= 64
    return bytes([(2 if kind == 2 else 3) | ((ln - 1) << 2)]) + off.to_bytes(kind, "little")


def block(elements: list[bytes], declared: int | None = None, content: bytes | None = None) -> bytes:
    """a raw block of the given elements; declared: its varint (default: len(content), which must then be given)"""
    return put_varint(len(content) if declared is None else declared) + b"".join(elements)


def frame(blocks: list[bytes], version: int = 1, compat: int = 1) -> bytes:
    """the snappy-java framing of the given raw blocks"""
    return MAGIC + struct.pack(">II", version, compat) + b"".join(struct.pack(">I", len(b)) + b for b in blocks)


def xerial(data: bytes, chunk: int = 32 << 10) -> bytes:
    """data as snappy-java's SnappyOutputStream writes it: chunks of `chunk` input bytes, each a raw block of Google snappy"""
    import snappy_ref as sr
    return frame([sr.compress(data[i:i + chunk]) for i in range(0, len(data), chunk)])


# ---- malformed --------------------------------------------------------------------------------------------------------
def malformed_blocks() -> dict[str, bytes]:
    """{class: raw block} that snappy refuses"""
    ab = lit(b"abcdefgh")
    return {
        "empty input": b"",
        "varint cut off": b"\x80",
        "varint cut off after 4 bytes": b"\x80\x80\x80\x80",
        "varint of 6 bytes": b"\x80\x80\x80\x80\x80\x00",
        "5th varint byte 16": b"\x80\x80\x80\x80\x10",
        "5th varint byte 0x8f": b"\x80\x80\x80\x80\x8f\x00",
        "varint ending the input, length 1": b"\x01",
        "literal cut off in its bytes": b"\x05" + lit(b"abcde")[:4],
        "literal cut off in a 1-byte length": b"\x41" + bytes([60 << 2]),
        "literal cut off in a 2-byte length": b"\x41" + bytes([61 << 2, 0x40]),
        "literal cut off in a 4-byte length": b"\x41" + bytes([63 << 2, 0x40, 0, 0]),
        "copy-1 cut off": b"\x0c" + ab + b"\x01",
        "copy-2 cut off": b"\x0c" + ab + b"\x0e\x08",
        "copy-4 cut off": b"\x0c" + ab + b"\x0f\x08\x00\x00",
        "tag cut off after a literal": block([ab], declared=8)[:-1],
        "copy-1 offset 0": block([ab, copy(0, 4, 1)], declared=12),
        "copy-2 offset 0": block([ab, copy(0, 4, 2)], declared=12),
        "copy-4 offset 0": block([ab, copy(0, 4, 4)], declared=12),
        "copy-1 offset one past the start": block([ab, copy(9, 4, 1)], declared=12),
        "copy-2 offset one past the start": block([ab, copy(9, 4, 2)], declared=12),
        "copy-4 offset one past the start": block([ab, copy(9, 4, 4)], declared=12),
        "copy at the start": block([copy(1, 4, 2)], declared=4),
        "output one short": block([ab, copy(8, 4, 2)], declared=13),
        "output one long": block([ab, copy(8, 4, 2)], declared=11),
        "literal one long": block([ab], declared=7),
        "nothing but a length": b"\x05",
    }


def malformed_framings() -> dict[str, bytes]:
    """{class: records section} framed by snappy-java and refused by the walk; their blocks are valid"""
    a = block([lit(b"hello snappy "), copy(13, 26, 2)], content=b"hello snappy " * 3)
    b = block([lit(b"xyz"), copy(3, 9, 1)], content=b"xyz" * 4)
    good = frame([a, b])
    return {
        "chunk length 0": frame([a]) + b"\x00\x00\x00\x00" + b,
        "chunk length past the end": good[:-1],
        "chunk length one past the end": frame([a]) + struct.pack(">I", len(b) + 1) + b,
        "1 byte left over": good + b"\x00",
        "3 bytes left over": good + b"\x00\x00\x01",
        "5 bytes left over": good + b"\x00\x00\x00\x02\x00",
        "second stream header mid-section": good + frame([a]),
        "header only (a raw block, which snappy refuses)": frame([]),
        "header and a cut-off length": frame([]) + b"\x00\x00\x00",
        "chunk declaring more than 22 times its size": frame([a, b"\xff\xff\x03" + lit(b"x")]),
    }


# ---- hand-written and mutated blocks ----------------------------------------------------------------------------------
def hand_blocks() -> dict[str, tuple[bytes, bytes]]:
    """{name: (raw block, its content)}: overlapping copies at offsets 1-8 of every copy kind, copy-4 (which Google's
    compressor never writes), literal lengths of every width, an empty literal of a wrapped 4-byte length, and the empty
    block"""
    out = {}
    seed = b"abcdefgh"
    for off in range(1, 9):
        for kind, ln in ((1, 11), (2, 64), (4, 40)):
            content = bytearray(seed[:off])
            for _ in range(ln):
                content.append(content[-off])
            out[f"copy-{kind} offset {off}"] = (block([lit(seed[:off]), copy(off, ln, kind)], content=bytes(content)), bytes(content))
    pad = bytes(range(256)) * 5
    for width in (1, 2, 3, 4):
        d = pad[:200 if width == 1 else 1000]
        out[f"literal of a {width}-byte length"] = (block([lit(d, width)], content=d), d)
    out["short literal of a 1-byte length"] = (block([lit(b"ab", 1)], content=b"ab"), b"ab")
    digits = b"0123456789" * 8
    content = digits[:74] + digits[:64] + b"12312" + b"!"
    out["copy-4 chain"] = (block([lit(b"0123456789"), copy(10, 64, 4), copy(74, 64, 4), copy(3, 5, 1), lit(b"!")], content=content), content)
    out["empty literal of length 0xffffffff + 1"] = (b"\x00" + bytes([63 << 2]) + b"\xff\xff\xff\xff", b"")
    out["empty block"] = (b"\x00", b"")
    out["5-byte varint of 0"] = (b"\x80\x80\x80\x80\x00", b"")
    out["5-byte varint of 3"] = (b"\x83\x80\x80\x80\x00" + lit(b"xyz"), b"xyz")
    return out


def mutations(srcs: list[bytes], seed: int = 9, flips: int = 3000, cuts: int = 300) -> list[bytes]:
    """`flips` blocks of srcs with one or two bit flips, then `cuts` truncations"""
    import random
    rng = random.Random(seed)
    out = []
    for _ in range(flips):
        z = bytearray(rng.choice(srcs))
        for _ in range(rng.randint(1, 2)):
            i = rng.randrange(len(z))
            z[i] ^= 1 << rng.randrange(8)
        out.append(bytes(z))
    for _ in range(cuts):
        z = rng.choice(srcs)
        out.append(z[:rng.randrange(0, len(z))])
    return out
