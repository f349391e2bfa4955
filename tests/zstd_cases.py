"""TEST INFRASTRUCTURE ONLY: the zstd frames the decoder is held against libzstd on.

  SETTINGS, DATA_SIZES, data()   the settings matrix and the inputs (tool envelopes, random bytes, one byte, text)
  frame(), block(), seq_block()  a small writer: frames of raw and RLE blocks, and compressed blocks with raw or RLE
                                 literals and RLE sequence modes (whose bitstream holds only extra bits, no FSE coding)
  parse()                        where the fields of a frame lie (headers, literals sections, sequences headers)
  malformed()                    {class: frame} of every malformed class; each is refused by libzstd
  mutations()                    seeded bit flips and truncations of ~20 frames

The classes that need a Huffman or FSE description come from editing libzstd output at the positions parse() finds."""
import random
import struct

import zstd_ref as zr

MAGIC = zr.MAGIC
SETTINGS = {
    "level-5": dict(level=-5), "level1": dict(level=1), "level3": dict(level=3), "level19": dict(level=19),
    "no_content_size": dict(level=3, content_size=False), "checksum": dict(level=3, checksum=True),
    "window_log10": dict(level=3, window_log=10), "ldm": dict(level=3, ldm=True),
    "target_cblock": dict(level=3, target_cblock=1340),
}
DATA_SIZES = (0, 1, 100, (64 << 10) - 1, 64 << 10, (64 << 10) + 1, (128 << 10) - 1, 128 << 10, (128 << 10) + 1, 1 << 20, 4 << 20)
KINDS = ("records", "random", "one_byte", "text")

# ---- XXH64 (seed 0), for the writer's checksums --------------------------------------------------------------------
_P1, _P2, _P3, _P4, _P5 = 0x9E3779B185EBCA87, 0xC2B2AE3D27D4EB4F, 0x165667B19E3779F9, 0x85EBCA77C2B2AE63, 0x27D4EB2F165667C5
_M = (1 << 64) - 1


def _rotl(x, r):
    return ((x << r) | (x >> (64 - r))) & _M


def _round(acc, v):
    return (_rotl((acc + v * _P2) & _M, 31) * _P1) & _M


def xxh64(b: bytes) -> int:
    n, i = len(b), 0
    if n >= 32:
        v = [(_P1 + _P2) & _M, _P2, 0, (-_P1) & _M]
        while i + 32 <= n:
            for k in range(4):
                v[k] = _round(v[k], struct.unpack_from("<Q", b, i + 8 * k)[0])
            i += 32
        h = (_rotl(v[0], 1) + _rotl(v[1], 7) + _rotl(v[2], 12) + _rotl(v[3], 18)) & _M
        for k in range(4):
            h = ((h ^ _round(0, v[k])) * _P1 + _P4) & _M
    else:
        h = _P5
    h = (h + n) & _M
    while i + 8 <= n:
        h = (_rotl(h ^ _round(0, struct.unpack_from("<Q", b, i)[0]), 27) * _P1 + _P4) & _M
        i += 8
    if i + 4 <= n:
        h = (_rotl(h ^ (struct.unpack_from("<I", b, i)[0] * _P1 & _M), 23) * _P2 + _P3) & _M
        i += 4
    while i < n:
        h = (_rotl(h ^ (b[i] * _P5 & _M), 11) * _P1) & _M
        i += 1
    h ^= h >> 33
    h = h * _P2 & _M
    h ^= h >> 29
    h = h * _P3 & _M
    return h ^ (h >> 32)


# ---- inputs ------------------------------------------------------------------------------------------------------------
def data(kind: str, n: int, seed: int = 0) -> bytes:
    import numpy as np
    rng = np.random.default_rng(seed + n)
    if kind == "records":
        from calfkit import synth
        recs = b"".join(synth.tool_events(200, seed=seed + 7))
        return (recs * (n // len(recs) + 1))[:n]
    if kind == "random":
        return rng.integers(0, 256, n, dtype=np.uint8).tobytes()
    if kind == "one_byte":
        return b"z" * n
    words = [b"the", b"tool", b"call", b"weather", b"sunny", b"in", b"paris", b"agent", b"reply", b"json"]
    out = bytearray()
    while len(out) < n:
        out += words[int(rng.integers(0, len(words)))] + (b" " if rng.integers(0, 8) else b"\n")
    return bytes(out[:n])


# ---- the writer --------------------------------------------------------------------------------------------------------
def header(fcs=None, single_segment=False, window_log=17, checksum=False, dict_id=None, reserved=False,
           window_byte=None) -> bytes:
    """a frame header: Frame_Content_Size `fcs` (None: absent), Single_Segment, a window descriptor of 2^window_log, the
    checksum flag, a Dictionary_ID (4 bytes) and the reserved bit when asked"""
    if single_segment:
        assert fcs is not None
    if fcs is None:
        fid, field = 0, b""
    elif single_segment and fcs < 256:
        fid, field = 0, bytes([fcs])
    elif 256 <= fcs < 65536 + 256:
        fid, field = 1, struct.pack("<H", fcs - 256)
    elif fcs < 1 << 32:
        fid, field = 2, struct.pack("<I", fcs)
    else:
        fid, field = 3, struct.pack("<Q", fcs)
    fhd = (fid << 6) | (32 if single_segment else 0) | (4 if checksum else 0) | (8 if reserved else 0) | (3 if dict_id is not None else 0)
    out = MAGIC + bytes([fhd])
    if not single_segment:
        out += bytes([window_byte if window_byte is not None else (window_log - 10) << 3])
    if dict_id is not None:
        out += struct.pack("<I", dict_id)
    return out + field


def block(last: bool, btype: int, payload: bytes, size: int | None = None) -> bytes:
    """a block: type 0 raw, 1 RLE (payload = its byte, size = its length), 2 compressed, 3 reserved"""
    if size is None:
        size = len(payload)
    return ((size << 3) | (btype << 1) | int(last)).to_bytes(3, "little") + payload


def frame(blocks: list[bytes], content: bytes | None = None, checksum: bool = False, **hk) -> bytes:
    """header + blocks (+ the XXH64 checksum of `content`)"""
    z = header(checksum=checksum, **hk) + b"".join(blocks)
    if checksum:
        z += struct.pack("<I", xxh64(content) & 0xFFFFFFFF)
    return z


def lit_header(btype: int, size: int) -> bytes:
    """a raw (0) or RLE (1) literals section header of `size`"""
    if size < 32:
        return bytes([(size << 3) | btype])
    if size < 4096:
        return ((size << 4) | (1 << 2) | btype).to_bytes(2, "little")
    return ((size << 4) | (3 << 2) | btype).to_bytes(3, "little")


class _Bits:
    """a forward bit writer; the decoder reads it back to front"""
    def __init__(self):
        self.v, self.n = 0, 0

    def add(self, val: int, nb: int):
        assert 0 <= val < (1 << nb) or nb == 0
        self.v |= val << self.n
        self.n += nb

    def close(self) -> bytes:
        self.add(1, 1)
        return self.v.to_bytes((self.n + 7) // 8, "little")


LL_BITS = [0] * 16 + [1, 1, 1, 1, 2, 2, 3, 3, 4, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16]
LL_BASE = list(range(16)) + [16, 18, 20, 22, 24, 28, 32, 40, 48, 64, 0x80, 0x100, 0x200, 0x400, 0x800, 0x1000, 0x2000,
                             0x4000, 0x8000, 0x10000]
ML_BITS = [0] * 32 + [1, 1, 1, 1, 2, 2, 3, 3, 4, 4, 5, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16]
ML_BASE = list(range(3, 35)) + [35, 37, 39, 41, 43, 47, 51, 59, 67, 83, 99, 0x83, 0x103, 0x203, 0x403, 0x803, 0x1003,
                                0x2003, 0x4003, 0x8003, 0x10003]


def seq_block(literals: bytes, seqs, ll_code: int, of_code: int, ml_code: int, rle_lits: bool = False,
              modes: int | None = None, extra_bits: int = 0) -> bytes:
    """a compressed block's payload: raw (or RLE) literals, then len(seqs) sequences in RLE mode for all three codes.
    seqs = [(literal length, Offset_Value, match length)]; each must fit its code.  `modes` overrides the modes byte;
    `extra_bits` adds unread bits to the bitstream"""
    lits = lit_header(1, len(literals)) + literals[:1] if rle_lits else lit_header(0, len(literals)) + literals
    n = len(seqs)
    if n == 0:
        return lits + b"\0"
    nb = bytes([n]) if n < 128 else bytes([(n >> 8) + 128, n & 255]) if n < 0x7F00 else b"\xff" + struct.pack("<H", n - 0x7F00)
    md = (1 << 6) | (1 << 4) | (1 << 2) if modes is None else modes
    bits = _Bits()
    bits.add(0, extra_bits)
    for ll, ofv, ml in reversed(seqs):
        bits.add(ll - LL_BASE[ll_code], LL_BITS[ll_code])
        bits.add(ml - ML_BASE[ml_code], ML_BITS[ml_code])
        bits.add(ofv - (1 << of_code), of_code)
    return lits + nb + bytes([md, ll_code, of_code, ml_code]) + bits.close()


# ---- a parse of libzstd frames, to edit them -------------------------------------------------------------------------
def parse(z: bytes) -> dict:
    """{"hdr": header bytes, "blocks": [dict(pos, type, size, last, and for compressed ones: lit_type, lit_streams, lh,
    L, C, huf (the Huffman description's offset or None), huf_size, seq (the sequences header's offset), nseq, modes_pos)]}"""
    fhd = z[4]
    ss, did, fid = (fhd >> 5) & 1, fhd & 3, fhd >> 6
    pos = 5 + (not ss) + [0, 1, 2, 4][did] + [0, 2, 4, 8][fid] + (1 if ss and not fid else 0)
    out = {"hdr": pos, "blocks": []}
    while pos + 3 <= len(z):
        bh = int.from_bytes(z[pos:pos + 3], "little")
        b = dict(pos=pos, type=(bh >> 1) & 3, size=bh >> 3, last=bh & 1)
        p = pos + 3
        if b["type"] == 2:
            s0 = z[p]
            lt, sf = s0 & 3, (s0 >> 2) & 3
            b["lit_type"] = lt
            if lt < 2:
                lh = 1 if sf in (0, 2) else 2 if sf == 1 else 3
                L = (int.from_bytes(z[p:p + lh], "little") >> (3 if lh == 1 else 4))
                C = L if lt == 0 else 1
                b.update(lh=lh, L=L, C=C, huf=None, huf_size=0, lit_streams=1)
            else:
                lhc = int.from_bytes(z[p:p + 5], "little")
                if sf <= 1:
                    lh, L, C = 3, (lhc >> 4) & 0x3FF, (lhc >> 14) & 0x3FF
                elif sf == 2:
                    lh, L, C = 4, (lhc >> 4) & 0x3FFF, (lhc >> 18) & 0x3FFF
                else:
                    lh, L, C = 5, (lhc >> 4) & 0x3FFFF, (lhc >> 22) & 0x3FFFF
                hs = 0
                if lt == 2:
                    hb = z[p + lh]
                    hs = 1 + hb if hb < 128 else 1 + (hb - 127 + 1) // 2
                b.update(lh=lh, L=L, C=C, huf=p + lh if lt == 2 else None, huf_size=hs, lit_streams=1 if sf == 0 else 4)
            q = p + b["lh"] + b["C"]
            b["seq"] = q
            n0 = z[q]
            k = 1 if n0 < 128 else 3 if n0 == 255 else 2
            b["nseq"] = n0 if n0 < 128 else (z[q + 1] + 0x7F00 + (z[q + 2] << 8)) if n0 == 255 else ((n0 - 128) << 8) + z[q + 1]
            b["modes_pos"] = q + k if n0 else None
        out["blocks"].append(b)
        pos = p + (1 if b["type"] == 1 else b["size"])
        if b["last"]:
            break
    return out


def _edit(z: bytes, pos: int, val: int) -> bytes:
    return z[:pos] + bytes([val]) + z[pos + 1:]


def _find(pred):
    """(frame, block) of the first libzstd frame of _libzstd_sources() with a block for which pred(frame, block,
    earlier blocks) holds"""
    for kw, d in _libzstd_sources():
        z = zr.compress(d, **kw)
        bl = parse(z)["blocks"]
        for i, b in enumerate(bl):
            if pred(z, b, bl[:i]):
                return z, b
    raise AssertionError("no libzstd frame with such a block")


def _libzstd_sources():
    txt = data("text", 60000, seed=3)
    rec = data("records", 60000, seed=4)
    return [(dict(level=lv, content_size=False), d) for lv in (19, 3, 1) for d in (txt, rec)]


def malformed() -> dict[str, bytes]:
    """{class: frame}: every malformed class, each refused by libzstd (asserted by the tests)"""
    content = b"hello zstd " * 20
    good_raw = frame([block(True, 0, content)], fcs=len(content), window_log=17, checksum=True, content=content)
    out = {}
    # frame
    out["wrong magic"] = b"\x28\xb5\x2f\xfe" + good_raw[4:]
    out["skippable frame"] = b"\x50\x2a\x4d\x18" + struct.pack("<I", 4) + b"skip" + good_raw
    out["reserved descriptor bit"] = frame([block(True, 0, content)], window_log=17, reserved=True)
    out["Dictionary_ID"] = frame([block(True, 0, content)], window_log=17, dict_id=7)
    out["windowLog 28"] = frame([block(True, 0, content)], window_log=28)
    out["window past 2^27 + 1"] = frame([block(True, 0, content)], window_byte=(17 << 3) | 1)
    out["Frame_Content_Size one short"] = frame([block(True, 0, content)], fcs=len(content) - 1, window_log=17)
    out["Frame_Content_Size one over"] = frame([block(True, 0, content)], fcs=len(content) + 1, window_log=17)
    out["single segment content size one over"] = frame([block(True, 0, content)], fcs=len(content) + 1, single_segment=True)
    # blocks
    out["block type 3"] = frame([block(True, 3, content)], window_log=17)
    big = b"r" * ((128 << 10) + 1)
    out["raw block past 128 KiB"] = frame([block(True, 0, big)], window_log=20)
    out["RLE block past 128 KiB"] = frame([block(True, 1, b"r", (128 << 10) + 1)], window_log=20)
    out["raw block past the window"] = frame([block(True, 0, b"w" * 1025)], window_log=10)
    out["RLE block past the content size"] = frame([block(True, 1, b"w", 300)], fcs=299, single_segment=True)
    out["no last block"] = frame([block(False, 0, content)], window_log=17)
    out["a trailing byte"] = good_raw + b"\0"
    out["a second frame"] = good_raw + good_raw
    out["wrong checksum"] = good_raw[:-1] + bytes([good_raw[-1] ^ 1])
    out["compressed block of one byte"] = frame([block(True, 2, b"\0")], window_log=17)
    # literals
    lits = b"abcdefgh" * 8
    out["raw literals past the block"] = frame([block(True, 2, lit_header(0, 200) + lits + b"\0")], window_log=17)
    out["RLE literals past the block maximum"] = frame([block(True, 2, lit_header(1, 2000) + b"x\0")], window_log=10)
    huf = lambda z, b, before: b["type"] == 2 and b["lit_type"] == 2
    z, b = _find(huf)
    out["Huffman weights above 12"] = z[:b["huf"]] + bytes([128 + 1, 0xFF]) + z[b["huf"] + 2:]
    out["Huffman weights not a power of 2"] = z[:b["huf"]] + bytes([128 + 3, 0x12, 0x20]) + z[b["huf"] + 3:]
    first4 = lambda z, b, before: huf(z, b, before) and b["lit_streams"] == 4 and not any(huf(z, e, ()) for e in before)
    z, b = _find(first4)
    j = b["huf"] + b["huf_size"]
    out["jump table past the literals"] = z[:j] + b"\xff\xff" + z[j + 2:]
    p = b["pos"] + 3
    lhc = int.from_bytes(z[p:p + b["lh"]], "little")
    shorter = (lhc - (1 << 4)).to_bytes(b["lh"], "little")
    out["Huffman streams one literal short"] = z[:p] + shorter + z[p + b["lh"]:]
    out["Treeless with no earlier table"] = _edit(z, p, (z[p] & ~3) | 3)
    # sequences
    good = seq_block(lits, [(8, 8, 4)], 8, 3, 1)
    out["Repeat with no earlier table"] = frame([block(True, 2, seq_block(lits, [(8, 8, 4)], 8, 3, 1, modes=(3 << 6) | 0x14))], window_log=17)
    z, b = _find(lambda z, b, before: b["type"] == 2 and b["modes_pos"] and (z[b["modes_pos"]] >> 6) == 2)
    m = b["modes_pos"] + 1
    out["FSE accuracy log too high"] = _edit(z, m, (z[m] & 0xF0) | 15)
    out["normalized count under-fills"] = _edit(z, m, (z[m] & 0xF0) | ((z[m] & 15) + 1))
    out["normalized count over-fills"] = _edit(z, m, (z[m] & 0xF0) | ((z[m] & 15) - 1)) if z[m] & 15 else _edit(z, m, (z[m] & 0xF0) | 4)
    out["RLE literal length code 36"] = frame([block(True, 2, good[:-5] + bytes([0x54, 36, 3, 1]) + good[-1:])], window_log=17)
    out["RLE offset code 32"] = frame([block(True, 2, good[:-5] + bytes([0x54, 8, 32, 1]) + good[-1:])], window_log=17)
    out["RLE match length code 53"] = frame([block(True, 2, good[:-5] + bytes([0x54, 8, 3, 53]) + good[-1:])], window_log=17)
    out["offset before the frame's output"] = frame([block(True, 2, seq_block(lits, [(8, 12, 4)], 8, 3, 1))], window_log=17)
    out["match past the block maximum"] = frame([block(True, 2, seq_block(b"ab" * 8, [(16, 5, 2000)], 16, 2, 46))], window_log=10)
    out["more literals consumed than decoded"] = frame([block(True, 2, seq_block(lits[:10], [(12, 8, 4)], 12, 3, 1))], window_log=17)
    out["bitstream not consumed exactly"] = frame([block(True, 2, seq_block(lits, [(8, 8, 4)], 8, 3, 1, extra_bits=9))], window_log=17)
    out["sequences section after no sequences"] = frame([block(True, 2, lit_header(0, 8) + lits[:8] + b"\0\0")], window_log=17)
    # truncation at every header boundary of a frame with every kind of block
    ref = truncation_source()
    for cut in sorted(boundaries(ref)):
        if 0 < cut < len(ref):
            out[f"truncated at {cut}"] = ref[:cut]
    return out


def truncation_source() -> bytes:
    """a checksummed libzstd frame of several blocks, with Huffman literals and FSE sequence tables"""
    d = data("text", 300000, seed=5)
    return zr.compress(d, level=3, checksum=True)


def boundaries(z: bytes) -> set[int]:
    """every header boundary of a frame: inside and after the frame header, each block header, literals header,
    Huffman description and sequences header, and the checksum"""
    p = parse(z)
    cuts = set(range(1, p["hdr"] + 1))
    for b in p["blocks"]:
        cuts.update({b["pos"] + 1, b["pos"] + 2, b["pos"] + 3})
        if b["type"] == 2:
            q = b["pos"] + 3
            cuts.update({q + 1, q + b["lh"]})
            if b["huf"] is not None:
                cuts.update({b["huf"] + 1, b["huf"] + b["huf_size"]})
            cuts.update({b["seq"], b["seq"] + 1})
            if b["modes_pos"]:
                cuts.update({b["modes_pos"], b["modes_pos"] + 1})
    cuts.update({len(z) - 4, len(z) - 1})
    return cuts


def mutation_sources() -> list[bytes]:
    """~20 frames of every shape the mutations start from"""
    srcs = []
    for i, (kind, n) in enumerate([("records", 3000), ("text", 5000), ("random", 600), ("records", 40000), ("text", 70000)]):
        d = data(kind, n, seed=40 + i)
        srcs += [zr.compress(d, level=3, checksum=True), zr.compress(d, level=19), zr.compress(d, level=-5, content_size=False),
                 zr.stream(d, piece=1500, flush=True, level=1)]
    return srcs


def mutations(seed: int = 7, flips: int = 5000, cuts: int = 500) -> list[tuple[bytes, bytes, list[int]]]:
    """[(mutated frame, its source, the flipped byte positions)]: `flips` frames with one or two bit flips, then `cuts`
    truncations (no positions)"""
    rng = random.Random(seed)
    srcs = mutation_sources()
    out = []
    for _ in range(flips):
        src = rng.choice(srcs)
        z, at = bytearray(src), []
        for _ in range(rng.randint(1, 2)):
            i = rng.randrange(len(z))
            z[i] ^= 1 << rng.randrange(8)
            at.append(i)
        out.append((bytes(z), src, at))
    for _ in range(cuts):
        z = rng.choice(srcs)
        out.append((z[:rng.randrange(1, len(z))], z, []))
    return out


def in_4stream_literals(src: bytes, at: list[int]) -> bool:
    """a position of `at` lies in a 4-stream Huffman literals section (header, tree description, jump table, streams) of
    the frame src"""
    spans = [(b["pos"] + 3, b["pos"] + 3 + b["lh"] + b["C"])
             for b in parse(src)["blocks"] if b["type"] == 2 and b["lit_type"] >= 2 and b["lit_streams"] == 4]
    return any(a <= i < e for a, e in spans for i in at)
