"""gzip members and raw deflate streams made here with the standard library's zlib, and by hand for the malformed classes
the inflate core (csrc/ck_inflate.cuh) refuses.  Shared by the CPU test of the host build (test_inflate_hostsim.py), the
device launcher's test (test_gpu_inflate.py) and the fetch tests (test_gpu_kafka_gzip_fetch.py).

zlib's verdict is the reference: a member is accepted when zlib.decompressobj(31) takes it whole — no error, the end of
the member reached, nothing after it — and a raw stream when decompressobj(-15) does."""
import struct
import zlib

import numpy as np

STRATEGIES = {"default": zlib.Z_DEFAULT_STRATEGY, "filtered": zlib.Z_FILTERED, "huffman_only": zlib.Z_HUFFMAN_ONLY,
              "rle": zlib.Z_RLE, "fixed": zlib.Z_FIXED}


def zlib_ref(data: bytes, wbits: int = 31):
    """what zlib inflates `data` to as one member (31) or one raw stream (-15), or None when it refuses it"""
    d = zlib.decompressobj(wbits)
    try:
        out = d.decompress(data)
    except zlib.error:
        return None
    return out if d.eof and not d.unused_data else None


def deflate(data: bytes, level=6, strategy=zlib.Z_DEFAULT_STRATEGY, wbits=-15, mem=8, flushes=()):
    """data compressed by zlib; flushes = [(offset, flush mode)] issued mid-stream"""
    c = zlib.compressobj(level, zlib.DEFLATED, wbits, mem, strategy)
    out, pos = b"", 0
    for at, mode in sorted(flushes):
        out += c.compress(data[pos:at]) + c.flush(mode)
        pos = at
    return out + c.compress(data[pos:]) + c.flush()


def member(raw: bytes, data: bytes, flg=0, extra=b"", name=b"", comment=b"", hcrc=None, crc=None, isize=None, mtime=0) -> bytes:
    """a gzip member around the raw deflate stream `raw` of `data`; hcrc: True = the right FHCRC, an int = that value"""
    h = bytes([0x1f, 0x8b, 8, flg]) + struct.pack("<I", mtime) + b"\x00\x03"
    if flg & 4:
        h += struct.pack("<H", len(extra)) + extra
    if flg & 8:
        h += name + b"\0"
    if flg & 16:
        h += comment + b"\0"
    if flg & 2:
        h += struct.pack("<H", (zlib.crc32(h) & 0xffff) if hcrc is None or hcrc is True else hcrc)
    return h + raw + struct.pack("<II", zlib.crc32(data) if crc is None else crc, (len(data) if isize is None else isize) & 0xffffffff)


def gzip_bytes(data: bytes, **kw) -> bytes:
    return member(deflate(data, **kw), data)


# ---- hand-built streams --------------------------------------------------------------------------------------------------
class Bits:
    """a DEFLATE bit writer: fields LSB first, Huffman codes first bit first"""
    def __init__(self):
        self.v, self.n = 0, 0

    def put(self, value, k):
        self.v |= (value & ((1 << k) - 1)) << self.n
        self.n += k
        return self

    def code(self, code, k):
        return self.put(int(format(code, f"0{k}b")[::-1], 2), k)

    def align(self):
        self.n = (self.n + 7) & ~7
        return self

    def bytes(self):
        return self.v.to_bytes((self.n + 7) // 8, "little")


def canonical(lens):
    """canonical codes of a list of lengths (0 = no code): {symbol: (code, length)}"""
    bl = [0] * 16
    for L in lens:
        if L:
            bl[L] += 1
    code, nxt = 0, [0] * 16
    for L in range(1, 16):
        code = (code + bl[L - 1]) << 1
        nxt[L] = code
    out = {}
    for s, L in enumerate(lens):
        if L:
            out[s] = (nxt[L], L)
            nxt[L] += 1
    return out


CL_ORDER = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]


def dynamic_block(lit_lens, dist_lens, symbols, final=1, cl_lens=None, cl_seq=None, hlit=None, hdist=None, hclen=None):
    """one dynamic block: the code lengths sent plainly (code-length symbols 0-15 of cl_lens, 4 bits each by default, or
    cl_seq = [(symbol, extra bits, extra value)]), then `symbols`: ints (literal / 256) or (length, distance) pairs"""
    b = Bits().put(final, 1).put(2, 2)
    nl, nd = len(lit_lens) if hlit is None else hlit, len(dist_lens) if hdist is None else hdist
    cl_lens = cl_lens or [4] * 16 + [0, 0, 0]
    hc = 19 if hclen is None else hclen
    b.put(nl - 257, 5).put(nd - 1, 5).put(hc - 4, 4)
    for i in range(hc):
        b.put(cl_lens[CL_ORDER[i]], 3)
    clc = canonical(cl_lens)
    seq = cl_seq if cl_seq is not None else [(L, 0, 0) for L in list(lit_lens) + list(dist_lens)]
    for sym, eb, ev in seq:
        b.code(*clc[sym])
        if eb:
            b.put(ev, eb)
    lc, dc = canonical(lit_lens), canonical(dist_lens)
    for s in symbols:
        if isinstance(s, int):
            b.code(*lc[s])
        else:
            _length_dist(b, lc, dc, *s)
    return b


def _length_dist(b, lc, dc, length, dist):
    lbase = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258]
    lext = [0] * 8 + [1] * 4 + [2] * 4 + [3] * 4 + [4] * 4 + [5] * 4 + [0]
    dbase = [1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097,
             6145, 8193, 12289, 16385, 24577]
    dext = [0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13]
    li = 28 if length == 258 else max(i for i in range(28) if lbase[i] <= length)
    b.code(*lc[257 + li]).put(length - lbase[li], lext[li])
    di = max(i for i in range(30) if dbase[i] <= dist)
    b.code(*dc[di]).put(dist - dbase[di], dext[di])


def fixed_block(symbols, final=1):
    """one fixed-code block of `symbols` (ints, including 286 / 287, or (length, distance) pairs; ("d", k) = distance code k)"""
    lens = [8] * 144 + [9] * 112 + [7] * 24 + [8] * 8
    lc, dc = canonical(lens), canonical([5] * 32)
    b = Bits().put(final, 1).put(1, 2)
    for s in symbols:
        if isinstance(s, int):
            b.code(*lc[s])
        elif s[0] == "d":                                       # length 3, then the raw distance code k
            b.code(*lc[257]).code(*dc[s[1]])
        else:
            _length_dist(b, lc, dc, *s)
    return b


def stored_block(data: bytes, final=1, nlen=None) -> Bits:
    b = Bits().put(final, 1).put(0, 2).align()
    for x in struct.pack("<HH", len(data), (~len(data) & 0xffff) if nlen is None else nlen):
        b.put(x, 8)
    for x in data:
        b.put(x, 8)
    return b


def _complete_lits():
    """litlen lengths: 'a' .. 'p' and EOB and length codes 257-261, a complete set"""
    lens = [0] * 286
    syms = [ord(c) for c in "abcdefghijklmnop"] + [256, 257, 258, 259, 260, 261]
    # 22 symbols: 10 of length 4 and 12 of length 5 -> 10/16 + 12/32 = 1
    for i, s in enumerate(syms):
        lens[s] = 4 if i < 10 else 5
    return lens


def malformed_streams():
    """{class: raw deflate stream} zlib refuses, built by hand; each differs from an accepted stream in the one point"""
    lits = _complete_lits()
    dist2 = [1, 1]
    ok_syms = [ord("a"), ord("b"), ord("c"), (4, 2), 256]
    out = {}
    # over-subscribed litlen: one more length-4 code
    over = list(lits)
    over[ord("q")] = 4
    out["over-subscribed litlen set"] = dynamic_block(over, dist2, ok_syms).bytes()
    # incomplete litlen: drop one code (more than the single one-bit code zlib allows)
    inc = list(lits)
    inc[ord("p")] = 0
    out["incomplete litlen set"] = dynamic_block(inc, dist2, ok_syms).bytes()
    out["over-subscribed distance set"] = dynamic_block(lits, [1, 1, 1], ok_syms).bytes()
    out["incomplete distance set"] = dynamic_block(lits, [1, 2, 0], [ord("a"), 256]).bytes()
    cl_over = [4] * 16 + [0, 0, 0]
    cl_over[17] = 4                                              # 17 codes of 4 bits
    out["over-subscribed code-length set"] = dynamic_block(lits, dist2, ok_syms, cl_lens=cl_over).bytes()
    cl_inc = [4] * 15 + [0, 0, 0, 0]                             # 15 codes of 4 bits (length 15 is never sent)
    out["incomplete code-length set"] = dynamic_block(lits, dist2, ok_syms, cl_lens=cl_inc).bytes()
    seq = [(L, 0, 0) for L in list(lits) + dist2]
    cl16 = [4] * 16 + [0, 0, 0]
    cl16[15], cl16[16] = 0, 4                                    # code 16 instead of 15
    out["repeat 16 with nothing before it"] = dynamic_block(lits, dist2, ok_syms, cl_lens=cl16,
                                                             cl_seq=[(16, 2, 0)] + seq).bytes()
    cl18 = [4] * 16 + [0, 0, 0]
    cl18[15], cl18[18] = 0, 4
    out["repeat past HLIT + HDIST"] = dynamic_block(lits, dist2, ok_syms, cl_lens=cl18,
                                                     cl_seq=seq[:-2] + [(18, 7, 127)]).bytes()
    noeob = list(lits)
    noeob[256], noeob[ord("q")] = 0, 5
    out["no end-of-block code"] = dynamic_block(noeob, dist2, [ord("a")]).bytes()
    out["litlen symbol 286"] = fixed_block([ord("a"), 286, 256]).bytes()
    out["litlen symbol 287"] = fixed_block([ord("a"), 287, 256]).bytes()
    out["distance symbol 30"] = fixed_block([ord("a")] * 40 + [("d", 30), 256]).bytes()
    out["distance symbol 31"] = fixed_block([ord("a")] * 40 + [("d", 31), 256]).bytes()
    out["distance before the output"] = fixed_block([ord("a"), ord("b"), (3, 3), 256]).bytes()
    out["BTYPE 3"] = Bits().put(1, 1).put(3, 2).put(0, 13).bytes()
    out["stored LEN != ~NLEN"] = stored_block(b"hello", nlen=0x1234).bytes()
    out["HLIT 287"] = dynamic_block(lits + [0], dist2, ok_syms).bytes()
    out["HDIST 31"] = dynamic_block(lits, dist2 + [0] * 29, ok_syms).bytes()
    good = fixed_block([ord(c) for c in "hello, hello, hello"] + [256]).bytes()
    out["ends early"] = good[:-2]
    out["no final block"] = fixed_block([ord("a"), 256], final=0).bytes()
    out["empty"] = b""
    return out


def accepted_edge_streams():
    """{name: raw deflate stream} zlib accepts at the edges the refusals above sit next to"""
    lits = _complete_lits()
    one = [0] * 257
    one[256] = 1                                                 # a litlen set of one one-bit code: EOB alone
    out = {
        "complete dynamic block": dynamic_block(lits, [1, 1], [ord("a"), ord("b"), ord("c"), (4, 2), 256]).bytes(),
        "single one-bit litlen code": dynamic_block(one, [0], [256]).bytes(),
        "no distance code": dynamic_block(lits, [0], [ord("a"), ord("b"), 256]).bytes(),
        "single one-bit distance code": dynamic_block(lits, [1], [ord("a"), (4, 1), 256]).bytes(),
        "empty stored block": stored_block(b"").bytes(),
        "distance = output": fixed_block([ord("a"), ord("b"), ord("c"), (3, 3), 256]).bytes(),
    }
    b = stored_block(b"stored bytes ", final=0)
    fb = fixed_block([ord(c) for c in "then fixed"] + [(20, 13), 256])
    b.put(fb.v, fb.n)
    out["stored then fixed"] = b.bytes()
    return out


def records_data(n=200, seed=1) -> bytes:
    from calfkit import synth
    return b"".join(synth.tool_events(n, seed=seed))


def far_match_data() -> bytes:
    """a 40 KB random block repeated: zlib must match at distance 32768 (a period of exactly 32 KB) with 258-byte lengths"""
    rng = np.random.default_rng(9)
    blk = rng.integers(0, 256, 32768, dtype=np.uint8).tobytes()
    return blk + blk + blk[:20000]
