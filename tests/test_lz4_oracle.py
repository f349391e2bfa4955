"""The LZ4 restatement the device's compressed frames are checked against (tests/kafka_lz4.py), pinned to the frames
liblz4 writes (tests/golden/lz4_frames.json, written by make_golden_lz4.py): every input comes back from every frame flag
and block size, XXH32 matches, corrupted frames are refused, and an LZ4 batch decompresses to the uncompressed batch."""
import base64
import json
import os
import struct

import pytest

import kafka_lz4 as lz
from make_golden_lz4 import inputs
from oracle import kafka_batch as kb

GOLDEN = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "lz4_frames.json")))
INPUTS = inputs()
FRAMES = [(f["variant"], f["input"], base64.b64decode(f["frame"])) for f in GOLDEN["frames"]]


def _frame(variant, name):
    return next(f for v, n, f in FRAMES if v == variant and n == name)


@pytest.mark.parametrize("variant,name", [(v, n) for v, n, _f in FRAMES])
def test_decompress_frame_reproduces_every_input(variant, name):
    assert lz.decompress_frame(_frame(variant, name)) == INPUTS[name]


def test_golden_covers_every_frame_flag_and_block_size():
    flg = {f[4] for _v, _n, f in FRAMES}
    bd = {f[5] for _v, _n, f in FRAMES}
    assert {0x60, 0x40, 0x70, 0x64, 0x68, 0x5C} <= flg          # default, linked, block / content checksum, size, all
    assert bd == {0x40, 0x50, 0x60, 0x70}                       # 64 KB, 256 KB, 1 MB, 4 MB blocks
    # liblz4's default descriptor is the one the device writes (for more than one block liblz4 links them by default,
    # FLG 0x40; the device's blocks are independent, as FLG 0x60 says)
    assert _frame("default", "records_20k")[:7] == _frame("independent", "period_251")[:7] == bytes.fromhex("04224D18604082")
    assert _frame("default", "period_251")[4] == 0x40
    # incompressible data: a stored block (bit 31 of the size)
    f = _frame("independent", "random_3k")
    assert struct.unpack_from("<I", f, 7)[0] == 0x80000000 | 3000


def test_xxh32_vectors():
    assert lz.xxh32(b"") == 0x02CC5D05
    for v in GOLDEN["xxh32"]:
        assert lz.xxh32(INPUTS[v["input"]]) == v["xxh32"], v["input"]
    assert (lz.xxh32(bytes([0x60, 0x40])) >> 8) & 0xFF == 0x82


def _blocks(frame):
    """(offset of the size word, size word) of every block of a frame without content size / dict id"""
    pos, out = 7, []
    bsum = frame[4] & 0x10
    while True:
        w = struct.unpack_from("<I", frame, pos)[0]
        if w == 0:
            return out
        out.append((pos, w))
        pos += 4 + (w & 0x7FFFFFFF) + (4 if bsum else 0)


def test_corrupted_frames_are_refused():
    f = bytearray(_frame("default", "records_20k"))
    bad = bytearray(f)
    bad[6] ^= 1
    with pytest.raises(ValueError, match="header checksum"):
        lz.decompress_frame(bytes(bad))
    g = bytearray(_frame("block_checksum", "records_20k"))
    pos, w = _blocks(g)[0]
    g[pos + 4 + 100] ^= 0x40
    with pytest.raises(ValueError, match="block checksum"):
        lz.decompress_frame(bytes(g))
    c = bytearray(_frame("content_checksum", "records_20k"))
    c[-1] ^= 1
    with pytest.raises(ValueError, match="content checksum"):
        lz.decompress_frame(bytes(c))


def _block(literals: bytes, off: int, ml: int, last: bytes):
    """a hand-made block of two sequences: literals + one match (< 19 bytes), then the last literals (< 15)"""
    return bytes([len(literals) << 4 | (ml - 4)]) + literals + struct.pack("<H", off) + bytes([len(last) << 4]) + last


def _frame_of(block: bytes) -> bytes:
    return bytes.fromhex("04224D18604082") + struct.pack("<I", len(block)) + block + b"\0\0\0\0"


def test_block_rules_are_enforced():
    ok = _block(b"abcdefgh", 8, 8, b"abcdefgh")                 # 8 literals, an 8-byte match, 8 literals
    assert lz.decompress_frame(_frame_of(ok)) == b"abcdefgh" * 3
    with pytest.raises(ValueError, match="offset 0"):
        lz.decompress_frame(_frame_of(_block(b"abcdefgh", 0, 8, b"abcdefgh")))
    with pytest.raises(ValueError, match="before the block"):
        lz.decompress_frame(_frame_of(_block(b"abcdefgh", 9, 8, b"abcdefgh")))
    with pytest.raises(ValueError, match="last 5 bytes"):       # the match ends 4 bytes before the end of the block
        lz.decompress_frame(_frame_of(_block(b"abcdefgh", 8, 8, b"abcd")))
    with pytest.raises(ValueError, match="12 bytes"):           # starts 11 bytes before the end, ends 7 before it
        lz.decompress_frame(_frame_of(_block(b"abcd", 4, 4, b"1234567")))
    with pytest.raises(ValueError, match="literals-only"):
        lz.decompress_frame(_frame_of(ok[:11]))                 # ends right after the match


def test_decompress_batch_equals_the_uncompressed_batch():
    """an LZ4 batch assembled from a golden frame (liblz4's frame of the records section of the first tool events)
    decompresses to encode_batch of the same records; a flipped bit fails its CRC"""
    from calfkit import synth
    recs = [kb.calfkit_record(r, f"corr-{i:06d}") for i, r in enumerate(synth.tool_events(80, seed=111))]
    n = next(n for n in range(1, len(recs) + 1) if len(kb.encode_batch(recs[:n])) - kb.HEADER_LEN == len(INPUTS["records_20k"]))
    want = kb.encode_batch(recs[:n], base_offset=7, base_timestamp=1767225600123)
    assert want[kb.HEADER_LEN:] == INPUTS["records_20k"]
    covered = struct.pack(">h", 3) + want[23:kb.HEADER_LEN] + _frame("independent", "records_20k")
    batch = want[:8] + struct.pack(">i", len(covered) + 9) + want[12:17] + struct.pack(">I", kb.crc32c(covered)) + covered
    assert len(batch) < len(want) // 3
    assert lz.decompress_batch(batch) == want
    bad = bytearray(batch)
    bad[-3] ^= 1
    with pytest.raises(ValueError, match="CRC32C"):
        lz.decompress_batch(bytes(bad))
