"""The shipped inflate core (csrc/ck_inflate.cuh) compiled by g++ (tests/inflate, one lane) against zlib: every gzip member
and raw deflate stream below inflates to exactly what zlib.decompressobj gives, or is refused exactly when zlib refuses
it — tool-stage records, cycled records (long matches) and random bytes (stored blocks), at every level, strategy,
window size and memLevel, with mid-stream flushes; hand-built headers with every FLG bit; matches at distance 32768 of
length 258; every malformed class built by hand; and seeded bit flips and truncations of valid members."""
import random
import zlib

import numpy as np
import pytest

import gzip_cases as gz
import inflate


def _data():
    from calfkit import synth
    recs = gz.records_data(120, seed=11)
    cyc = b"".join(synth.tool_events(6, seed=12)) * 40
    rnd = np.random.default_rng(13).integers(0, 256, 70000, dtype=np.uint8).tobytes()
    return {"records": recs, "cycled": cyc, "random": rnd}


DATA = _data()


def check_member(z: bytes):
    want = gz.zlib_ref(z, 31)
    assert inflate.member(z) == want
    return want


def check_raw(s: bytes):
    want = gz.zlib_ref(s, -15)
    got, used = inflate.inflate(s, 1 << 22)
    assert (got if got is not None and used == len(s) else None) == want
    return want


@pytest.mark.parametrize("name", list(DATA))
@pytest.mark.parametrize("level", range(10))
def test_levels(name, level):
    data = DATA[name]
    assert check_member(gz.gzip_bytes(data, level=level)) == data


@pytest.mark.parametrize("strategy", list(gz.STRATEGIES))
@pytest.mark.parametrize("name", list(DATA))
def test_strategies(strategy, name):
    data = DATA[name]
    for level in (1, 6, 9):
        assert check_member(gz.gzip_bytes(data, level=level, strategy=gz.STRATEGIES[strategy])) == data


@pytest.mark.parametrize("wbits", range(9, 16))
@pytest.mark.parametrize("mem", [1, 9])
def test_window_bits_and_mem_level(wbits, mem):
    for data in DATA.values():
        assert check_member(gz.member(gz.deflate(data, level=9, wbits=-wbits, mem=mem), data)) == data


@pytest.mark.parametrize("mode", ["Z_SYNC_FLUSH", "Z_FULL_FLUSH", "Z_BLOCK"])
def test_mid_stream_flushes(mode):
    m = getattr(zlib, mode)
    for data in DATA.values():
        fl = [(k, m) for k in (1, 100, len(data) // 3, len(data) // 2, len(data) - 1)]
        assert check_member(gz.member(gz.deflate(data, flushes=fl), data)) == data


@pytest.mark.parametrize("flg", range(32))
def test_header_flags(flg):
    """every combination of FTEXT, FHCRC, FEXTRA, FNAME and FCOMMENT (with the right FHCRC), and the wrong FHCRC"""
    data = DATA["records"][:5000]
    raw = gz.deflate(data)
    kw = dict(extra=b"AB\x04\x00test", name=b"records.json", comment=b"a comment")
    assert check_member(gz.member(raw, data, flg=flg, **kw)) == data
    if flg & 2:
        right = zlib.crc32(gz.member(raw, data, flg=flg, **kw)[:-(len(raw) + 10)]) & 0xffff
        assert check_member(gz.member(raw, data, flg=flg, hcrc=right ^ 0x100, **kw)) is None


@pytest.mark.parametrize("bit", [0x20, 0x40, 0x80])
def test_reserved_flag_bits_are_refused(bit):
    data = b"hello"
    assert check_member(gz.member(gz.deflate(data), data, flg=bit)) is None


def test_bad_magic_method_and_trailer():
    data = DATA["records"][:3000]
    z = gz.gzip_bytes(data)
    assert check_member(z) == data
    for i, v in ((0, 0x1e), (1, 0x8a), (2, 7)):
        assert check_member(z[:i] + bytes([v]) + z[i + 1:]) is None
    raw = gz.deflate(data)
    assert check_member(gz.member(raw, data, crc=zlib.crc32(data) ^ 1)) is None
    assert check_member(gz.member(raw, data, isize=len(data) + 1)) is None
    assert check_member(gz.member(raw, data, isize=len(data) - 1)) is None
    assert check_member(z + b"\0") is None
    assert check_member(z + z) is None                           # a second member follows
    assert check_member(gz.gzip_bytes(b"")) == b""


def test_distance_32768_and_length_258():
    data = gz.far_match_data()
    raw = gz.deflate(data, level=9)
    assert check_member(gz.member(raw, data)) == data
    # the same by hand: 32768 literals, then 258-byte matches at distance 32768
    blk = data[:32768]
    syms = list(blk) + [(258, 32768)] * 10 + [256]
    b = gz.fixed_block(syms)
    want = blk + blk[:2580]
    assert check_raw(b.bytes()) == want
    assert check_raw(gz.fixed_block(list(blk[:-1]) + [(258, 32768), 256]).bytes()) is None


@pytest.mark.parametrize("name", list(gz.malformed_streams()))
def test_malformed_raw_streams(name):
    s = gz.malformed_streams()[name]
    assert gz.zlib_ref(s, -15) is None
    assert check_raw(s) is None


@pytest.mark.parametrize("name", list(gz.accepted_edge_streams()))
def test_accepted_edge_streams(name):
    s = gz.accepted_edge_streams()[name]
    want = gz.zlib_ref(s, -15)
    assert want is not None and check_raw(s) == want


def test_malformed_members():
    """each malformed stream inside a member whose trailer is right for what zlib inflated before it failed"""
    for s in gz.malformed_streams().values():
        assert check_member(gz.member(s, b"abc")) is None


def test_bit_flips_and_truncations():
    rng = random.Random(2026)
    base = [gz.gzip_bytes(DATA["records"][:4000], level=lv) for lv in (1, 6, 9)] + \
        [gz.gzip_bytes(DATA["cycled"][:6000], strategy=zlib.Z_FIXED), gz.gzip_bytes(DATA["random"][:3000], level=0),
         gz.member(gz.deflate(b"x"), b"x", flg=30, extra=b"ex", name=b"n", comment=b"c")]
    accepted = refused = 0
    for it in range(4000):
        z = bytearray(rng.choice(base))
        if it % 5 == 4:
            z = z[:rng.randrange(len(z))]
        else:
            for _ in range(rng.randint(1, 3)):
                i = rng.randrange(len(z))
                z[i] ^= 1 << rng.randrange(8)
        if check_member(bytes(z)) is None:
            refused += 1
        else:
            accepted += 1
    assert refused > 1000
    # raw streams: flips inside the Huffman data reach the table build and the symbol decode
    raws = [gz.deflate(DATA["records"][:4000], level=lv) for lv in (1, 9)] + [gz.deflate(DATA["cycled"][:5000], strategy=zlib.Z_FIXED)]
    for it in range(4000):
        s = bytearray(rng.choice(raws))
        for _ in range(rng.randint(1, 2)):
            i = rng.randrange(len(s))
            s[i] ^= 1 << rng.randrange(8)
        check_raw(bytes(s))
