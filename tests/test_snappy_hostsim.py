"""The snappy decoder (csrc/ck_snappy.cuh) built by g++ as one lane (tests/snappydec), held on the CPU against Google snappy
(pyarrow's, tests/snappy_ref.py) and against the plain restatement (tests/kafka_snappy.py): raw blocks of 1 B to 4 MiB
over tool envelopes, random bytes, one repeated byte and low-entropy text; hand-written blocks with overlapping copies at
offsets 1-8 of every copy kind, copy-4 and every literal-length width; every malformed block; the varint edge cases;
snappy-java framed sections of 32 KB and 1 KB chunks and every malformed framing; and seeded bit flips and truncations.
The verdict and the bytes must be identical."""
import pytest

import kafka_snappy as ks
import snappy_ref as sr
import snappydec
import zstd_cases as zc

SIZES = (1, 2, 59, 60, 61, 100, (32 << 10) - 1, 32 << 10, (64 << 10) + 1, 1 << 20, 4 << 20)


def host(z: bytes):
    """what the host build makes of the raw block z as the fetch path runs it: the walk reads its varint (and refuses a
    length past CK_SN_RATIO times the block), the decoder fills exactly that many bytes"""
    n = snappydec.declared(z)
    if n is None or n > ks.RATIO * len(z):
        return None
    return snappydec.decode_block(z, n)


@pytest.mark.parametrize("kind", zc.KINDS)
def test_blocks_1b_to_4mb(kind):
    sr.need()
    for n in SIZES:
        d = zc.data(kind, n, seed=21)
        z = sr.compress(d)
        assert sr.decompress(z) == d
        assert host(z) == d and ks.decompress_block(z) == d, n
        assert snappydec.walk(z) == [(0, len(z), n)]


def test_hand_written_blocks():
    for name, (z, content) in ks.hand_blocks().items():
        assert ks.decompress_block(z) == content, name
        assert host(z) == content, name
        if sr.available():
            assert sr.decompress(z) == content, name


def test_malformed_blocks():
    for name, z in ks.malformed_blocks().items():
        assert ks.decompress_block(z) is None, name
        assert host(z) is None, name
        assert snappydec.decode_block(z, (ks.varint(z) or (0, 0))[0]) is None, name
        if sr.available():
            assert sr.decompress(z) is None, name


def test_varint_edges():
    """a 5th varint byte of 15 and of 16, a varint of 6 bytes, a varint that ends the input (length 0 and 1): the host
    build's reading and pyarrow's verdict agree"""
    sr.need()
    cases = {b"\x80\x80\x80\x80\x00": b"", b"\x00": b"", b"\x01": None, b"\x80\x80\x80\x80\x10": None,
             b"\x80\x80\x80\x80\x0f": None, b"\x80\x80\x80\x80\x80\x00": None, b"\x80": None, b"": None}
    for z, want in cases.items():
        assert sr.decompress(z) == want, z
        assert host(z) == want and ks.decompress_block(z) == want, z
    assert snappydec.declared(b"\x80\x80\x80\x80\x0f") == 0xF0000000 and snappydec.declared(b"\x80\x80\x80\x80\x10") is None


def test_slot_other_than_the_declared_length_is_refused():
    sr.need()
    d = zc.data("text", 5000, seed=22)
    z = sr.compress(d)
    assert snappydec.decode_block(z, 5000) == d
    assert snappydec.decode_block(z, 4999) is None and snappydec.decode_block(z, 5001) is None


@pytest.mark.parametrize("chunk", [32 << 10, 1 << 10])
def test_framed_sections(chunk):
    sr.need()
    for n in (1, 1000, 32 << 10, (32 << 10) + 1, 300000):
        d = zc.data("records", n, seed=23)
        sec = ks.xerial(d, chunk)
        w = snappydec.walk(sec)
        assert w == ks.walk(sec) and len(w) == (n + chunk - 1) // chunk
        assert sum(dl for _o, _l, dl in w) == n
        assert snappydec.decode_section(sec) == d == ks.decompress_section(sec)


def test_malformed_framings():
    for name, sec in ks.malformed_framings().items():
        assert ks.walk(sec) is None or ks.decompress_section(sec) is None, name
        assert snappydec.decode_section(sec) is None, name
        assert snappydec.walk(sec) == ks.walk(sec), name
    hdr = ks.malformed_framings()["header only (a raw block, which snappy refuses)"]
    assert len(hdr) == 16 and not ks.framed(hdr)
    if sr.available():
        assert sr.decompress(hdr) is None


def test_mutations():
    """3,000 blocks with one or two bit flips and 300 truncations: accepted exactly when snappy accepts, with its bytes"""
    sr.need()
    srcs = [sr.compress(zc.data(k, n, seed=24)) for k in zc.KINDS for n in (40, 700, 5000)]
    srcs += [z for z, _c in ks.hand_blocks().values() if len(z) > 1]
    accepted = 0
    for z in ks.mutations(srcs):
        want = sr.decompress(z)
        assert host(z) == want == ks.decompress_block(z), z[:16].hex()
        accepted += want is not None
    assert 0 < accepted < 3300
