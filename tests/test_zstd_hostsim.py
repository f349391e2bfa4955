"""The zstd decoder (csrc/ck_zstd.cuh) built by g++ as one lane (tests/zstdec), held against libzstd on the CPU: every
setting of the matrix over tool envelopes, random bytes, one repeated byte and low-entropy text of 0 B to 4 MiB, a
streamed frame, the writer's raw / RLE / sequence frames, every malformed class, and seeded bit flips and truncations.
The verdict and the bytes must be identical, with one characterized exception (see test_mutations)."""
import pytest

import zstd_cases as zc
import zstd_ref as zr
import zstdec


def check(z: bytes):
    want = zr.decompress(z)
    got = zstdec.decode(z)
    assert got == want, (len(z), want is None, got is None)
    return want


def test_library_version():
    assert zr.version() == "1.5.5"


@pytest.mark.parametrize("setting", list(zc.SETTINGS))
@pytest.mark.parametrize("kind", zc.KINDS)
def test_settings_matrix(setting, kind):
    for n in zc.DATA_SIZES:
        if n >= 1 << 20 and setting in ("level19", "target_cblock"):
            continue                     # slow to compress; their shapes are covered below 1 MiB
        d = zc.data(kind, n, seed=11)
        z = zr.compress(d, **zc.SETTINGS[setting])
        assert check(z) == d


@pytest.mark.parametrize("flush", [False, True])
def test_streamed_frames(flush):
    """the streaming shape (no content size, a window descriptor: windowLog 21 at level 3), with and without flushes"""
    d = zc.data("records", 300000, seed=12)
    z = zr.stream(d, piece=7000, flush=flush, level=3)
    assert not (z[4] & 0x20) and (z[4] >> 6) == 0 and (z[5] >> 3) + 10 == 21
    assert check(z) == d


def test_writer_frames():
    content = b"hello zstd " * 20
    lits = b"abcdefgh" * 8
    frames = {
        "raw, content size, checksum": zc.frame([zc.block(True, 0, content)], fcs=len(content), window_log=17, checksum=True, content=content),
        "RLE then raw": zc.frame([zc.block(False, 1, b"q", 5000), zc.block(True, 0, b"xyz")], window_log=17),
        "empty, single segment": zc.frame([zc.block(True, 0, b"")], fcs=0, single_segment=True),
        "sequences, RLE modes": zc.frame([zc.block(True, 2, zc.seq_block(lits, [(8, 8, 4), (8, 9, 4)], 8, 3, 1))], window_log=17),
        "sequences, RLE literals": zc.frame([zc.block(True, 2, zc.seq_block(b"x" * 40, [(8, 8, 4)], 8, 3, 1, rle_lits=True))], window_log=17),
        "no sequences": zc.frame([zc.block(True, 2, zc.lit_header(0, 8) + lits[:8] + b"\0")], window_log=17),
        "reserved bits of the modes byte (libzstd 1.5.5 ignores them)":
            zc.frame([zc.block(True, 2, zc.seq_block(lits, [(8, 8, 4)], 8, 3, 1, modes=0x55))], window_log=17),
    }
    for name, z in frames.items():
        assert check(z) is not None, name
    assert check(zc.frame([zc.block(True, 1, b"a", 0)], fcs=0, single_segment=True)) is None   # RLE's input byte past a 0-byte maximum


def test_malformed_classes():
    mal = zc.malformed()
    assert len(mal) >= 60
    for name, z in mal.items():
        assert zr.decompress(z) is None, name
        assert zstdec.decode(z) is None, name
        assert zstdec.decode(z, cap=(zstdec.bound(z) or 0) + 4096) is None, name   # a slot not the bound is refused too


def test_mutations():
    """5,000 frames with one or two bit flips and 500 truncations of 20 frames: the same verdict and bytes as libzstd.
    The one exception: libzstd decodes 4-stream Huffman literals with a double-symbol decoder when its speed heuristic
    picks it, and that decoder lets a stream end inexactly on its last symbol; so a frame with a flip inside such a section may pass
    libzstd (with garbage literals) where this decoder, which requires every stream to end exactly, refuses it"""
    muts = zc.mutations()
    assert len(muts) == 5500
    lenient = 0
    for z, src, at in muts:
        want, got = zr.decompress(z), zstdec.decode(z)
        if got == want:
            continue
        assert got is None and want is not None and zc.in_4stream_literals(src, at), (len(z), at)
        lenient += 1
    assert lenient < len(muts) // 20
