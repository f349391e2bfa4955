"""The LZ4 block decoder on its own (ck_lz4_decode_block, csrc/ck_lz4.cuh, through tests/lz4dec), held against the CPU
restatement tests/kafka_lz4.decompress_block on 1 B - 4 MB blocks: the blocks liblz4 wrote into the golden frames (linked
ones decoded behind their frame's earlier output), blocks from the device's own compressor (ck_lz4_block), hand-made
blocks at the format's edges, and every malformed class the decoder refuses.  A block decodes to exactly what the
restatement gives, or is refused exactly when the restatement raises."""
import base64
import json
import os
import struct

import numpy as np
import pytest

import kafka_lz4 as lz
from make_golden_lz4_batches import load as load_batches

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture(autouse=True)
def _cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def _len_bytes(n):
    out = b""
    while n >= 255:
        out += b"\xff"
        n -= 255
    return out + bytes([n])


def seq(lit: bytes, off: int = 0, ml: int = 0) -> bytes:
    """one sequence; ml 0: the literals-only last sequence"""
    ll, mc = len(lit), (ml - 4 if ml else 0)
    tok = (min(ll, 15) << 4) | min(mc, 15)
    out = bytes([tok]) + (_len_bytes(ll - 15) if ll >= 15 else b"") + lit
    if ml:
        out += struct.pack("<H", off) + (_len_bytes(mc - 15) if mc >= 15 else b"")
    return out


def frame_blocks(frame: bytes):
    """(block data, history, block max) of every compressed block of an LZ4 frame, history = the frame's output before
    the block when its blocks are linked (at most 64 KB), empty when independent"""
    flg, bd = frame[4], frame[5]
    bmax = lz.BLOCK_MAX[(bd >> 4) & 7]
    pos = 6 + (8 if flg & 8 else 0) + 1
    out, got = bytearray(), []
    while (w := struct.unpack_from("<I", frame, pos)[0]):
        size = w & 0x7FFFFFFF
        data = frame[pos + 4:pos + 4 + size]
        pos += 4 + size + (4 if flg & 0x10 else 0)
        if w >> 31:
            out += data
            continue
        hist = b"" if flg & 0x20 else bytes(out[-65535:])
        got.append((data, hist, bmax))
        lz.decompress_block(data, out, bmax, len(hist))
    return got


def expected(block, hist, bmax):
    out = bytearray(hist)
    try:
        lz.decompress_block(block, out, bmax, len(hist))
    except ValueError:
        return None
    return bytes(out[len(hist):])


def run_device(cases):
    """cases: [(block, history, block max)] -> [decoded bytes or None]"""
    import torch
    import lz4dec
    res = [None] * len(cases)
    for bmax in sorted({c[2] for c in cases}):
        idx = [i for i, c in enumerate(cases) if c[2] == bmax]
        blocks = [cases[i][0] for i in idx]
        hists = [cases[i][1] for i in idx]
        soff = np.concatenate(([0], np.cumsum([len(b) for b in blocks]))).astype(np.int64)
        regions = [len(h) + bmax for h in hists]
        doff = np.concatenate(([0], np.cumsum(regions))).astype(np.int64)
        host_dst = np.zeros(int(doff[-1]) + 256, dtype=np.uint8)
        for k, h in enumerate(hists):
            host_dst[doff[k]:doff[k] + len(h)] = np.frombuffer(h, dtype=np.uint8)
        src = torch.from_numpy(np.frombuffer(b"".join(blocks) + b"\0" * 256, dtype=np.uint8).copy()).cuda()
        dst = torch.from_numpy(host_dst).cuda()
        d_soff, d_doff = torch.from_numpy(soff).cuda(), torch.from_numpy(doff).cuda()
        d_hist = torch.tensor([len(h) for h in hists], dtype=torch.int32).cuda()
        out_len = torch.zeros(len(blocks), dtype=torch.int64, device="cuda")
        assert lz4dec.lib().lz4dec_blocks(src.data_ptr(), d_soff.data_ptr(), len(blocks), dst.data_ptr(), d_doff.data_ptr(),
                                          d_hist.data_ptr(), bmax, out_len.data_ptr()) == 0
        data, lens = dst.cpu().numpy(), out_len.cpu().numpy()
        for k, i in enumerate(idx):
            n = int(lens[k])
            a = int(doff[k]) + len(hists[k])
            res[i] = None if n < 0 else data[a:a + n].tobytes()
    return res


def check(cases):
    got = run_device(cases)
    for i, c in enumerate(cases):
        assert got[i] == expected(*c), (i, len(c[0]), len(c[1]), c[2])


def test_liblz4_golden_blocks():
    """every compressed block liblz4 wrote into the golden frames and batches: 64 KB to 4 MB blocks, linked ones behind
    their frame's earlier output"""
    cases = []
    for f in json.load(open(os.path.join(GOLDEN, "lz4_frames.json")))["frames"]:
        cases += frame_blocks(base64.b64decode(f["frame"]))
    for _n, _s, batch in load_batches():
        cases += frame_blocks(batch[61:])
    assert any(len(h) for _b, h, _m in cases) and {m for _b, _h, m in cases} == set(lz.BLOCK_MAX.values())
    assert max(len(expected(*c)) for c in cases) > 1 << 20
    check(cases)


def test_device_compressor_blocks():
    """blocks ck_lz4_block (through tests/lz4sim) made of records, runs, periods and random bytes, 13 B - 64 KB"""
    import torch
    import lz4sim
    from calfkit import synth
    rng = np.random.default_rng(77)
    recs = b"".join(synth.tool_events(200, seed=78))
    raw = []
    for n in (13, 14, 17, 32, 100, 1000, 4096, 30000, 65535, 65536):
        raw += [b"q" * n, recs[:n], (bytes(range(7)) * (n // 7 + 1))[:n], rng.integers(0, 4, n, dtype=np.uint8).tobytes()]
    off = np.concatenate(([0], np.cumsum([len(b) for b in raw]))).astype(np.int64)
    src = torch.from_numpy(np.frombuffer(b"".join(raw) + b"\0" * 256, dtype=np.uint8).copy()).cuda()
    dst = torch.zeros(int(off[-1]) + 256, dtype=torch.uint8, device="cuda")
    out_len = torch.zeros(len(raw), dtype=torch.int32, device="cuda")
    assert lz4sim.lib().lz4sim_blocks(src.data_ptr(), torch.from_numpy(off).cuda().data_ptr(), len(raw), dst.data_ptr(),
                                      out_len.data_ptr()) == 0
    data, lens = dst.cpu().numpy().tobytes(), out_len.cpu().numpy()
    cases = [(data[off[i]:off[i] + int(lens[i])], b"", 65536) for i in range(len(raw)) if lens[i]]
    assert len(cases) > len(raw) // 2
    got = run_device(cases)
    comp = [b for i, b in enumerate(raw) if lens[i]]
    assert got == comp


def test_edge_blocks():
    """1 B, literal lengths of 14 / 15 / 270 bytes, overlapping matches of every offset 1 - 40, an offset of 65535 into
    history, and a 4 MB block (one long overlapping match) at the 4 MB block maximum"""
    cases = [(seq(b"x"), b"", 65536), (seq(b"a" * 14), b"", 65536), (seq(b"b" * 15), b"", 65536), (seq(b"c" * 270), b"", 65536)]
    for off in range(1, 41):
        lit = bytes(range(65, 65 + off))
        cases.append((seq(lit, off, 300 + off) + seq(b"0123456789ab"), b"", 65536))
    hist = np.random.default_rng(5).integers(0, 256, 65535, dtype=np.uint8).tobytes()
    cases.append((seq(b"hd", 65535, 40) + seq(b"tail-literals"), hist, 65536))
    big = 4 << 20
    cases.append((seq(b"z", 1, big - 1 - 12) + seq(b"twelve bytes"), b"", big))
    check(cases)
    assert expected(*cases[-1]) == b"z" * (big - 12) + b"twelve bytes"


MALFORMED = {
    "empty block": b"",
    "offset 0": seq(b"abcd", 0, 8) + seq(b"0123456789ab"),
    "offset before the output": seq(b"abcd", 5, 8) + seq(b"0123456789ab"),
    "literal run past the block": seq(b"abcdef")[:-2],
    "literal length past the block": bytes([0xF0, 255, 255]),
    "truncated offset": seq(b"abcd", 4, 8)[:-1],
    "match length past the block": bytes([0x1F]) + b"a" + struct.pack("<H", 1) + b"\xff",
    "block larger than block max": seq(b"a", 1, 70000) + seq(b"0123456789ab"),
    "ends after a match": seq(b"abcd", 4, 20),
    "last match nearer than 12 bytes to the end": seq(b"abcd", 4, 20) + seq(b"0123"),
    "match into the last 5 bytes": seq(b"abcd", 4, 20) + seq(b"012"),
}


@pytest.mark.parametrize("name", list(MALFORMED))
def test_malformed_blocks_are_refused(name):
    block = MALFORMED[name]
    assert expected(block, b"", 65536) is None
    assert run_device([(block, b"", 65536)]) == [None]


def test_offset_past_history_is_refused():
    """behind 100 bytes of history an offset may reach 102 bytes back (2 literals first), not 103"""
    hist = bytes(range(100))
    cases = [(seq(b"ab", 103, 8) + seq(b"0123456789ab"), hist, 65536), (seq(b"ab", 102, 8) + seq(b"0123456789ab"), hist, 65536)]
    assert expected(*cases[0]) is None and expected(*cases[1]) == b"ab" + hist[:8] + b"0123456789ab"
    check(cases)
