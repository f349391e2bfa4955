"""Fetch responses holding LZ4 batches (attributes 3), decoded on the device (ck_rb_lz4_kernel, csrc/ck_kafka.cuh): the
records of an LZ4 batch read, through the host view, exactly as tests/kafka_lz4.decompress_batch and the Kafka oracle give
them, and walk exactly as the same batch submitted uncompressed; a Worker lane consumes the LZ4 frames another engine's
frame pass wrote as it consumes the uncompressed ones; a mixed fetch marks exactly its malformed LZ4 batches and its gzip
batch bad; the fetch buffer grows; the same fetch gives the same results; an uncompressed fetch afterwards takes the
path it always took."""
import struct

import numpy as np
import pytest

import kafka_lz4 as lz
from make_golden_lz4_batches import load as load_batches, uncompressed, with_section
from oracle import kafka_batch as kb

pytestmark = pytest.mark.gpu

GOLDEN = load_batches()


@pytest.fixture(autouse=True)
def _cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def tool_engine(max_in=64 << 20):
    from calfkit.engine import BatchEngine
    e = BatchEngine(0, max_records=1 << 15, max_in_bytes=max_in)
    configure(e)
    return e


def configure(e):
    from calfkit.engine import ToolTemplate
    e.register_topics(["tool.get_weather.input", "tool.get_weather.output", "weather_agent.input"], num_partitions=8)
    e.set_tool_node("tool.get_weather.output", ToolTemplate.from_format("It's sunny in {location}"))


def spans(ix, i):
    """(value, key, correlation id) of record i through the host view of the last fetch"""
    d = ix["data"]
    val = d[int(ix["val_off"][i]):int(ix["val_off"][i]) + int(ix["val_len"][i])].tobytes()
    key = None if ix["key_len"][i] < 0 else d[int(ix["key_off"][i]):int(ix["key_off"][i]) + int(ix["key_len"][i])].tobytes()
    corr = None if ix["corr_len"][i] < 0 else d[int(ix["corr_off"][i]):int(ix["corr_off"][i]) + int(ix["corr_len"][i])].tobytes()
    return val, key, corr


def oracle_spans(batch_bytes):
    return [(r.value, r.key, dict(r.headers).get("correlation_id")) for r in kb.decode_batches(batch_bytes)]


def submit(e, buf):
    n = e.submit_recordbatch(np.frombuffer(bytes(buf), dtype=np.uint8))
    e.tool_plan()
    out = e.fetch()
    return n, e._rb, out


def publishes(out):
    return [(p.topic, p.key, p.payload) for p in out.publishes()]


@pytest.mark.parametrize("name", [n for n, _s, _b in GOLDEN])
def test_golden_batch_spans_and_columns(name):
    """every golden LZ4 batch: value / key / correlation_id spans equal the oracle's records of the decompressed batch, and
    the walker's columns and the publishes equal those of the same batch submitted uncompressed"""
    _n, spec, batch = next(c for c in GOLDEN if c[0] == name)
    plain = uncompressed(spec)
    assert lz.decompress_batch(batch) == plain
    want = oracle_spans(plain)
    e = tool_engine()
    try:
        n, ix, out = submit(e, batch)
        assert n == len(want) and ix["bad"].sum() == 0
        base = ix["data"].base
        assert base >= len(batch) and all(int(o) >= base for o in ix["val_off"])
        assert [spans(ix, i) for i in range(n)] == want
        cols, pubs = out.cols.copy(), publishes(out)
        n2, ix2, out2 = submit(e, plain)
        assert n2 == n and ix2["bad"].sum() == 0 and isinstance(ix2["data"], np.ndarray)
        assert [spans(ix2, i) for i in range(n)] == want
        assert (out2.cols == cols).all() and publishes(out2) == pubs
    finally:
        e.close()


# ---- LZ4 frames made here: a literals-only block (valid), and the malformed classes ----------------------------------
def lit_block(data: bytes) -> bytes:
    ll = len(data)
    out = bytes([min(ll, 15) << 4])
    if ll >= 15:
        r = ll - 15
        out += b"\xff" * (r // 255) + bytes([r % 255])
    return out + data


def lz4_frame(blocks, flg=0x60, bd=0x40, content=None, csum=None, extra=b"", end=True, dict_id=None):
    """an LZ4 frame: blocks = [(size word, data)]; HC is recomputed over whatever the descriptor holds"""
    desc = bytes([flg, bd]) + (struct.pack("<Q", len(content)) if flg & 8 else b"") + (struct.pack("<I", dict_id) if dict_id is not None else b"")
    out = struct.pack("<I", lz.MAGIC) + desc + bytes([(lz.xxh32(desc) >> 8) & 0xFF])
    for w, d in blocks:
        out += struct.pack("<I", w) + d
    if end:
        out += b"\0\0\0\0"
    if flg & 4:
        out += struct.pack("<I", lz.xxh32(content) if csum is None else csum)
    return out + extra


def tool_batches(n_batches, per, seed):
    from calfkit import synth
    recs = synth.tool_events(n_batches * per, seed=seed)
    out = []
    for b in range(n_batches):
        krecs = [kb.calfkit_record(r, f"id-{seed}-{b}-{i}", keyed=i % 3 != 2) for i, r in enumerate(recs[b * per:(b + 1) * per])]
        out.append(kb.encode_batch(krecs, base_offset=100 * b, base_timestamp=1767225600000 + b))
    return out


def malformed(batch):
    """{class: LZ4 batch} for one uncompressed batch (its records section is small: one 64 KB block); every CRC32C is valid"""
    sec = batch[61:]
    assert 40 < len(sec) < 60000
    seq = lambda lit, off, ml: bytes([(min(len(lit), 15) << 4) | min(ml - 4, 15)]) + \
        (b"" if len(lit) < 15 else b"\xff" * ((len(lit) - 15) // 255) + bytes([(len(lit) - 15) % 255])) + lit + struct.pack("<H", off) + \
        (b"" if ml - 4 < 15 else b"\xff" * ((ml - 19) // 255) + bytes([(ml - 19) % 255]))  # noqa: E731
    good = lit_block(sec)
    frames = {
        "offset 0": lz4_frame([(len(b := seq(sec[:20], 0, 8) + lit_block(sec[28:])), b)]),
        "offset before the output": lz4_frame([(len(b := seq(sec[:20], 21, 8) + lit_block(sec[28:])), b)]),
        "literal run past the block": lz4_frame([(len(good) - 5, good[:-5])]),
        "block size past the frame": lz4_frame([(len(good) + 9, good)]),
        "size word larger than blockMax": lz4_frame([(0x80000000 | 65537, sec + b"\0" * (65537 - len(sec)))]),
        "block decodes larger than blockMax": lz4_frame([(len(b := seq(sec[:1], 1, 70000) + lit_block(sec[1:13])), b)]),
        "wrong HC": None,
        "wrong content checksum": lz4_frame([(len(good), good)], flg=0x64, content=sec, csum=lz.xxh32(sec) ^ 1),
        "dictionary id": lz4_frame([(len(good), good)], flg=0x61, dict_id=7),
        "missing end mark": lz4_frame([(len(good), good)], end=False),
        "bytes after the end mark": lz4_frame([(len(good), good)], extra=b"\0"),
    }
    f = bytearray(lz4_frame([(len(good), good)]))
    f[6] ^= 0x55
    frames["wrong HC"] = bytes(f)
    out = {}
    for k, fr in frames.items():
        if k != "dictionary id":                                # the restatement decodes it against an empty dictionary;
            with pytest.raises(ValueError):                     # Kafka never sets one, and the device refuses it
                lz.decompress_frame(fr)
        out[k] = with_section(batch, fr)
    return out


def test_mixed_fetch():
    """uncompressed batches, LZ4 batches (liblz4's and literals-only ones), a gzip batch, every malformed LZ4 class with a
    valid CRC32C, and a truncated tail, in one fetch submitted once: exactly the malformed and gzip batches' records are
    CK_BAD_FRAME, every other record reads and walks as the oracle says"""
    from calfkit.engine._lib import CK_BAD_FRAME, COL
    plain = tool_batches(3, 30, seed=501)
    lit_src = tool_batches(2, 20, seed=502)
    lz_lit = [with_section(b, lz4_frame([(len(lb := lit_block(b[61:])), lb)])) for b in lit_src]
    gold = [b for n, _s, b in GOLDEN if n in ("b64k_linked", "b64k_all_flags")]
    gz_src = tool_batches(1, 10, seed=503)[0]
    bad_src = tool_batches(1, 12, seed=504)[0]
    # (batch in the fetch, whether its records are good, the uncompressed batch it stands for)
    parts = [(b, True, b) for b in plain[:2]] + [(b, True, s) for b, s in zip(lz_lit, lit_src)] + \
        [(b, True, lz.decompress_batch(b)) for b in gold] + [(with_section(gz_src, gz_src[61:], codec=1), False, gz_src)] + \
        [(plain[2], True, plain[2])] + [(b, False, bad_src) for b in malformed(bad_src).values()]
    buf = b"".join(p for p, _ok, _s in parts) + plain[0][:45]       # a truncated tail
    want, ok = [], []
    for _p, good, src in parts:
        recs = oracle_spans(src)
        want += recs
        ok += [good] * len(recs)
    e = tool_engine()
    try:
        n, ix, out = submit(e, buf)
        assert n == len(want)
        ok = np.array(ok)
        assert (ix["bad"] == ~ok).all()
        st = out.cols[COL["STATUS"]]
        assert (st[~ok] == CK_BAD_FRAME).all() and not (st[ok] == CK_BAD_FRAME).any()
        for i in np.nonzero(ok)[0]:
            assert spans(ix, int(i)) == want[i]
    finally:
        e.close()


def test_grow_determinism_and_unchanged_path():
    """a small LZ4 fetch, then one whose bound (4 MB blocks) exceeds the fetch buffer: the second decodes right after the
    buffer grew; the same fetch twice gives identical columns and publishes; an uncompressed fetch afterwards gives what a
    fresh engine gives, with the same kernel launches"""
    small = next(b for n, _s, b in GOLDEN if n == "b64k_content_size")
    big_name, big_spec, big = next(c for c in GOLDEN if c[0] == "b4m_content_checksum")
    e, fresh = tool_engine(), tool_engine()
    try:
        n, ix, _out = submit(e, small)
        assert ix["bad"].sum() == 0
        runs = []
        for _ in range(2):
            n, ix, out = submit(e, big + small)
            assert ix["bad"].sum() == 0
            assert [spans(ix, i) for i in range(n)] == oracle_spans(uncompressed(big_spec)) + oracle_spans(lz.decompress_batch(small))
            runs.append((out.cols.copy(), publishes(out), ix["data"].decoded.copy()))
        assert (runs[0][0] == runs[1][0]).all() and runs[0][1] == runs[1][1] and (runs[0][2] == runs[1][2]).all()
        plain = b"".join(tool_batches(3, 40, seed=505))
        l0, f0 = e.launch_count(), fresh.launch_count()
        n, ix, out = submit(e, plain)
        n2, ix2, out2 = submit(fresh, plain)
        assert e.launch_count() - l0 == fresh.launch_count() - f0
        assert isinstance(ix["data"], np.ndarray)
        for k in ("val_off", "val_len", "key_off", "key_len", "corr_off", "corr_len", "bad"):
            assert (ix[k] == ix2[k]).all(), k
        assert (out.cols == out2.cols).all() and publishes(out) == publishes(out2)
    finally:
        e.close()
        fresh.close()


@pytest.mark.parametrize("nparts", [8, 1000])
@pytest.mark.parametrize("window", [64 << 10, 1 << 20])
def test_lane_consumes_lz4_frames_of_a_tool_step(nparts, window):
    """engine A frames a config-2-shaped tool step with compression on and off; each set of frames, concatenated, is one
    fetch response for a Worker lane B.  B reads every record as A published it, and B's publishes — topic, key,
    payload — are the same byte for byte for the LZ4 fetch and the uncompressed one"""
    from calfkit import synth
    from calfkit.engine.lane import FetchArena, Lane, PinnedPool
    from test_gpu_kafka_frames import tool_engine as frame_engine, tool_step
    recs = synth.tool_events(3000, seed=511) + synth.tool_events(200, seed=512, size=4000, jitter=3000)
    got = {}
    for codec in (None, "lz4"):
        a = frame_engine(nparts)
        try:
            a.set_frame_compression(codec)
            _out, frames = tool_step(a, recs, window)
            fetch = b"".join(f.tobytes() for _t, _p, f, _n in frames)
            values = [r.value for t, _p, f, _n in frames
                      for r in kb.decode_batches(lz.decompress_batch(f.tobytes()) if codec else f.tobytes())]
        finally:
            a.close()
        assert (fetch[22] & 7) == (3 if codec else 0)
        pool = PinnedPool()
        lane = Lane(0, configure, pool, max_records=1 << 14, max_in_bytes=64 << 20)
        try:
            lane.submit(FetchArena.of(fetch, pool))
            batch = lane.collect()
            src = batch.source
            assert src.n == len(values) and src.bad.sum() == 0
            assert [src.record(i) for i in range(src.n)] == values
            if codec:
                assert lane.d2h_bytes >= src.data.decoded.nbytes > 0
            got[codec] = [(t, k, p) for t, k, p, _j in batch.iter_records()]
            batch.release()
        finally:
            lane.close()
            pool.close()
    assert got["lz4"] == got[None]
