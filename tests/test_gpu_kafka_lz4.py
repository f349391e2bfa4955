"""LZ4-compressed frames built on the device (ck_set_option 3 = 3, csrc/ck_kafka.cuh): every frame is a batch with
attributes 3 whose records section is one LZ4 frame (04224D18 60 40 82, independent 64 KB blocks), its CRC32C is valid over
the compressed bytes, and decompressed (tests/kafka_lz4.py, pinned to liblz4 in tests/test_lz4_oracle.py) it equals, byte
for byte, the uncompressed frame the Kafka oracle expects — with the plan, frame order, topic, partition and record counts
of the uncompressed pass.  Where the GPU machine has liblz4, LZ4F_decompress decodes every frame as well."""
import ctypes
import ctypes.util
import struct

import numpy as np
import pytest

import kafka_lz4 as lz
from test_gpu_kafka_frames import FRAME_TOPICS, TS, check_frames, groups_of, tool_engine, tool_step

pytestmark = pytest.mark.gpu

LZ4_HDR = bytes.fromhex("04224D18604082")


@pytest.fixture(autouse=True)
def _cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def _liblz4():
    name = ctypes.util.find_library("lz4")
    if not name:
        return None
    L = ctypes.CDLL(name)
    L.LZ4F_createDecompressionContext.argtypes = [ctypes.POINTER(ctypes.c_void_p), ctypes.c_uint]
    L.LZ4F_freeDecompressionContext.argtypes = [ctypes.c_void_p]
    L.LZ4F_decompress.restype = ctypes.c_size_t
    L.LZ4F_decompress.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.POINTER(ctypes.c_size_t), ctypes.c_char_p,
                                  ctypes.POINTER(ctypes.c_size_t), ctypes.c_void_p]
    L.LZ4F_isError.argtypes = [ctypes.c_size_t]
    return L


LIBLZ4 = _liblz4()


def liblz4_decompress(frame: bytes, size: int) -> bytes:
    """a second decoder: liblz4's LZ4F_decompress over a whole LZ4 frame of `size` content bytes"""
    ctx = ctypes.c_void_p()
    assert LIBLZ4.LZ4F_createDecompressionContext(ctypes.byref(ctx), 100) == 0
    try:
        out = ctypes.create_string_buffer(size + 1)
        got, pos = bytearray(), 0
        while True:
            dst_n, src_n = ctypes.c_size_t(len(out)), ctypes.c_size_t(len(frame) - pos)
            r = LIBLZ4.LZ4F_decompress(ctx, out, ctypes.byref(dst_n), frame[pos:], ctypes.byref(src_n), None)
            assert not LIBLZ4.LZ4F_isError(r), r
            got += out.raw[:dst_n.value]
            pos += src_n.value
            if r == 0:
                break
            assert src_n.value or dst_n.value
        assert pos == len(frame)
        return bytes(got)
    finally:
        LIBLZ4.LZ4F_freeDecompressionContext(ctx)


def blocks_of(section: bytes):
    """(size word, data) of every block of a device LZ4 frame"""
    pos, out = 7, []
    while True:
        w = struct.unpack_from("<I", section, pos)[0]
        if w == 0:
            assert pos + 4 == len(section)
            return out
        out.append((w, section[pos + 4:pos + 4 + (w & 0x7FFFFFFF)]))
        pos += 4 + (w & 0x7FFFFFFF)


def check_lz4_frame(f: bytes) -> bytes:
    """the checks every compressed frame meets; returns its uncompressed equivalent"""
    from oracle import kafka_batch as kb
    assert struct.unpack_from(">h", f, 21)[0] == 3                   # attributes: LZ4, CreateTime
    assert f[kb.HEADER_LEN:kb.HEADER_LEN + 7] == LZ4_HDR
    assert kb.crc32c(f[kb.CRC_FROM:]) == struct.unpack_from(">I", f, 17)[0]
    u = lz.decompress_batch(f)
    nblk = len(blocks_of(f[kb.HEADER_LEN:]))
    assert nblk == -(-(len(u) - kb.HEADER_LEN) // 65536)              # one block per 64 KB of records
    assert len(f) <= len(u) + 4 * nblk + 11
    if LIBLZ4 is not None:
        assert liblz4_decompress(f[kb.HEADER_LEN:], len(u) - kb.HEADER_LEN) == u[kb.HEADER_LEN:]
    return u


def decompressed(frames):
    """Frames of an LZ4 pass -> [(topic, partition, uncompressed frame as uint8, records)] after check_lz4_frame"""
    return [(t, p, np.frombuffer(check_lz4_frame(f.tobytes()), dtype=np.uint8), n) for t, p, f, n in frames]


def snapshot(frames):
    return frames.table.copy(), frames.data.tobytes()


def tool_recs():
    from calfkit import synth
    return synth.tool_events(1500, seed=91) + synth.tool_events(150, seed=92, size=None, full_history=True) + \
        synth.tool_events(200, seed=93, size=9000, jitter=8000)


@pytest.mark.parametrize("nparts,window", [(8, 4 << 10), (8, 64 << 10), (8, 1 << 20), (1000, 1 << 20)])
def test_tool_step_lz4_frames_match_oracle(nparts, window):
    """config-2-shaped tool steps: the compressed frames decompress to the oracle's frames, in the uncompressed pass's
    order with its table; the same step twice gives identical bytes; option 3 back to 0 gives the uncompressed pass"""
    recs = tool_recs()
    e = tool_engine(nparts)
    try:
        out, plain = tool_step(e, recs, window)
        plain = snapshot(plain)
        e.set_frame_compression("lz4")
        out, frames = tool_step(e, recs, window)
        groups = groups_of(out, FRAME_TOPICS, nparts)
        check_frames(decompressed(frames), groups, window, nparts)
        for k in ("topic_id", "partition", "n_records", "first"):
            assert (frames.table[k] == plain[0][k]).all()
        comp, raw = int(frames.table["length"].sum()), int(plain[0]["length"].sum())
        if window == 1 << 20:
            assert comp * 3 <= raw, (comp, raw)                  # liblz4 reaches 1/6 on these records
        first = snapshot(frames)
        _out, again = tool_step(e, recs, window)
        assert again.data.tobytes() == first[1] and (again.table == first[0]).all()
        e.set_frame_compression(None)
        _out, back = tool_step(e, recs, window)
        assert back.data.tobytes() == plain[1] and (back.table == plain[0]).all()
    finally:
        e.close()


def _record_value(section_len: int, fill) -> bytes:
    """a value whose unkeyed record without a correlation id (offsetDelta 0) is exactly section_len bytes"""
    from oracle import kafka_batch as kb
    n = section_len - 40
    while True:
        v = fill(n)
        r = len(kb.encode_record(kb.KRecord(v, None, [("content-type", b"application/json")]), 0, 0))
        if r == section_len:
            return v
        n += section_len - r


def _json_fill(n: int) -> bytes:
    from calfkit import synth
    src = b"".join(synth.tool_events(max(1, n // 900 + 1), seed=131))
    return (src * (n // len(src) + 1))[:n]


def _record_form(e, values, window=1 << 20, keyed=False):
    """values as records of one topic through the record form: compressed frames checked, decompressed frames against
    the oracle; returns (compressed frames, uncompressed frames)"""
    from oracle import kafka_batch as kb
    from test_gpu_parity import _murmur2
    records = [(v, f"k{i}".encode() if keyed else None, None) for i, v in enumerate(values)]
    e.set_frame_bytes(window)
    e.set_frame_compression("lz4")
    e.encode_frames_records("weather_agent.input", records, TS)
    frames = e.fetch_frames()
    dec = decompressed(frames)
    groups = {}
    for value, key, _cid in records:
        part = (_murmur2(key) & 0x7FFFFFFF) % e.num_partitions if key is not None else -1
        groups.setdefault(("weather_agent.input", part), []).append(kb.KRecord(value, key, [("content-type", b"application/json")]))
    check_frames(dec, {g: groups[g] for g in sorted(groups, key=lambda g: g[1])}, window, e.num_partitions)
    return frames, dec


def _case(name):
    """(values, window, keyed) of a record-form case"""
    rng = np.random.default_rng(132)
    base = rng.integers(0, 256, 65536, dtype=np.uint8).tobytes()
    if name.startswith("section_"):                              # one record whose records section is that long
        return [_record_value(int(name[8:]), _json_fill)], 1 << 20, False
    return {"five_mib": ([_json_fill(50_000 + 37 * i) for i in range(104)], 6 << 20, False),
            "one_byte": ([b"a" * 300_000], 1 << 20, False),
            "period_65535": ([(base[:65535] * 4)[:200_000]], 1 << 20, False),
            "period_65536": ([(base * 4)[:200_000]], 1 << 20, False),
            "short": ([b"", b"x", b"ab" * 7], 1 << 20, False),
            "random": ([rng.integers(0, 256, int(n), dtype=np.uint8).tobytes() for n in rng.integers(1, 40_000, 60)], 256 << 10, True),
            }[name]


@pytest.mark.parametrize("name", ["section_65535", "section_65536", "section_65537", "section_131085", "five_mib", "one_byte",
                                  "period_65535", "period_65536", "short", "random"])
def test_record_form_lz4_frames(name):
    """records sections of 64 KB - 1, 64 KB, 64 KB + 1 and 128 KB + 13 bytes, a 5 MiB frame, one repeated byte (matches
    reach the block end), periods at the offset limit, short values, and random values (stored blocks only)"""
    values, window, keyed = _case(name)
    e = tool_engine(8)
    try:
        frames, dec = _record_form(e, values, window, keyed)
        if name.startswith("section_"):
            assert len(frames) == 1 and len(dec[0][2]) == 61 + int(name[8:]) and len(frames.frame(0)) * 3 < len(dec[0][2])
        if name == "five_mib":
            assert len(frames) == 1 and len(dec[0][2]) > 5 << 20
        if name == "one_byte":
            assert len(frames.frame(0)) < 3000
        if name == "random":
            assert all(w >> 31 for _t, _p, f, _n in frames for w, _d in blocks_of(f.tobytes()[61:]))
    finally:
        e.close()


def test_grow_path_rewrites_everything():
    """frames larger than the first frame buffer: compressible ones (the scratch of the uncompressed frames is too small,
    the compressed frames fit) and then random ones (the frame buffer is too small) are written again into grown buffers"""
    from calfkit.engine import BatchEngine
    rng = np.random.default_rng(134)
    e = BatchEngine(0, max_records=64, max_in_bytes=24 << 20, max_out_bytes=1 << 20)
    try:
        e.register_topics(["weather_agent.input"], num_partitions=8)
        cap = 2 * e.max_out + 160 * 2 * e.max_payloads + 4096
        for kind in ("json", "random"):
            values = [_json_fill(150_000 + i) if kind == "json" else rng.integers(0, 256, 150_000, dtype=np.uint8).tobytes()
                      for i in range(40)]
            assert sum(map(len, values)) > 2 * cap
            _record_form(e, values, window=1 << 20, keyed=True)
    finally:
        e.close()


def test_encode_recordbatch_with_lz4():
    from calfkit import synth
    from oracle import kafka_batch as kb
    recs = synth.tool_events(4000, seed=71) + synth.tool_events(300, seed=72, size=None, full_history=True)
    e = tool_engine(8, max_records=1 << 15)
    try:
        b = synth.pack(recs)
        e.submit(b.data, b.offsets)
        e.tool_plan()
        out = e.fetch()
        groups = groups_of(out, ["weather_agent.input", "tool.get_weather.output"], 8)
        tid = e.topic_ids["weather_agent.input"]
        live = np.nonzero(out.pubs["payload"] != 0xFFFFFFFF)[0]
        e.set_frame_compression("lz4")
        for part in (0, 5):
            idx = live[(out.pubs["topic_id"][live] == tid) & (out.pubs["partition"][live] == part)]
            frame = e.encode_recordbatch(idx, base_offset=5000 + part, timestamp_ms=TS).tobytes()
            want = kb.encode_batch(groups[("weather_agent.input", part)], base_offset=5000 + part, base_timestamp=TS)
            assert check_lz4_frame(frame) == want
            assert len(frame) * 3 < len(want)
        from calfkit.exceptions import EngineError
        with pytest.raises(EngineError, match="zstd"):
            e.set_frame_compression("zstd")
        with pytest.raises(EngineError, match="codec"):
            e._check(e.lib.ck_set_option(e.h, 3, 2))
    finally:
        e.close()


def _worker_frames(buf, codec):
    """one Worker over the fetch response `buf` with frame sinks on both output topics; returns the (topic, partition, key,
    value) of every record framed, after decompression when compressed"""
    import asyncio
    import tools_def
    from calfkit import Client, Worker, agent_tool
    from calfkit.engine.lane import FetchArena, PinnedPool
    from oracle import kafka_batch as kb
    client = Client.connect("localhost", compression_type=codec)
    pool = PinnedPool()
    client.broker.produce_fetch("tool.get_weather.input", FetchArena.of(buf, pool))
    got, n_lz4 = [], [0]

    def on_frame(topic, part, frame, n):
        f = frame.tobytes()
        if codec == "lz4":
            f = check_lz4_frame(f)
            n_lz4[0] += 1
        else:
            assert f[22] & 7 == 0
        recs = kb.decode_batches(f)
        assert len(recs) == n
        got.extend((topic, part, r.key, r.value) for r in recs)
    for t in ("weather_agent.input", "tool.get_weather.output"):
        client.broker.frame_sink(t, on_frame)
    node_def = agent_tool(tools_def.get_weather, device_template="It's sunny in {location}")
    worker = Worker(client, nodes=[node_def], batch_records=256, batch_bytes=8 << 20, lanes=3, route_topics=["weather_agent.input"])
    asyncio.run(worker.run(until_idle=True))
    stats = dict(worker.stats)
    worker.close()
    pool.close()
    return sorted(got, key=repr), stats, n_lz4[0]


def test_worker_lz4_frames_equal_the_uncompressed_worker():
    """Worker.run over fetch responses with MemoryBroker(compression_type="lz4") and frame sinks: lane frames and the
    record form (records the device declines are framed by flush_frames) decompress to what the same Worker frames
    with compression off"""
    from calfkit import synth
    from test_gpu_kafka import frames_of
    recs = synth.tool_events(1200, seed=101) + synth.tool_events(100, seed=102, size=None, full_history=True)
    recs[7] = recs[7].replace(b'"args":{"location":"', b'"args":"{\\"location\\":\\"').replace(b'"},"tool_call_id"', b'\\"}","tool_call_id"', 1)
    buf, _krecs = frames_of(recs, [40] * 30 + [100])
    plain, st, _n = _worker_frames(buf, None)
    comp, st2, n_lz4 = _worker_frames(buf, "lz4")
    assert comp == plain and len(plain) >= len(recs)
    assert st2["host_fallback"] == st["host_fallback"] == 1 and n_lz4 > 0


def test_block_compressor_alone():
    """ck_lz4_block (csrc/ck_lz4.cuh) through tests/lz4sim: 1 B - 64 KB blocks of one byte, random bytes, periodic bytes
    and records, and blocks whose one match ends 12, 5, 13 or 4 bytes before the end, decoded by the oracle; a block
    comes back only when it shrank, and the same blocks give the same bytes"""
    import lz4sim
    import torch
    rng = np.random.default_rng(135)
    rand = lambda n: rng.integers(0, 256, n, dtype=np.uint8).tobytes()  # noqa: E731
    blocks = []
    for n in (1, 2, 12, 13, 14, 16, 17, 31, 32, 33, 64, 100, 255, 256, 1000, 4096, 65535, 65536):
        blocks += [b"z" * n, rand(n), (b"0123456789abcdef" * (n // 16 + 1))[:n], _json_fill(n)]
    for n in (60, 1000, 65536):
        for tail in (12, 5, 13, 4):
            head = rand(20)
            blocks.append(head + rand(n - 40 - tail) + head + rand(tail))
    blocks += [(rand(p) * (65536 // p + 1))[:65536] for p in (1, 3, 7, 251, 4096, 30000)]
    off = np.concatenate(([0], np.cumsum([len(b) for b in blocks]))).astype(np.int64)
    src = torch.from_numpy(np.frombuffer(b"".join(blocks) + b"\0" * 256, dtype=np.uint8).copy()).cuda()
    d_off = torch.from_numpy(off).cuda()
    runs = []
    for _ in range(2):
        dst = torch.zeros(int(off[-1]) + 256, dtype=torch.uint8, device="cuda")
        out_len = torch.zeros(len(blocks), dtype=torch.int32, device="cuda")
        assert lz4sim.lib().lz4sim_blocks(src.data_ptr(), d_off.data_ptr(), len(blocks), dst.data_ptr(), out_len.data_ptr()) == 0
        runs.append((dst.cpu().numpy().tobytes(), out_len.cpu().numpy()))
    assert runs[0][0] == runs[1][0] and (runs[0][1] == runs[1][1]).all()
    data, lens = runs[0]
    for i, b in enumerate(blocks):
        z = int(lens[i])
        assert z < len(b) or z == 0
        if z:
            out = bytearray()
            lz.decompress_block(data[off[i]:off[i] + z], out, 65536)
            assert bytes(out) == b, i
    assert (lens > 0).sum() > len(blocks) // 3 and all(int(lens[i]) == 0 for i, b in enumerate(blocks) if len(b) < 13)
