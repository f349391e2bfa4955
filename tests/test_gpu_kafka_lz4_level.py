"""LZ4 frames at a compression level (ck_set_option 4, Kafka's compression.lz4.level): levels 1 and 2 build the frames
of the default parse byte for byte, levels 3 and up the hash-chain parse (ck_lz4_block_hc), whose frames decompress to
the uncompressed pass's frames, are deterministic, and are never larger in total than the default parse's."""
import asyncio
import struct

import numpy as np
import pytest

import kafka_lz4 as lz
from test_gpu_kafka_frames import FRAME_TOPICS, TS, tool_engine, tool_step
from test_gpu_kafka_lz4 import LIBLZ4, LZ4_HDR, _json_fill, check_lz4_frame, liblz4_decompress, snapshot, tool_recs

pytestmark = pytest.mark.gpu

DEPTH_CAP = 256                                               # CK_LZ_HC_DEPTH_CAP, reached at level 9


@pytest.fixture(autouse=True)
def _cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def _hc_blocks(blocks, depth):
    """every block through ck_lz4_block_hc at `depth` (tests/lz4hc), its chains full of stale entries: (bytes, lengths)"""
    import lz4hc
    import torch
    off = np.concatenate(([0], np.cumsum([len(b) for b in blocks]))).astype(np.int64)
    src = torch.from_numpy(np.frombuffer(b"".join(blocks) + b"\0" * 256, dtype=np.uint8).copy()).cuda()
    d_off = torch.from_numpy(off).cuda()
    dst = torch.zeros(int(off[-1]) + 256, dtype=torch.uint8, device="cuda")
    out_len = torch.zeros(len(blocks), dtype=torch.int32, device="cuda")
    chains = torch.randint(-32768, 32767, (len(blocks) * 65536,), dtype=torch.int16, device="cuda")
    assert lz4hc.lib().lz4hc_blocks(src.data_ptr(), d_off.data_ptr(), len(blocks), dst.data_ptr(), out_len.data_ptr(),
                                         chains.data_ptr(), depth) == 0
    return dst.cpu().numpy().tobytes(), out_len.cpu().numpy(), off


def test_hash_chain_block_compressor_alone():
    """ck_lz4_block_hc at every depth from 1 to the cap over 1 B - 64 KB blocks of one byte, random bytes (stored raw),
    periodic bytes, periods at the offset limit and config-2 JSON, and blocks whose one match ends 12, 5, 13 or 4 bytes
    before the end: each block decodes through the oracle (which enforces the block rules) and, as a one-block LZ4
    frame, through liblz4 where it is installed; the same blocks give the same bytes"""
    rng = np.random.default_rng(141)
    rand = lambda n: rng.integers(0, 256, n, dtype=np.uint8).tobytes()  # noqa: E731
    blocks, random = [], set()
    for n in (1, 2, 12, 13, 14, 16, 17, 31, 32, 33, 64, 100, 255, 256, 1000, 4096, 65535, 65536):
        random.add(len(blocks) + 1)
        blocks += [b"z" * n, rand(n), (b"0123456789abcdef" * (n // 16 + 1))[:n], _json_fill(n)]
    for n in (60, 1000, 65536):
        for tail in (12, 5, 13, 4):
            head = rand(20)
            blocks.append(head + rand(n - 40 - tail) + head + rand(tail))
    base = rand(65535)
    blocks += [(base * 2)[:65536], (base[:30000] * 3)[:65536]]
    blocks += [(rand(p) * (65536 // p + 1))[:65536] for p in (1, 3, 7, 251, 4096)]
    depth = 1
    while depth <= DEPTH_CAP:
        data, lens, off = _hc_blocks(blocks, depth)
        again = _hc_blocks(blocks, depth)
        assert data == again[0] and (lens == again[1]).all()
        for i, b in enumerate(blocks):
            z = int(lens[i])
            assert z < len(b) or z == 0
            if len(b) < 13 or (i in random and len(b) >= 64):
                assert z == 0, (depth, i)
            if not z:
                continue
            blk = data[off[i]:off[i] + z]
            out = bytearray()
            lz.decompress_block(blk, out, 65536)
            assert bytes(out) == b, (depth, i)
            if LIBLZ4 is not None:
                assert liblz4_decompress(LZ4_HDR + struct.pack("<I", z) + blk + b"\0" * 4, len(b)) == b
        assert int(lens[-5]) and int(lens[-5]) < 300                # one repeated byte: matches run to the block end
        depth *= 2


def _frames(fr):
    return [(t, p, f.tobytes(), n) for t, p, f, n in fr]


@pytest.mark.parametrize("nparts,window", [(8, 4 << 10), (8, 64 << 10), (8, 1 << 20), (1000, 4 << 10), (1000, 64 << 10), (1000, 1 << 20)])
def test_tool_step_levels(nparts, window):
    """config-2-shaped tool steps at levels 1, 3, 6, 9, 12 and 17: levels 1 and 2 (and the level set back to none) give the
    bytes of a pass that sets no level; from 3, every frame decompresses to the uncompressed pass's frame (header
    fields equal apart from attributes, batchLength and CRC), two passes give the same bytes, the total is no larger
    than the default parse's, and levels above the cap give the cap's frames"""
    recs = tool_recs()
    e = tool_engine(nparts)
    try:
        _out, plain = tool_step(e, recs, window)
        plain_tab, plain_frames = plain.table.copy(), _frames(plain)
        e.set_frame_compression("lz4")
        _out, f0 = tool_step(e, recs, window)
        default = snapshot(f0)
        total0 = int(default[0]["length"].sum())
        by_level = {}
        for level in (1, 2, 3, 6, 9, 12, 17):
            e.set_frame_compression("lz4", level)
            _out, fr = tool_step(e, recs, window)
            snap = snapshot(fr)
            by_level[level] = snap
            if level < 3:
                assert snap[1] == default[1] and (snap[0] == default[0]).all(), level
                continue
            for k in ("topic_id", "partition", "n_records", "first"):
                assert (snap[0][k] == plain_tab[k]).all()
            got = _frames(fr)
            assert len(got) == len(plain_frames)
            for (t, p, f, n), (t0, p0, f0_, n0) in zip(got, plain_frames):
                assert (t, p, n) == (t0, p0, n0) and check_lz4_frame(f) == f0_
            assert int(snap[0]["length"].sum()) <= total0, (level, int(snap[0]["length"].sum()), total0)
            _out, again = tool_step(e, recs, window)
            assert again.data.tobytes() == snap[1] and (again.table == snap[0]).all()
        assert by_level[12][1] == by_level[17][1] == by_level[9][1]
        e.set_frame_compression("lz4")
        _out, back = tool_step(e, recs, window)
        assert back.data.tobytes() == default[1] and (back.table == default[0]).all()
    finally:
        e.close()


def _record_pass(e, values, level, window=1 << 20):
    records = [(v, f"k{i}".encode(), None) for i, v in enumerate(values)]
    e.set_frame_bytes(window)
    e.set_frame_compression("lz4", level)
    e.encode_frames_records("weather_agent.input", records, TS)
    fr = e.fetch_frames()
    return snapshot(fr), _frames(fr)


@pytest.mark.parametrize("kind", ["json", "random"])
def test_grow_paths_at_level_9(kind):
    """frames larger than the first buffers at level 9: compressible records (the scratch of the uncompressed frames
    grows) and random ones (the frame buffer grows) are written again at the pass's level, byte for byte what the same
    pass gives when it fits the first time; they decompress to the default parse's frames"""
    from calfkit.engine import BatchEngine
    rng = np.random.default_rng(142)
    e = BatchEngine(0, max_records=64, max_in_bytes=24 << 20, max_out_bytes=1 << 20)
    try:
        e.register_topics(["weather_agent.input"], num_partitions=8)
        cap = 2 * e.max_out + 160 * 2 * e.max_payloads + 4096
        values = [_json_fill(150_000 + i) if kind == "json" else rng.integers(0, 256, 150_000, dtype=np.uint8).tobytes()
                  for i in range(40)]
        assert sum(map(len, values)) > 2 * cap
        grown, grown_frames = _record_pass(e, values, 9)
        fit, _f = _record_pass(e, values, 9)
        assert fit[1] == grown[1] and (fit[0] == grown[0]).all()
        _default, default_frames = _record_pass(e, values, None)
        assert [check_lz4_frame(f) for _t, _p, f, _n in grown_frames] == [check_lz4_frame(f) for _t, _p, f, _n in default_frames]
    finally:
        e.close()


def test_encode_recordbatch_at_a_level():
    """ck_encode_recordbatch at level 9 gives a frame that decompresses to the oracle's; the level back to none gives the
    default parse's frame again; the ABI refuses level 18 naming it"""
    from calfkit import synth
    from calfkit.exceptions import EngineError
    from oracle import kafka_batch as kb
    from test_gpu_kafka_frames import groups_of
    recs = synth.tool_events(4000, seed=143) + synth.tool_events(300, seed=144, size=None, full_history=True)
    e = tool_engine(8, max_records=1 << 15)
    try:
        b = synth.pack(recs)
        e.submit(b.data, b.offsets)
        e.tool_plan()
        out = e.fetch()
        groups = groups_of(out, FRAME_TOPICS, 8)
        tid = e.topic_ids["weather_agent.input"]
        live = np.nonzero(out.pubs["payload"] != 0xFFFFFFFF)[0]
        for part in (0, 5):
            idx = live[(out.pubs["topic_id"][live] == tid) & (out.pubs["partition"][live] == part)]
            want = kb.encode_batch(groups[("weather_agent.input", part)], base_offset=7000 + part, base_timestamp=TS)
            e.set_frame_compression("lz4")
            default = e.encode_recordbatch(idx, base_offset=7000 + part, timestamp_ms=TS).tobytes()
            e.set_frame_compression("lz4", 9)
            frame = e.encode_recordbatch(idx, base_offset=7000 + part, timestamp_ms=TS).tobytes()
            assert check_lz4_frame(frame) == want
            e.set_frame_compression("lz4")
            assert e.encode_recordbatch(idx, base_offset=7000 + part, timestamp_ms=TS).tobytes() == default
        with pytest.raises(EngineError, match="18"):
            e._check(e.lib.ck_set_option(e.h, 4, 18))
    finally:
        e.close()


def _run_worker(level, idempotent):
    """a Worker over tool inputs with frame sinks on its output topics and on "b.input", where each tick produces tool
    inputs for a second Worker; the "b.input" frames, fed back through produce_fetch, are that Worker's input.
    Returns (the first Worker's framed records, the second Worker's outputs, every frame of the sink log)"""
    import tools_def
    from calfkit import Client, Worker, agent_tool
    from calfkit import synth
    from calfkit.broker import Record
    from calfkit.engine.lane import FetchArena, PinnedPool
    from oracle import kafka_batch as kb
    kw = {"compression_type": "lz4"}
    if level is not None:
        kw["compression_level"] = level
    if idempotent:
        kw["enable_idempotence"] = True
    client = Client.connect("localhost", **kw)
    broker = client.broker
    recs = synth.tool_events(1200, seed=145)
    recs[7] = recs[7].replace(b'"args":{"location":"', b'"args":"{\\"location\\":\\"').replace(b'"},"tool_call_id"', b'\\"}","tool_call_id"', 1)
    broker.produce_batch([Record("tool.get_weather.input", r) for r in recs])
    b_recs = synth.tool_events(600, seed=146)
    log = []
    for t in FRAME_TOPICS + ["b.input"]:
        broker.frame_sink(t, lambda topic, part, f, n: log.append((topic, part, f.tobytes(), n)))

    def tool_worker(c):
        node = agent_tool(tools_def.get_weather, device_template="It's sunny in {location}")
        return Worker(c, nodes=[node], batch_records=128, batch_bytes=8 << 20, lanes=2, route_topics=["weather_agent.input"])
    w = tool_worker(client)
    real_step, ticks = w.step, [0]

    def step():
        k = ticks[0]
        ticks[0] += 1
        more = b_recs[40 * k:40 * (k + 1)]
        for j, r in enumerate(more):
            broker.produce(Record("b.input", r, f"k{j}".encode() if j % 3 else None))
        return real_step() + len(more)
    w.step = step
    asyncio.run(w.run(until_idle=True))
    w.close()
    first = sorted((t, r.key, r.value) for t, _p, f, _n in log if t != "b.input" for r in kb.decode_batches(check_lz4_frame(f)))

    parts, buf = [], b""
    for p in sorted({p for t, p, _f, _n in log if t == "b.input"}, key=repr):
        parts.append((len(buf), []))
        off = 0
        for t, p2, f, n in log:
            if t == "b.input" and p2 == p:
                buf += struct.pack(">q", off) + f[8:]
                off += n
    client2 = Client.connect("localhost")
    pool = PinnedPool()
    client2.broker.produce_fetch("tool.get_weather.input", FetchArena.of(buf, pool, partitions=parts))
    got = []
    for t in FRAME_TOPICS:
        client2.broker.sink(t, lambda b, idx, t=t: got.extend((t, k, p) for (_t, k, p, _j) in b.iter_records(idx)))
    w2 = tool_worker(client2)
    asyncio.run(w2.run(until_idle=True))
    for t in FRAME_TOPICS:
        got += [(t, r.key, r.value) for r in client2.broker.poll_batch((t,), 100000)]
    w2.close()
    pool.close()
    return first, sorted(got), log


def test_worker_run_at_level_9():
    """Worker.run with compression_type="lz4", compression_level=9: lane frames and record-form frames are LZ4 batches of
    the hash-chain parse that decompress to the records of the level-0 run; fed back through produce_fetch, the
    "b.input" frames give a second Worker the same outputs as the level-0 run's; with enable_idempotence the
    baseSequence patch leaves every CRC valid and the sequences contiguous per partition"""
    from oracle import kafka_batch as kb
    first0, second0, _log0 = _run_worker(None, False)
    first9, second9, log9 = _run_worker(9, True)
    assert first9 == first0 and len(first0) >= 1200
    assert second9 == second0 and len(second0) >= 600
    nxt = {}
    for t, p, f, n in log9:
        assert kb.crc32c(f[kb.CRC_FROM:]) == struct.unpack_from(">I", f, 17)[0] and f[22] & 7 == 3
        pid, _epoch, seq = struct.unpack_from(">qhi", f, 43)
        assert pid >= 0 and seq == nxt.get((t, p), 0)
        nxt[(t, p)] = seq + n
