"""Fetch responses holding zstd batches (attributes 4), decoded on the device (ck_rb_zstd_kernel, csrc/ck_kafka.cuh):
the records of every golden zstd batch read, through the host view, exactly as the Kafka oracle gives those of the
uncompressed batch, and walk and publish exactly as that batch submitted uncompressed; a mixed fetch marks exactly its
malformed zstd and its snappy batches bad; an empty frame is accepted where a refused header with the same empty slot is
not; each codec present adds one launch; the fetch buffer grows; the same fetch gives the same results; a Lane and
Worker.run consume zstd fetches as they consume plain ones."""
import os
import sys

import numpy as np
import pytest

import gzip_cases as gz
import zstd_cases as zc
import zstd_ref as zr
from make_golden_lz4_batches import load as load_lz4, with_section
from oracle import kafka_batch as kb
from test_gpu_kafka_lz4_fetch import oracle_spans, publishes, spans, submit, tool_batches, tool_engine

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
from make_golden_zstd_batches import WORKER, load, load_worker, uncompressed  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def zstd_batch(batch: bytes, **kw) -> bytes:
    """`batch` with its records section as one zstd frame (libzstd, level 3 unless kw says otherwise)"""
    return with_section(batch, zr.compress(batch[61:], **(kw or dict(level=3))), codec=4)


@pytest.mark.parametrize("name", [n for n, _s, _b in load()])
def test_golden_batch_spans_and_columns(name):
    spec, batch = {n: (s, b) for n, s, b in load()}[name]
    plain = uncompressed(spec)
    want = oracle_spans(plain)
    e = tool_engine()
    try:
        n, ix, out = submit(e, batch)
        assert n == len(want) and ix["bad"].sum() == 0
        assert [spans(ix, i) for i in range(n)] == want
        if n:
            base = ix["data"].base
            assert base >= len(batch) and all(int(o) >= base for o in ix["val_off"])
        cols, pubs = out.cols.copy(), publishes(out)
        n2, ix2, out2 = submit(e, plain)
        assert n2 == n and ix2["bad"].sum() == 0
        assert (out2.cols == cols).all() and publishes(out2) == pubs
    finally:
        e.close()


def malformed(batch):
    """{class: zstd batch} for one uncompressed batch; every CRC32C is valid"""
    out = {k: with_section(batch, z, codec=4) for k, z in zc.malformed().items()}
    good = zr.compress(batch[61:], level=3, checksum=True)
    for cut in (5, 9, len(good) - 4):
        out[f"records frame cut at {cut}"] = with_section(batch, good[:cut], codec=4)
    out["records frame with a flipped checksum"] = with_section(batch, good[:-1] + bytes([good[-1] ^ 0x80]), codec=4)
    return out


def test_mixed_fetch():
    """uncompressed, golden LZ4, gzip and zstd batches, every malformed zstd class with a valid CRC32C, a snappy batch and
    a truncated tail, in one fetch submitted once: exactly the malformed and snappy batches' records are CK_BAD_FRAME"""
    zr.need()
    from calfkit.engine._lib import CK_BAD_FRAME, COL
    import kafka_lz4 as lz
    plain = tool_batches(3, 30, seed=811)
    zs_src = tool_batches(3, 20, seed=812)
    gold = [b for n, _s, b in load_lz4() if n in ("b64k_linked", "b64k_all_flags")]
    bad_src = tool_batches(1, 12, seed=813)[0]
    other = tool_batches(2, 9, seed=814)
    parts = [(b, True, b) for b in plain[:2]] + \
        [(zstd_batch(b, level=lv, checksum=True), True, b) for b, lv in zip(zs_src, (-5, 3, 19))] + \
        [(b, True, lz.decompress_batch(b)) for b in gold] + \
        [(with_section(other[0], gz.gzip_bytes(other[0][61:]), codec=1), True, other[0])] + \
        [(b, True, uncompressed(spec)) for _n, spec, b in load()[:2]] + \
        [(plain[2], True, plain[2])] + \
        [(b, False, bad_src) for b in malformed(bad_src).values()] + \
        [(with_section(other[1], zr.compress(other[1][61:]), codec=2), False, other[1])]
    buf = b"".join(p for p, _ok, _s in parts) + plain[0][:45]
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


def test_empty_frame_is_not_a_refused_slot():
    """an empty frame has an empty slot, like a refused header, and still decodes (0 bytes); the refused header with the
    same empty slot is refused, and so is a batch that claims records of an empty frame"""
    import test_gpu_zstd as tz
    empty_ok = zc.frame([zc.block(True, 0, b"")], fcs=0, single_segment=True)
    refused = b"\x28\xb5\x2f\xfe" + empty_ok[4:]
    assert tz.run_device([empty_ok, refused], [0, 0]) == [b"", None]
    src = tool_batches(2, 5, seed=815)
    empty = kb.encode_batch([], base_offset=7, base_timestamp=1767225600000)
    frame_of = lambda b: with_section(b, zc.frame([zc.block(True, 0, b[61:])], window_log=17), codec=4)
    e = tool_engine()
    try:
        n, ix, _out = submit(e, frame_of(src[0]) + with_section(empty, empty_ok, codec=4) + frame_of(src[1]))
        assert n == 10 and ix["bad"].sum() == 0
        assert [spans(ix, i) for i in range(10)] == oracle_spans(src[0]) + oracle_spans(src[1])
        n, ix, _out = submit(e, frame_of(src[0]) + with_section(empty, refused, codec=4) + frame_of(src[1]))
        assert n == 10 and ix["bad"].sum() == 0
        n, ix, _out = submit(e, with_section(src[0], empty_ok, codec=4) + frame_of(src[1]))
        assert n == 10 and list(ix["bad"]) == [1] * 5 + [0] * 5
        assert [spans(ix, i) for i in range(5, 10)] == oracle_spans(src[1])
    finally:
        e.close()


def test_launch_counts():
    """against a fetch with no compressed batch: zstd-only adds one launch whatever the batch count; LZ4 + gzip + zstd
    adds three"""
    plain = b"".join(tool_batches(3, 10, seed=821))
    lz_b = [b for n, _s, b in load_lz4() if n == "b64k_independent"][0]
    gz_b = with_section(tool_batches(1, 10, seed=822)[0], gz.gzip_bytes(tool_batches(1, 10, seed=822)[0][61:]), codec=1)
    zss = [b for _n, _s, b in load()[:3]]
    e = tool_engine()
    try:
        def launches(buf):
            l0 = e.launch_count()
            submit(e, buf)
            return e.launch_count() - l0
        base = launches(plain)
        assert launches(plain + zss[0]) == base + 1
        assert launches(plain + b"".join(zss)) == base + 1
        assert launches(plain + zss[0] + lz_b + gz_b + zss[1]) == base + 3
        assert launches(plain) == base
    finally:
        e.close()


def test_grow_and_determinism():
    """a small zstd fetch, then the golden section of more than 4 MB, which outgrows the fetch buffer: it decodes right
    after the buffer grew; the same fetch twice gives identical columns, publishes and decoded slots"""
    g = {n: (s, b) for n, s, b in load()}
    small_spec, small = g["level3"]
    big_spec, big = g["over_4mb"]
    assert len(uncompressed(big_spec)) > 4 << 20
    e = tool_engine()
    try:
        _n, ix, _out = submit(e, small)
        assert ix["bad"].sum() == 0
        runs = []
        for _ in range(2):
            n, ix, out = submit(e, big + small)
            assert ix["bad"].sum() == 0
            assert [spans(ix, i) for i in range(n)] == oracle_spans(uncompressed(big_spec)) + oracle_spans(uncompressed(small_spec))
            runs.append((out.cols.copy(), publishes(out), ix["data"].decoded.copy()))
        assert (runs[0][0] == runs[1][0]).all() and runs[0][1] == runs[1][1] and (runs[0][2] == runs[1][2]).all()
    finally:
        e.close()


def zstd_frames(fetch: bytes, streamed: bool) -> bytes:
    """every frame of a fetch response with its records section recompressed to one zstd frame at level 3: one-shot
    (content size, single segment when small) or streamed in pieces (no content size, a window descriptor)"""
    out, pos = [], 0
    while pos + 12 <= len(fetch):
        end = pos + 12 + int.from_bytes(fetch[pos + 8:pos + 12], "big")
        f = fetch[pos:end]
        sec = zr.stream(f[61:], piece=16384, level=3) if streamed else zr.compress(f[61:], level=3)
        out.append(with_section(f, sec, codec=4))
        pos = end
    return b"".join(out)


@pytest.mark.parametrize("nparts", [8, 1000])
@pytest.mark.parametrize("window", [64 << 10, 1 << 20])
def test_lane_consumes_zstd_frames_of_a_tool_step(nparts, window):
    """engine A frames a config-2-shaped tool step; its frames, recompressed by libzstd in both header shapes, are one
    fetch response each for a Worker lane B, whose publishes equal those of the uncompressed fetch"""
    zr.need()
    from calfkit import synth
    from calfkit.engine.lane import FetchArena, Lane, PinnedPool
    from test_gpu_kafka_frames import tool_engine as frame_engine, tool_step
    from test_gpu_kafka_lz4_fetch import configure
    recs = synth.tool_events(3000, seed=841) + synth.tool_events(200, seed=842, size=4000, jitter=3000)
    a = frame_engine(nparts)
    try:
        _out, frames = tool_step(a, recs, window)
        plain = b"".join(f.tobytes() for _t, _p, f, _n in frames)
        values = [r.value for _t, _p, f, _n in frames for r in kb.decode_batches(f.tobytes())]
    finally:
        a.close()
    got = {}
    for codec, fetch in (("none", plain), ("oneshot", zstd_frames(plain, False)), ("streamed", zstd_frames(plain, True))):
        assert (fetch[22] & 7) == (0 if codec == "none" else 4)
        pool = PinnedPool()
        lane = Lane(0, configure, pool, max_records=1 << 14, max_in_bytes=64 << 20)
        try:
            lane.submit(FetchArena.of(fetch, pool))
            batch = lane.collect()
            src = batch.source
            assert src.n == len(values) and src.bad.sum() == 0
            assert [src.record(i) for i in range(src.n)] == values
            if codec != "none":
                assert lane.d2h_bytes >= src.data.decoded.nbytes > 0
            got[codec] = [(t, k, p) for t, k, p, _j in batch.iter_records()]
            batch.release()
        finally:
            lane.close()
            pool.close()
    assert got["oneshot"] == got["none"] and got["streamed"] == got["none"]


def test_worker_run_consumes_a_zstd_fetch():
    """the golden worker fetch through broker.produce_fetch and Worker.run, one of its batches corrupt (a checksummed
    frame with a flipped bit, which libzstd refuses too): the output equals the oracle's tool-node outputs for every record
    outside that batch, and stats["rejected"] counts exactly its records"""
    import tools_def
    from calfkit import synth
    from oracle import port
    from test_gpu_kafka_frames import _worker_run
    recs = synth.tool_events(WORKER["batches"] * WORKER["per"], seed=WORKER["seed"])
    lo, hi = WORKER["corrupt"] * WORKER["per"], (WORKER["corrupt"] + 1) * WORKER["per"]
    got, _parts, st = _worker_run(b"".join(load_worker()), False)
    node = port.ToolNode.of(tools_def.get_weather)
    want = sorted((t, kk, pl) for i, r in enumerate(recs) if not lo <= i < hi for (t, kk, _c, pl) in port.tool_node_event(node, r))
    assert sorted(got) == want
    assert st["records"] == len(recs) and st["rejected"] == hi - lo
