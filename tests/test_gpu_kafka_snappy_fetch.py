"""Fetch responses holding snappy batches (attributes 2), decoded on the device a warp per chunk (ck_rb_snappy_kernel,
csrc/ck_kafka.cuh): the records of every golden snappy batch read, through the host view, exactly as the Kafka oracle gives
those of the uncompressed batch, and walk and publish exactly as that batch submitted uncompressed; a mixed fetch of all
five codecs marks exactly its malformed snappy batches bad; a fetch without snappy launches what it did before and snappy
adds one launch; the fetch buffer and the chunk table grow; the same fetch gives the same results; a Lane and Worker.run
consume snappy fetches as they consume plain ones; under read_committed a committed snappy batch decodes and an aborted
one is skipped and never decoded."""
import os
import sys

import numpy as np
import pytest

import gzip_cases as gz
import kafka_snappy as ks
import kafka_txn as kt
import snappy_ref as sr
from make_golden_lz4_batches import load as load_lz4, with_section
from oracle import kafka_batch as kb
from test_gpu_kafka_lz4_fetch import oracle_spans, publishes, spans, submit, tool_batches, tool_engine

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
from make_golden_snappy_batches import WORKER, load, load_worker, uncompressed  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def snappy_batch(batch: bytes, chunk: int | None = 32 << 10) -> bytes:
    """`batch` with its records section in snappy: framed in chunks of `chunk` bytes, or one raw block (chunk None)"""
    sec = batch[61:]
    return with_section(batch, sr.compress(sec) if chunk is None else ks.xerial(sec, chunk), codec=2)


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
    """{class: snappy batch} for one uncompressed batch; every CRC32C is valid.  The malformed blocks as raw-block
    sections, the malformed framings, and the batch's own section framed and then cut, flipped or mis-declared"""
    out = {f"raw block: {k}": with_section(batch, z, codec=2) for k, z in ks.malformed_blocks().items()}
    out.update({f"framing: {k}": with_section(batch, s, codec=2) for k, s in ks.malformed_framings().items()})
    good = ks.xerial(batch[61:], 1 << 10)
    w = ks.walk(good)
    assert len(w) > 2
    out["records section cut inside its last chunk"] = with_section(batch, good[:-3], codec=2)
    off, ln, _d = w[1]
    z = sr.compress(batch[61:])
    out["records block declaring one byte more"] = with_section(batch, ks.put_varint(len(batch) - 60) + z[len(ks.put_varint(len(batch) - 61)):], codec=2)
    second = good[off:off + ln]
    n = ks.varint(second)
    bad = ks.put_varint(n[0] - 1) + second[n[1]:]
    out["second chunk declaring one byte less"] = with_section(batch, good[:off - 4] + len(bad).to_bytes(4, "big") + bad + good[off + ln:], codec=2)
    out["records empty, batch claims records"] = with_section(batch, b"\x00", codec=2)
    for k, v in out.items():
        assert ks.decompress_section(v[61:]) != batch[61:], k
    return out


def test_mixed_fetch():
    """uncompressed, golden LZ4, gzip, zstd and snappy batches (raw and framed), every malformed snappy class with a valid
    CRC32C and a truncated tail, in one fetch submitted once: exactly the malformed snappy batches' records are
    CK_BAD_FRAME"""
    sr.need()
    import zstd_ref as zr
    zr.need()
    from calfkit.engine._lib import CK_BAD_FRAME, COL
    import kafka_lz4 as lz
    plain = tool_batches(3, 30, seed=861)
    sn_src = tool_batches(3, 20, seed=862)
    gold = [b for n, _s, b in load_lz4() if n in ("b64k_linked", "b64k_all_flags")]
    bad_src = tool_batches(1, 40, seed=863)[0]
    other = tool_batches(2, 9, seed=864)
    parts = [(b, True, b) for b in plain[:2]] + \
        [(snappy_batch(b, c), True, b) for b, c in zip(sn_src, (None, 32 << 10, 1 << 10))] + \
        [(b, True, lz.decompress_batch(b)) for b in gold] + \
        [(with_section(other[0], gz.gzip_bytes(other[0][61:]), codec=1), True, other[0])] + \
        [(with_section(other[1], zr.compress(other[1][61:], level=3), codec=4), True, other[1])] + \
        [(b, True, uncompressed(spec)) for _n, spec, b in load()[:5]] + \
        [(plain[2], True, plain[2])] + \
        [(b, False, bad_src) for b in malformed(bad_src).values()]
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


def test_launch_counts():
    """against a fetch with no compressed batch: snappy adds one launch whatever the batch and chunk count; LZ4 + gzip +
    zstd + snappy adds four; a fetch without snappy launches what it launched before"""
    plain = b"".join(tool_batches(3, 10, seed=871))
    lz_b = [b for n, _s, b in load_lz4() if n == "b64k_independent"][0]
    g = tool_batches(1, 10, seed=872)[0]
    gz_b = with_section(g, gz.gzip_bytes(g[61:]), codec=1)
    from make_golden_zstd_batches import load as load_zstd
    zs_b = load_zstd()[0][2]
    sns = [b for _n, _s, b in load()]
    e = tool_engine()
    try:
        def launches(buf):
            l0 = e.launch_count()
            submit(e, buf)
            return e.launch_count() - l0
        base = launches(plain)
        assert launches(plain + sns[0]) == base + 1
        assert launches(plain + b"".join(sns)) == base + 1
        assert launches(plain + sns[0] + lz_b + gz_b + zs_b + sns[4]) == base + 4
        assert launches(plain + lz_b + gz_b + zs_b) == base + 3
        assert launches(plain) == base
    finally:
        e.close()


def test_grow_and_determinism():
    """a small snappy fetch, then the golden framed section of more than 4 MB with a section of 1 KB chunks that outgrows
    the chunk table (more than 1,024 chunks): it decodes right after the fetch buffer and the chunk table grew; the same
    fetch twice gives identical columns, publishes and decoded slots"""
    sr.need()
    from calfkit import synth
    g = {n: (s, b) for n, s, b in load()}
    small_spec, small = g["xerial_1k"]
    big_spec, big = g["over_4mb_xerial_32k"]
    recs = synth.tool_events(1400, seed=873)
    many_src = kb.encode_batch([kb.calfkit_record(r, f"m-{i}", keyed=True) for i, r in enumerate(recs)], base_offset=9, base_timestamp=1767225600000)
    many = snappy_batch(many_src, 1 << 10)
    assert len(ks.walk(many[61:])) > 1024
    e = tool_engine()
    try:
        _n, ix, _out = submit(e, small)
        assert ix["bad"].sum() == 0
        runs = []
        for _ in range(2):
            n, ix, out = submit(e, big + many + small)
            assert ix["bad"].sum() == 0
            assert [spans(ix, i) for i in range(n)] == oracle_spans(uncompressed(big_spec)) + oracle_spans(many_src) + oracle_spans(uncompressed(small_spec))
            runs.append((out.cols.copy(), publishes(out), ix["data"].decoded.copy()))
        assert (runs[0][0] == runs[1][0]).all() and runs[0][1] == runs[1][1] and (runs[0][2] == runs[1][2]).all()
    finally:
        e.close()


def snappy_frames(fetch: bytes, chunk) -> bytes:
    """every frame of a fetch response with its records section in snappy (framed in `chunk` bytes, or one raw block)"""
    out, pos = [], 0
    while pos + 12 <= len(fetch):
        end = pos + 12 + int.from_bytes(fetch[pos + 8:pos + 12], "big")
        out.append(snappy_batch(fetch[pos:end], chunk))
        pos = end
    return b"".join(out)


@pytest.mark.parametrize("nparts", [8, 1000])
def test_lane_consumes_snappy_frames_of_a_tool_step(nparts):
    """engine A frames a config-2-shaped tool step in 1 MiB frames; its frames in both snappy shapes are one fetch response
    each for a Worker lane B, whose publishes equal those of the uncompressed fetch"""
    sr.need()
    from calfkit import synth
    from calfkit.engine.lane import FetchArena, Lane, PinnedPool
    from test_gpu_kafka_frames import tool_engine as frame_engine, tool_step
    from test_gpu_kafka_lz4_fetch import configure
    recs = synth.tool_events(3000, seed=881) + synth.tool_events(200, seed=882, size=4000, jitter=3000)
    a = frame_engine(nparts)
    try:
        _out, frames = tool_step(a, recs, 1 << 20)
        plain = b"".join(f.tobytes() for _t, _p, f, _n in frames)
        values = [r.value for _t, _p, f, _n in frames for r in kb.decode_batches(f.tobytes())]
    finally:
        a.close()
    got = {}
    for codec, fetch in (("none", plain), ("raw", snappy_frames(plain, None)), ("xerial", snappy_frames(plain, 32 << 10))):
        assert (fetch[22] & 7) == (0 if codec == "none" else 2)
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
    assert got["raw"] == got["none"] and got["xerial"] == got["none"]


def test_worker_run_consumes_a_snappy_fetch():
    """the golden worker fetch through broker.produce_fetch and Worker.run, one of its batches corrupt (a block with a
    flipped bit, which snappy refuses too): the output equals the oracle's tool-node outputs for every record outside that
    batch, and stats["rejected"] counts exactly its records"""
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


def submit_txn(e, buf, partitions):
    n = e.submit_recordbatch(np.frombuffer(bytes(buf), dtype=np.uint8), partitions=partitions)
    e.tool_plan()
    return n, e._rb, e.fetch()


def test_read_committed_over_snappy_batches():
    """a log whose data batches are snappy (raw and framed) under transactions: at read_committed the committed ones
    decode as they do outside a transaction, and the aborted ones, a malformed section among them, are skipped and never
    decoded (a fetch of aborted snappy batches only has no decoded region and launches what a plain fetch launches).  The
    host's rule (the g++ build of ck_txn.h) gives the log the verdicts the restatement gives its uncompressed twin"""
    sr.need()
    import txnmask
    from calfkit.engine._lib import CK_SKIPPED, COL
    A, B = 51, 52
    src = tool_batches(6, 6, seed=891)
    log, twin, deliver = [], [], []
    aborted, off = [(A, 0)], 0
    for i in range(4):                   # producer A: aborted, sections raw, framed, framed, malformed
        b = kt.txn_batch([kb.KRecord(r.value, r.key, r.headers) for r in kb.decode_batches(src[i])], off, A)
        sec = [sr.compress(b[61:]), ks.xerial(b[61:]), ks.xerial(b[61:], 1 << 10), b"\x05\x01"][i]
        log.append(with_section(b, sec, codec=2))
        twin.append(b)
        deliver += [False] * 6
        off += 6
    for i in (4, 5):                     # producer B: committed, raw and framed
        b = kt.txn_batch([kb.KRecord(r.value, r.key, r.headers) for r in kb.decode_batches(src[i])], off, B)
        log.append(snappy_batch(b, None if i == 4 else 32 << 10))
        twin.append(b)
        deliver += [True] * 6
        off += 6
    for pid, ctype in ((A, kt.ABORT), (B, kt.COMMIT)):
        c = kt.control_batch(off, pid, ctype)
        log.append(c)
        twin.append(c)
        deliver.append(False)
        off += 1
    fetch, plain_twin = b"".join(log), b"".join(twin)
    parts = [(0, aborted)]
    for rc in (False, True):
        assert txnmask.verdicts(fetch, parts, rc) == kt.verdicts(plain_twin, parts, rc)
    extra = tool_batches(1, 6, seed=892)[0]
    aborted_only = b"".join(log[:4]) + log[6] + extra
    e = tool_engine()
    e.set_isolation_level("read_committed")
    try:
        n, ix, out = submit_txn(e, fetch, parts)
        d = np.array(deliver)
        assert n == len(deliver)
        assert (ix["bad"][~d] == 2).all() and (ix["bad"][d] == 0).all()
        assert (out.cols[COL["STATUS"]][~d] == CK_SKIPPED).all()
        assert [spans(ix, int(i)) for i in np.nonzero(d)[0]] == oracle_spans(src[4]) + oracle_spans(src[5])
        l0 = e.launch_count()
        n, ix, _out = submit_txn(e, aborted_only, parts)
        l1 = e.launch_count()
        assert n == 31 and (ix["bad"][:25] == 2).all() and (ix["bad"][25:] == 0).all()
        assert isinstance(ix["data"], np.ndarray)                  # no decoded region: nothing was sized or decoded
        assert [spans(ix, i) for i in range(25, 31)] == oracle_spans(extra)
        submit(e, extra)
        assert l1 - l0 == e.launch_count() - l1
        # read_uncommitted delivers them: the valid sections decode, the malformed one is a bad frame
        e.set_isolation_level("read_uncommitted")
        n, ix, _out = submit_txn(e, fetch, parts)
        bad = np.array(ix["bad"])
        assert (bad[:18] == 0).all() and (bad[18:24] == 1).all() and (bad[24:36] == 0).all() and (bad[36:] == 2).all()
        assert [spans(ix, i) for i in range(18)] == oracle_spans(src[0]) + oracle_spans(src[1]) + oracle_spans(src[2])
    finally:
        e.close()
