"""Fetch responses holding transactional and control batches (KIP-98), consumed on the device: over seeded random logs
every record's status and span is what the restatement of the rule (tests/kafka_txn.py) says, at both isolation levels;
aborted gzip, LZ4 and zstd batches, their compressed sections corrupt or not, are skipped and never decoded while the
committed ones decode; a fetch with no control batch and no mask launches what it launched before; a Lane consumes a
config-2 tool step rewritten as transactions under read_committed; Worker.run publishes the oracle's outputs for the
committed records only, counts the rest as skipped and logs nothing as rejected."""
import logging

import numpy as np
import pytest

import gzip_cases as gz
import kafka_txn as kt
from make_golden_lz4_batches import with_section
from oracle import kafka_batch as kb
from test_gpu_kafka_lz4_fetch import lit_block, lz4_frame, malformed as lz4_malformed, oracle_spans, publishes, spans, tool_batches, \
    tool_engine

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def submit(e, buf, partitions=None):
    n = e.submit_recordbatch(np.frombuffer(bytes(buf), dtype=np.uint8), partitions=partitions)
    e.tool_plan()
    return n, e._rb, e.fetch()


def tool_records(seed):
    """make_records for kafka_txn.random_log: config-2 tool events as calfkit writes them"""
    from calfkit import synth
    state = {"k": 0}

    def make(n, tag):
        recs = synth.tool_events(n, seed=seed * 1000 + state["k"])
        state["k"] += 1
        return [kb.calfkit_record(r, f"{tag}-{i}", keyed=i % 3 != 2) for i, r in enumerate(recs)]
    return make


def expected(buf, partitions, read_committed):
    """per record: (verdict, its oracle spans or None)"""
    out = []
    for (s, e), v in zip(kt.batches(buf), kt.verdicts(buf, partitions, read_committed)):
        f = buf[s:e]
        cnt = kt.record_counts(f)[0]
        recs = oracle_spans(f) if v == kt.DELIVER else [None] * cnt
        assert len(recs) == cnt
        out += [(v, r) for r in recs]
    return out


@pytest.mark.parametrize("level", ["read_uncommitted", "read_committed"])
def test_random_logs_status_and_spans(level):
    from calfkit.engine._lib import CK_BAD_FRAME, CK_SKIPPED, COL
    e = tool_engine()
    e.set_isolation_level(level)
    try:
        seen = {kt.DELIVER: 0, kt.BAD: 0, kt.SKIP: 0}
        for seed in range(40):
            buf, parts = kt.random_log(seed, make_records=tool_records(seed), n_events=30)
            want = expected(buf, parts, level == "read_committed")
            n, ix, out = submit(e, buf, partitions=parts)
            assert n == len(want), seed
            st = out.cols[COL["STATUS"]]
            for i, (v, rec) in enumerate(want):
                seen[v] += 1
                assert int(ix["bad"][i]) == v, (seed, i)
                if v == kt.DELIVER:
                    assert spans(ix, i) == rec and st[i] not in (CK_BAD_FRAME, CK_SKIPPED), (seed, i)
                else:
                    assert st[i] == (CK_SKIPPED if v == kt.SKIP else CK_BAD_FRAME) and ix["val_len"][i] == 0, (seed, i)
                    assert ix["key_len"][i] == -1 and ix["corr_len"][i] == -1
            assert all(want[p.record][0] == kt.DELIVER for p in out.publishes())
        assert min(seen.values()) > 100
    finally:
        e.close()


def test_walked_delivered_records_equal_the_plain_fetch_of_them():
    """the columns and publishes of the delivered records of a read_committed fetch equal those of the same records in a
    plain fetch of only the delivered batches"""
    from calfkit.engine._lib import COL
    buf, parts = kt.random_log(77, make_records=tool_records(77), n_events=40)
    v = kt.verdicts(buf, parts, True)
    plain = b"".join(buf[s:e] for (s, e), x in zip(kt.batches(buf), v) if x == kt.DELIVER)
    e = tool_engine()
    e.set_isolation_level("read_committed")
    try:
        _n, _ix, out = submit(e, buf, partitions=parts)
        keep = np.array([x == kt.DELIVER for x, _r in expected(buf, parts, True)])
        cols = out.cols[:, keep].copy()
        pubs = sorted((t, k, p) for t, k, p in publishes(out))
        _n2, _ix2, out2 = submit(e, plain)
        assert (out2.cols[COL["STATUS"]] == cols[COL["STATUS"]]).all() and (out2.cols[COL["ACTION"]] == cols[COL["ACTION"]]).all()
        assert sorted(publishes(out2)) == pubs and len(pubs) > 0
    finally:
        e.close()


def compressed(batch, codec, corrupt=False):
    """`batch` (transactional, uncompressed) with its records section compressed: gzip 1, LZ4 3, zstd 4; corrupt: a
    malformed section under a valid CRC32C"""
    sec = batch[61:]
    if codec == 1:
        z = gz.gzip_bytes(sec)
        z = z[:10] + bytes([z[10] ^ 0xFF]) + z[11:] if corrupt else z
    elif codec == 3:
        if corrupt:
            return lz4_malformed(batch)["offset 0"]
        z = lz4_frame([(len(b := lit_block(sec)), b)])
    else:
        import zstd_ref as zr
        zr.need()
        z = zr.compress(sec, level=3, checksum=True)
        z = z[:-1] + bytes([z[-1] ^ 0x80]) if corrupt else z
    return with_section(batch, z, codec=codec)


def test_aborted_compressed_batches_are_skipped_and_never_decoded():
    """aborted gzip, LZ4 and zstd batches (a valid and a corrupt section each) are skipped, and a fetch holding no other
    compressed batch has no decoded region and launches what a plain fetch launches; committed compressed batches of the
    same producers decode as they do outside a transaction"""
    from calfkit.engine._lib import CK_SKIPPED, COL
    A, B = 41, 42
    src = tool_batches(8, 6, seed=931)
    off, log, aborted, deliver = 0, [], [], []
    for i, codec in enumerate((1, 3, 4)):
        for corrupt in (False, True):
            b = kt.txn_batch([kb.KRecord(r.value, r.key, r.headers) for r in kb.decode_batches(src[2 * i + corrupt])], off, A)
            aborted.append((A, off))
            log.append(compressed(b, codec, corrupt))
            off += 6
            log.append(kt.control_batch(off, A, kt.ABORT))
            off += 1
            deliver += [False] * 7
    plain_part = kt.txn_batch([kb.KRecord(r.value, r.key, r.headers) for r in kb.decode_batches(src[6])], off, B)
    log.append(plain_part)
    deliver += [True] * 6
    off += 6
    log.append(kt.control_batch(off, B, kt.COMMIT))
    deliver.append(False)
    fetch = b"".join(log)
    e = tool_engine()
    e.set_isolation_level("read_committed")
    try:
        n, ix, out = submit(e, fetch, partitions=[(0, aborted)])
        assert n == len(deliver)
        d = np.array(deliver)
        assert (ix["bad"][~d] == 2).all() and (ix["bad"][d] == 0).all()
        assert (out.cols[COL["STATUS"]][~d] == CK_SKIPPED).all()
        assert isinstance(ix["data"], np.ndarray)                  # no decoded region: nothing was sized or decoded
        assert [spans(ix, int(i)) for i in np.nonzero(d)[0]] == oracle_spans(src[6])
        l0 = e.launch_count()
        submit(e, fetch, partitions=[(0, aborted)])
        l1 = e.launch_count()
        submit(e, plain_part)
        assert l1 - l0 == e.launch_count() - l1
        # read_uncommitted delivers the same batches: they decode (the corrupt ones are bad frames), as outside a transaction
        e.set_isolation_level("read_uncommitted")
        n, ix, out = submit(e, fetch, partitions=[(0, aborted)])
        bad = np.array(ix["bad"])
        for k in range(6):
            rows = slice(7 * k, 7 * k + 6)
            if k % 2:
                assert (bad[rows] == 1).all()
            else:
                assert (bad[rows] == 0).all()
                assert [spans(ix, i) for i in range(7 * k, 7 * k + 6)] == oracle_spans(src[k])
            assert bad[7 * k + 6] == 2                              # the marker: skipped at both levels
        assert ix["data"].decoded.nbytes > 0
    finally:
        e.close()


def test_launch_counts_unchanged_without_control_batches_or_mask():
    """a plain fetch launches the same kernels at both isolation levels, with or without aborted transactions that hide
    nothing; control batches and a mask that hides batches add no launch"""
    plain = b"".join(tool_batches(3, 10, seed=951))
    A = 5
    log = [kt.txn_batch([kb.KRecord(r.value, r.key, r.headers) for r in kb.decode_batches(b)], 100 * i, A) for i, b in enumerate(tool_batches(3, 10, seed=952))]
    txn = b"".join(log[:2]) + kt.control_batch(150, A, kt.ABORT) + log[2]
    e = tool_engine()
    try:
        def launches(buf, **kw):
            l0 = e.launch_count()
            submit(e, buf, **kw)
            return e.launch_count() - l0
        base = launches(plain)
        e.set_isolation_level("read_committed")
        assert launches(plain) == base
        assert launches(plain, partitions=[(0, [(99, 10 ** 6)])]) == base
        assert launches(txn, partitions=[(0, [(A, 0)])]) == base
        e.set_isolation_level("read_uncommitted")
        assert launches(txn) == base and launches(plain) == base
    finally:
        e.close()


def test_mask_must_cover_the_fetch():
    from calfkit.exceptions import EngineError
    e = tool_engine()
    try:
        e.set_fetch_hidden(np.zeros(2, np.uint8))
        with pytest.raises(EngineError):
            submit(e, b"".join(tool_batches(3, 4, seed=961)))
        n, ix, _out = submit(e, b"".join(tool_batches(3, 4, seed=961)))       # the mask went with the failed call
        assert n == 12 and ix["bad"].sum() == 0
    finally:
        e.close()


def tool_step_fetch(abort_share, seed):
    """the events of a config-2-shaped tool step framed by engine A (its record form, 64 KB frames), as transactions
    with commits and aborts: (fetch, aborted entries, the uncompressed fetch of the committed frames only)"""
    from calfkit import synth
    from test_gpu_kafka_frames import TS, tool_engine as frame_engine
    recs = synth.tool_events(3000, seed=seed) + synth.tool_events(200, seed=seed + 1, size=4000, jitter=3000)
    a = frame_engine(8)
    try:
        a.set_frame_bytes(64 << 10)
        items = []
        for r in recs:
            k = r.index(b'"correlation_id":"') + 18
            c = r[k:r.index(b'"', k)].decode()
            items.append((r, c.encode(), c))
        a.encode_frames_records("tool.get_weather.input", items, TS)
        frames = a.fetch_frames()
        fr = [frames.frame(i).tobytes() for i in range(len(frames))]
    finally:
        a.close()
    fetch, entries, aborted = kt.transactional_fetch(fr, abort_share, seed)
    assert any(aborted) and not all(aborted)
    return fetch, entries, b"".join(f for f, ab in zip(fr, aborted) if not ab)


def test_lane_consumes_a_transactional_tool_step_read_committed():
    """a Lane at read_committed over the transactional fetch, split at every fourth frame like a broker poll would,
    publishes what a Lane publishes over the committed frames alone"""
    from calfkit.engine.lane import FetchArena, Lane, PinnedPool
    from test_gpu_kafka_lz4_fetch import configure
    fetch, entries, committed = tool_step_fetch(0.3, seed=971)

    def run(arena, level):
        pool = PinnedPool()
        lane = Lane(0, lambda e: (configure(e), e.set_isolation_level(level)), pool, max_records=1 << 14, max_in_bytes=64 << 20)
        got, skipped = [], 0
        try:
            nf = len(arena.frames()[1])
            for a in range(0, nf, 4):
                lane.submit(arena.slice_frames(a, a + 4 if a + 4 < nf else None))
                batch = lane.collect()
                skipped += int((batch.source.bad == 2).sum())
                assert (batch.source.bad != 1).all()
                got += [(t, k, p) for t, k, p, _j in batch.iter_records()]
                batch.release()
        finally:
            lane.close()
            pool.close()
        return got, skipped
    got, skipped = run(FetchArena.of(fetch, aborted_transactions=entries), "read_committed")
    want, none = run(FetchArena.of(committed), "read_committed")
    assert got == want and none == 0 and skipped > 0
    got_ru, _s = run(FetchArena.of(fetch, aborted_transactions=entries), "read_uncommitted")
    assert len(got_ru) > len(got)


def test_worker_run_publishes_only_committed_records(caplog):
    import asyncio
    import tools_def
    from calfkit import Client, Worker, agent_tool, synth
    from oracle import port
    recs = synth.tool_events(600, seed=981)
    per = 20
    src = [kb.encode_batch([kb.calfkit_record(r, f"w-{b}-{i}", keyed=i % 3 != 2) for i, r in enumerate(recs[b * per:(b + 1) * per])])
           for b in range(len(recs) // per)]
    fetch, entries, aborted = kt.transactional_fetch(src, 0.3, seed=982)
    node_def = agent_tool(tools_def.get_weather, device_template="It's sunny in {location}")
    client = Client.connect("localhost")
    client.broker.produce_fetch("tool.get_weather.input", fetch, aborted_transactions=entries)
    got = []
    for t in ("weather_agent.input", "tool.get_weather.output"):
        client.broker.sink(t, lambda b, idx, t=t: got.extend((t, k, p) for (_t, k, p, _j) in b.iter_records(idx)))
    worker = Worker(client, nodes=[node_def], batch_records=64, batch_bytes=8 << 20, lanes=3, route_topics=["weather_agent.input"],
                    extra_subscribe_kwargs={"isolation_level": "read_committed"})
    with caplog.at_level(logging.ERROR):
        asyncio.run(worker.run(until_idle=True))
    for t in ("weather_agent.input", "tool.get_weather.output"):
        got += [(t, r.key, r.value) for r in client.broker.poll_batch((t,), 10000)]
    stats = dict(worker.stats)
    worker.close()
    node = port.ToolNode.of(tools_def.get_weather)
    kept = [r for b, ab in enumerate(aborted) if not ab for r in recs[b * per:(b + 1) * per]]
    want = sorted((t, kk, pl) for r in kept for (t, kk, _c, pl) in port.tool_node_event(node, r))
    assert sorted(got) == want
    markers = sum(1 for s, _e in kt.batches(fetch) if fetch[s + 22] & kt.CONTROL)
    assert stats["skipped"] == per * sum(aborted) + markers
    assert stats["rejected"] == 0 and stats["records"] == len(recs) + markers
    assert "rejected" not in caplog.text
