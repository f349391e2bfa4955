"""Fetch responses holding gzip batches (attributes 1), inflated on the device (ck_rb_gzip_kernel, csrc/ck_kafka.cuh): the
records of a gzip batch read, through the host view, exactly as the Kafka oracle gives those of the uncompressed batch,
and walk and publish exactly as that batch submitted uncompressed, for every zlib setting and header variant; a mixed
fetch marks exactly its malformed gzip, snappy and zstd batches bad; each codec present adds one launch; the fetch buffer
grows; the same fetch gives the same results; a Lane and Worker.run consume gzip fetches as they consume plain ones."""
import zlib

import numpy as np
import pytest

import gzip_cases as gz
from make_golden_lz4_batches import load as load_batches, with_section
from oracle import kafka_batch as kb
from test_gpu_kafka_lz4_fetch import oracle_spans, publishes, spans, submit, tool_batches, tool_engine

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def gzip_batch(batch: bytes, **kw) -> bytes:
    """`batch` with its records section as one gzip member (zlib, level 6 unless kw says otherwise)"""
    return with_section(batch, gz.gzip_bytes(batch[61:], **kw), codec=1)


SETTINGS = {f"level{lv}": dict(level=lv) for lv in (0, 1, 6, 9)}
SETTINGS.update({s: dict(strategy=v) for s, v in gz.STRATEGIES.items() if s != "default"})
SETTINGS.update({"wbits9_mem1": dict(wbits=-9, mem=1), "sync_flush": dict(flushes=[(300, zlib.Z_SYNC_FLUSH), (5000, zlib.Z_FULL_FLUSH)])})
HEADERS = {"plain": {}, "all_flags_hcrc": dict(flg=30, extra=b"KF\x02\x00ab", name=b"batch", comment=b"kafka", hcrc=True),
           "fname": dict(flg=8, name=b"records.bin")}


@pytest.mark.parametrize("header", list(HEADERS))
@pytest.mark.parametrize("setting", list(SETTINGS))
def test_gzip_batch_spans_and_columns(setting, header):
    kw = dict(SETTINGS[setting])
    plain = tool_batches(1, 40, seed=601)[0]
    sec = plain[61:]
    if "flushes" in kw:
        kw["flushes"] = [(min(a, len(sec) - 1), m) for a, m in kw["flushes"]]
    batch = with_section(plain, gz.member(gz.deflate(sec, **kw), sec, **HEADERS[header]), codec=1)
    assert gz.zlib_ref(batch[61:]) == sec
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
        assert n2 == n and ix2["bad"].sum() == 0
        assert (out2.cols == cols).all() and publishes(out2) == pubs
    finally:
        e.close()


def malformed(batch):
    """{class: gzip batch} for one uncompressed batch; every CRC32C is valid"""
    sec = batch[61:]
    raw = gz.deflate(sec)
    good = gz.member(raw, sec)
    out = {k: gz.member(s, sec) for k, s in gz.malformed_streams().items()}
    out.update({
        "bad magic": b"\x1f\x8c" + good[2:],
        "reserved flag bit": gz.member(raw, sec, flg=0x20),
        "wrong FHCRC": gz.member(raw, sec, flg=2, hcrc=1),
        "wrong CRC32": gz.member(raw, sec, crc=zlib.crc32(sec) ^ 4),
        "ISIZE one short": gz.member(raw, sec, isize=len(sec) - 1),
        "implausible ISIZE": gz.member(raw, sec, isize=1032 * len(raw) + 1),
        "ISIZE past the 32-bit split": gz.member(raw, sec, isize=0x7fffffff),
        "shorter than header + trailer": good[:17],
        "a second member": good + gz.gzip_bytes(b""),
        "a byte after the trailer": good + b"\0",
        "truncated": good[:-9],
    })
    for k, z in out.items():
        assert gz.zlib_ref(z) is None, k
    return {k: with_section(batch, z, codec=1) for k, z in out.items()}


def test_mixed_fetch():
    """uncompressed, golden LZ4 and gzip batches, every malformed gzip class with a valid CRC32C, a snappy and a zstd
    batch, and a truncated tail, in one fetch submitted once: exactly the malformed, snappy and zstd batches' records are
    CK_BAD_FRAME, every other record reads and walks as the oracle says"""
    from calfkit.engine._lib import CK_BAD_FRAME, COL
    plain = tool_batches(3, 30, seed=611)
    gz_src = tool_batches(3, 20, seed=612)
    gold = [b for n, _s, b in load_batches() if n in ("b64k_linked", "b64k_all_flags")]
    import kafka_lz4 as lz
    bad_src = tool_batches(1, 12, seed=613)[0]
    other = tool_batches(2, 9, seed=614)
    parts = [(b, True, b) for b in plain[:2]] + [(gzip_batch(b, level=lv), True, b) for b, lv in zip(gz_src, (1, 6, 9))] + \
        [(b, True, lz.decompress_batch(b)) for b in gold] + [(plain[2], True, plain[2])] + \
        [(b, False, bad_src) for b in malformed(bad_src).values()] + \
        [(with_section(other[0], gz.gzip_bytes(other[0][61:]), codec=2), False, other[0]),
         (with_section(other[1], gz.gzip_bytes(other[1][61:]), codec=4), False, other[1])]
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


def test_empty_member_is_not_a_refused_slot():
    """a member of ISIZE 0 has an empty slot, like a refused one, and still decodes: the device parses the member itself
    (tests/inflate's member mode: 0 bytes, not a refusal) and a batch of no records around it leaves its neighbours as
    they are; a member whose header is refused, given the same empty slot, is refused, and so is a batch that claims
    records of an empty member"""
    import inflate as inf
    empty_ok = gz.gzip_bytes(b"")
    refused = b"\x1f\x8c" + empty_ok[2:]
    assert run_members([empty_ok, refused, gz.gzip_bytes(b"abc")], [0, 0, 3]) == [0, -1, 3]
    assert inf.member(empty_ok) == b"" and inf.member(refused) is None
    src = tool_batches(2, 5, seed=615)
    empty = kb.encode_batch([], base_offset=7, base_timestamp=1767225600000)
    assert len(empty) == 61
    e = tool_engine()
    try:
        n, ix, _out = submit(e, gzip_batch(src[0]) + with_section(empty, empty_ok, codec=1) + gzip_batch(src[1]))
        assert n == 10 and ix["bad"].sum() == 0
        assert [spans(ix, i) for i in range(10)] == oracle_spans(src[0]) + oracle_spans(src[1])
        n, ix, _out = submit(e, with_section(src[0], empty_ok, codec=1) + gzip_batch(src[1]))
        assert n == 10 and list(ix["bad"]) == [1] * 5 + [0] * 5
        assert [spans(ix, i) for i in range(5, 10)] == oracle_spans(src[1])
    finally:
        e.close()


def run_members(members, caps):
    """ck_gz_decode on the device (everything the gzip kernel checks but the CRC32): inflated length or -1 per member"""
    import torch
    import inflate as inf
    soff = np.concatenate(([0], np.cumsum([len(m) for m in members]))).astype(np.int64)
    doff = np.concatenate(([0], np.cumsum(caps))).astype(np.int64)
    src = torch.from_numpy(np.frombuffer(b"".join(members) + b"\0" * 256, dtype=np.uint8).copy()).cuda()
    dst = torch.zeros(int(doff[-1]) + 256, dtype=torch.uint8, device="cuda")
    out_len = torch.zeros(len(members), dtype=torch.int64, device="cuda")
    used = torch.zeros(len(members), dtype=torch.int64, device="cuda")
    assert inf.lib().inflate_members(src.data_ptr(), torch.from_numpy(soff).cuda().data_ptr(), len(members), dst.data_ptr(),
                                     torch.from_numpy(doff).cuda().data_ptr(), out_len.data_ptr()) == 0
    return [int(x) for x in out_len.cpu().numpy()]


def test_launch_counts():
    """against a fetch with no compressed batch: an LZ4-only fetch adds one launch, a gzip-only fetch one, a fetch with
    both two, whatever the number of batches of each codec"""
    plain = b"".join(tool_batches(3, 10, seed=621))
    lz_b = [b for n, _s, b in load_batches() if n == "b64k_independent"][0]
    gzs = [gzip_batch(b) for b in tool_batches(3, 10, seed=622)]
    e = tool_engine()
    try:
        def launches(buf):
            l0 = e.launch_count()
            submit(e, buf)
            return e.launch_count() - l0
        base = launches(plain)
        assert launches(plain + lz_b) == base + 1
        assert launches(plain + lz_b + lz_b) == base + 1
        assert launches(plain + gzs[0]) == base + 1
        assert launches(plain + b"".join(gzs)) == base + 1
        assert launches(plain + gzs[0] + lz_b + gzs[1]) == base + 2
        assert launches(plain) == base
    finally:
        e.close()


def test_grow_and_determinism():
    """a small gzip fetch, then one whose ISIZEs exceed the fetch buffer: the second inflates right after the buffer grew;
    the same fetch twice gives identical columns, publishes and decoded slots"""
    from calfkit import synth
    small = gzip_batch(tool_batches(1, 10, seed=631)[0])
    recs = synth.tool_events(8, seed=632, size=8000)
    big_plain = kb.encode_batch([kb.calfkit_record(recs[i % 8], f"big-{i}", keyed=i % 3 != 0) for i in range(600)],
                                base_offset=5, base_timestamp=1767225600000)
    big = gzip_batch(big_plain, level=9)
    assert len(big_plain) > 4 << 20 and len(big) < len(big_plain) // 20
    e = tool_engine()
    try:
        _n, ix, _out = submit(e, small)
        assert ix["bad"].sum() == 0
        runs = []
        for _ in range(2):
            n, ix, out = submit(e, big + small)
            assert ix["bad"].sum() == 0
            assert [spans(ix, i) for i in range(n)] == oracle_spans(big_plain) + oracle_spans(tool_batches(1, 10, seed=631)[0])
            runs.append((out.cols.copy(), publishes(out), ix["data"].decoded.copy()))
        assert (runs[0][0] == runs[1][0]).all() and runs[0][1] == runs[1][1] and (runs[0][2] == runs[1][2]).all()
    finally:
        e.close()


def gzip_frames(fetch: bytes) -> bytes:
    """every frame of a fetch response with its records section recompressed to one gzip member (level 6)"""
    out, pos = [], 0
    while pos + 12 <= len(fetch):
        end = pos + 12 + int.from_bytes(fetch[pos + 8:pos + 12], "big")
        out.append(gzip_batch(fetch[pos:end]))
        pos = end
    return b"".join(out)


@pytest.mark.parametrize("nparts", [8, 1000])
@pytest.mark.parametrize("window", [64 << 10, 1 << 20])
def test_lane_consumes_gzip_frames_of_a_tool_step(nparts, window):
    """engine A frames a config-2-shaped tool step; its frames, recompressed to gzip on the host, are one fetch response
    for a Worker lane B.  B reads every record as A published it, and B's publishes equal those of the uncompressed fetch"""
    from calfkit import synth
    from calfkit.engine.lane import FetchArena, Lane, PinnedPool
    from test_gpu_kafka_frames import tool_engine as frame_engine, tool_step
    from test_gpu_kafka_lz4_fetch import configure
    recs = synth.tool_events(3000, seed=641) + synth.tool_events(200, seed=642, size=4000, jitter=3000)
    a = frame_engine(nparts)
    try:
        _out, frames = tool_step(a, recs, window)
        plain = b"".join(f.tobytes() for _t, _p, f, _n in frames)
        values = [r.value for _t, _p, f, _n in frames for r in kb.decode_batches(f.tobytes())]
    finally:
        a.close()
    got = {}
    for codec, fetch in (("none", plain), ("gzip", gzip_frames(plain))):
        assert (fetch[22] & 7) == (1 if codec == "gzip" else 0)
        pool = PinnedPool()
        lane = Lane(0, configure, pool, max_records=1 << 14, max_in_bytes=64 << 20)
        try:
            lane.submit(FetchArena.of(fetch, pool))
            batch = lane.collect()
            src = batch.source
            assert src.n == len(values) and src.bad.sum() == 0
            assert [src.record(i) for i in range(src.n)] == values
            if codec == "gzip":
                assert lane.d2h_bytes >= src.data.decoded.nbytes > 0
            got[codec] = [(t, k, p) for t, k, p, _j in batch.iter_records()]
            batch.release()
        finally:
            lane.close()
            pool.close()
    assert got["gzip"] == got["none"]


def test_worker_run_consumes_a_gzip_fetch():
    """a gzip fetch through broker.produce_fetch and Worker.run, one of its batches corrupt (a flipped bit in its deflate
    stream, the CRC32C recomputed): the output equals the oracle's tool-node outputs for every record outside that batch,
    and stats["rejected"] counts exactly its records"""
    import json
    import tools_def
    from calfkit import synth
    from oracle import port
    from test_gpu_kafka_frames import _worker_run
    recs = synth.tool_events(600, seed=651)
    sizes = [40] * 15
    out, k = [], 0
    lo = hi = 0
    for bi, sz in enumerate(sizes):
        chunk = [kb.calfkit_record(r, json.loads(r)["context"]["deps"]["correlation_id"], keyed=(j % 4 != 0))
                 for j, r in enumerate(recs[k:k + sz])]
        plain = kb.encode_batch(chunk, base_offset=1000 + k, base_timestamp=1767225600000 + bi)
        z = bytearray(gz.gzip_bytes(plain[61:]))
        if bi == 6:
            z[len(z) // 2] ^= 0x10
            assert gz.zlib_ref(bytes(z)) is None
            lo, hi = k, k + sz
        out.append(with_section(plain, bytes(z), codec=1))
        k += sz
    got, _parts, st = _worker_run(b"".join(out), False)
    node = port.ToolNode.of(tools_def.get_weather)
    want = sorted((t, kk, pl) for i, r in enumerate(recs) if not lo <= i < hi for (t, kk, _c, pl) in port.tool_node_event(node, r))
    assert sorted(got) == want
    assert st["records"] == len(recs) and st["rejected"] == hi - lo
