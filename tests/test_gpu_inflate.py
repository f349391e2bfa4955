"""The inflate core on the device alone (ck_inflate, csrc/ck_inflate.cuh, through tests/inflate: a warp per stream, its
tables in shared memory), held against zlib and against the g++ build of the same source on raw deflate streams of
1 B to 4 MB — records, cycled records, random bytes, runs, at several levels and strategies, with flushes — and on every
malformed class: the same bytes, or the same refusal."""
import zlib

import numpy as np
import pytest

import gzip_cases as gz
import inflate

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def run_device(streams, caps):
    import torch
    soff = np.concatenate(([0], np.cumsum([len(s) for s in streams]))).astype(np.int64)
    doff = np.concatenate(([0], np.cumsum(caps))).astype(np.int64)
    src = torch.from_numpy(np.frombuffer(b"".join(streams) + b"\0" * 256, dtype=np.uint8).copy()).cuda()
    dst = torch.zeros(int(doff[-1]) + 256, dtype=torch.uint8, device="cuda")
    d_soff, d_doff = torch.from_numpy(soff).cuda(), torch.from_numpy(doff).cuda()
    out_len = torch.zeros(len(streams), dtype=torch.int64, device="cuda")
    used = torch.zeros(len(streams), dtype=torch.int64, device="cuda")
    assert inflate.lib().inflate_streams(src.data_ptr(), d_soff.data_ptr(), len(streams), dst.data_ptr(), d_doff.data_ptr(),
                                         out_len.data_ptr(), used.data_ptr()) == 0
    data, lens, us = dst.cpu().numpy(), out_len.cpu().numpy(), used.cpu().numpy()
    res = []
    for i, s in enumerate(streams):
        n = int(lens[i])
        res.append(None if n < 0 or int(us[i]) != len(s) else data[doff[i]:doff[i] + n].tobytes())
    return res


def check(streams, cap_of=lambda want, s: (len(want) if want is not None else 1 << 16)):
    wants = [gz.zlib_ref(s, -15) for s in streams]
    caps = [cap_of(w, s) for w, s in zip(wants, streams)]
    got = run_device(streams, caps)
    for i, s in enumerate(streams):
        h, used = inflate.inflate(s, caps[i])
        host = h if h is not None and used == len(s) else None
        assert got[i] == wants[i] == host, (i, len(s), wants[i] is None, got[i] is None, host is None)
    return wants


def test_streams_1b_to_4mb():
    from calfkit import synth
    rng = np.random.default_rng(21)
    recs = b"".join(synth.tool_events(3000, seed=22))
    cyc = b"".join(synth.tool_events(8, seed=23)) * 500
    streams = []
    for n in (1, 2, 7, 100, 1000, 4096, 65535, 65536, 100000, 1 << 20, 4 << 20):
        for data in (recs[:n] if n <= len(recs) else (recs * (n // len(recs) + 1))[:n], (cyc * (n // len(cyc) + 1))[:n],
                     rng.integers(0, 256, min(n, 300000), dtype=np.uint8).tobytes(), b"z" * n):
            for level, strat in ((0, 0), (1, 0), (6, 0), (9, 0), (6, zlib.Z_FIXED), (6, zlib.Z_HUFFMAN_ONLY), (6, zlib.Z_RLE)):
                if n >= 1 << 20 and (level, strat) not in ((6, 0), (1, 0)):
                    continue
                streams.append(gz.deflate(data, level=level, strategy=strat))
    streams.append(gz.deflate(recs, flushes=[(1000, zlib.Z_SYNC_FLUSH), (5000, zlib.Z_FULL_FLUSH), (9000, zlib.Z_BLOCK)]))
    streams.append(gz.deflate(gz.far_match_data(), level=9))
    wants = check(streams)
    assert all(w is not None for w in wants) and max(len(w) for w in wants) == 4 << 20


def test_malformed_and_edge_streams():
    mal = list(gz.malformed_streams().values())
    edge = list(gz.accepted_edge_streams().values())
    wants = check(mal + edge)
    assert all(w is None for w in wants[:len(mal)]) and all(w is not None for w in wants[len(mal):])


def test_output_past_the_capacity_is_refused():
    data = gz.records_data(50, seed=24)
    s = gz.deflate(data)
    assert run_device([s, s, s], [len(data), len(data) - 1, 0]) == [data, None, None if data else b""]


def test_bit_flips():
    import random
    rng = random.Random(25)
    base = [gz.deflate(gz.records_data(40, seed=26), level=lv) for lv in (1, 9)]
    streams = []
    for _ in range(3000):
        s = bytearray(rng.choice(base))
        for _ in range(rng.randint(1, 2)):
            i = rng.randrange(len(s))
            s[i] ^= 1 << rng.randrange(8)
        streams.append(bytes(s))
    check(streams)
