"""The zstd decoder on the device alone (ck_zs_decode, csrc/ck_zstd.cuh, through tests/zstdec: a warp per frame, its
tables in shared memory), held against libzstd and against the g++ build of the same source on frames of 1 B to 4 MB
over the settings matrix, on every malformed class and on a seeded subset of the mutations: the same bytes, or the same
refusal (the mutations keep the one characterized exception of tests/test_zstd_hostsim.py)."""
import numpy as np
import pytest

import zstd_cases as zc
import zstd_ref as zr
import zstdec

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def run_device(frames, caps=None):
    """each frame decoded on the device into a slot of its host bound (or caps[i]): bytes or None"""
    import torch
    if caps is None:
        caps = [zstdec.bound(z) or 0 for z in frames]
    soff = np.concatenate(([0], np.cumsum([len(z) for z in frames]))).astype(np.int64)
    doff = np.concatenate(([0], np.cumsum(caps))).astype(np.int64)
    src = torch.from_numpy(np.frombuffer(b"".join(frames) + b"\0" * 256, dtype=np.uint8).copy()).cuda()
    dst = torch.zeros(int(doff[-1]) + 256, dtype=torch.uint8, device="cuda")
    out_len = torch.zeros(len(frames), dtype=torch.int64, device="cuda")
    assert zstdec.lib().zstd_frames(src.data_ptr(), torch.from_numpy(soff).cuda().data_ptr(), len(frames), dst.data_ptr(),
                                    torch.from_numpy(doff).cuda().data_ptr(), out_len.data_ptr()) == 0
    data, lens = dst.cpu().numpy(), out_len.cpu().numpy()
    return [None if lens[i] < 0 else data[doff[i]:doff[i] + lens[i]].tobytes() for i in range(len(frames))]


def test_frames_1b_to_4mb():
    zr.need()
    frames, datas = [], []
    for n in (1, 2, 100, 1000, 65535, 65536, 131073, 1 << 20, 4 << 20):
        for kind in zc.KINDS:
            for name, kw in zc.SETTINGS.items():
                if n >= 1 << 20 and name not in ("level1", "level3", "checksum", "no_content_size"):
                    continue
                d = zc.data(kind, n, seed=31)
                frames.append(zr.compress(d, **kw))
                datas.append(d)
    d = zc.data("records", 300000, seed=32)
    frames.append(zr.stream(d, piece=7000, flush=True, level=3, checksum=True))
    datas.append(d)
    got = run_device(frames)
    for i, z in enumerate(frames):
        assert got[i] == datas[i] == zstdec.decode(z), (i, len(z))
    assert max(len(d) for d in datas) == 4 << 20


def test_malformed_classes():
    mal = zc.malformed()
    got = run_device(list(mal.values()))
    for (name, z), g in zip(mal.items(), got):
        assert g is None and zstdec.decode(z) is None and zr.decompress(z) is None, name


def test_slot_other_than_the_bound_is_refused():
    zr.need()
    d = zc.data("text", 5000, seed=33)
    z = zr.compress(d, level=3)
    b = zstdec.bound(z)
    assert run_device([z, z, z], [b, b + 1, 0]) == [d, None, None]


def test_mutations_subset():
    zr.need()
    muts = zc.mutations()[::5]
    got = run_device([z for z, _s, _a in muts])
    for (z, src, at), g in zip(muts, got):
        host = zstdec.decode(z)
        assert g == host
        want = zr.decompress(z)
        assert g == want or (g is None and want is not None and zc.in_4stream_literals(src, at))
