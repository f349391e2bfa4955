"""The snappy block decoder on the device alone (ck_sn_decode_block, csrc/ck_snappy.cuh, through tests/snappydec: a warp per
raw block), held against the g++ build of the same source and against Google snappy (pyarrow's) on the blocks the CPU suite
uses: 1 B to 4 MiB blocks of every data kind, the hand-written blocks (overlapping copies at offsets 1-8, copy-4, every
literal-length width), every malformed block, the chunks of framed sections, and a seeded subset of the mutations: the same
bytes, or the same refusal."""
import numpy as np
import pytest

import kafka_snappy as ks
import snappy_ref as sr
import snappydec
import zstd_cases as zc
from test_snappy_hostsim import SIZES, host

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def run_device(blocks, caps=None):
    """each raw block decoded on the device into a slot of its declared length (or caps[i]): bytes or None"""
    import torch
    if caps is None:
        caps = [d if (d := snappydec.declared(z)) is not None and d <= ks.RATIO * len(z) else 0 for z in blocks]
    soff = np.concatenate(([0], np.cumsum([len(z) for z in blocks]))).astype(np.int64)
    doff = np.concatenate(([0], np.cumsum(caps))).astype(np.int64)
    src = torch.from_numpy(np.frombuffer(b"".join(blocks) + b"\0" * 256, dtype=np.uint8).copy()).cuda()
    dst = torch.zeros(int(doff[-1]) + 256, dtype=torch.uint8, device="cuda")
    out_len = torch.zeros(len(blocks), dtype=torch.int64, device="cuda")
    assert snappydec.lib().snappy_blocks(src.data_ptr(), torch.from_numpy(soff).cuda().data_ptr(), len(blocks), dst.data_ptr(),
                                         torch.from_numpy(doff).cuda().data_ptr(), out_len.data_ptr()) == 0
    data, lens = dst.cpu().numpy(), out_len.cpu().numpy()
    return [None if lens[i] < 0 else data[doff[i]:doff[i] + lens[i]].tobytes() for i in range(len(blocks))]


def test_blocks_1b_to_4mb():
    sr.need()
    blocks, datas = [], []
    for kind in zc.KINDS:
        for n in SIZES:
            d = zc.data(kind, n, seed=21)
            blocks.append(sr.compress(d))
            datas.append(d)
    got = run_device(blocks)
    for i, z in enumerate(blocks):
        assert got[i] == datas[i] == host(z), (i, len(z))
    assert max(len(d) for d in datas) == 4 << 20


def test_hand_written_and_malformed_blocks():
    hand = ks.hand_blocks()
    mal = ks.malformed_blocks()
    got = run_device([z for z, _c in hand.values()] + list(mal.values()))
    for (name, (z, content)), g in zip(hand.items(), got):
        assert g == content == host(z), name
    for (name, z), g in zip(mal.items(), got[len(hand):]):
        assert g is None and host(z) is None, name


def test_framed_chunks():
    """every chunk of framed sections of 32 KB and 1 KB chunks, decoded side by side as the fetch path decodes them"""
    sr.need()
    d = zc.data("records", 300000, seed=25)
    blocks, want = [], []
    for chunk in (32 << 10, 1 << 10):
        sec = ks.xerial(d, chunk)
        for off, ln, _dl in ks.walk(sec):
            blocks.append(sec[off:off + ln])
        want.append(d)
    got = run_device(blocks)
    assert b"".join(got) == b"".join(want)


def test_slot_other_than_the_declared_length_is_refused():
    sr.need()
    d = zc.data("text", 5000, seed=22)
    z = sr.compress(d)
    assert run_device([z, z, z], [5000, 5001, 4999]) == [d, None, None]


def test_mutations_subset():
    sr.need()
    srcs = [sr.compress(zc.data(k, n, seed=24)) for k in zc.KINDS for n in (40, 700, 5000)]
    srcs += [z for z, _c in ks.hand_blocks().values() if len(z) > 1]
    muts = ks.mutations(srcs)[::3]
    got = run_device(muts)
    for z, g in zip(muts, got):
        assert g == host(z) == sr.decompress(z)
