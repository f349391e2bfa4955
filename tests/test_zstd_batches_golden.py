"""tests/golden/zstd_batches.json (written by make_golden_zstd_batches.py with libzstd 1.5.5) against its seeds: every
batch's records section, one zstd frame, decodes with the host build of the device decoder (tests/zstdec) to exactly
the records section of the same batch uncompressed, and with libzstd too when it is present.  The golden-driven checks
never skip; only the libzstd one does when the library is missing."""
import os
import sys

import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))

import zstdec  # noqa: E402
from make_golden_zstd_batches import CASES, WORKER, load, load_worker, uncompressed, worker_batches  # noqa: E402


def test_file_covers_the_cases():
    import json
    from make_golden_zstd_batches import GOLDEN
    g = json.load(open(GOLDEN))
    assert g["libzstd"] == "1.5.5"
    assert [n for n, _s, _b in load()] == [c[0] for c in CASES]
    assert os.path.getsize(GOLDEN) < 160_000


@pytest.mark.parametrize("name", [c[0] for c in CASES])
def test_golden_batch_decodes_to_its_records(name):
    spec, batch = {n: (s, b) for n, s, b in load()}[name]
    plain = uncompressed(spec)
    assert batch[22] & 7 == 4 and batch[:8] == plain[:8]
    z = batch[61:]
    assert zstdec.bound(z) is not None
    assert zstdec.decode(z) == plain[61:]
    if name == "over_4mb":
        assert len(plain) > 4 << 20
    if name == "streamed_flushes":
        assert not (z[4] & 0x20) and z[4] >> 6 == 0              # no content size, a window descriptor


def test_golden_batches_with_libzstd():
    import zstd_ref as zr
    zr.need()
    for name, spec, batch in load():
        assert zr.decompress(batch[61:]) == uncompressed(spec)[61:], name


def test_worker_fetch():
    """the Worker.run fetch: every batch decodes to its seeded records but the corrupt one, which is refused"""
    got = load_worker()
    want = worker_batches()
    assert len(got) == WORKER["batches"]
    for i, (g, w) in enumerate(zip(got, want)):
        d = zstdec.decode(g[61:])
        assert (d is None) if i == WORKER["corrupt"] else (d == w[61:]), i
