"""tests/golden/snappy_batches.json (written by make_golden_snappy_batches.py with pyarrow's snappy) against its seeds:
every batch's records section, a raw snappy block or snappy-java framed chunks, decodes with the plain restatement
(tests/kafka_snappy.py) and with the host build of the device decoder (tests/snappydec) to exactly the records section of
the same batch uncompressed, and with pyarrow too when it is present.  The golden-driven checks never skip; only the
pyarrow one does when pyarrow is missing."""
import os
import sys

import pytest

import kafka_snappy as ks
import snappydec

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))

from make_golden_snappy_batches import CASES, WORKER, load, load_worker, uncompressed, worker_batches  # noqa: E402


def test_file_covers_the_cases():
    import json
    from make_golden_snappy_batches import GOLDEN
    g = json.load(open(GOLDEN))
    assert g["pyarrow"] == "24.0.0"
    assert [n for n, _s, _b in load()] == [c[0] for c in CASES]
    assert os.path.getsize(GOLDEN) < 200_000


@pytest.mark.parametrize("name", [c[0] for c in CASES])
def test_golden_batch_decodes_to_its_records(name):
    spec, batch = {n: (s, b) for n, s, b in load()}[name]
    prefs = {c[0]: c[2] for c in CASES}[name]
    plain = uncompressed(spec)
    assert batch[22] & 7 == 2 and batch[:8] == plain[:8]
    sec = batch[61:]
    assert ks.framed(sec) == (prefs["shape"] == "xerial")
    w = ks.walk(sec)
    assert snappydec.walk(sec) == w
    if prefs["shape"] == "xerial":
        assert len(w) == (len(plain) - 61 + prefs["chunk"] - 1) // prefs["chunk"]
        assert all(dl == prefs["chunk"] for _o, _l, dl in w[:-1])
    assert ks.decompress_section(sec) == plain[61:]
    assert snappydec.decode_section(sec) == plain[61:]
    if name == "empty":
        assert sec == b"\x00"
    if name.startswith("over_4mb"):
        assert len(plain) > 4 << 20


def test_golden_batches_with_pyarrow():
    import snappy_ref as sr
    sr.need()
    for name, spec, batch in load():
        sec = batch[61:]
        got = b"".join(sr.decompress(sec[o:o + n]) for o, n, _d in ks.walk(sec))
        assert got == uncompressed(spec)[61:], name


def test_worker_fetch():
    """the Worker.run fetch: every batch decodes to its seeded records but the corrupt one, which is refused"""
    got = load_worker()
    want = worker_batches()
    assert len(got) == WORKER["batches"]
    for i, (g, w) in enumerate(zip(got, want)):
        assert ks.framed(g[61:])
        d = snappydec.decode_section(g[61:])
        assert d == ks.decompress_section(g[61:])
        assert (d is None) if i == WORKER["corrupt"] else (d == w[61:]), i
