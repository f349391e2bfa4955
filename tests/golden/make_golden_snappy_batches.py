"""Writes tests/golden/snappy_batches.json: Kafka RecordBatch v2 batches with attributes 2 (snappy) whose blocks Google
snappy (as pyarrow bundles it) compressed: raw-block sections (librdkafka's and sarama's shape), snappy-java framed
sections of 32 KB chunks (the default of Java's producer, kafka-python and aiokafka) and of 1 KB chunks, an empty records
section (a raw block holding only the varint 0), and sections of more than 4 MB in both shapes.  Only the compressed
batches are stored, each gzipped and then base64-encoded: snappy's output of repetitive records is itself repetitive, and
gzip keeps the 4 MB cases small.  Their records are rebuilt from seeds as the LZ4 golden file's are
(make_golden_lz4_batches.records / uncompressed).

It also holds `worker_fetch`: 10 batches of 20 tool events (seed 661), framed in 32 KB chunks, the seventh with one bit of
a block flipped so that snappy refuses it, for the Worker.run test of tests/test_gpu_kafka_snappy_fetch.py.

    python tests/golden/make_golden_snappy_batches.py       (needs pyarrow; the tests only read the JSON)
"""
import base64
import gzip
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [HERE, os.path.join(HERE, ".."), os.path.join(HERE, "..", "..", "calfkit-sdk_b200"), os.path.join(HERE, "..", "..")]

from make_golden_lz4_batches import TS, uncompressed, with_section  # noqa: E402

GOLDEN = os.path.join(HERE, "snappy_batches.json")
CASES = [
    ("raw_small", {"n": 16, "seed": 751}, dict(shape="raw")),
    ("raw_cycle", {"n": 60, "seed": 752, "cycle": 8}, dict(shape="raw")),
    ("xerial_32k", {"n": 60, "seed": 753, "cycle": 8}, dict(shape="xerial", chunk=32 << 10)),
    ("xerial_32k_one_chunk", {"n": 12, "seed": 754}, dict(shape="xerial", chunk=32 << 10)),
    ("xerial_1k", {"n": 30, "seed": 755}, dict(shape="xerial", chunk=1 << 10)),
    ("incompressible_raw", {"n": 1, "seed": 756, "random": 3000}, dict(shape="raw")),
    ("incompressible_xerial_1k", {"n": 2, "seed": 757, "random": 3000}, dict(shape="xerial", chunk=1 << 10)),
    ("empty", {"n": 0, "seed": 758}, dict(shape="raw")),
    ("over_4mb_raw", {"n": 560, "seed": 759, "cycle": 8, "size": 8000}, dict(shape="raw")),
    ("over_4mb_xerial_32k", {"n": 560, "seed": 760, "cycle": 8, "size": 8000}, dict(shape="xerial", chunk=32 << 10)),
]
WORKER = {"batches": 10, "per": 20, "seed": 661, "corrupt": 6}


def section(raw_section: bytes, prefs: dict) -> bytes:
    import kafka_snappy as ks
    import snappy_ref as sr
    if prefs["shape"] == "raw":
        return sr.compress(raw_section)
    return ks.xerial(raw_section, prefs["chunk"])


def worker_batches() -> list[bytes]:
    """the worker_fetch batches, rebuilt uncompressed"""
    import json as js
    from calfkit import synth
    from oracle import kafka_batch as kb
    recs = synth.tool_events(WORKER["batches"] * WORKER["per"], seed=WORKER["seed"])
    out = []
    for bi in range(WORKER["batches"]):
        chunk = recs[bi * WORKER["per"]:(bi + 1) * WORKER["per"]]
        krecs = [kb.calfkit_record(r, js.loads(r)["context"]["deps"]["correlation_id"], keyed=(j % 4 != 0)) for j, r in enumerate(chunk)]
        out.append(kb.encode_batch(krecs, base_offset=2000 + bi * WORKER["per"], base_timestamp=TS + bi))
    return out


def load():
    """[(name, spec, compressed batch)] of the golden file"""
    g = json.load(open(GOLDEN))
    return [(c["name"], c["records"], _unpack(c["batch"])) for c in g["batches"]]


def load_worker() -> list[bytes]:
    return [_unpack(b) for b in json.load(open(GOLDEN))["worker_fetch"]]


def _pack(b: bytes) -> str:
    return base64.b64encode(gzip.compress(b, mtime=0)).decode()


def _unpack(s: str) -> bytes:
    return gzip.decompress(base64.b64decode(s))


def main():
    import kafka_snappy as ks
    import snappy_ref as sr
    from oracle import kafka_batch as kb
    out = []
    for name, spec, prefs in CASES:
        raw = uncompressed(spec)
        sec = section(raw[kb.HEADER_LEN:], prefs)
        assert ks.decompress_section(sec) == raw[kb.HEADER_LEN:], name
        for off, ln, _d in ks.walk(sec):
            assert sr.decompress(sec[off:off + ln]) is not None, name
        out.append({"name": name, "records": spec, "setting": prefs,
                    "batch": _pack(with_section(raw, sec, codec=2))})
    wf = []
    for bi, plain in enumerate(worker_batches()):
        z = bytearray(ks.xerial(plain[kb.HEADER_LEN:], 32 << 10))
        if bi == WORKER["corrupt"]:
            (off, ln, _d), = ks.walk(bytes(z))
            flip = off + ln // 2
            while True:                  # the first bit flip from the block's middle on that snappy refuses
                z[flip] ^= 0x10
                if sr.decompress(bytes(z[off:off + ln])) is None:
                    break
                z[flip] ^= 0x10
                flip += 1
            assert ks.decompress_section(bytes(z)) is None
        wf.append(_pack(with_section(plain, bytes(z), codec=2)))
    with open(GOLDEN, "w") as fh:
        json.dump({"pyarrow": sr.version(), "worker": WORKER, "batches": out, "worker_fetch": wf}, fh, indent=0)
        fh.write("\n")


if __name__ == "__main__":
    main()
