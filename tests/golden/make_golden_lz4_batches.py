"""Writes tests/golden/lz4_batches.json: Kafka RecordBatch v2 batches with attributes 3 (LZ4) whose records sections the
system liblz4 (LZ4F_compressFrame) compressed, across block sizes of 64 KB to 4 MB, linked and independent blocks, block
checksums, content checksums and content size on and off, and one incompressible section (stored blocks).
Only the compressed batches are stored (base64).  The records — calfkit tool-stage envelopes from the seeded generator,
encoded by oracle/kafka_batch.py — are made again from their seeds: `uncompressed(case)` gives the batch each one
decompresses to (tests/test_lz4_batches_golden.py, tests/test_gpu_kafka_lz4_fetch.py).

    python tests/golden/make_golden_lz4_batches.py        (needs liblz4; the tests only read the JSON)
"""
import base64
import json
import os
import struct
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [HERE, os.path.join(HERE, "..", "..", "calfkit-sdk_b200"), os.path.join(HERE, "..", "..")]

TS = 1767225600123
GOLDEN = os.path.join(HERE, "lz4_batches.json")

# name, records, compressFrame preferences.  Records: n distinct tool events; or (cycle k) k distinct events of `size`
# bytes repeated, with their own correlation ids and offsets, so that sections of 1 MB and more compress to a few KB and
# linked blocks match across their boundaries; or (random) values of random bytes, the incompressible section.  liblz4
# lowers the block maximum to fit the input: a 256 KB / 1 MB / 4 MB case needs more than 64 KB / 256 KB / 1 MB of records
CASES = [
    ("b64k_independent", {"n": 55, "seed": 301}, {}),
    ("b64k_linked", {"n": 60, "seed": 302, "cycle": 8}, {"linked": True}),
    ("b64k_block_checksum", {"n": 60, "seed": 303, "cycle": 8}, {"block_sum": True}),
    ("b64k_content_checksum", {"n": 60, "seed": 304, "cycle": 8}, {"content_sum": True}),
    ("b64k_content_size", {"n": 60, "seed": 305, "cycle": 8}, {"content_size": True}),
    ("b64k_all_flags", {"n": 60, "seed": 306, "cycle": 8}, {"linked": True, "block_sum": True, "content_sum": True, "content_size": True}),
    ("b256k_independent", {"n": 60, "seed": 307, "cycle": 8}, {"block_id": 5}),
    ("b256k_linked_checksums", {"n": 40, "seed": 308, "cycle": 8, "size": 8000}, {"block_id": 5, "linked": True, "block_sum": True, "content_sum": True}),
    ("b1m", {"n": 36, "seed": 309, "cycle": 8, "size": 8000}, {"block_id": 6}),
    ("b4m_content_checksum", {"n": 136, "seed": 310, "cycle": 8, "size": 8000}, {"block_id": 7, "content_sum": True, "content_size": True}),
    ("incompressible", {"n": 1, "seed": 311, "random": 3000}, {"block_sum": True}),
]


def records(spec: dict):
    """the oracle records of a case, rebuilt from its seed"""
    from calfkit import synth
    from oracle import kafka_batch as kb
    n, seed = spec["n"], spec["seed"]
    if spec.get("random"):
        rng = np.random.default_rng(seed)
        vals = [rng.integers(0, 256, spec["random"], dtype=np.uint8).tobytes() for _ in range(n)]
    elif spec.get("cycle"):
        distinct = synth.tool_events(spec["cycle"], seed=seed, size=spec.get("size", 1152))
        vals = [distinct[i % len(distinct)] for i in range(n)]
    else:
        vals = synth.tool_events(n, seed=seed)
    return [kb.calfkit_record(v, f"corr-{seed}-{i:06d}", keyed=i % 5 != 4) for i, v in enumerate(vals)]


def uncompressed(spec: dict) -> bytes:
    from oracle import kafka_batch as kb
    return kb.encode_batch(records(spec), base_offset=spec["seed"], base_timestamp=TS)


def with_section(batch: bytes, section: bytes, codec: int = 3) -> bytes:
    """`batch` (uncompressed v2) with its records section [61, end) replaced by `section`, attributes codec `codec`,
    batchLength and CRC32C recomputed"""
    from oracle import kafka_batch as kb
    attrs = (struct.unpack_from(">h", batch, 21)[0] & ~7) | codec
    covered = struct.pack(">h", attrs) + batch[23:kb.HEADER_LEN] + section
    return batch[:8] + struct.pack(">i", len(covered) + 9) + batch[12:17] + struct.pack(">I", kb.crc32c(covered)) + covered


def load():
    """[(name, spec, compressed batch)] of the golden file"""
    g = json.load(open(GOLDEN))
    return [(c["name"], c["records"], base64.b64decode(c["batch"])) for c in g["batches"]]


def main():
    from oracle import kafka_batch as kb
    from make_golden_lz4 import compress, lib
    L = lib()
    out = []
    for name, spec, prefs in CASES:
        raw = uncompressed(spec)
        section = compress(L, raw[kb.HEADER_LEN:], **prefs)
        out.append({"name": name, "records": spec, "batch": base64.b64encode(with_section(raw, section)).decode()})
    with open(GOLDEN, "w") as fh:
        json.dump({"liblz4": L.LZ4_versionString().decode(), "batches": out}, fh, indent=0)
        fh.write("\n")


if __name__ == "__main__":
    main()
