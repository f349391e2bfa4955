"""Writes tests/golden/zstd_batches.json: Kafka RecordBatch v2 batches with attributes 4 (zstd) whose records sections
libzstd 1.5.5 compressed, across levels -5, 1, 3 and 19, content size off, checksum on, a small window, long-distance
matching, targetCBlockSize, a streamed frame with flushes, and sections of raw blocks and of RLE blocks written by
tests/zstd_cases.py; sections from empty to more than 4 MB.  Only the compressed batches are stored (base64); their
records are rebuilt from seeds as the LZ4 golden file's are (make_golden_lz4_batches.records / uncompressed).

It also holds `worker_fetch`: 10 batches of 20 tool events (seed 651), checksummed frames at level 3, the seventh with
one bit of its frame flipped (libzstd refuses it), for the Worker.run test of tests/test_gpu_kafka_zstd_fetch.py.

    python tests/golden/make_golden_zstd_batches.py       (needs libzstd; the tests only read the JSON)
"""
import base64
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [HERE, os.path.join(HERE, ".."), os.path.join(HERE, "..", "..", "calfkit-sdk_b200"), os.path.join(HERE, "..", "..")]

from make_golden_lz4_batches import TS, uncompressed, with_section  # noqa: E402

GOLDEN = os.path.join(HERE, "zstd_batches.json")
CASES = [
    ("level-5", {"n": 16, "seed": 701}, dict(level=-5)),
    ("level1", {"n": 16, "seed": 702}, dict(level=1)),
    ("level3", {"n": 16, "seed": 703}, dict(level=3)),
    ("level19", {"n": 16, "seed": 704}, dict(level=19)),
    ("no_content_size", {"n": 60, "seed": 705, "cycle": 8}, dict(level=3, content_size=False)),
    ("checksum", {"n": 60, "seed": 706, "cycle": 8}, dict(level=3, checksum=True)),
    ("window_log10", {"n": 20, "seed": 707, "cycle": 8}, dict(level=3, window_log=10, checksum=True)),
    ("ldm", {"n": 200, "seed": 708, "cycle": 8, "size": 8000}, dict(level=3, ldm=True)),
    ("target_cblock", {"n": 12, "seed": 709}, dict(level=3, target_cblock=1340)),
    ("streamed_flushes", {"n": 60, "seed": 710, "cycle": 8}, dict(stream=True, level=3, checksum=True)),
    ("raw_blocks", {"n": 6, "seed": 711}, dict(writer="raw")),
    ("rle_blocks", {"n": 3, "seed": 712}, dict(writer="rle")),
    ("empty", {"n": 0, "seed": 713}, dict(level=3, checksum=True)),
    ("over_4mb", {"n": 560, "seed": 714, "cycle": 8, "size": 8000}, dict(level=3, checksum=True)),
]
WORKER = {"batches": 10, "per": 20, "seed": 651, "corrupt": 6}


def section(raw_section: bytes, prefs: dict) -> bytes:
    import zstd_cases as zc
    import zstd_ref as zr
    prefs = dict(prefs)
    w = prefs.pop("writer", None)
    if w == "raw":                       # raw blocks of at most 4 KB, window 64 KB
        parts = [raw_section[i:i + 4096] for i in range(0, len(raw_section), 4096)] or [b""]
        return zc.frame([zc.block(i == len(parts) - 1, 0, p) for i, p in enumerate(parts)], window_log=16)
    if w == "rle":                       # every run of 2 or more equal bytes an RLE block, the rest raw blocks
        blocks, i, lit = [], 0, bytearray()
        while i < len(raw_section):
            j = i
            while j < len(raw_section) and raw_section[j] == raw_section[i]:
                j += 1
            if j - i >= 2:
                if lit:
                    blocks.append((0, bytes(lit), len(lit)))
                    lit = bytearray()
                blocks.append((1, raw_section[i:i + 1], j - i))
            else:
                lit += raw_section[i:j]
            i = j
        if lit:
            blocks.append((0, bytes(lit), len(lit)))
        return zc.frame([zc.block(k == len(blocks) - 1, t, p, s) for k, (t, p, s) in enumerate(blocks)],
                        fcs=len(raw_section), window_log=16, checksum=True, content=raw_section)
    if prefs.pop("stream", False):
        return zr.stream(raw_section, piece=3000, flush=True, **prefs)
    return zr.compress(raw_section, **prefs)


def worker_batches() -> list[bytes]:
    """the worker_fetch batches, rebuilt: (uncompressed batches, their records' values)"""
    import json as js
    from calfkit import synth
    from oracle import kafka_batch as kb
    recs = synth.tool_events(WORKER["batches"] * WORKER["per"], seed=WORKER["seed"])
    out = []
    for bi in range(WORKER["batches"]):
        chunk = recs[bi * WORKER["per"]:(bi + 1) * WORKER["per"]]
        krecs = [kb.calfkit_record(r, js.loads(r)["context"]["deps"]["correlation_id"], keyed=(j % 4 != 0)) for j, r in enumerate(chunk)]
        out.append(kb.encode_batch(krecs, base_offset=1000 + bi * WORKER["per"], base_timestamp=TS + bi))
    return out


def load():
    """[(name, spec, compressed batch)] of the golden file"""
    g = json.load(open(GOLDEN))
    return [(c["name"], c["records"], base64.b64decode(c["batch"])) for c in g["batches"]]


def load_worker() -> list[bytes]:
    return [base64.b64decode(b) for b in json.load(open(GOLDEN))["worker_fetch"]]


def main():
    from oracle import kafka_batch as kb
    import zstd_ref as zr
    out = []
    for name, spec, prefs in CASES:
        raw = uncompressed(spec)
        sec = section(raw[kb.HEADER_LEN:], prefs)
        assert zr.decompress(sec) == raw[kb.HEADER_LEN:], name
        out.append({"name": name, "records": spec, "setting": {k: v for k, v in prefs.items()},
                    "batch": base64.b64encode(with_section(raw, sec, codec=4)).decode()})
    wf = []
    for bi, plain in enumerate(worker_batches()):
        z = bytearray(zr.compress(plain[kb.HEADER_LEN:], level=3, checksum=True))
        if bi == WORKER["corrupt"]:
            z[len(z) // 2] ^= 0x10
            assert zr.decompress(bytes(z)) is None
        wf.append(base64.b64encode(with_section(plain, bytes(z), codec=4)).decode())
    with open(GOLDEN, "w") as fh:
        json.dump({"libzstd": zr.version(), "worker": WORKER, "batches": out, "worker_fetch": wf}, fh, indent=0)
        fh.write("\n")


if __name__ == "__main__":
    main()
