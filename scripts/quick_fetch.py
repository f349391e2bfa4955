"""Cost of consuming LZ4, gzip, zstd and snappy fetch responses on a config-2 step (device-template tool node, 1M events), engine level.

The step's tool events are framed once by the record form of the frame pass (ck_encode_frames_records), uncompressed and
with LZ4 (ck_set_option 3 = 3), as a producer would write them to the tool's input topic; the gzip fetch is the same
step's uncompressed frames with every records section recompressed on the host by zlib at level 6 (the level Java's
GZIPOutputStream uses), one member per batch; the zstd fetch is the same with every records section recompressed by
libzstd at level 3 (Kafka's default zstd level) and fed to it in 64 KB pieces, so that its frames carry no content size
(the zstd leg is left out, and reported as not measured, when libzstd.so.1 cannot be loaded).  The snappy fetches are the
same with every records section recompressed by Google snappy (pyarrow's): framed by snappy-java in 32 KB chunks, as Java's
producer, kafka-python and aiokafka write them, and as one raw block per batch, as librdkafka and sarama write them (both
legs are left out, and reported as not measured, without pyarrow).  The legs, alternating, two runs each, consume one of
those fetch responses per step:
  plain  ck_submit_recordbatch over the uncompressed frames + plan + the copies a Lane makes (results, record index)
  lz4    the same over the LZ4 frames: their records sections are decoded on the device, and the decoded region is
         copied back with the results (ck_fetch_rb_decoded_async)
  gzip   the same over the gzip frames (inflated on the device)
  zstd   the same over the zstd frames (decoded on the device)
  snappy the same over the snappy-java framed frames (decoded on the device, a warp per 32 KB chunk)
  snappy_raw  the same over the raw-block snappy frames (a warp per batch: each batch is one block)
  txn    the uncompressed frames as transactions of four interleaved producers, each followed by its commit or abort
         marker (about 10 % of the frames aborted), consumed read_committed: the mask of the whole fetch is computed once
         (ck_fetch_txn_mask) and handed to every step (ck_set_fetch_hidden); the aborted and control batches' records
         are skipped (CK_SKIPPED), so the leg's "skipped_records" are not walked
Per leg: step time (CUDA events around the whole step, copies included), the fetch and walk kernels (profile timer
"walk": CRC, decode, split, fields and the walker), each decode alone (walk of the leg minus walk of plain), events/s,
and H2D / D2H bytes per step.  Prints one JSON line with the card name and power limit read in the same run.

    python scripts/quick_fetch.py [events]
"""
import ctypes as C
import json
import os
import struct
import subprocess
import sys
import time
import zlib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "calfkit-sdk_b200"))
import numpy as np  # noqa: E402
import torch  # noqa: E402
from calfkit import synth  # noqa: E402
from calfkit.engine import BatchEngine, ToolTemplate  # noqa: E402
from calfkit.engine._lib import PUB_DTYPE, ptr  # noqa: E402
from calfkit.engine.lane import PinnedBuffer  # noqa: E402

TOPICS = ["tool.get_weather.input", "tool.get_weather.output", "weather_agent.input"]
n = int(sys.argv[1]) if len(sys.argv) > 1 else 1_000_000
recs = synth.tool_events(n, seed=0)


def corr_of(r: bytes) -> str:
    k = r.index(b'"correlation_id":"') + 18
    return r[k:r.index(b'"', k)].decode()


items = [(r, c.encode(), c) for r, c in ((r, corr_of(r)) for r in recs)]
fetch = {}
fr = BatchEngine(0, max_records=n, max_in_bytes=sum(len(r) for r in recs) + 64 * n + 4096)
fr.register_topics(TOPICS, num_partitions=8)
for codec in (None, "lz4"):
    fr.set_frame_compression(codec)
    fr.encode_frames_records("tool.get_weather.input", items, 1767225600000)
    frames = fr.fetch_frames()
    fetch["lz4" if codec else "plain"] = b"".join(frames.frame(i).tobytes() for i in range(len(frames)))
fr.close()
del items


def gzip_frames(buf: bytes) -> bytes:
    """every frame's records section [61, end) as one gzip member (zlib level 6), attributes codec 1, CRC32C recomputed"""
    from oracle import kafka_batch as kb
    out, pos = [], 0
    while pos + 12 <= len(buf):
        end = pos + 12 + int.from_bytes(buf[pos + 8:pos + 12], "big")
        f = buf[pos:end]
        c = zlib.compressobj(6, zlib.DEFLATED, 31)
        sec = c.compress(f[61:]) + c.flush()
        covered = struct.pack(">h", (struct.unpack_from(">h", f, 21)[0] & ~7) | 1) + f[23:61] + sec
        out.append(f[:8] + struct.pack(">i", len(covered) + 9) + f[12:17] + struct.pack(">I", kb.crc32c(covered)) + covered)
        pos = end
    return b"".join(out)


sys.path.insert(0, ROOT)
fetch["gzip"] = gzip_frames(fetch["plain"])
sys.path.insert(0, os.path.join(ROOT, "tests"))
import zstd_ref  # noqa: E402


def zstd_frames(buf: bytes) -> bytes:
    """every frame's records section as one zstd frame (libzstd level 3, streamed in 64 KB pieces), attributes codec 4"""
    from oracle import kafka_batch as kb
    out, pos = [], 0
    while pos + 12 <= len(buf):
        end = pos + 12 + int.from_bytes(buf[pos + 8:pos + 12], "big")
        f = buf[pos:end]
        sec = zstd_ref.stream(f[61:], piece=64 << 10, level=3)
        covered = struct.pack(">h", (struct.unpack_from(">h", f, 21)[0] & ~7) | 4) + f[23:61] + sec
        out.append(f[:8] + struct.pack(">i", len(covered) + 9) + f[12:17] + struct.pack(">I", kb.crc32c(covered)) + covered)
        pos = end
    return b"".join(out)


if zstd_ref.lib() is not None:
    fetch["zstd"] = zstd_frames(fetch["plain"])
import snappy_ref  # noqa: E402


def snappy_frames(buf: bytes, chunk) -> bytes:
    """every frame's records section in snappy, attributes codec 2: framed in `chunk`-byte chunks, or one raw block (None)"""
    import kafka_snappy
    from oracle import kafka_batch as kb
    out, pos = [], 0
    while pos + 12 <= len(buf):
        end = pos + 12 + int.from_bytes(buf[pos + 8:pos + 12], "big")
        f = buf[pos:end]
        sec = snappy_ref.compress(f[61:]) if chunk is None else kafka_snappy.xerial(f[61:], chunk)
        covered = struct.pack(">h", (struct.unpack_from(">h", f, 21)[0] & ~7) | 2) + f[23:61] + sec
        out.append(f[:8] + struct.pack(">i", len(covered) + 9) + f[12:17] + struct.pack(">I", kb.crc32c(covered)) + covered)
        pos = end
    return b"".join(out)


if snappy_ref.available():
    fetch["snappy"] = snappy_frames(fetch["plain"], 32 << 10)
    fetch["snappy_raw"] = snappy_frames(fetch["plain"], None)
import kafka_txn  # noqa: E402
from calfkit.engine.batch import fetch_txn_mask  # noqa: E402
_starts = [0]
while _starts[-1] + 12 <= len(fetch["plain"]):
    _starts.append(_starts[-1] + 12 + int.from_bytes(fetch["plain"][_starts[-1] + 8:_starts[-1] + 12], "big"))
fetch["txn"], txn_aborted, _ab = kafka_txn.transactional_fetch([fetch["plain"][a:b] for a, b in zip(_starts, _starts[1:])], 0.1, seed=7)
txn_mask = fetch_txn_mask(np.frombuffer(fetch["txn"], dtype=np.uint8), [(0, txn_aborted)])
LEGS = [k for k in ("plain", "lz4", "gzip", "zstd", "snappy", "snappy_raw", "txn") if k in fetch]

e = BatchEngine(0, max_records=n + len(_starts) + 64, max_in_bytes=len(fetch["txn"]) + 4096)
e.register_topics(TOPICS, num_partitions=8)
e.set_tool_node("tool.get_weather.output", ToolTemplate.from_format("It's sunny in {location}"))
pinned = {}
for k, v in fetch.items():
    pinned[k] = PinnedBuffer(len(v))
    pinned[k].array[:len(v)] = np.frombuffer(v, dtype=np.uint8)
b_out = PinnedBuffer(e.max_out + 64)
b_off, b_len = PinnedBuffer(8 * (e.max_payloads + 1)), PinnedBuffer(4 * e.max_payloads)
b_pubs = PinnedBuffer(PUB_DTYPE.itemsize * 2 * e.max_records)
b_rb = PinnedBuffer(16 * e.max_records + 64)
b_dec = {}
st = torch.cuda.ExternalStream(e.stream_ptr())


def step(name: str) -> tuple[int, int]:
    buf = pinned[name]
    nrec = C.c_uint32(0)
    if name == "txn":
        e.set_fetch_hidden(txn_mask)
    e._check(e.lib.ck_submit_recordbatch(e.h, ptr(buf.array), buf.nbytes, C.byref(nrec)))
    e.n = m = nrec.value
    e.tool_plan()
    nb, npay, npub = e.out_size()
    e._check(e.lib.ck_fetch_output_async(e.h, ptr(b_out.array), b_out.nbytes, ptr(b_off.array), ptr(b_len.array), ptr(b_pubs.array)))
    e._check(e.lib.ck_fetch_rb_index_async(e.h, ptr(b_rb.array), ptr(b_rb.array[8 * m:]), None, None, None, None, ptr(b_rb.array[12 * m:])))
    d2h = nb + 8 * (npay + 1) + 4 * npay + PUB_DTYPE.itemsize * npub + 16 * m
    base, dn = C.c_uint64(0), C.c_uint64(0)
    e._check(e.lib.ck_fetch_rb_decoded_async(e.h, None, 0, C.byref(base), C.byref(dn)))
    if dn.value:
        if name not in b_dec or b_dec[name].nbytes < dn.value:
            b_dec[name] = PinnedBuffer(dn.value)
        e._check(e.lib.ck_fetch_rb_decoded_async(e.h, ptr(b_dec[name].array), b_dec[name].nbytes, None, None))
        d2h += dn.value
    e.sync()
    return buf.nbytes, d2h


def leg(name: str, steps: int = 5) -> dict:
    step(name)
    m = e.n
    flags = b_rb.array[12 * m:16 * m].view(np.uint32)
    bad, skipped = int((flags == 1).sum()), int((flags == 2).sum())
    e.profile(True)
    e.profile_read()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record(st)
    for _ in range(steps):
        h2d, d2h = step(name)
    ev1.record(st)
    torch.cuda.synchronize()
    prof = e.profile_read()
    e.profile(False)
    ms = ev0.elapsed_time(ev1) / steps
    return {"step_ms": round(ms, 3), "walk_kernel_ms": round(prof["walk"][0] / steps, 3), "events_per_s": round(n / ms * 1e3),
            "h2d_bytes_per_step": h2d, "d2h_bytes_per_step": d2h, "bad_records": bad,
            "skipped_records": skipped}


q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
res = {"events": n, "gpu": q.stdout.strip(), "libzstd": zstd_ref.version() if "zstd" in fetch else None,
       "pyarrow_snappy": snappy_ref.version() if "snappy" in fetch else None,
       "fetch_bytes": {k: len(v) for k, v in fetch.items()}, "runs": []}
t0 = time.time()
for _ in range(2):
    for name in LEGS:
        res["runs"].append({"leg": name, **leg(name)})
res["wall_s"] = round(time.time() - t0, 1)
walk = {k: min(r["walk_kernel_ms"] for r in res["runs"] if r["leg"] == k) for k in LEGS}
res["lz4_decode_ms"] = round(walk["lz4"] - walk["plain"], 3)
res["gzip_decode_ms"] = round(walk["gzip"] - walk["plain"], 3)
res["zstd_decode_ms"] = round(walk["zstd"] - walk["plain"], 3) if "zstd" in walk else "not measured"
for k in ("snappy", "snappy_raw"):
    res[f"{k}_decode_ms"] = round(walk[k] - walk["plain"], 3) if k in walk else "not measured"
res["txn_walk_minus_plain_ms"] = round(walk["txn"] - walk["plain"], 3)
res["txn_aborted_frames"] = f"{sum(_ab)} of {len(_ab)}"
res["decoded_bytes"] = {k: int(b.nbytes) for k, b in b_dec.items()}
print(json.dumps(res))
