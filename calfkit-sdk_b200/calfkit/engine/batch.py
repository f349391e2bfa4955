"""BatchEngine: the host side of one CUDA stream's worth of the hot path.

One engine = one `ck_handle` (device buffers + stream).  It replaces, batch-wise, the reference's
per-record sandwich  bytes-in -> Envelope -> handler -> _publish_action -> bytes-out
(reference calfkit/nodes/base.py:149-164, calfkit/worker/worker.py:45-53) for the node kinds the
reference ships (@agent_tool nodes, Agent fan-out).  All decoding, routing and encoding happens in
the CUDA kernels behind the C-ABI; this class only moves buffers and interprets result tables.
"""
from __future__ import annotations

import ctypes as C
import json
import os
import string
from dataclasses import dataclass
from typing import Iterator, Sequence

import numpy as np

from calfkit.engine import _lib
from calfkit.engine._lib import COL, FRAME_DTYPE, NUM_COLS, PUB_DTYPE, ptr
from calfkit.exceptions import EngineError

# frame codecs the device builds, by the name Kafka clients use (KafkaBroker(compression_type=...)) -> Kafka's codec id
FRAME_CODECS = {None: 0, "lz4": 3}
# the levels of LZ4 frames (Kafka's compression.lz4.level, KIP-390): 1 .. 17; None is the default parse
LZ4_LEVELS = range(1, 18)


def check_compression_level(level) -> int | None:
    """`level` when it is None or an int in LZ4_LEVELS; else EngineError naming it"""
    if level is not None and (type(level) is not int or level not in LZ4_LEVELS):
        raise EngineError(f"compression level {level!r} is not supported (None or an int in 1 .. 17)")
    return level

# what a Kafka consumer's `isolation_level` takes: read_committed hides the records of aborted transactions (csrc/ck_txn.h)
ISOLATION_LEVELS = ("read_uncommitted", "read_committed")


def txn_partitions(aborted_transactions=None, partitions=None) -> list[tuple[int, list[tuple[int, int]], int]]:
    """the partition model of a fetch response's record set: [(byte start of the partition's batches, its AbortedTransactions
    [(producer id, first offset), ...], its partition id), ...] in byte order; `aborted_transactions` alone: one partition,
    the whole record set, partition 0.  An entry given as (start, aborted) without an id is partition r, its place in
    the list"""
    if aborted_transactions is not None and partitions is not None:
        raise EngineError("give aborted_transactions (one partition) or partitions, not both")
    if partitions is None:
        partitions = [(0, aborted_transactions or [])]
    return [(int(e[0]), [(int(pid), int(first)) for pid, first in e[1]], int(e[2]) if len(e) > 2 else r)
            for r, e in enumerate(partitions)]


def fetch_txn_mask(buf: np.ndarray, partitions) -> np.ndarray:
    """per complete batch of the record set `buf`: 1 where a read_committed consumer skips it, a transactional batch of an
    aborted producer (ck_fetch_txn_mask; control batches are skipped by the engine itself)"""
    lib = _lib.load()
    starts = np.asarray([e[0] for e in partitions], dtype=np.uint64)
    runs = np.asarray([r for r, e in enumerate(partitions) for _e in e[1]], dtype=np.uint32)
    pids = np.asarray([pid for e in partitions for pid, _f in e[1]], dtype=np.int64)
    firsts = np.asarray([first for e in partitions for _p, first in e[1]], dtype=np.int64)
    cap = buf.nbytes // 61 + 1
    mask, nb = np.zeros(cap, dtype=np.uint8), C.c_uint32(0)
    if lib.ck_fetch_txn_mask(ptr(buf), buf.nbytes, ptr(starts), len(starts), ptr(runs), ptr(pids), ptr(firsts), len(runs),
                             ptr(mask), cap, C.byref(nb)):
        raise EngineError(lib.ck_last_error(None).decode())
    return mask[:nb.value]


def fetch_positions(buf: np.ndarray, partitions) -> tuple[dict[int, int], np.ndarray]:
    """where a consumer of the record set `buf` (a fetch, or a slice of one with its partition model) resumes: ({partition
    id: lastOffset + 1 of its last complete batch} for every partition a complete batch of buf belongs to, lastOffset + 1
    of each complete batch).  Every batch counts, delivered, skipped or bad (ck_fetch_positions reads only the headers)"""
    lib = _lib.load()
    starts = np.asarray([e[0] for e in partitions], dtype=np.uint64)
    nxt = np.empty(len(starts), dtype=np.int64)
    cap = buf.nbytes // 61 + 1
    per_batch, nb = np.empty(cap, dtype=np.int64), C.c_uint32(0)
    if lib.ck_fetch_positions(ptr(buf), buf.nbytes, ptr(starts), len(starts), ptr(nxt), ptr(per_batch), cap, C.byref(nb)):
        raise EngineError(lib.ck_last_error(None).decode())
    out = {}
    for e, x in zip(partitions, nxt.tolist()):
        if x >= 0:
            out[e[2]] = x
    return out, per_batch[:nb.value]


@dataclass
class ToolTemplate:
    """A tool whose return value is a pure string template of its string arguments, e.g. the
    quickstart's get_weather: f"It's sunny in {location}" (reference
    examples/quickstart/weather_tool.py:9-12).  Such tools are evaluated on the device: the JSON
    return value is assembled from pre-escaped literal pieces and the raw (already canonically
    escaped) argument strings, so no host round trip is needed.  Anything else stays a host tool."""
    kinds: list[int]          # 0 literal, 1 argument
    pieces: list[bytes]       # literal bytes (JSON-escaped) or the argument's key name

    @classmethod
    def from_format(cls, fmt: str) -> "ToolTemplate":
        kinds, pieces = [], []
        parsed = list(string.Formatter().parse(fmt))
        lit_acc = '"'
        for literal, field, spec, conv in parsed:
            lit_acc += json.dumps(literal, ensure_ascii=False)[1:-1]
            if field is not None:
                if spec or conv or not field.isidentifier():
                    raise ValueError(f"unsupported template field {field!r}")
                kinds.append(0); pieces.append(lit_acc.encode()); lit_acc = ""
                kinds.append(1); pieces.append(json.dumps(field, ensure_ascii=False)[1:-1].encode())
        lit_acc += '"'
        kinds.append(0); pieces.append(lit_acc.encode())
        return cls(kinds, pieces)


@dataclass
class Publish:
    topic: str
    key: bytes | None
    payload: bytes
    record: int
    partition: int


class _SpanOffsets:
    """offsets[i], offsets[i+1] of records that do NOT lie back to back (values inside raw Kafka frames): indexing i gives
    the start, and BatchOutput takes the end from `end(i)`"""
    def __init__(self, off: np.ndarray, ln: np.ndarray):
        self.off, self.ln = off, ln

    def __getitem__(self, i):
        return self.off[i]

    def end(self, i):
        return int(self.off[i]) + int(self.ln[i])

    def __len__(self):
        return len(self.off) + 1


class FetchBytes:
    """the bytes value offsets of a fetch response index: offsets below len(raw) lie in the raw response, offsets from
    `base` on in the gzip, snappy, LZ4 and zstd batches' decoded records sections, `decoded` (ck_fetch_rb_decoded_async).  Sliced like an array"""
    def __init__(self, raw: np.ndarray, base: int, decoded: np.ndarray):
        self.raw, self.base, self.decoded = raw, int(base), decoded

    def __getitem__(self, s: slice) -> np.ndarray:
        a, b = int(s.start or 0), int(s.stop)
        if a >= self.base:
            return self.decoded[a - self.base:b - self.base]
        if b > len(self.raw):
            raise IndexError(f"span [{a}, {b}) runs past the raw bytes ({len(self.raw)}) and starts before the decoded ones ({self.base})")
        return self.raw[a:b]

    @property
    def nbytes(self) -> int:
        return int(self.raw.nbytes + self.decoded.nbytes)


class BatchOutput:
    """Result of one plan+emit: unique payloads + the publish table that references them."""

    def __init__(self, engine: "BatchEngine", out: np.ndarray, out_off: np.ndarray, out_len: np.ndarray, pubs: np.ndarray,
                 in_data: np.ndarray | None, in_off: np.ndarray | None, cols: np.ndarray | None, overlay=None):
        self.engine, self.out, self.out_off, self.out_len, self.pubs = engine, out, out_off, out_len, pubs
        self.in_data, self.in_off, self.cols = in_data, in_off, cols
        self.overlay = overlay          # (bytes, off[n], len[n]): canonical re-emissions of non-canonical inputs

    def record_bytes(self, r: int) -> np.ndarray:
        """the bytes the column spans of record r refer to: its canonical re-emission if it has one"""
        if self.overlay is not None and self.overlay[1][r] >= 0:
            o = int(self.overlay[1][r])
            return self.overlay[0][o:o + int(self.overlay[2][r])]
        if isinstance(self.in_off, _SpanOffsets):
            return self.in_data[int(self.in_off[r]):self.in_off.end(r)]
        return self.in_data[self.in_off[r]:self.in_off[r + 1]]

    def payload(self, i: int) -> bytes:
        return self.out[self.out_off[i]:self.out_off[i] + self.out_len[i]].tobytes()

    def live(self) -> np.ndarray:
        return self.pubs[self.pubs["payload"] != 0xFFFFFFFF]

    def topic_of(self, p) -> str:
        if p["topic_id"] >= 0:
            return self.engine.topic_names[int(p["topic_id"])]
        rec = self.record_bytes(int(p["record"]))
        raw = rec[int(p["topic_off"]):int(p["topic_off"]) + int(p["topic_len"])].tobytes()
        return json.loads(b'"' + raw + b'"')

    def key_of(self, p) -> bytes | None:
        if not p["has_key"]:
            return None
        r = int(p["record"])
        o = int(self.cols[COL["CORR_OFF"], r])
        raw = self.record_bytes(r)[o:o + int(self.cols[COL["CORR_LEN"], r])].tobytes()
        return json.loads(b'"' + raw + b'"').encode()

    def publishes(self) -> Iterator[Publish]:
        for p in self.live():
            yield Publish(self.topic_of(p), self.key_of(p), self.payload(int(p["payload"])), int(p["record"]),
                          int(p["partition"]))


def patch_base_sequence(frame: np.ndarray, seq: int) -> None:
    """write baseSequence `seq` into a RecordBatch v2 frame (uint8 array, in place) and patch its CRC32C by linearity
    (ck_crc32c_patch: O(log length), however long the frame)"""
    new = np.frombuffer((seq & 0xFFFFFFFF).to_bytes(4, "big"), dtype=np.uint8)
    old = frame[SEQ_AT:SEQ_AT + 4].copy()
    crc = C.c_uint32(int.from_bytes(frame[17:21].tobytes(), "big"))
    lib = _lib.load()
    if lib.ck_crc32c_patch(C.byref(crc), len(frame) - 21, SEQ_AT - 21, ptr(old), ptr(new)):
        raise EngineError(lib.ck_last_error(None).decode())
    frame[SEQ_AT:SEQ_AT + 4] = new
    frame[17:21] = np.frombuffer(crc.value.to_bytes(4, "big"), dtype=np.uint8)


def control_batch(producer_id: int, producer_epoch: int, commit: bool, timestamp_ms: int, base_offset: int = 0) -> np.ndarray:
    """the COMMIT or ABORT marker the broker appends to a partition when a transaction ends (ck_encode_control_batch)"""
    lib = _lib.load()
    out, n = np.empty(78, dtype=np.uint8), C.c_uint64(0)
    if lib.ck_encode_control_batch(base_offset, timestamp_ms, producer_id, producer_epoch, 1 if commit else 0, ptr(out), out.nbytes, C.byref(n)):
        raise EngineError(lib.ck_last_error(None).decode())
    return out[:n.value]


SEQ_AT = 53                    # baseSequence i32 in a RecordBatch v2 header (producerId i64 at 43, producerEpoch i16 at 51)


class Frames:
    """Kafka RecordBatch v2 frames of one frame pass, produce-ready: `table` (FRAME_DTYPE: topic id, partition, records,
    first record, offset, length) and the frame bytes back to back in `data`.  Partition -1 holds unkeyed records: the
    producer client picks their partition (with sticky partitions set, BatchEngine.set_sticky_partitions, they have one)."""

    def __init__(self, table: np.ndarray, data: np.ndarray, topic_names: dict[int, str], on_release=None):
        self.table, self.data, self.topic_names, self._on_release = table, data, topic_names, on_release

    def release(self) -> None:
        if self._on_release is not None:
            cb, self._on_release = self._on_release, None
            cb()

    def __len__(self) -> int:
        return len(self.table)

    def frame(self, i: int) -> np.ndarray:
        o = int(self.table["offset"][i])
        return self.data[o:o + int(self.table["length"][i])]

    def __iter__(self) -> Iterator[tuple[str, int | None, np.ndarray, int]]:
        """(topic, partition or None, frame bytes, records) per frame"""
        for i, e in enumerate(self.table):
            p = int(e["partition"])
            yield self.topic_names[int(e["topic_id"])], (p if p >= 0 else None), self.frame(i), int(e["n_records"])


def json_content(s: str) -> bytes:
    """a string as the content of a JSON string, the spelling the device unescapes (the envelope's own spelling)"""
    return json.dumps(s, ensure_ascii=False)[1:-1].encode()


_M64 = (1 << 64) - 1


def _splitmix64(x: int) -> int:
    x = (x + 0x9E3779B97F4A7C15) & _M64
    x = ((x ^ (x >> 30)) * 0xBF58476D1CE4E5B9) & _M64
    x = ((x ^ (x >> 27)) * 0x94D049BB133111EB) & _M64
    return x ^ (x >> 31)


def device_uuid7_hex(unix_ms: int, seed: int, index: int) -> str:
    """The frame id the fan-out kernel writes for payload slot `index` (csrc/ck_kernels.cuh
    ck_uuid7_hex) — exposed so parity tests can inject the same ids into the oracle."""
    r0, r1 = _splitmix64((seed + 2 * index) & _M64), _splitmix64((seed + 2 * index + 1) & _M64)
    hi = ((unix_ms & 0xFFFFFFFFFFFF) << 16) | 0x7000 | (r0 & 0xFFF)
    lo = (0x2 << 62) | (r1 & 0x3FFFFFFFFFFFFFFF)
    return f"{hi:016x}{lo:016x}"


def bind_host_to_gpu(device: int) -> list[int] | None:
    """Pin the calling process to the CPUs NVML reports as local to `device` (same socket / NUMA node), so
    that pinned staging buffers allocated afterwards are first-touched next to the GPU's PCIe root.  With
    one worker process per GPU this keeps eight concurrent H2D/D2H streams off the inter-socket link.
    Returns the CPU list, or None when NVML is unavailable (nothing is changed then)."""
    try:
        import pynvml
        pynvml.nvmlInit()
        vis = os.environ.get("CUDA_VISIBLE_DEVICES")
        idx = int(vis.split(",")[device]) if vis and all(x.strip().isdigit() for x in vis.split(",")) else device
        hnd = pynvml.nvmlDeviceGetHandleByIndex(idx)
        words = pynvml.nvmlDeviceGetCpuAffinity(hnd, (os.cpu_count() + 63) // 64)
        cpus = [64 * w + b for w, m in enumerate(words) for b in range(64) if (int(m) >> b) & 1]
        cpus = [c for c in cpus if c in os.sched_getaffinity(0)]
        if cpus:
            os.sched_setaffinity(0, cpus)
            return cpus
    except Exception:
        pass
    return None


class BatchEngine:
    def __init__(self, device: int = 0, max_records: int = 1 << 16, max_in_bytes: int = 128 << 20,
                 max_out_bytes: int | None = None, max_aux_bytes: int | None = None, max_payloads: int | None = None):
        self.lib = _lib.load()
        self.max_records, self.max_in = max_records, max_in_bytes
        self.max_payloads = max_payloads if max_payloads is not None else max_records
        self.max_out = max_out_bytes if max_out_bytes is not None else max_in_bytes + 528 * max_records
        self.max_aux = max_aux_bytes if max_aux_bytes is not None else max(1 << 20, max_in_bytes // 4, 32 * self.max_payloads)
        h = C.c_void_p()
        if self.lib.ck_create(device, self.max_in, self.max_out, max_records, self.max_payloads, self.max_aux, C.byref(h)):
            raise EngineError(self.lib.ck_last_error(None).decode())
        self.h = h
        self.topic_names: dict[int, str] = {}
        self.topic_ids: dict[str, int] = {}
        self.num_partitions = 0
        self.n = 0
        self._in_data = self._in_off = self._rb_raw = None
        self.frame_topics: list[str] = []
        self.read_committed = False
        self.skipped = 0                # records of the fetches submitted so far that were not delivered (CK_SKIPPED)

    # ------------------------------------------------------------------------------------------
    def close(self) -> None:
        if getattr(self, "h", None):
            self.lib.ck_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc: int) -> None:
        if rc:
            raise EngineError(self.lib.ck_last_error(self.h).decode())

    # ------------------------------------------------------------------------------------------
    def register_topics(self, names: Sequence[str], num_partitions: int = 0) -> dict[str, int]:
        """topic string -> id table on the device (ids are positions in `names`, de-duplicated)."""
        uniq = list(dict.fromkeys(names))
        blob = b"".join(n.encode() for n in uniq)
        offs = np.zeros(len(uniq) + 1, dtype=np.uint32)
        np.cumsum([len(n.encode()) for n in uniq], out=offs[1:])
        ids = np.arange(len(uniq), dtype=np.int32)
        b = np.frombuffer(blob, dtype=np.uint8) if blob else np.zeros(1, dtype=np.uint8)
        self._check(self.lib.ck_register_topics(self.h, ptr(b), ptr(offs), len(uniq), ptr(ids), num_partitions))
        self.topic_names = dict(enumerate(uniq))
        self.topic_ids = {n: i for i, n in enumerate(uniq)}
        self.num_partitions = num_partitions
        return self.topic_ids

    def set_tool_node(self, publish_topic: str | None, template: ToolTemplate | None = None) -> None:
        pid = -1
        if publish_topic is not None:
            if publish_topic not in self.topic_ids:
                raise EngineError(f"publish topic {publish_topic!r} is not registered")
            pid = self.topic_ids[publish_topic]
        if template is None:
            self._check(self.lib.ck_set_tool_node(self.h, pid, 0, None, None, None))
            return
        kinds = np.asarray(template.kinds, dtype=np.uint32)
        blob = np.frombuffer(b"".join(template.pieces) or b"\0", dtype=np.uint8)
        offs = np.zeros(len(template.pieces) + 1, dtype=np.uint32)
        np.cumsum([len(p) for p in template.pieces], out=offs[1:])
        self._check(self.lib.ck_set_tool_node(self.h, pid, len(kinds), ptr(kinds), ptr(blob), ptr(offs)))

    def set_agent_node(self, agent_name: str, callback_topic: str, publish_topic: str | None,
                       registry: dict[str, str]) -> None:
        """registry: tool_name -> the tool node's subscribe_topics[0] (reference nodes/agent.py:71-75)."""
        missing = [t for t in list(registry.values()) + ([publish_topic] if publish_topic else []) if t not in self.topic_ids]
        if missing:
            raise EngineError(f"topics not registered: {missing}")
        esc = lambda s: json.dumps(s, ensure_ascii=False)[1:-1].encode()   # noqa: E731  spliced inside JSON strings
        names = [esc(k) for k in registry]
        topics = [esc(v) for v in registry.values()]
        nb = np.frombuffer(b"".join(names) or b"\0", dtype=np.uint8)
        tb = np.frombuffer(b"".join(topics) or b"\0", dtype=np.uint8)
        no = np.zeros(len(names) + 1, dtype=np.uint32); np.cumsum([len(x) for x in names], out=no[1:])
        to = np.zeros(len(topics) + 1, dtype=np.uint32); np.cumsum([len(x) for x in topics], out=to[1:])
        an, cb = esc(agent_name), esc(callback_topic)
        anb, cbb = np.frombuffer(an, dtype=np.uint8), np.frombuffer(cb, dtype=np.uint8)
        pid = self.topic_ids[publish_topic] if publish_topic else -1
        self._check(self.lib.ck_set_agent_node(self.h, pid, ptr(anb), len(an), ptr(cbb), len(cb), ptr(nb), ptr(no),
                                               ptr(tb), ptr(to), len(names)))
        ids = np.asarray([self.topic_ids[v] for v in registry.values()] or [0], dtype=np.uint32)
        self._check(self.lib.ck_set_agent_tool_topic_ids(self.h, self.topic_ids.get(callback_topic, -1), ptr(ids), len(registry)))

    def fanout_plan(self, unix_ms: int, seed: int, max_fanout: int = 128, sequential: bool = False) -> None:
        """list[Call] / Call of the pending tool calls; sequential: first pending only (agent.py:94-108)."""
        self._check(self.lib.ck_fanout_plan(self.h, unix_ms, seed, max_fanout, 1 if sequential else 0))

    def tailcall_plan(self, unix_ms: int, seed: int) -> None:
        """TailCall to the agent's own subscribe topic (agent.py:171-175)."""
        self._check(self.lib.ck_tailcall_plan(self.h, unix_ms, seed))

    def set_bucketing(self, on: bool = True) -> None:
        """bucket every submitted batch by record length before the walk (topics with mixed record sizes / shapes)"""
        self._check(self.lib.ck_set_option(self.h, 1, 1 if on else 0))

    # ---- aggregation gate on the device (csrc/ck_gate.cuh; reference nodes/agent.py:57-68) ---------------------------
    def gate_create(self, max_entries: int = 1 << 14, max_slots: int | None = None, arena_bytes: int = 128 << 20) -> None:
        """the device holds two arenas of arena_bytes (and two entry and slot arrays): gate_compact moves between them"""
        max_slots = max_slots if max_slots is not None else 16 * max_entries
        self._check(self.lib.ck_gate_create(self.h, max_entries, max_slots, arena_bytes))
        self.gate_max_entries, self.gate_max_slots, self.gate_arena_bytes = max_entries, max_slots, arena_bytes

    def gate_register(self, min_pending: int = 2) -> None:
        """after fanout_plan: every record that went out as list[Call] becomes a pending entry of the gate"""
        self._check(self.lib.ck_gate_register(self.h, min_pending))

    def gate_arrive(self, stamp_base: int) -> None:
        """run the gate over the submitted batch of arrivals; ACTION afterwards: SILENT / GATE_COMPLETE / GATE_PASS"""
        self._check(self.lib.ck_gate_arrive(self.h, stamp_base))

    def gate_stats(self) -> dict[str, int]:
        """`failures`: fan-outs the last gate_register could not hold, and tool returns or merges of the last gate_arrive
        the arena could not hold (those records are declined); the next register / arrive call starts again from 0"""
        out = np.zeros(5, dtype=np.uint64)
        self._check(self.lib.ck_gate_stats(self.h, ptr(out)))
        return dict(zip(["entries_used", "slots_used", "arena_used", "live", "failures"], (int(x) for x in out)))

    def gate_compact(self, room: int = 0, force: bool = False) -> bool:
        """give back what finished fan-outs used once entries, slots or arena bytes in use pass half of what the gate
        holds, or once fewer than `room` entries are left (the records of a batch about to be registered); always with
        force.  Returns whether it compacted"""
        st = self.gate_stats()
        if not (force or 2 * st["entries_used"] > self.gate_max_entries or 2 * st["slots_used"] > self.gate_max_slots
                or 2 * st["arena_used"] > self.gate_arena_bytes or st["entries_used"] + room > self.gate_max_entries):
            return False
        self._check(self.lib.ck_gate_compact(self.h))
        return True

    def gate_reset(self) -> None:
        self._check(self.lib.ck_gate_reset(self.h))

    # ------------------------------------------------------------------------------------------
    def submit(self, data: np.ndarray, offsets: np.ndarray) -> None:
        """H2D + decode of a host batch (uint8 bytes, int64 offsets[n+1]); asynchronous."""
        assert data.dtype == np.uint8 and offsets.dtype == np.int64
        self.n = len(offsets) - 1
        self._in_data, self._in_off = data, offsets
        self._check(self.lib.ck_submit(self.h, ptr(data), ptr(offsets), self.n))

    def set_isolation_level(self, level: str) -> None:
        """what the fetches submitted from now on deliver, as a Kafka consumer's `isolation_level` says: "read_uncommitted"
        (the default) every record but the control batches' markers, "read_committed" also not the records of aborted
        transactions (those a fetch names in its AbortedTransactions).  Records not delivered get status CK_SKIPPED"""
        if level not in ISOLATION_LEVELS:
            raise EngineError(f"isolation_level {level!r}: expected one of {ISOLATION_LEVELS}")
        self.read_committed = level == "read_committed"

    def set_fetch_hidden(self, mask: np.ndarray) -> None:
        """the read_committed mask (fetch_txn_mask, or its slice) of the next fetch submitted"""
        mask = np.ascontiguousarray(mask, dtype=np.uint8)
        self._check(self.lib.ck_set_fetch_hidden(self.h, ptr(mask), len(mask)))

    def submit_recordbatch(self, buf: np.ndarray, aborted_transactions=None, partitions=None) -> int:
        """H2D + CRC32C check + (gzip / snappy / LZ4 / zstd batches) decode + record split + field decode + walk of a fetch response's record set
        (concatenated Kafka RecordBatch v2 frames, uncompressed, gzip, snappy, LZ4 or zstd); returns the number of records.  Column spans are
        relative to each VALUE.  Control batches are skipped; under read_committed so are the aborted transactions' batches, from
        `aborted_transactions` [(producer id, first offset), ...] of a one-partition record set or `partitions` (txn_partitions)"""
        assert buf.dtype == np.uint8
        parts = txn_partitions(aborted_transactions, partitions)
        if self.read_committed and any(e[1] for e in parts):
            self.set_fetch_hidden(fetch_txn_mask(buf, parts))
        n = C.c_uint32(0)
        self._check(self.lib.ck_submit_recordbatch(self.h, ptr(buf), buf.nbytes, C.byref(n)))
        self.n = n.value
        self._rb_raw = buf
        idx = self.rb_index()
        # the host-side view of the batch for result decoding: record i = data[val_off[i] : val_off[i] + val_len[i]]
        self._in_data, self._in_off = idx["data"], _SpanOffsets(idx["val_off"], idx["val_len"])
        self._rb = idx
        self.skipped += int(np.count_nonzero(idx["bad"] == 2))
        return self.n

    @property
    def fetch_index(self) -> dict[str, np.ndarray]:
        """rb_index() of the fetch submit_recordbatch submitted last, as that call read it"""
        return self._rb

    def rb_index(self) -> dict[str, np.ndarray]:
        """where value / key / the correlation_id header of every record lie (len -1 = absent), and under "data" the bytes
        those offsets index: the submitted buffer, or a FetchBytes when the fetch held gzip, snappy, LZ4 or zstd batches"""
        n = self.n
        out = {"val_off": np.zeros(n, np.int64), "val_len": np.zeros(n, np.uint32), "key_off": np.zeros(n, np.int64),
               "key_len": np.zeros(n, np.int32), "corr_off": np.zeros(n, np.int64), "corr_len": np.zeros(n, np.int32),
               "bad": np.zeros(n, np.uint32)}
        if n:
            self._check(self.lib.ck_fetch_rb_index(self.h, *[ptr(out[k]) for k in ("val_off", "val_len", "key_off", "key_len", "corr_off", "corr_len", "bad")]))
        base, nbytes = C.c_uint64(0), C.c_uint64(0)
        self._check(self.lib.ck_fetch_rb_decoded_async(self.h, None, 0, C.byref(base), C.byref(nbytes)))
        out["data"] = self._rb_raw
        if nbytes.value:
            dec = np.empty(nbytes.value, dtype=np.uint8)
            self._check(self.lib.ck_fetch_rb_decoded_async(self.h, ptr(dec), dec.nbytes, None, None))
            self.sync()
            out["data"] = FetchBytes(self._rb_raw, base.value, dec)
        return out

    def encode_recordbatch(self, pub_indices: np.ndarray, base_offset: int = 0, timestamp_ms: int = 0) -> np.ndarray:
        """one Kafka RecordBatch v2 frame holding the publishes `pub_indices` of the current plan (one topic-partition, in
        send order), built on the device"""
        idx = np.ascontiguousarray(pub_indices, dtype=np.uint32)
        cap = self.max_out + 256 * self.max_payloads + 4096
        buf = np.empty(cap, dtype=np.uint8)
        used = C.c_uint64(0)
        self._check(self.lib.ck_encode_recordbatch(self.h, ptr(idx), len(idx), base_offset, timestamp_ms, ptr(buf), cap, C.byref(used)))
        return buf[:used.value]

    # ---- produce-ready frames: one frame pass per step (csrc/ck_kafka.cuh) -------------------------------------------
    def set_frame_topics(self, topics: Sequence[str]) -> None:
        """the registered topics whose publishes encode_frames frames"""
        missing = [t for t in topics if t not in self.topic_ids]
        if missing:
            raise EngineError(f"frame topics not registered: {missing}")
        ids = np.asarray([self.topic_ids[t] for t in topics] or [0], dtype=np.int32)
        self._check(self.lib.ck_set_frame_topics(self.h, ptr(ids), len(topics)))
        self.frame_topics = list(topics)

    def set_frame_bytes(self, window: int) -> None:
        """the frame split window W: a frame holds at most 61 + W + one record bytes (default 1 MiB)"""
        self._check(self.lib.ck_set_option(self.h, 2, window))

    def set_frame_compression(self, codec: str | None, level: int | None = None) -> None:
        """the codec of the frames the frame passes build: None (uncompressed, the default) or "lz4" (Kafka codec 3: the
        records section of every frame is one LZ4 frame of independent 64 KB blocks, compressed on the device).  `level`
        (compression.lz4.level, 1 .. 17; None: the default parse) picks the LZ4 parse: 1 and 2 give the default's bytes,
        3 and up a hash-chain search that deepens with the level (ck_set_option 4).  It has no effect on other codecs"""
        check_compression_level(level)
        if codec not in FRAME_CODECS:
            raise EngineError(f"frame compression {codec!r} is not supported (None or 'lz4')")
        self._check(self.lib.ck_set_option(self.h, 3, FRAME_CODECS[codec]))
        self._check(self.lib.ck_set_option(self.h, 4, level or 0))

    def set_producer(self, pid: int, epoch: int, transactional: bool = False) -> None:
        """the producer fields of the frames the following passes build (ck_set_producer): pid -1 none (producerId and
        producerEpoch -1, the default); else the idempotent producer (pid, epoch), with attributes bit 4 when transactional.
        baseSequence stays -1: the broker writes it at hand-off (patch_base_sequence)"""
        flags = 0 if pid < 0 else 1 | (2 if transactional else 0)
        self._check(self.lib.ck_set_producer(self.h, pid, epoch if pid >= 0 else -1, flags))

    def set_sticky_partitions(self, sticky: dict[str, int] | None) -> None:
        """topic -> the partition its unkeyed publishes join in the following passes (ck_set_sticky_partitions); None or {}:
        they stay the partition -1 group"""
        sticky = sticky or {}
        missing = [t for t in sticky if t not in self.topic_ids]
        if missing:
            raise EngineError(f"sticky partitions of topics not registered: {missing}")
        parts = np.full(max([self.topic_ids[t] + 1 for t in sticky] or [0]), -1, dtype=np.int32)
        for t, p in sticky.items():
            parts[self.topic_ids[t]] = p
        self._check(self.lib.ck_set_sticky_partitions(self.h, ptr(parts) if len(parts) else None, len(parts)))

    def encode_frames(self, timestamp_ms: int) -> None:
        """queue the frame pass over the current plan: every live publish to a frame topic, grouped by (topic, partition)
        in send order, as frames with baseOffset 0 and baseTimestamp timestamp_ms (asynchronous; fetch_frames reads them)"""
        self._check(self.lib.ck_encode_frames(self.h, timestamp_ms))

    def encode_frames_records(self, topic: str, records: Sequence[tuple[bytes, bytes | None, str | None]], timestamp_ms: int) -> None:
        """queue the frame pass over records a host path produced for `topic`: (value, key or None, correlation id or None)
        each; keyed records go to partition murmur2(key) % num_partitions, as the plan's publishes do"""
        if topic not in self.topic_ids:
            raise EngineError(f"topic {topic!r} is not registered")
        parts, desc, pos = [], np.full((len(records), 6), -1, dtype=np.int64), 0
        for i, (value, key, corr) in enumerate(records):
            for f, b in enumerate((value, None if key is None else json_content(key.decode()), None if corr is None else json_content(corr))):
                if b is None:
                    continue
                desc[i, 2 * f], desc[i, 2 * f + 1] = pos, len(b)
                parts.append(b)
                pos += len(b)
        blob = np.frombuffer(b"".join(parts) or b"\0", dtype=np.uint8)
        self._frame_src = (blob, desc)                   # the copies to the device read them after this call returns
        self._check(self.lib.ck_encode_frames_records(self.h, self.topic_ids[topic], ptr(blob), pos, ptr(desc), len(records), timestamp_ms))

    def frames_size(self) -> tuple[int, int]:
        """(frames, bytes) of the last frame pass; waits for it"""
        nf, nb = C.c_uint32(), C.c_uint64()
        self._check(self.lib.ck_frames_size(self.h, C.byref(nf), C.byref(nb)))
        return nf.value, nb.value

    def fetch_frames(self, pool=None) -> Frames:
        """the frames of the last frame pass, copied to the host (waits).  With a PinnedPool (engine.lane) they land in
        page-locked buffers taken from it; Frames.release() gives them back"""
        nf, nb = self.frames_size()
        if pool is None:
            table, data, bufs = np.zeros(nf, dtype=FRAME_DTYPE), np.empty(max(nb, 1), dtype=np.uint8), ()
        else:
            bufs = (pool.take(FRAME_DTYPE.itemsize * nf + 64), pool.take(nb + 64))
            table, data = bufs[0].view(FRAME_DTYPE, nf), bufs[1].array
        self._check(self.lib.ck_fetch_frames_async(self.h, ptr(table), nf, ptr(data), data.nbytes))
        self.sync()
        return Frames(table, data[:nb], self.topic_names, on_release=(lambda: [pool.give(b) for b in bufs]) if bufs else None)

    def submit_device(self, dev_data, dev_off, n: int, host_data: np.ndarray | None = None,
                      host_off: np.ndarray | None = None) -> None:
        """decode a batch already resident in HBM (torch tensors or raw device addresses)."""
        self.n = n
        self._in_data, self._in_off = host_data, host_off
        a = dev_data if isinstance(dev_data, int) else ptr(dev_data)
        b = dev_off if isinstance(dev_off, int) else ptr(dev_off)
        self._check(self.lib.ck_submit_device(self.h, a, b, n))

    def tool_args(self) -> tuple[np.ndarray, np.ndarray]:
        """(blob, offsets[n+1]): the `args` JSON of every record that reaches the tool (host tools)."""
        self._check(self.lib.ck_tool_args(self.h))
        out, off, ln, _ = self._fetch(want_pubs=False)
        return out, off, ln

    def tool_plan(self, aux: np.ndarray | None = None, aux_off: np.ndarray | None = None) -> None:
        self._check(self.lib.ck_tool_plan(self.h, ptr(aux), ptr(aux_off)))

    def reply_plan(self, mode: int = 0) -> None:
        """client reply decode (client/deserialize.py:55-89): payload i = output value JSON; mode 0 auto, 1 text, 2 data"""
        self._check(self.lib.ck_reply_plan(self.h, mode))

    def return_plan(self) -> None:
        self._check(self.lib.ck_return_plan(self.h))

    def tool_plan_device(self, dev_aux, dev_aux_off) -> None:
        self._check(self.lib.ck_tool_plan_device(self.h, ptr(dev_aux), ptr(dev_aux_off)))

    def launch_count(self) -> int:
        """kernels launched by this engine so far"""
        return int(self.lib.ck_launch_count(self.h))

    def sync(self) -> None:
        self._check(self.lib.ck_sync(self.h))

    def columns(self) -> np.ndarray:
        cols = np.empty((NUM_COLS, self.n), dtype=np.uint32)
        if self.n:
            self._check(self.lib.ck_fetch_columns(self.h, ptr(cols)))
        return cols

    def out_size(self) -> tuple[int, int, int]:
        nb, npay, npub = C.c_uint64(), C.c_uint32(), C.c_uint32()
        self._check(self.lib.ck_out_size(self.h, C.byref(nb), C.byref(npay), C.byref(npub)))
        return nb.value, npay.value, npub.value

    def _fetch(self, want_pubs: bool = True, out_buf: np.ndarray | None = None, off_buf: np.ndarray | None = None,
               len_buf: np.ndarray | None = None, pubs_buf: np.ndarray | None = None):
        """D2H of the results.  The optional *_buf arrays let a caller land everything in pinned memory it
        owns (required for copies that overlap with the other PCIe direction)."""
        nb, npay, npub = self.out_size()
        out = out_buf if out_buf is not None else np.empty(max(nb, 1), dtype=np.uint8)
        off = off_buf[:npay + 1] if off_buf is not None else np.zeros(npay + 1, dtype=np.int64)
        ln = len_buf[:npay] if len_buf is not None else np.zeros(npay, dtype=np.uint32)
        npub_eff = npub if want_pubs else 0
        pubs = pubs_buf[:npub_eff] if pubs_buf is not None else np.zeros(npub_eff, dtype=PUB_DTYPE)
        self._check(self.lib.ck_fetch_output(self.h, ptr(out), out.nbytes, ptr(off) if npay else None,
                                             ptr(ln) if npay else None, ptr(pubs) if npub_eff else None))
        return out[:nb], off, ln, pubs

    def fetch(self, out_buf: np.ndarray | None = None, with_columns: bool = True) -> BatchOutput:
        out, off, ln, pubs = self._fetch(out_buf=out_buf)
        cols = self.columns() if with_columns else None
        return BatchOutput(self, out, off, ln, pubs, self._in_data, self._in_off, cols, self.overlay())

    def overlay(self):
        """(bytes, off[n], len[n]) of the canonicalised records of the current batch, or None if there are none"""
        if not self.n:
            return None
        off = np.empty(self.n, dtype=np.int64)
        ln = np.empty(self.n, dtype=np.uint32)
        buf = np.empty(self.max_in + 256, dtype=np.uint8)
        used = C.c_uint64(0)
        self._check(self.lib.ck_fetch_overlay(self.h, ptr(buf), buf.nbytes, ptr(off), ptr(ln), C.byref(used)))
        if not (off >= 0).any():
            return None
        return buf[:used.value], off, ln

    # ------------------------------------------------------------------------------------------
    def stream_ptr(self) -> int:
        return int(self.lib.ck_stream(self.h))

    def device_buffers(self) -> dict[str, int]:
        ps = [C.c_void_p() for _ in range(5)]
        self._check(self.lib.ck_device_buffers(self.h, *[C.byref(p) for p in ps]))
        return dict(zip(["in", "in_off", "out", "out_off", "cols"], [p.value for p in ps]))

    def profile(self, enable: bool) -> None:
        self._check(self.lib.ck_profile(self.h, int(enable)))

    def profile_read(self, reset: bool = True) -> dict[str, tuple[float, int]]:
        ms = np.zeros(_lib.NUM_KERNELS, dtype=np.float32)
        cnt = np.zeros(_lib.NUM_KERNELS, dtype=np.uint32)
        self._check(self.lib.ck_profile_read(self.h, ptr(ms), ptr(cnt), int(reset)))
        return {k: (float(ms[i]), int(cnt[i])) for i, k in enumerate(_lib.KERNELS)}

    # ------------------------------------------------------------------------------------------
    def run_tool_batch(self, data: np.ndarray, offsets: np.ndarray, host_tool=None) -> BatchOutput:
        """Convenience: one full tool-node step over a host batch.  `host_tool(args_json: bytes) ->
        result_json: bytes` is used when the node has no device template."""
        self.submit(data, offsets)
        if host_tool is None:
            self.tool_plan()
        else:
            blob, off, ln = self.tool_args()
            results = [host_tool(blob[off[i]:off[i] + ln[i]].tobytes()) if ln[i] else b"" for i in range(self.n)]
            aux_off = np.zeros(self.n + 1, dtype=np.int64)
            np.cumsum([len(r) for r in results], out=aux_off[1:])
            aux = np.frombuffer(b"".join(results) or b"\0", dtype=np.uint8)
            self.tool_plan(aux, aux_off)
        return self.fetch()
