"""TEST INFRASTRUCTURE ONLY — Kafka transactions (message format v2, KIP-98) restated in plain Python: the control record
schema, a writer of transactional and control batches built on oracle.kafka_batch, the consume rule the device path
implements (csrc/ck_txn.h), and seeded random transactional logs.

  control batch      attributes bit 5 (0x20), one record: key = version i16 | type i16 (0 ABORT, 1 COMMIT),
                     value = version i16 | coordinatorEpoch i32; producerId / producerEpoch of the transaction it ends
  transactional      attributes bit 4 (0x10), producerId i64 at byte 43, producerEpoch i16 at 51, baseSequence i32 at 53
  the rule           per partition, over its batches in order (the Java consumer's fetch loop):
                       a batch failing its framing (magic 2, a known codec, the CRC32C) is bad and changes nothing;
                       a control batch that is compressed, holds recordsCount != 1, whose record does not span its records
                       section, or whose key is shorter than 4 bytes or of negative version is bad and changes nothing;
                       else the aborted transactions whose first offset <= the batch's lastOffset join `aborted`;
                       a control batch is skipped, and an ABORT marker removes its producer from `aborted`;
                       read_committed: a transactional batch of a producer in `aborted` is skipped;
                       anything else is delivered
"""
from __future__ import annotations

import random
import struct

from oracle import kafka_batch as kb

ABORT, COMMIT = 0, 1
TRANSACTIONAL, CONTROL = 0x10, 0x20
DELIVER, BAD, SKIP = 0, 1, 2


def _recrc(b: bytes) -> bytes:
    return b[:17] + struct.pack(">I", kb.crc32c(b[kb.CRC_FROM:])) + b[21:]


def with_attrs(batch: bytes, attrs: int) -> bytes:
    """`batch` with its attributes replaced (CRC32C recomputed)"""
    return _recrc(batch[:21] + struct.pack(">h", attrs) + batch[23:])


def txn_batch(records: list[kb.KRecord], base_offset: int, producer_id: int, producer_epoch: int = 0, base_sequence: int = 0,
              transactional: bool = True, base_timestamp: int = 1767225600000) -> bytes:
    """an uncompressed data batch of `producer_id`; transactional: attributes bit 4"""
    b = kb.encode_batch(records, base_offset=base_offset, base_timestamp=base_timestamp, producer_id=producer_id,
                        producer_epoch=producer_epoch, base_sequence=base_sequence)
    return with_attrs(b, TRANSACTIONAL) if transactional else b


def control_key(ctype: int, version: int = 0) -> bytes:
    return struct.pack(">hh", version, ctype)


def control_value(coordinator_epoch: int = 0, version: int = 0) -> bytes:
    return struct.pack(">hi", version, coordinator_epoch)


def control_batch(base_offset: int, producer_id: int, ctype: int, producer_epoch: int = 0, key: bytes | None = None,
                  extra_records: int = 0) -> bytes:
    """a control batch ending the transaction of `producer_id` (ctype ABORT / COMMIT); key: another key in its record;
    extra_records: more records after the marker (malformed)"""
    recs = [kb.KRecord(control_value(), control_key(ctype) if key is None else key)] + \
        [kb.KRecord(control_value(), control_key(ctype)) for _ in range(extra_records)]
    b = kb.encode_batch(recs, base_offset=base_offset, base_timestamp=1767225600000, producer_id=producer_id,
                        producer_epoch=producer_epoch, base_sequence=-1)
    return with_attrs(b, TRANSACTIONAL | CONTROL)


def batches(buf: bytes) -> list[tuple[int, int]]:
    """(start, end) of every complete batch of a record set (a truncated tail is not one)"""
    out, pos = [], 0
    while pos + 12 <= len(buf):
        blen = struct.unpack_from(">i", buf, pos + 8)[0]
        if blen < 49 or pos + 12 + blen > len(buf):
            break
        out.append((pos, pos + 12 + blen))
        pos += 12 + blen
    return out


def _framed(f: bytes) -> bool:
    codec = f[22] & 7
    return f[16] == 2 and codec in (0, 1, 3, 4) and kb.crc32c(f[kb.CRC_FROM:]) == struct.unpack_from(">I", f, 17)[0]


def control_type(f: bytes) -> int | None:
    """the marker type of a well-formed control batch, None for a malformed one"""
    if not _framed(f) or f[22] & 7 or struct.unpack_from(">i", f, 57)[0] != 1:
        return None
    try:
        length, p = kb.get_varint(f, kb.HEADER_LEN)
        if length < 0 or p + length != len(f):
            return None
        p += 1
        _ts, p = kb.get_varint(f, p)
        _od, p = kb.get_varint(f, p)
        klen, p = kb.get_varint(f, p)
    except (IndexError, ValueError):
        return None
    if klen < 4 or p + klen > len(f):
        return None
    version, ctype = struct.unpack_from(">hh", f, p)
    return None if version < 0 else ctype


def verdicts(buf: bytes, partitions, read_committed: bool) -> list[int]:
    """DELIVER / BAD / SKIP for every complete batch of the record set; partitions = [(byte start, [(pid, first offset)])]"""
    out = []
    run, aborted, pending = -1, set(), []
    for start, end in batches(buf):
        while run + 1 < len(partitions) and partitions[run + 1][0] <= start:
            run += 1
            aborted, pending = set(), sorted(partitions[run][1], key=lambda e: e[1])
        f = buf[start:end]
        control = bool(f[22] & CONTROL)
        if not _framed(f) or (control and control_type(f) is None):
            out.append(BAD)
            continue
        last = struct.unpack_from(">q", f, 0)[0] + struct.unpack_from(">i", f, 23)[0]
        pid = struct.unpack_from(">q", f, 43)[0]
        while pending and pending[0][1] <= last:
            aborted.add(pending.pop(0)[0])
        if control:
            if control_type(f) == ABORT:
                aborted.discard(pid)
            out.append(SKIP)
        elif read_committed and f[22] & TRANSACTIONAL and pid in aborted:
            out.append(SKIP)
        else:
            out.append(DELIVER)
    return out


def record_counts(buf: bytes) -> list[int]:
    return [struct.unpack_from(">i", buf, s + 57)[0] for s, _e in batches(buf)]


# ---- seeded random transactional logs ------------------------------------------------------------------------------
def _records(rng: random.Random, n: int, tag: str) -> list[kb.KRecord]:
    out = []
    for i in range(n):
        cid = f"{tag}-{i}-{rng.randrange(1 << 30):x}"
        val = ('{"k":"%s","pad":"%s"}' % (cid, "x" * rng.randrange(0, 40))).encode()
        out.append(kb.calfkit_record(val, cid, keyed=rng.random() < 0.7))
    return out


def random_partition(rng: random.Random, tag: str, n_events: int = 40, make_records=None) -> tuple[bytes, list[tuple[int, int]]]:
    """one partition's batches and its AbortedTransactions: several producers with interleaved transactions (commits and
    aborts, markers past the end), non-transactional batches, aborted entries no batch reaches, offsets that jump back,
    malformed control batches and batches with a bad CRC"""
    make_records = make_records or (lambda n, t: _records(rng, n, t))
    pids = [rng.randrange(1, 1 << 40) for _ in range(rng.randint(1, 4))]
    open_txn: dict[int, int] = {}                      # pid -> first offset of its open transaction
    aborted: list[tuple[int, int]] = []
    off = rng.randrange(0, 1000)
    out = []
    for ev in range(n_events):
        pid = rng.choice(pids)
        r = rng.random()
        if r < 0.06:
            off = max(0, off - rng.randrange(1, 30))   # non-monotone offsets
        if pid in open_txn and r < 0.3:
            ctype = ABORT if rng.random() < 0.5 else COMMIT
            if ctype == ABORT:
                aborted.append((pid, open_txn[pid]))
            del open_txn[pid]
            m = rng.random()
            if m < 0.1:
                out.append(control_batch(off, pid, ctype, key=control_key(ctype)[:rng.randrange(0, 4)]))   # short key
            elif m < 0.15:
                out.append(control_batch(off, pid, ctype, extra_records=1))
            elif m < 0.2:
                b = control_batch(off, pid, ctype)
                out.append(b[:17] + struct.pack(">I", struct.unpack_from(">I", b, 17)[0] ^ 1) + b[21:])   # bad CRC
            elif m < 0.25:
                out.append(control_batch(off, pid, rng.choice([2, 7, -1])))      # unknown type
            elif m < 0.3:
                out.append(control_batch(off, pid, ctype, key=control_key(ctype, version=rng.choice([1, 3, -1]))))
            else:
                out.append(control_batch(off, pid, ctype))
            off += 1
            continue
        n = rng.randint(1, 4)
        txn = rng.random() < 0.8
        if txn and pid not in open_txn:
            open_txn[pid] = off
        b = txn_batch(make_records(n, f"{tag}-{ev}"), off, pid if txn or rng.random() < 0.5 else -1, transactional=txn)
        if rng.random() < 0.05:
            b = b[:-1] + bytes([b[-1] ^ 0x40])                                   # bad CRC
        out.append(b)
        off += n
    for pid, first in open_txn.items():                # abort markers past the end of the fetch
        if rng.random() < 0.5:
            aborted.append((pid, first))
    for _ in range(rng.randint(0, 2)):                 # entries no batch reaches
        aborted.append((rng.choice(pids), off + rng.randrange(1, 100)))
    rng.shuffle(aborted)
    return b"".join(out), aborted


def random_log(seed: int, make_records=None, n_events: int = 40) -> tuple[bytes, list[tuple[int, list[tuple[int, int]]]]]:
    """a record set of one to three partitions, maybe with a truncated tail, and its partitions"""
    rng = random.Random(seed)
    buf, parts = b"", []
    for p in range(rng.randint(1, 3)):
        data, ab = random_partition(rng, f"s{seed}p{p}", n_events, make_records)
        parts.append((len(buf), ab))
        buf += data
    if rng.random() < 0.3:
        cut = batches(buf)[0]
        buf += buf[cut[0]:cut[1]][:rng.randrange(12, cut[1] - cut[0])]
    return buf, parts


# ---- a producer's frames rewritten as transactions ------------------------------------------------------------------
def retxn(frame: bytes, base_offset: int, producer_id: int) -> bytes:
    """`frame` with its baseOffset and producerId replaced and the transactional bit set (CRC32C recomputed natively:
    frames of a step are large)"""
    import txnmask
    f = struct.pack(">q", base_offset) + frame[8:21] + struct.pack(">h", struct.unpack_from(">h", frame, 21)[0] | TRANSACTIONAL) + \
        frame[23:43] + struct.pack(">q", producer_id) + frame[51:]
    return f[:17] + struct.pack(">I", txnmask.crc32c(f[kb.CRC_FROM:])) + f[21:]


def transactional_fetch(frames: list[bytes], abort_share: float, seed: int, producers: int = 4):
    """the frames of a record set as the transactions of `producers` producers, interleaved: frame i joins the open
    transaction of producer i % producers, which then ends (a commit or, with probability abort_share, an abort marker)
    with probability 1/2; whatever is open at the end is ended too.  Returns (record set, its AbortedTransactions,
    aborted[i] for every frame)"""
    rng = random.Random(seed)
    pids = [1000 + 17 * p for p in range(producers)]
    out, aborted, entries, members = [], [], [], {}
    off = 0

    def end(p):
        nonlocal off
        first, idx = members.pop(p)
        abort = rng.random() < abort_share
        if abort:
            entries.append((pids[p], first))
            for i in idx:
                aborted[i] = True
        out.append(control_batch(off, pids[p], ABORT if abort else COMMIT))
        off += 1

    for i, f in enumerate(frames):
        p = i % producers
        aborted.append(False)
        members.setdefault(p, (off, []))[1].append(i)
        out.append(retxn(f, off, pids[p]))
        off += struct.unpack_from(">i", f, 57)[0]
        if rng.random() < 0.5:
            end(p)
    for p in list(members):
        end(p)
    return b"".join(out), entries, aborted
