// Kafka transactions on the consume side (message format v2, KIP-98): which batches of a fetch response's record set a
// consumer does not deliver.  Host code only, no device dependency: ck_submit_recordbatch uses it for the control batches
// of every fetch, and ck_fetch_txn_mask for the read_committed mask of a whole fetch before it is split over engines.
//
// Two attributes bits of the batch header matter (attributes i16 at byte 21, so its low byte is byte 22):
//   0x20 control batch: one record whose key is (version i16, type i16), type 0 = ABORT, 1 = COMMIT; its value
//        (version i16, coordinatorEpoch i32) is not read.  Every consumer skips it, at both isolation levels.
//   0x10 transactional batch: its records belong to the transaction of producerId (i64 at byte 43).
// The rule, per partition of the record set, over its batches in order (the Java consumer's fetch loop):
//   aborted = {}; pending = the partition's aborted transactions (producer id, first offset) sorted by first offset
//   for each batch:
//     a batch that fails its framing (magic 2, a known codec, the CRC32C) is bad: its records are bad frames, no state change
//     while pending and pending[0].first_offset <= batch.lastOffset (baseOffset + lastOffsetDelta): aborted += pop(pending)
//     control batch: skipped; an ABORT marker removes batch.producerId from aborted, any other type changes nothing
//     transactional batch of a producer in aborted (read_committed only): skipped
//     else delivered
// A control batch that is compressed, holds recordsCount != 1, whose one record does not span its records section, or
// whose key is shorter than 4 bytes or has a negative version, is bad and changes no state.  The Java consumer raises on
// such a batch instead; here it is one more bad frame.  A producer whose abort marker lies past the end of the fetch stays
// aborted to its end.  The broker never returns data past the partition's last stable offset to a read_committed fetch,
// so a transaction still open there is not this code's concern.
#ifndef CK_TXN_H
#define CK_TXN_H

#include <stdint.h>

#include <algorithm>
#include <set>
#include <vector>

#define CK_TXN_TRANSACTIONAL 0x10u
#define CK_TXN_CONTROL 0x20u
#define CK_TXN_ABORT 0                    // control record type of an abort marker
enum { CK_TXN_SHOW = 0, CK_TXN_BAD = 1, CK_TXN_HIDE = 2 };   // per-batch flag: delivered / bad frame / skipped

static inline uint32_t ck_txn_be32(const uint8_t* p) { return ((uint32_t)p[0] << 24) | ((uint32_t)p[1] << 16) | ((uint32_t)p[2] << 8) | p[3]; }
static inline int64_t ck_txn_be64(const uint8_t* p) { return (int64_t)(((uint64_t)ck_txn_be32(p) << 32) | ck_txn_be32(p + 4)); }

// end of the complete frame at pos (12 + batchLength bytes, at least a header), 0 when none starts there: the end of the
// record set or a truncated trailing frame, which a fetch response may carry
static inline uint64_t ck_txn_frame_end(const uint8_t* buf, uint64_t n, uint64_t pos) {
    if (pos + 12 > n) return 0;
    uint32_t blen = ck_txn_be32(buf + pos + 8);
    uint64_t end = pos + 12 + (uint64_t)blen;
    return (int32_t)blen < 49 || end > n ? 0 : end;
}

static inline uint32_t ck_txn_crc32c(const uint8_t* p, uint64_t n) {
    static const std::vector<uint32_t> t = [] {
        std::vector<uint32_t> v(256);
        for (uint32_t i = 0; i < 256; i++) {
            uint32_t c = i;
            for (int k = 0; k < 8; k++) c = (c >> 1) ^ ((c & 1u) ? 0x82F63B78u : 0u);
            v[i] = c;
        }
        return v;
    }();
    uint32_t c = 0xffffffffu;
    for (uint64_t i = 0; i < n; i++) c = t[(c ^ p[i]) & 0xffu] ^ (c >> 8);
    return ~c;
}

// a(x) * b(x) mod P(x) over GF(2), CRC32C's reflected representation (bit 31 = x^0)
static inline uint32_t ck_txn_gf_mul(uint32_t a, uint32_t b) {
    uint32_t p = 0;
    for (uint32_t m = 0x80000000u; m; m >>= 1) {
        if (a & m) p ^= b;
        b = (b & 1u) ? (b >> 1) ^ 0x82F63B78u : b >> 1;
    }
    return p;
}

// The CRC32C of a span of len bytes whose CRC was crc, after its 4 bytes at pos changed from old4 to new4.  The CRC is
// affine in the message, so the change adds the CRC (zero init, no final xor) of the message that is zero but for
// old4 ^ new4 at pos.  Leading zeros do not move that CRC and each trailing zero byte multiplies it by x^8, so it is the
// CRC of the 4 delta bytes times x^(8 (len - pos - 4)) mod P: O(log len), whatever the span's length
static inline uint32_t ck_txn_crc32c_patch(uint32_t crc, uint64_t len, uint64_t pos, const uint8_t* old4, const uint8_t* new4) {
    uint32_t d = 0;                                             // raw CRC of the 4 delta bytes
    for (int i = 0; i < 4; i++) {
        d ^= (uint8_t)(old4[i] ^ new4[i]);
        for (int k = 0; k < 8; k++) d = (d >> 1) ^ ((d & 1u) ? 0x82F63B78u : 0u);
    }
    uint32_t p = 0x80000000u, sq = 0x00800000u;                 // x^0, x^8
    for (uint64_t n = len - pos - 4; n; n >>= 1) {
        if (n & 1u) p = ck_txn_gf_mul(sq, p);
        sq = ck_txn_gf_mul(sq, sq);
    }
    return crc ^ ck_txn_gf_mul(p, d);
}

// the checks the device makes of every batch: magic 2, codec none / gzip / snappy / LZ4 / zstd, and (check_crc) the CRC32C
static inline bool ck_txn_framed(const uint8_t* f, uint64_t flen, bool check_crc) {
    uint32_t codec = f[22] & 7u;
    if (f[16] != 2 || codec > 4) return false;
    return !check_crc || ck_txn_crc32c(f + 21, flen - 21) == ck_txn_be32(f + 17);
}

// a zig-zag varint of at most 10 bytes whose unsigned value fits in 64 bits: a 10th byte above 1 is refused
static inline bool ck_txn_varint(const uint8_t* p, uint64_t& pos, uint64_t end, int64_t& out) {
    uint64_t u = 0;
    for (uint32_t shift = 0;; shift += 7) {
        if (pos >= end) return false;
        uint8_t b = p[pos++];
        if (shift == 63 && b > 1) return false;
        u |= (uint64_t)(b & 0x7f) << shift;
        if (!(b & 0x80)) break;
    }
    out = (int64_t)(u >> 1) ^ -(int64_t)(u & 1);
    return true;
}

// a control batch f[0..flen): CK_TXN_HIDE and its marker's type in *type when it is well formed (see above), else CK_TXN_BAD
static inline int ck_txn_control(const uint8_t* f, uint64_t flen, int* type) {
    if (!ck_txn_framed(f, flen, true) || (f[22] & 7u) || ck_txn_be32(f + 57) != 1) return CK_TXN_BAD;
    uint64_t pos = 61;
    int64_t len, v, klen;
    if (!ck_txn_varint(f, pos, flen, len) || len < 0 || (uint64_t)len != flen - pos) return CK_TXN_BAD;
    pos += 1;                                                   // record attributes
    if (!ck_txn_varint(f, pos, flen, v) || !ck_txn_varint(f, pos, flen, v) || !ck_txn_varint(f, pos, flen, klen)) return CK_TXN_BAD;
    if (klen < 4 || (uint64_t)klen > flen - pos) return CK_TXN_BAD;
    int16_t version = (int16_t)((f[pos] << 8) | f[pos + 1]);
    if (version < 0) return CK_TXN_BAD;
    *type = (int16_t)((f[pos + 2] << 8) | f[pos + 3]);
    return CK_TXN_HIDE;
}

// The control batch the broker appends when producer (pid, epoch) ends its transaction on a partition: type CK_TXN_ABORT
// or 1 (COMMIT), attributes transactional | control, baseSequence -1, one record of offsetDelta 0 whose key is (version 0,
// type) and whose value is (version 0, coordinatorEpoch 0), no headers.  CK_TXN_CONTROL_LEN bytes into out; ck_txn_control
// accepts it
#define CK_TXN_CONTROL_LEN 78u
static inline void ck_txn_put_be(uint8_t* p, uint64_t v, int n) { for (int i = n - 1; i >= 0; i--, v >>= 8) p[i] = (uint8_t)v; }
static inline void ck_txn_control_batch(uint8_t* out, int64_t base_offset, int64_t timestamp_ms, int64_t pid, int16_t epoch, int16_t type) {
    static const uint8_t rec[17] = {32, 0, 0, 0, 8, 0, 0, 0, 0, 12, 0, 0, 0, 0, 0, 0, 0};   // 16-byte body (varint 32)
    uint8_t* f = out;
    ck_txn_put_be(f, (uint64_t)base_offset, 8);
    ck_txn_put_be(f + 8, CK_TXN_CONTROL_LEN - 12, 4);          // batchLength
    ck_txn_put_be(f + 12, 0, 4);                                // partitionLeaderEpoch
    f[16] = 2;
    ck_txn_put_be(f + 21, CK_TXN_TRANSACTIONAL | CK_TXN_CONTROL, 2);
    ck_txn_put_be(f + 23, 0, 4);                                // lastOffsetDelta
    ck_txn_put_be(f + 27, (uint64_t)timestamp_ms, 8);
    ck_txn_put_be(f + 35, (uint64_t)timestamp_ms, 8);
    ck_txn_put_be(f + 43, (uint64_t)pid, 8);
    ck_txn_put_be(f + 51, (uint16_t)epoch, 2);
    ck_txn_put_be(f + 53, 0xffffffffu, 4);                      // baseSequence -1
    ck_txn_put_be(f + 57, 1, 4);
    for (int i = 0; i < 17; i++) f[61 + i] = rec[i];
    ck_txn_put_be(f + 61 + 7, (uint16_t)type, 2);               // key: version 0 (bytes 5, 6), type
    ck_txn_put_be(f + 17, ck_txn_crc32c(f + 21, CK_TXN_CONTROL_LEN - 21), 4);
}

// The read_committed mask of a whole record set buf[0..n): mask[b] = 1 for each complete batch b the rule above skips
// because it is a transactional batch of an aborted producer, else 0 (control batches included: ck_submit_recordbatch
// flags those itself).  Partition r is the run of batches that start in [run_start[r], run_start[r + 1]) (the last run:
// to the end); its aborted transactions are the entries k with abort_run[k] = r.  The CRC32C of a data batch is checked
// only where it matters, when the batch would move aborted transactions into the set.  Returns the number of complete
// batches (mask is written up to cap of them), or -1 when the runs are not in order or an entry names no run
static inline int64_t ck_txn_mask(const uint8_t* buf, uint64_t n, const uint64_t* run_start, uint32_t nruns,
                                  const uint32_t* abort_run, const int64_t* abort_pid, const int64_t* abort_first, uint32_t naborts,
                                  uint8_t* mask, uint64_t cap) {
    for (uint32_t r = 1; r < nruns; r++)
        if (run_start[r] < run_start[r - 1]) return -1;
    std::vector<uint32_t> order(naborts);
    for (uint32_t k = 0; k < naborts; k++) {
        if (abort_run[k] >= nruns) return -1;
        order[k] = k;
    }
    std::stable_sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) {
        return abort_run[a] != abort_run[b] ? abort_run[a] < abort_run[b] : abort_first[a] < abort_first[b];
    });
    std::set<int64_t> aborted;
    uint32_t next = 0;                                          // first entry of order not yet moved into `aborted`
    int64_t run = -1;
    uint64_t pos = 0, end;
    int64_t b = 0;
    for (; (end = ck_txn_frame_end(buf, n, pos)) != 0; pos = end, b++) {
        while (run + 1 < (int64_t)nruns && run_start[run + 1] <= pos) {
            run++;
            aborted.clear();
            while (next < naborts && abort_run[order[next]] < run) next++;   // a run no batch started in
        }
        uint8_t m = 0;
        const uint8_t* f = buf + pos;
        uint64_t flen = end - pos;
        int64_t last = ck_txn_be64(f) + (int32_t)ck_txn_be32(f + 23), pid = ck_txn_be64(f + 43);
        bool control = f[22] & CK_TXN_CONTROL;
        auto due = [&] { return next < naborts && abort_run[order[next]] == run && abort_first[order[next]] <= last; };
        int type = -1;
        if (ck_txn_framed(f, flen, control || due()) && (!control || ck_txn_control(f, flen, &type) == CK_TXN_HIDE)) {
            while (due()) aborted.insert(abort_pid[order[next++]]);
            if (control) {
                if (type == CK_TXN_ABORT) aborted.erase(pid);
            } else if ((f[22] & CK_TXN_TRANSACTIONAL) && aborted.count(pid)) {
                m = 1;
            }
        }
        if ((uint64_t)b < cap) mask[b] = m;
    }
    return b;
}

// The consumed positions of a record set buf[0..n) with the partition runs above: next[r] = lastOffset + 1 (baseOffset +
// lastOffsetDelta + 1) of the last complete batch that starts in run r, or -1 when none does; batch_next[b] (up to cap of
// them, null: not wanted) the same of batch b.  Every complete batch moves its partition's position, delivered or not:
// control batches, aborted transactions' batches and batches that fail their framing or CRC32C alike, as the Java
// consumer advances past them.  Only the 61-byte headers are read.  Returns the number of complete batches, or -1 when
// the runs are not in order
static inline int64_t ck_txn_positions(const uint8_t* buf, uint64_t n, const uint64_t* run_start, uint32_t nruns,
                                       int64_t* next, int64_t* batch_next, uint64_t cap) {
    for (uint32_t r = 0; r < nruns; r++) {
        if (r && run_start[r] < run_start[r - 1]) return -1;
        next[r] = -1;
    }
    int64_t run = -1;
    uint64_t pos = 0, end;
    int64_t b = 0;
    for (; (end = ck_txn_frame_end(buf, n, pos)) != 0; pos = end, b++) {
        while (run + 1 < (int64_t)nruns && run_start[run + 1] <= pos) run++;
        int64_t nx = ck_txn_be64(buf + pos) + (int32_t)ck_txn_be32(buf + pos + 23) + 1;
        if (run >= 0) next[run] = nx;
        if (batch_next && (uint64_t)b < cap) batch_next[b] = nx;
    }
    return b;
}

#endif  // CK_TXN_H
