// Kafka RecordBatch v2 framing on the device (SURVEY.md section 8f row 1).
//
// Reference: done by aiokafka underneath broker.subscriber(...) / broker.publish(...) (calfkit/worker/worker.py:45-53,
// calfkit/nodes/base.py:82-87; faststream[kafka] -> aiokafka, third-party, absent from the image).  Format restated in
// oracle/kafka_batch.py from the published protocol (message format v2) and pinned there to known-answer vectors.
//
// decode (a fetch response's record set = concatenated frames, copied to HBM as it arrived):
//   ck_rb_crc_kernel     warp per batch: CRC32C (Castagnoli) of the covered bytes [21, end) — every lane runs a
//                        slicing-by-4 table CRC over its own contiguous chunk, the 32 partial CRCs are folded with
//                        GF(2) polynomial arithmetic (crc(A||B) = crc(A) * x^(8|B|) mod P  xor  crc(B));
//   ck_rb_lz4_kernel     (a fetch holding LZ4 batches only) warp per LZ4 batch: its records section, one LZ4 frame, decoded
//                        into the batch's slot behind the raw bytes (ck_lz4.cuh)
//   ck_rb_gzip_kernel    (a fetch holding gzip batches only) warp per gzip batch: its records section, one gzip member,
//                        inflated into the batch's slot (ck_inflate.cuh) and checked against the trailer's CRC32
//   ck_rb_zstd_kernel    (a fetch holding zstd batches only) warp per zstd batch: its records section, one zstd frame,
//                        decoded into the batch's slot (ck_zstd.cuh)
//   ck_rb_snappy_kernel  (a fetch holding snappy batches only) warp per snappy chunk, over the chunks of all the fetch's
//                        snappy batches: each raw snappy block decoded into its place in its batch's slot (ck_snappy.cuh)
//   ck_rb_split_kernel   thread per batch: hop from record to record (each starts with its own varint length)
//                        (a batch the host flagged skipped — a control batch, or under read_committed a transactional
//                        batch of an aborted producer, ck_txn.h — passes the CRC check, is neither decoded nor split, and
//                        its records come out CK_SKIPPED)
//   ck_rb_fields_kernel  thread per record: zig-zag varints -> key span, value span, the `correlation_id` header span
// The walker then reads every value where it lies inside the buffer (ck_view.len): the raw bytes, or a compressed batch's
// decoded slot.  No per-record slicing on the host.
//
// encode (produce): the publishes of a step to the frame topics, grouped by (topic, partition), become frames in one
// asynchronous pass (ck_fr_*_kernel, below); ck_encode_recordbatch is its one-group case
#ifndef CK_KAFKA_CUH
#define CK_KAFKA_CUH

#include "ck_lz4.cuh"
#include "ck_inflate.cuh"
#include "ck_zstd.cuh"
#include "ck_snappy.cuh"

#define CK_CRC_POLY 0x82F63B78u      // CRC32C (Castagnoli), reflected
#define CK_CRC32_POLY 0xEDB88320u    // CRC32 (IEEE), reflected: gzip's
#define CK_RB_HEADER 61u
#define CK_RB_CRC_FROM 21u
#define CK_RB_GZIP 1u                // attributes & 7: Kafka's codec ids of gzip
#define CK_RB_SNAPPY 2u              // snappy
#define CK_RB_LZ4 3u                 // LZ4
#define CK_RB_ZSTD 4u                // and zstd

// ---- CRC32 ------------------------------------------------------------------------------------------------------------
// Generic over the reflected polynomial P: CRC32C (Castagnoli, the batch CRC) by default, CRC32 (IEEE, the gzip trailer)
// for the gzip decode.  Four 256-entry tables (slicing-by-4) built in shared memory by the block itself
template <u32 P = CK_CRC_POLY>
__device__ __forceinline__ void ck_crc_tables(u32* t /* [4][256] */) {
    for (u32 i = threadIdx.x; i < 256; i += blockDim.x) {
        u32 c = i;
#pragma unroll
        for (int k = 0; k < 8; k++) c = (c >> 1) ^ ((c & 1u) ? P : 0u);
        t[i] = c;
    }
    __syncthreads();
    for (u32 i = threadIdx.x; i < 256; i += blockDim.x) {
        u32 c = t[i];
#pragma unroll
        for (int k = 1; k < 4; k++) { c = (c >> 8) ^ t[c & 0xffu]; t[k * 256 + i] = c; }
    }
    __syncthreads();
}
// finalised CRC of p[0..n) (init / xor-out all ones) with the tables of its polynomial.  LDG: words read through the
// read-only cache; false for bytes the same kernel wrote
template <bool LDG = true>
__device__ __forceinline__ u32 ck_crc_span(const u32* __restrict__ t, const u8* __restrict__ p, u32 n) {
    u32 c = 0xffffffffu;
    while (n && ((uintptr_t)p & 3u)) { c = t[(c ^ *p++) & 0xffu] ^ (c >> 8); n--; }
    const u32* w = (const u32*)p;
    for (; n >= 4; n -= 4) {
        c ^= LDG ? __ldg(w++) : *w++;
        c = t[768 + (c & 0xffu)] ^ t[512 + ((c >> 8) & 0xffu)] ^ t[256 + ((c >> 16) & 0xffu)] ^ t[c >> 24];
    }
    p = (const u8*)w;
    while (n--) c = t[(c ^ *p++) & 0xffu] ^ (c >> 8);
    return ~c;
}
// a(x) * b(x) mod P(x), reflected representation (bit 31 = x^0)
template <u32 P = CK_CRC_POLY>
__device__ __forceinline__ u32 ck_gf_mul(u32 a, u32 b) {
    u32 p = 0;
#pragma unroll 4
    for (u32 m = 0x80000000u; m; m >>= 1) {
        if (a & m) p ^= b;
        b = (b & 1u) ? (b >> 1) ^ P : b >> 1;
    }
    return p;
}
// x^(8 n) mod P
template <u32 P = CK_CRC_POLY>
__device__ __forceinline__ u32 ck_gf_xpow8(unsigned long long n) {
    u32 p = 0x80000000u;                       // x^0
    u32 sq = 0x00800000u;                      // x^8
    while (n) { if (n & 1ull) p = ck_gf_mul<P>(sq, p); sq = ck_gf_mul<P>(sq, sq); n >>= 1; }
    return p;
}
template <u32 P = CK_CRC_POLY>
__device__ __forceinline__ u32 ck_crc_combine(u32 crc_a, u32 crc_b, u32 xpow_len_b) { return ck_gf_mul<P>(xpow_len_b, crc_a) ^ crc_b; }

// the CRC of one span by one warp (all lanes return it): lane 0 takes the odd-sized head so that every other lane holds
// exactly `chunk` bytes and the tree fold shifts by multiples of one precomputed power
template <u32 P = CK_CRC_POLY, bool LDG = true>
__device__ __forceinline__ u32 ck_crc_warp(const u32* __restrict__ t, const u8* __restrict__ p, u32 n, u32 lane) {
    u32 chunk = (n >> 5) & ~3u;
    u32 head = n - 31u * chunk;
    u32 c = lane == 0 ? ck_crc_span<LDG>(t, p, head) : (chunk ? ck_crc_span<LDG>(t, p + head + (lane - 1) * chunk, chunk) : 0u);
    if (!chunk) return __shfl_sync(0xffffffffu, c, 0);
    u32 xp = ck_gf_xpow8<P>(chunk);            // x^(8 chunk); squared at every level: right blocks hold 1, 2, 4, 8, 16 chunks
#pragma unroll
    for (u32 s = 1; s < 32; s <<= 1) {
        u32 right = __shfl_down_sync(0xffffffffu, c, s);
        if ((lane & (2 * s - 1)) == 0) c = ck_crc_combine<P>(c, right, xp);
        xp = ck_gf_mul<P>(xp, xp);
    }
    return __shfl_sync(0xffffffffu, c, 0);
}

__device__ __forceinline__ u32 ck_be32(const u8* p) { return ((u32)p[0] << 24) | ((u32)p[1] << 16) | ((u32)p[2] << 8) | p[3]; }
__device__ __forceinline__ void ck_put_be32(u8* p, u32 v) { p[0] = v >> 24; p[1] = v >> 16; p[2] = v >> 8; p[3] = v; }
__device__ __forceinline__ void ck_put_be64(u8* p, unsigned long long v) { ck_put_be32(p, (u32)(v >> 32)); ck_put_be32(p + 4, (u32)v); }

// ---- decode -------------------------------------------------------------------------------------------------------------
// batch_off[b] .. batch_off[b+1]: frame b inside buf (indexed by the host: the frames chain through their own length field)
// batch_bad[b] afterwards: 0 delivered, 1 bad (CK_TXN_BAD), 2 skipped (CK_TXN_HIDE): the host's flag (ck_txn.h; NULL: none
// flagged) for a batch that passes the check, 1 for one that does not
__global__ void __launch_bounds__(256)
ck_rb_crc_kernel(const u8* __restrict__ buf, const long long* __restrict__ batch_off, const u32* __restrict__ flag, u32 nb,
                 u32* __restrict__ batch_bad) {
    __shared__ u32 t[1024];
    ck_crc_tables(t);
    u32 w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (w >= nb) return;
    const u8* f = buf + batch_off[w];
    u32 flen = (u32)(batch_off[w + 1] - batch_off[w]);
    u32 bad = 0;
    u32 codec = flen >= CK_RB_HEADER ? f[22] & 7u : 0u;
    if (flen < CK_RB_HEADER || f[16] != 2 || codec > CK_RB_ZSTD) bad = 1;   // not magic 2 / a codec id Kafka does not define
    else {
        u32 c = ck_crc_warp(t, f + CK_RB_CRC_FROM, flen - CK_RB_CRC_FROM, lane);
        if (c != ck_be32(f + 17)) bad = 1;
    }
    if (lane == 0) batch_bad[w] = bad ? 1u : flag ? flag[w] : 0u;
}

// a zig-zag varint of at most 10 bytes whose unsigned value fits in 64 bits (a 10th byte above 1 is refused, as an exact
// 64-bit reader refuses it); non-minimal encodings are accepted
__device__ __forceinline__ bool ck_varint(const u8* __restrict__ p, u32& pos, u32 end, long long& out) {
    unsigned long long u = 0; u32 shift = 0;
    for (;;) {
        if (pos >= end) return false;
        u8 b = p[pos++];
        if (shift == 63 && b > 1) return false;
        u |= (unsigned long long)(b & 0x7f) << shift;
        if (!(b & 0x80)) break;
        shift += 7;
    }
    out = (long long)(u >> 1) ^ -(long long)(u & 1);
    return true;
}

__device__ __forceinline__ bool ck_rb_is_lz4(const u8* __restrict__ buf, const long long* __restrict__ batch_off, u32 b) {
    return (buf[batch_off[b] + 22] & 7u) == CK_RB_LZ4;
}
// a batch whose records section is decoded into a slot: gzip, snappy, LZ4 or zstd
__device__ __forceinline__ bool ck_rb_is_decoded(const u8* __restrict__ buf, const long long* __restrict__ batch_off, u32 b) {
    u32 codec = buf[batch_off[b] + 22] & 7u;
    return codec == CK_RB_GZIP || codec == CK_RB_SNAPPY || codec == CK_RB_LZ4 || codec == CK_RB_ZSTD;
}

// warp per batch of a fetch that holds LZ4 batches; the uncompressed ones and those the CRC check refused are skipped.
// dec_off[b] .. dec_off[b+1]: the slot of batch b in buf, behind the raw bytes, sized by the host's walk of its block chain
// (ck_lz_walk; an empty slot: a chain the host could not walk).  The records section of the batch is one LZ4 frame; its
// blocks decode in order into the slot (linked blocks reach back into the frame's earlier output there), with the header
// checksum, block checksums, content checksum and content size verified where the frame carries them.  dec_len[b] = the
// decoded length; a frame that is malformed in any way, or does not fit its slot, marks its batch bad
__global__ void __launch_bounds__(256)
ck_rb_lz4_kernel(u8* __restrict__ buf, const long long* __restrict__ batch_off, const long long* __restrict__ dec_off, u32 nb,
                 u32* __restrict__ batch_bad, u32* __restrict__ dec_len) {
    u32 w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (w >= nb || batch_bad[w] || !ck_rb_is_lz4(buf, batch_off, w)) return;
    const u8* z = buf + batch_off[w] + CK_RB_HEADER;
    unsigned long long zn = (unsigned long long)(batch_off[w + 1] - batch_off[w]) - CK_RB_HEADER;
    u8* out = buf + dec_off[w];
    unsigned long long cap = (unsigned long long)(dec_off[w + 1] - dec_off[w]), bound = 0, op = 0;
    ck_lz_desc d;
    u32 nblk;
    bool ok = cap && ck_lz_parse_desc(z, zn, d) && ck_lz_walk(z, zn, d, &nblk, &bound) && bound <= cap;
    unsigned long long pos = ok ? d.hdr_len : 0;
    while (ok) {                                               // the walk checked the chain: every size word lies in the frame
        u32 word = ck_lz_le32(z + pos), sz = word & 0x7FFFFFFFu;
        pos += 4;
        if (!word) break;
        const u8* blk = z + pos;
        if (d.block_sum && ck_xxh32_warp(blk, sz, 0, lane) != ck_lz_le32(blk + sz)) { ok = false; break; }
        if (word >> 31) {                                      // stored raw
            if (op + sz > cap) { ok = false; break; }
            for (u32 i = lane; i < sz; i += 32) out[op + i] = blk[i];
            op += sz;
        } else {
            long long r = ck_lz4_decode_block(blk, sz, out, op, d.linked ? 0ull : op, cap, d.block_max, lane);
            if (r < 0) { ok = false; break; }
            op += (unsigned long long)r;
        }
        __syncwarp();
        pos += sz + (d.block_sum ? 4u : 0u);
    }
    __syncwarp();
    if (ok && d.content_sum) ok = ck_xxh32_warp(out, (u32)op, 0, lane) == ck_lz_le32(z + pos);
    if (ok && d.has_size) ok = d.content_size == op;
    if (lane == 0) { dec_len[w] = ok ? (u32)op : 0u; if (!ok) batch_bad[w] = 1; }
}

// warp per batch of a fetch that holds gzip batches (CK_GZ_WARPS per block, each with its Huffman tables in shared memory);
// the others and those the CRC check refused are skipped.  dec_off[b] .. dec_off[b+1]: the slot of batch b, as many bytes
// as the member's ISIZE says (ck_gz_member on the host).  The records section is one gzip member: its header parsed again,
// its deflate stream inflated into the slot (ck_gz_decode: zlib's verdict on every block), the trailer right behind the
// final block and ending at the batch's end, the output exactly ISIZE bytes, and the CRC32 of the output (the warp fold
// over the IEEE tables) equal to the trailer's.  The host refuses a member by giving it an empty slot; a member of
// ISIZE 0 gets one too, so the slot's size is no verdict: the decode parses the member itself and refuses unless the slot
// is exactly ISIZE bytes.  dec_len[b] = the inflated length; anything else marks the batch bad
#define CK_GZ_WARPS 4u
__global__ void __launch_bounds__(32 * CK_GZ_WARPS)
ck_rb_gzip_kernel(u8* buf, const long long* __restrict__ batch_off, const long long* __restrict__ dec_off, u32 nb,
                  u32* __restrict__ batch_bad, u32* __restrict__ dec_len) {
    __shared__ u32 t[1024];
    __shared__ ck_gz_ws ws[CK_GZ_WARPS];
    ck_crc_tables<CK_CRC32_POLY>(t);
    u32 wi = threadIdx.x >> 5, w = blockIdx.x * CK_GZ_WARPS + wi, lane = threadIdx.x & 31;
    if (w >= nb || batch_bad[w] || (buf[batch_off[w] + 22] & 7u) != CK_RB_GZIP) return;
    const u8* z = buf + batch_off[w] + CK_RB_HEADER;
    unsigned long long zn = (unsigned long long)(batch_off[w + 1] - batch_off[w]) - CK_RB_HEADER;
    u8* out = buf + dec_off[w];
    long long r = ck_gz_decode(z, zn, out, (unsigned long long)(dec_off[w + 1] - dec_off[w]), ws[wi], lane);
    __syncwarp();
    bool ok = r >= 0 && ck_crc_warp<CK_CRC32_POLY, false>(t, out, (u32)r, lane) == ck_gz_le32(z + zn - 8);
    if (lane == 0) { dec_len[w] = ok ? (u32)r : 0u; if (!ok) batch_bad[w] = 1; }
}

// warp per batch of a fetch that holds zstd batches (CK_ZS_WARPS per block, each with its Huffman and sequence tables in
// shared memory); the others and those the CRC check refused are skipped.  dec_off[b] .. dec_off[b+1]: the slot of batch
// b, sized by the host's walk of the frame's blocks (ck_zs_walk: raw and RLE blocks their size, compressed blocks
// Block_Maximum_Size), so that every compressed block has room for its literals at the end of its reservation.  The
// records section is one zstd frame: its header parsed and its blocks walked again, and refused unless the walk's bound is
// the slot's size (the host gives an empty slot to a frame it refuses, and a valid frame of empty blocks has one too),
// then decoded into the slot (ck_zs_decode: libzstd's verdict on every block), its output equal to Frame_Content_Size
// when the frame carries one and its XXH64 (four lanes, one accumulator each) to the checksum when present, the frame
// ending exactly at the batch's end.  dec_len[b] = the decoded length; anything else marks the batch bad
#define CK_ZS_WARPS 3u
__global__ void __launch_bounds__(32 * CK_ZS_WARPS)
ck_rb_zstd_kernel(u8* buf, const long long* __restrict__ batch_off, const long long* __restrict__ dec_off, u32 nb,
                  u32* __restrict__ batch_bad, u32* __restrict__ dec_len) {
    __shared__ ck_zs_ws ws[CK_ZS_WARPS];
    u32 wi = threadIdx.x >> 5, w = blockIdx.x * CK_ZS_WARPS + wi, lane = threadIdx.x & 31;
    if (w >= nb || batch_bad[w] || (buf[batch_off[w] + 22] & 7u) != CK_RB_ZSTD) return;
    const u8* z = buf + batch_off[w] + CK_RB_HEADER;
    unsigned long long zn = (unsigned long long)(batch_off[w + 1] - batch_off[w]) - CK_RB_HEADER;
    long long r = ck_zs_decode(z, zn, buf + dec_off[w], (unsigned long long)(dec_off[w + 1] - dec_off[w]), ws[wi], lane);
    if (lane == 0) { dec_len[w] = r >= 0 ? (u32)r : 0u; if (r < 0) batch_bad[w] = 1; }
}

// warp per chunk of a fetch that holds snappy batches: ch[0, nc) lists every raw snappy block of every snappy batch the
// host delivers (ck_sn_next: one for a raw-block section, one per chunk of a framed one), each with its place in its
// batch's slot.  dec_off[b] .. dec_off[b+1]: the slot of batch b, exactly the sum of its blocks' declared lengths.  A batch
// the host could not walk (or whose slot would pass the 32-bit lengths of the record split) has an empty slot and one
// entry of no input, which every decode refuses.  A batch the CRC check refused is skipped; a block that snappy refuses
// or that does not decode to exactly its declared length marks its batch bad; the batch's first block writes dec_len[b]
#define CK_SN_WARPS 8u
__global__ void __launch_bounds__(32 * CK_SN_WARPS)
ck_rb_snappy_kernel(u8* buf, const ck_sn_chunk* __restrict__ ch, u32 nc, const long long* __restrict__ dec_off,
                    u32* __restrict__ batch_bad, u32* __restrict__ dec_len) {
    u32 w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (w >= nc) return;
    const ck_sn_chunk c = ch[w];
    if (*(volatile u32*)(batch_bad + c.batch)) return;         // only ever set to 1 by the other chunks: any read is safe
    long long slot = dec_off[c.batch];
    if (c.out_off == 0 && lane == 0) dec_len[c.batch] = (u32)(dec_off[c.batch + 1] - slot);
    long long r = ck_sn_decode_block(buf + c.in_off, c.in_len, buf + slot + c.out_off, c.out_len, lane);
    if (r < 0 && lane == 0) batch_bad[c.batch] = 1;
}

// thread per batch: where does each record start.  rec_base[b] = records in the batches before b (host prefix sum of
// the recordsCount header fields); a batch whose records do not add up to its records section is marked bad.  The records
// section is [batch_off[b] + 61, batch_off[b+1]) of the raw bytes, or for a gzip, snappy, LZ4 or zstd batch (dec_off given) its decoded
// slot [dec_off[b], dec_off[b] + dec_len[b])
__global__ void __launch_bounds__(128)
ck_rb_split_kernel(const u8* __restrict__ buf, const long long* __restrict__ batch_off, const long long* __restrict__ dec_off,
                   const u32* __restrict__ dec_len, const u32* __restrict__ rec_base, u32 nb,
                   u32* __restrict__ batch_bad, long long* __restrict__ rec_pos, u32* __restrict__ rec_batch) {
    u32 b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= nb) return;
    u32 r0 = rec_base[b], cnt = rec_base[b + 1] - r0, st = batch_bad[b];
    bool ok = !st;                                              // a bad or skipped batch: its records get no span
    long long lo = batch_off[b] + CK_RB_HEADER, hi = batch_off[b + 1];
    if (ok && dec_off && ck_rb_is_decoded(buf, batch_off, b)) { lo = dec_off[b]; hi = lo + dec_len[b]; }
    const u8* f = buf + lo;
    u32 flen = (u32)(hi - lo);
    u32 pos = 0;
    for (u32 k = 0; k < cnt; k++) {
        rec_batch[r0 + k] = b;
        if (!ok) { rec_pos[r0 + k] = -1; continue; }
        rec_pos[r0 + k] = lo + pos;
        long long len;
        // the length compared in 64 bits: narrowed first, 2^32 + L would pass as L
        if (!ck_varint(f, pos, flen, len) || len < 0 || (unsigned long long)len > flen - pos) { ok = false; rec_pos[r0 + k] = -1; continue; }
        pos += (u32)len;
    }
    if (ok && pos != flen) ok = false;
    if (!ok && !st) batch_bad[b] = 1;
}

// thread per record.  Every length is compared with the bytes left in the record as a 64-bit quantity before it is
// narrowed; a negative key or value length is null, a negative header count or header key length is refused.  A refused
// record keeps no span
__global__ void __launch_bounds__(128)
ck_rb_fields_kernel(const u8* __restrict__ buf, long long buf_len, const long long* __restrict__ rec_pos, const u32* __restrict__ rec_batch,
                    const u32* __restrict__ batch_bad, u32 n,
                    long long* __restrict__ val_off, u32* __restrict__ val_len, long long* __restrict__ key_off, int* __restrict__ key_len,
                    long long* __restrict__ corr_off, int* __restrict__ corr_len, u32* __restrict__ rec_bad) {
    u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    val_off[i] = 0; val_len[i] = 0; key_off[i] = 0; key_len[i] = -1; corr_off[i] = 0; corr_len[i] = -1;
    long long rp = rec_pos[i];
    u32 st = batch_bad[rec_batch[i]];
    if (rp < 0 || st) { rec_bad[i] = st == 2u ? 2u : 1u; return; }
    const u8* p = buf + rp;
    u32 end = (u32)min((long long)0x7fffffff, buf_len - rp), pos = 0;
    long long len, t;
    bool ok = ck_varint(p, pos, end, len);
    u32 rec_end = pos + (u32)len;
    if (ok) end = rec_end;
    pos += 1;                                                   // attributes
    ok = ok && ck_varint(p, pos, end, t) && ck_varint(p, pos, end, t);       // timestampDelta, offsetDelta
    // after a varint is read, pos <= end
    ok = ok && ck_varint(p, pos, end, t);                       // key
    ok = ok && (t < 0 || (unsigned long long)t <= end - pos);
    if (ok && t >= 0) { key_off[i] = rp + pos; key_len[i] = (int)t; pos += (u32)t; }
    ok = ok && ck_varint(p, pos, end, t);                       // value
    ok = ok && (t < 0 || (unsigned long long)t <= end - pos);
    if (ok && t >= 0) { val_off[i] = rp + pos; val_len[i] = (u32)t; pos += (u32)t; }
    long long nh = 0;
    ok = ok && ck_varint(p, pos, end, nh) && nh >= 0;
    for (long long hcount = 0; ok && hcount < nh; hcount++) {
        long long kl, vl;
        ok = ck_varint(p, pos, end, kl) && kl >= 0 && (unsigned long long)kl <= end - pos;
        if (!ok) break;
        u32 kpos = pos; pos += (u32)kl;
        ok = ck_varint(p, pos, end, vl) && (vl < 0 || (unsigned long long)vl <= end - pos);
        if (!ok) break;
        bool is_corr = (kl == 14);                              // "correlation_id" (FastStream's header)
        const char* want = "correlation_id";
        for (u32 b = 0; is_corr && b < 14; b++) is_corr = (p[kpos + b] == (u8)want[b]);
        if (vl >= 0) { if (is_corr) { corr_off[i] = rp + pos; corr_len[i] = (int)vl; } pos += (u32)vl; }
    }
    ok = ok && pos == rec_end;
    rec_bad[i] = ok ? 0u : 1u;
    if (!ok) { val_off[i] = 0; val_len[i] = 0; key_off[i] = 0; key_len[i] = -1; corr_off[i] = 0; corr_len[i] = -1; }
}

// rec_bad[i]: 1 the record's batch failed a check, 2 the consumer does not deliver it (a control batch, or an aborted
// transaction's batch under read_committed).  Both have no span, so the walker passed over them as empty records
__global__ void __launch_bounds__(256)
ck_rb_mark_bad_kernel(const u32* __restrict__ rec_bad, u32 n, u32* __restrict__ cols, u32 stride) {
    u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n && rec_bad[i]) cols[(size_t)CK_COL_STATUS * stride + i] = rec_bad[i] == 2u ? CK_SKIPPED : CK_BAD_FRAME;
}

// ---- encode -------------------------------------------------------------------------------------------------------------
// Every live publish to a frame topic of the current plan (or every record of a small host-produced batch) becomes one
// record of a frame, in one pass queued on the stream (nothing in it waits for the host):
//   source   thread per publish / record: its value, key and correlation id (ck_fitem) and its group key (frame topic,
//            partition + 1); partition -1 (unkeyed) is a group of its own per topic, the producer client picks its partition,
//            unless the host gave the topic a sticky partition for the pass (idempotent produce: a sequence exists only per
//            partition), which the unkeyed publishes then join before the key is built
//   group    stable LSD radix sort by the group key (group_sort, ck_group.cuh): one run per group, send order kept
//   split    s_k = encoded size of record k with offsetDelta = its rank in the group, P_k = exclusive prefix of s inside the
//            group; record k starts a frame when it heads its group or floor(P_k / W) != floor(P_{k-1} / W), W = frame_bytes.
//            The real records of a frame (offsetDelta = rank in the frame) are no larger than their s_k, so a frame holds at
//            most 61 + W + one record bytes
//   size     exact sizes -> scan -> byte offset of every record; frames lie back to back, each behind its 61-byte header
//   table    thread per frame: frame table entry (topic id, partition, offset, length, records), header, CRC chunk count
//   write    warp per record: varint header, key, value, the headers calfkit's publishes carry
//   crc      warp per 16 KB chunk of any frame (chunk -> frame by binary search over the chunk scan), fold per frame
// Key and correlation id are JSON string content as they lie in the envelope: written unescaped (ck_key_byte), the bytes
// correlation_id.encode() gives and ck_murmur2_key hashes.
__device__ __forceinline__ u32 ck_varint_size(long long v) {
    unsigned long long u = ((unsigned long long)v << 1) ^ (unsigned long long)(v >> 63);
    u32 n = 1;
    while (u >= 0x80) { u >>= 7; n++; }
    return n;
}
__device__ __forceinline__ u32 ck_put_varint(u8* p, long long v) {
    unsigned long long u = ((unsigned long long)v << 1) ^ (unsigned long long)(v >> 63);
    u32 n = 0;
    while (u >= 0x80) { p[n++] = (u8)(u | 0x80); u >>= 7; }
    p[n++] = (u8)u;
    return n;
}
// what calfkit's publishes carry (SURVEY.md Appendix A): key = correlation id bytes when keyed, headers
// content-type: application/json and correlation_id (FastStream)
#define CK_RB_CT_HDR 30u             // varint(12) "content-type" varint(16) "application/json" = 1 + 12 + 1 + 16
#define CK_RB_NONE 0xffffffffu       // absent key / correlation id
#define CK_RB_CRC_CHUNK 16384u

struct ck_fitem {                    // one record to frame
    const u8* val; const u8* key; const u8* corr;
    u32 val_len;
    u32 key_raw, key_len;            // JSON string content: bytes in the source, bytes unescaped (CK_RB_NONE: no key)
    u32 corr_raw, corr_len;          // same for the correlation_id header (CK_RB_NONE: no header)
    int32_t topic_id, partition;
};
// the producer fields of a pass's frame headers (ck_set_producer): none = producerId -1, producerEpoch -1, attributes 0;
// idempotent = the producer's id and epoch; transactional = those and attributes bit 4.  baseSequence is always -1 here: the
// host writes each frame's sequence when it hands the frame out, and patches the CRC32C (ck_crc32c_patch)
struct ck_producer { long long pid; int epoch; u32 attr; };
struct ck_frame_ent {                // one frame of the frame table (mirrors ck_frame in include/calfkit_b200.h)
    int32_t topic_id, partition;     // partition -1: unkeyed records, the producer client picks the partition
    uint32_t n_records, first;       // records, first record in group order
    long long offset, length;        // bytes in the frame buffer
};

__device__ __forceinline__ u32 ck_unescaped_len(const u8* p, u32 raw) {
    if (raw == CK_RB_NONE) return CK_RB_NONE;
    GRd r; r.init(p, raw);
    u32 n = 0;
    for (u32 q = 0; q < raw; n++) ck_key_byte(r, q);
    return n;
}
// body length of a record whose offsetDelta is `rank` (timestampDelta 0)
__device__ __forceinline__ u32 ck_rb_measure(const ck_fitem& it, u32 rank) {
    u32 body = 1 + 1 + ck_varint_size(rank);                                    // attributes, timestampDelta 0, offsetDelta
    body += it.key_len != CK_RB_NONE ? ck_varint_size(it.key_len) + it.key_len : 1;   // key (or null)
    body += ck_varint_size(it.val_len) + it.val_len;
    body += 1 + CK_RB_CT_HDR;                                                   // header count, content-type
    if (it.corr_len != CK_RB_NONE) body += 1 + 14 + ck_varint_size(it.corr_len) + it.corr_len;
    return body;
}
__device__ __forceinline__ u32 ck_rb_encoded_size(const ck_fitem& it, u32 rank) { u32 b = ck_rb_measure(it, rank); return ck_varint_size(b) + b; }

// source: publishes idx[i] (NULL: publish i) of the plan.  frame_slot[topic id] = index of the frame topic or -1; NULL: one
// group for all of them (ck_encode_recordbatch).  Unframed slots get the key `excl`, which sorts last.  sticky[topic id]
// (n_sticky of them; NULL: none): the partition the topic's unkeyed publishes go to in this pass, -1 none
__global__ void __launch_bounds__(256)
ck_fr_src_pubs_kernel(ck_view vw, const ck_pub* __restrict__ pubs, const u32* __restrict__ idx, u32 n, const u32* __restrict__ pay_len,
                      const long long* __restrict__ out_off, const u8* __restrict__ out, const u32* __restrict__ cols, u32 stride,
                      const int32_t* __restrict__ frame_slot, u32 n_slots, u32 nparts, u32 excl,
                      const int32_t* __restrict__ sticky, u32 n_sticky, ck_fitem* __restrict__ items, u32* __restrict__ gkey) {
    u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    ck_pub p = pubs[idx ? idx[i] : i];
    int slot = -1;
    if (p.payload != 0xffffffffu) slot = !frame_slot ? 0 : (p.topic_id >= 0 && (u32)p.topic_id < n_slots ? frame_slot[p.topic_id] : -1);
    if (slot < 0) { gkey[i] = excl; return; }
    ck_fitem it;
    u32 rl; const u8* rec = ck_rec(vw, p.record, rl);
    u32 co = cols[(size_t)CK_COL_CORR_OFF * stride + p.record], cl = cols[(size_t)CK_COL_CORR_LEN * stride + p.record];
    it.val = out + out_off[p.payload]; it.val_len = pay_len[p.payload];
    it.corr = rec + co; it.corr_raw = cl; it.corr_len = ck_unescaped_len(it.corr, cl);
    it.key = it.corr; it.key_raw = p.has_key ? cl : CK_RB_NONE; it.key_len = p.has_key ? it.corr_len : CK_RB_NONE;
    it.topic_id = p.topic_id; it.partition = p.has_key ? p.partition : -1;
    if (!p.has_key && sticky && (u32)p.topic_id < n_sticky) it.partition = sticky[p.topic_id];
    items[i] = it;
    gkey[i] = frame_slot ? (u32)slot * (nparts + 1) + (u32)(it.partition + 1) : 0u;
}

// source: records a host path produced for one topic.  desc[i] = {value off, len, key off, len, correlation id off, len}
// into blob (len -1: absent); key and id are JSON string content, the partition is the plan's: murmur2(key) % nparts, or
// for an unkeyed record `sticky` (the topic's sticky partition of the pass; -1: none)
__global__ void __launch_bounds__(256)
ck_fr_src_recs_kernel(const u8* __restrict__ blob, const long long* __restrict__ desc, u32 n, int32_t topic_id, u32 nparts,
                      int32_t sticky, ck_fitem* __restrict__ items, u32* __restrict__ gkey) {
    u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const long long* d = desc + 6 * (size_t)i;
    ck_fitem it;
    it.val = blob + d[0]; it.val_len = (u32)d[1];
    it.key = blob + (d[3] >= 0 ? d[2] : 0); it.key_raw = d[3] >= 0 ? (u32)d[3] : CK_RB_NONE; it.key_len = ck_unescaped_len(it.key, it.key_raw);
    it.corr = blob + (d[5] >= 0 ? d[4] : 0); it.corr_raw = d[5] >= 0 ? (u32)d[5] : CK_RB_NONE; it.corr_len = ck_unescaped_len(it.corr, it.corr_raw);
    int part = sticky;
    if (it.key_raw != CK_RB_NONE && nparts) { GRd r; r.init(it.key, it.key_raw); part = (int)((ck_murmur2_key(r, 0, it.key_raw) & 0x7fffffffu) % nparts); }
    it.topic_id = topic_id; it.partition = part;
    items[i] = it;
    gkey[i] = (u32)(part + 1);
}

__device__ __forceinline__ u32 ck_fr_src(const u32* order, u32 k) { return order ? order[k] : k; }

// head[k]: record k (in group order) starts a group; *n_live = records that are framed (they sort before the rest)
__global__ void __launch_bounds__(256)
ck_fr_heads_kernel(const u32* __restrict__ order, const u32* __restrict__ gkey, u32 n, u32 excl, u32* __restrict__ head, u32* __restrict__ n_live) {
    u32 k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    u32 key = gkey[ck_fr_src(order, k)];
    bool live = key != excl;
    head[k] = live && (k == 0 || gkey[ck_fr_src(order, k - 1)] != key);
    if (live && (k + 1 == n || gkey[ck_fr_src(order, k + 1)] == excl)) *n_live = k + 1;
}
// first[id] = k for every k that starts group / frame id (scan = exclusive scan of flag)
__global__ void __launch_bounds__(256)
ck_fr_first_kernel(const u32* __restrict__ flag, const long long* __restrict__ scan, u32 n, u32* __restrict__ first) {
    u32 k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k < n && flag[k]) first[scan[k]] = k;
}
// encoded size of record k with offsetDelta = its rank in its group / frame
__global__ void __launch_bounds__(256)
ck_fr_size_kernel(const u32* __restrict__ order, const ck_fitem* __restrict__ items, const u32* __restrict__ flag,
                  const long long* __restrict__ scan, const u32* __restrict__ first, u32 n, const u32* __restrict__ n_live, u32* __restrict__ size) {
    u32 k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    if (k >= *n_live) { size[k] = 0; return; }
    u32 id = (u32)(scan[k] + flag[k]) - 1;
    size[k] = ck_rb_encoded_size(items[ck_fr_src(order, k)], k - first[id]);
}
// the split rule (see above); S = exclusive scan of the group-rank sizes
__global__ void __launch_bounds__(256)
ck_fr_split_kernel(const u32* __restrict__ head, const long long* __restrict__ gscan, const u32* __restrict__ gfirst,
                   const long long* __restrict__ S, u32 n, const u32* __restrict__ n_live, unsigned long long window, u32* __restrict__ fstart) {
    u32 k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    if (k >= *n_live) { fstart[k] = 0; return; }
    if (head[k]) { fstart[k] = 1; return; }
    long long base = S[gfirst[gscan[k] - 1]];
    fstart[k] = (unsigned long long)(S[k] - base) / window != (unsigned long long)(S[k - 1] - base) / window;
}

__device__ __forceinline__ void ck_rb_put_header(u8* __restrict__ f, unsigned long long total, u32 n, long long base_offset, long long ts,
                                                 const ck_producer& prod) {
    ck_put_be64(f, (unsigned long long)base_offset);
    ck_put_be32(f + 8, (u32)(total - 12));
    ck_put_be32(f + 12, 0);                                  // partitionLeaderEpoch
    f[16] = 2;
    ck_put_be32(f + 17, 0);                                  // crc: folded in last
    f[21] = 0; f[22] = (u8)prod.attr;                        // attributes: no compression, CreateTime, transactional or not
    ck_put_be32(f + 23, n - 1);                              // lastOffsetDelta
    ck_put_be64(f + 27, (unsigned long long)ts);
    ck_put_be64(f + 35, (unsigned long long)ts);
    ck_put_be64(f + 43, (unsigned long long)prod.pid);       // producerId (-1: none)
    f[51] = (u8)(prod.epoch >> 8); f[52] = (u8)prod.epoch;   // producerEpoch (-1: none)
    ck_put_be32(f + 53, 0xffffffffu);                        // baseSequence -1
    ck_put_be32(f + 57, n);
}
// thread per frame (F = exclusive scan of the frame starts, R = of the exact sizes; both n + 1 long).  A frame that does not
// fit the buffer is listed but not written: the size query reports the overflow
__global__ void __launch_bounds__(256)
ck_fr_table_kernel(const u32* __restrict__ order, const ck_fitem* __restrict__ items, const u32* __restrict__ ffirst,
                   const long long* __restrict__ F, const long long* __restrict__ R, u32 n, const u32* __restrict__ n_live,
                   long long base_offset, long long ts, ck_producer prod, unsigned long long cap, ck_frame_ent* __restrict__ table, u8* __restrict__ frames,
                   u32* __restrict__ chunks) {
    u32 f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= n) return;
    u32 nf = (u32)F[n];
    if (f >= nf) { chunks[f] = 0; return; }
    u32 a = ffirst[f], b = f + 1 < nf ? ffirst[f + 1] : *n_live;
    ck_frame_ent e;
    const ck_fitem& it = items[ck_fr_src(order, a)];
    e.topic_id = it.topic_id; e.partition = it.partition; e.n_records = b - a; e.first = a;
    e.offset = R[a] + (long long)CK_RB_HEADER * f; e.length = CK_RB_HEADER + R[b] - R[a];
    table[f] = e;
    bool fits = (unsigned long long)(e.offset + e.length) <= cap;
    chunks[f] = fits ? (u32)((e.length - CK_RB_CRC_FROM + CK_RB_CRC_CHUNK - 1) / CK_RB_CRC_CHUNK) : 0u;
    if (fits) ck_rb_put_header(frames + e.offset, (unsigned long long)e.length, b - a, base_offset, ts, prod);
}

// key / header value: JSON string content written unescaped (warp copy when it holds no escape)
__device__ __forceinline__ void ck_fr_put_str(u8* __restrict__ d, const u8* __restrict__ src, u32 raw, u32 len, u32 lane) {
    if (raw == len) { for (u32 b = lane; b < len; b += 32) d[b] = src[b]; return; }
    if (lane == 0) { GRd r; r.init(src, raw); u32 o = 0; for (u32 q = 0; q < raw;) d[o++] = (u8)ck_key_byte(r, q); }
}
// warp per record: every lane computes the same layout, lane 0 writes the small pieces, the warp copies key / value / id
__global__ void __launch_bounds__(256)
ck_fr_write_kernel(const u32* __restrict__ order, const ck_fitem* __restrict__ items, const u32* __restrict__ fstart,
                   const long long* __restrict__ F, const u32* __restrict__ ffirst, const long long* __restrict__ R, u32 n,
                   const u32* __restrict__ n_live, unsigned long long cap, u8* __restrict__ frames) {
    u32 k = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (k >= n || k >= *n_live) return;
    u32 f = (u32)(F[k] + fstart[k]) - 1, a = ffirst[f];
    unsigned long long at = (unsigned long long)R[a] + (unsigned long long)CK_RB_HEADER * (f + 1) + (unsigned long long)(R[k] - R[a]);
    if (at + (unsigned long long)(R[k + 1] - R[k]) > cap) return;
    const ck_fitem it = items[ck_fr_src(order, k)];
    u32 rank = k - a;
    u8* d = frames + at;
    u32 pos = 0, kpos = 0, vpos = 0, cpos = 0;
    u8 tmp[10];
    u32 m = ck_put_varint(tmp, ck_rb_measure(it, rank)); if (lane == 0) for (u32 b = 0; b < m; b++) d[pos + b] = tmp[b]; pos += m;
    if (lane == 0) { d[pos] = 0; d[pos + 1] = 0; } pos += 2;                                  // attributes, timestampDelta = 0
    m = ck_put_varint(tmp, rank); if (lane == 0) for (u32 b = 0; b < m; b++) d[pos + b] = tmp[b]; pos += m;
    if (it.key_len != CK_RB_NONE) {
        m = ck_put_varint(tmp, it.key_len); if (lane == 0) for (u32 b = 0; b < m; b++) d[pos + b] = tmp[b]; pos += m; kpos = pos; pos += it.key_len;
    } else { if (lane == 0) d[pos] = 1; pos += 1; }                                            // zig-zag(-1) = null key
    m = ck_put_varint(tmp, it.val_len); if (lane == 0) for (u32 b = 0; b < m; b++) d[pos + b] = tmp[b]; pos += m; vpos = pos; pos += it.val_len;
    bool has_corr = it.corr_len != CK_RB_NONE;
    if (lane == 0) {
        d[pos] = has_corr ? 4 : 2;                                                            // 2 headers (1 without an id)
        d[pos + 1] = 24; const char* a = "content-type"; for (u32 b = 0; b < 12; b++) d[pos + 2 + b] = (u8)a[b];
        d[pos + 14] = 32; const char* j = "application/json"; for (u32 b = 0; b < 16; b++) d[pos + 15 + b] = (u8)j[b];
        if (has_corr) { d[pos + 31] = 28; const char* c = "correlation_id"; for (u32 b = 0; b < 14; b++) d[pos + 32 + b] = (u8)c[b]; }
    }
    pos += 1 + CK_RB_CT_HDR;
    if (has_corr) {
        pos += 15;
        m = ck_put_varint(tmp, it.corr_len); if (lane == 0) for (u32 b = 0; b < m; b++) d[pos + b] = tmp[b]; pos += m; cpos = pos;
        ck_fr_put_str(d + cpos, it.corr, it.corr_raw, it.corr_len, lane);
    }
    if (it.key_len != CK_RB_NONE) ck_fr_put_str(d + kpos, it.key, it.key_raw, it.key_len, lane);
    ck_warp_copy(d + vpos, it.val, it.val_len, lane);
}

// CRC32C of every frame: warps stride over the chunks of all frames (C = exclusive scan of the per-frame chunk counts)
__global__ void __launch_bounds__(256)
ck_fr_crc_chunks_kernel(const ck_frame_ent* __restrict__ table, const long long* __restrict__ C, const long long* __restrict__ F, u32 n,
                        const u8* __restrict__ frames, u32* __restrict__ partial) {
    __shared__ u32 t[1024];
    ck_crc_tables(t);
    u32 lane = threadIdx.x & 31, nw = (gridDim.x * blockDim.x) >> 5;
    u32 nf = (u32)F[n];
    unsigned long long total = (unsigned long long)C[n];
    for (unsigned long long c = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; c < total; c += nw) {
        u32 lo = 0, hi = nf;                                   // last frame whose first chunk is <= c
        while (hi - lo > 1) { u32 mid = (lo + hi) >> 1; if ((unsigned long long)C[mid] <= c) lo = mid; else hi = mid; }
        ck_frame_ent e = table[lo];
        unsigned long long start = (c - (unsigned long long)C[lo]) * CK_RB_CRC_CHUNK, covered = (unsigned long long)e.length - CK_RB_CRC_FROM;
        u32 len = (u32)min((unsigned long long)CK_RB_CRC_CHUNK, covered - start);
        u32 crc = ck_crc_warp(t, frames + e.offset + CK_RB_CRC_FROM + start, len, lane);
        if (lane == 0) partial[c] = crc;
    }
}
__global__ void __launch_bounds__(256)
ck_fr_crc_fold_kernel(const ck_frame_ent* __restrict__ table, const long long* __restrict__ C, const long long* __restrict__ F, u32 n,
                      const u32* __restrict__ partial, u8* __restrict__ frames) {
    u32 f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= n || f >= (u32)F[n]) return;
    u32 c0 = (u32)C[f], nc = (u32)(C[f + 1] - C[f]);
    if (!nc) return;
    ck_frame_ent e = table[f];
    unsigned long long covered = (unsigned long long)e.length - CK_RB_CRC_FROM;
    u32 xp = ck_gf_xpow8(CK_RB_CRC_CHUNK);
    u32 c = 0;                                               // crc of the empty prefix
    for (u32 k = 0; k < nc; k++) {
        unsigned long long start = (unsigned long long)k * CK_RB_CRC_CHUNK;
        u32 len = (u32)min((unsigned long long)CK_RB_CRC_CHUNK, covered - start);
        c = ck_crc_combine(c, partial[c0 + k], len == CK_RB_CRC_CHUNK ? xp : ck_gf_xpow8(len));
    }
    ck_put_be32(frames + e.offset + 17, c);
}

// ---- LZ4 compression of the frames (ck_set_option 3 = 3) ------------------------------------------------------------------
// With the option on, the table and write kernels above build the uncompressed frames in a scratch buffer, and this stage
// turns each into a batch with attributes 3 (LZ4): header | 7-byte LZ4 frame header | blocks | end mark 00000000, where
// the records section [61, end) of the uncompressed frame is cut into independent blocks of 64 KB (the last one shorter):
//   blocks   thread per frame: block count; its scan gives every frame its first block
//   lz4      warp per block (ck_lz4_block, or ck_lz4_block_hc at a compression level of 3 and up, ck_set_option 4):
//            compressed bytes into a slot at the block's own offset in a second scratch region, or none when they would not
//            be smaller (the block is then stored raw, bit 31 of its size set)
//   size     block sizes -> scan; frame lengths -> scan -> offsets of the compressed frames
//   gather   warp per block: size word + bytes into the frame buffer; then thread per frame: header (attributes 3,
//            batchLength), LZ4 frame header, end mark, the frame table's offset / length and the CRC chunk count
// The CRC kernels above then run over the compressed frames.
// LZ4 frame descriptor as liblz4's LZ4F_compressFrame writes it with default preferences: magic 0x184D2204, FLG 0x60
// (version 01, independent blocks, no checksums, no content size), BD 0x40 (64 KB blocks), HC = (xxh32(FLG BD) >> 8) & 0xFF
#define CK_LZ_FRAME_HDR 7u
#define CK_LZ_OVERHEAD (CK_LZ_FRAME_HDR + 4u)   // frame header + end mark

// frame holding block b: the last frame whose first block is <= b (B = exclusive scan of the block counts)
__device__ __forceinline__ u32 ck_lz_frame_of(const long long* __restrict__ B, u32 nf, unsigned long long b) {
    u32 lo = 0, hi = nf;
    while (hi - lo > 1) { u32 mid = (lo + hi) >> 1; if ((unsigned long long)B[mid] <= b) lo = mid; else hi = mid; }
    return lo;
}
// thread per frame of the uncompressed frames (raw_cap: their buffer; frames that did not fit it get no block)
__global__ void __launch_bounds__(256)
ck_lz_blocks_kernel(const ck_frame_ent* __restrict__ table, const long long* __restrict__ F, u32 n, unsigned long long raw_cap,
                    u32* __restrict__ nblk) {
    u32 f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= n) return;
    u32 k = 0;
    if (f < (u32)F[n]) {
        ck_frame_ent e = table[f];
        if ((unsigned long long)(e.offset + e.length) <= raw_cap) k = (u32)((e.length - CK_RB_HEADER + CK_LZ_BLOCK - 1) / CK_LZ_BLOCK);
    }
    nblk[f] = k;
}
// warps stride over the block slots 0 .. bmax: bsize[b] = 4 + bytes of block b as it goes out (0 past the last block).
// depth 0: the greedy parse (ck_lz4_block); else the hash-chain parse (ck_lz4_block_hc) with the chain of warp slot w at
// chains + w * CK_LZ_BLOCK
template <bool HC>
__device__ __forceinline__ void ck_lz_compress_warps(const ck_frame_ent* __restrict__ table, const long long* __restrict__ B,
                                                     const long long* __restrict__ F, u32 n, const u8* __restrict__ raw,
                                                     u8* __restrict__ slots, u32 bmax, u32* __restrict__ bsize,
                                                     uint16_t* __restrict__ chains, u32 depth) {
    __shared__ uint16_t tabs[CK_LZ_WARPS][1u << CK_LZ_HBITS];
    u32 lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = gridDim.x * CK_LZ_WARPS;
    u32 nf = (u32)F[n];
    unsigned long long total = (unsigned long long)B[n];
    for (u32 b = blockIdx.x * CK_LZ_WARPS + wid; b < bmax; b += nw) {
        if (b >= total) { if (lane == 0) bsize[b] = 0; continue; }
        u32 f = ck_lz_frame_of(B, nf, b);
        ck_frame_ent e = table[f];
        unsigned long long at = (unsigned long long)e.offset + CK_RB_HEADER + (b - (unsigned long long)B[f]) * CK_LZ_BLOCK;
        u32 len = (u32)min((unsigned long long)CK_LZ_BLOCK, (unsigned long long)(e.offset + e.length) - at);
        u32 z = HC ? ck_lz4_block_hc(raw + at, len, slots + at, tabs[wid], chains + (size_t)(blockIdx.x * CK_LZ_WARPS + wid) * CK_LZ_BLOCK, depth, lane)
                   : ck_lz4_block(raw + at, len, slots + at, tabs[wid], lane);
        if (lane == 0) bsize[b] = 4u + (z ? z : len);
    }
}
__global__ void __launch_bounds__(CK_LZ_WARPS * 32)
ck_lz_compress_kernel(const ck_frame_ent* __restrict__ table, const long long* __restrict__ B, const long long* __restrict__ F, u32 n,
                      const u8* __restrict__ raw, u8* __restrict__ slots, u32 bmax, u32* __restrict__ bsize) {
    ck_lz_compress_warps<false>(table, B, F, n, raw, slots, bmax, bsize, nullptr, 0);
}
// the hash-chain parse runs on a fixed grid of CK_LZ_HC_CTAS_PER_SM CTAs per SM: one chain of CK_LZ_BLOCK u16 per warp
#define CK_LZ_HC_CTAS_PER_SM 2u
__global__ void __launch_bounds__(CK_LZ_WARPS * 32)
ck_lz_compress_hc_kernel(const ck_frame_ent* __restrict__ table, const long long* __restrict__ B, const long long* __restrict__ F, u32 n,
                         const u8* __restrict__ raw, u8* __restrict__ slots, u32 bmax, u32* __restrict__ bsize,
                         uint16_t* __restrict__ chains, u32 depth) {
    ck_lz_compress_warps<true>(table, B, F, n, raw, slots, bmax, bsize, chains, depth);
}
// thread per frame: compressed length (0: the frame has no blocks, it did not fit the scratch buffer); S = scan of bsize
__global__ void __launch_bounds__(256)
ck_lz_size_kernel(const long long* __restrict__ B, const long long* __restrict__ S, u32 n, u32* __restrict__ clen) {
    u32 f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= n) return;
    clen[f] = B[f + 1] > B[f] ? CK_RB_HEADER + CK_LZ_OVERHEAD + (u32)(S[B[f + 1]] - S[B[f]]) : 0u;
}
// warp per block: its size word and bytes at their place in the compressed frame (Z = scan of clen)
__global__ void __launch_bounds__(256)
ck_lz_gather_kernel(const ck_frame_ent* __restrict__ table, const long long* __restrict__ B, const long long* __restrict__ F, u32 n,
                    const long long* __restrict__ S, const u32* __restrict__ bsize, const long long* __restrict__ Z,
                    const u32* __restrict__ clen, const u8* __restrict__ raw, const u8* __restrict__ slots, unsigned long long cap,
                    u8* __restrict__ frames) {
    u32 lane = threadIdx.x & 31, nw = (gridDim.x * blockDim.x) >> 5;
    u32 nf = (u32)F[n];
    unsigned long long total = (unsigned long long)B[n];
    for (unsigned long long b = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; b < total; b += nw) {
        u32 f = ck_lz_frame_of(B, nf, b);
        if ((unsigned long long)Z[f] + clen[f] > cap) continue;
        ck_frame_ent e = table[f];
        unsigned long long at = (unsigned long long)e.offset + CK_RB_HEADER + (b - (unsigned long long)B[f]) * CK_LZ_BLOCK;
        u32 len = (u32)min((unsigned long long)CK_LZ_BLOCK, (unsigned long long)(e.offset + e.length) - at);
        u32 z = bsize[b] - 4u;
        bool stored = z == len;
        u8* d = frames + Z[f] + CK_RB_HEADER + CK_LZ_FRAME_HDR + (S[b] - S[B[f]]);
        if (lane == 0) { u32 w = stored ? (z | 0x80000000u) : z; d[0] = (u8)w; d[1] = (u8)(w >> 8); d[2] = (u8)(w >> 16); d[3] = (u8)(w >> 24); }
        ck_warp_copy(d + 4, (stored ? raw : slots) + at, z, lane);
    }
}
// thread per frame: batch header (codec 3, batchLength of the compressed frame; producer fields as the uncompressed frame
// has them), LZ4 frame header and end mark; the
// table entry moves to the compressed frame; CRC chunk count as ck_fr_table_kernel gives it (0: not written)
__global__ void __launch_bounds__(256)
ck_lz_head_kernel(ck_frame_ent* __restrict__ table, const long long* __restrict__ F, u32 n, const long long* __restrict__ Z,
                  const u32* __restrict__ clen, const u8* __restrict__ raw, unsigned long long cap, u8* __restrict__ frames,
                  u32* __restrict__ chunks) {
    u32 f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= n) return;
    if (f >= (u32)F[n]) { chunks[f] = 0; return; }
    ck_frame_ent e = table[f];
    u32 len = clen[f];
    bool fits = len && (unsigned long long)Z[f] + len <= cap;
    chunks[f] = fits ? (len - CK_RB_CRC_FROM + CK_RB_CRC_CHUNK - 1) / CK_RB_CRC_CHUNK : 0u;
    if (fits) {
        u8* d = frames + Z[f];
        const u8* s = raw + e.offset;
#pragma unroll 1
        for (u32 i = 0; i < CK_RB_HEADER; i++) d[i] = s[i];
        ck_put_be32(d + 8, len - 12u);
        d[22] = s[22] | CK_RB_LZ4;                           // attributes: LZ4, CreateTime, the transactional bit kept
        ck_put_be32(d + CK_RB_HEADER, 0x04224D18u);          // magic 0x184D2204, little-endian
        d[CK_RB_HEADER + 4] = 0x60; d[CK_RB_HEADER + 5] = 0x40; d[CK_RB_HEADER + 6] = 0x82;   // FLG, BD, HC
        ck_put_be32(d + len - 4, 0u);
    }
    e.offset = Z[f]; e.length = len;
    table[f] = e;
}

#endif  // CK_KAFKA_CUH
