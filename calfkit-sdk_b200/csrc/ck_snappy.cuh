// Snappy records sections decoded by one warp per chunk, for the snappy batches of fetch responses (ck_rb_snappy_kernel,
// ck_kafka.cuh).  The one parse of the format.  Depends on nothing else of the device code, and compiles with g++ as well
// (one "lane", no warp): the block varint and the section walk are __host__ __device__, because the host sizes each batch's
// slot and lists its chunks from them (ck_submit_recordbatch), and the block decoder is the same source on both sides, so
// that the CPU suite holds it against Google snappy (tests/test_snappy_hostsim.py).
//
// A snappy batch's records section (attributes & 7 == 2) has one of two shapes, told apart as librdkafka's reader does:
//   snappy-java ("xerial") framing, written by Java's producer, kafka-python and aiokafka: a section longer than 16 bytes
//     that starts with 82 'SNAPPY' 00.  The two big-endian version words behind the magic are stepped over unchecked; then
//     chunks, each a big-endian u32 length c (1 <= c <= the bytes left) and one raw snappy block of c bytes, tiling the rest
//     of the section exactly.  Java's SnappyInputStream also skips a second stream header where a chunk length is expected
//     (concatenated streams); no Kafka client writes one, and here its first word reads as a length above 2^31: refused.
//   one raw snappy block covering the whole section (librdkafka, sarama): anything else.
// A raw block is what Google snappy's RawUncompress accepts: the decoded length as a varint32 (at most 5 bytes, a 5th byte
// below 16), then elements to the end of the input:
//   literal  tag 00: length (tag >> 2) + 1, or for tag >> 2 >= 60 a little-endian length of (tag >> 2) - 59 bytes, plus 1
//            (computed in 32 bits, as snappy does: a 4-byte length of 0xffffffff is a literal of 0 bytes)
//   copy-1   tag 01: length 4 + ((tag >> 2) & 7), offset (tag >> 5) << 8 | next byte
//   copy-2   tag 10: length (tag >> 2) + 1, offset LE16
//   copy-4   tag 11: length (tag >> 2) + 1, offset LE32
// refused on an element cut off by the end of the input, offset 0 or reaching before the block's first byte, and output
// past the declared length or ending short of it.  A section's chunks decode independently: a copy reaches back into its
// own block's output only.  Every chunk states its decoded length, so the host places every chunk's output before any
// kernel runs and the device decodes a warp per chunk.
#ifndef CK_SNAPPY_CUH
#define CK_SNAPPY_CUH

#include <stdint.h>
typedef uint8_t u8;
typedef uint32_t u32;

#ifdef __CUDACC__
#define CK_SN_HD __host__ __device__ __forceinline__
#define CK_SN_DEV __device__ __forceinline__
#define CK_SN_LANES 32u
#else
#define CK_SN_HD inline
#define CK_SN_DEV inline
#define CK_SN_LANES 1u
#endif
#ifdef __CUDA_ARCH__
#define CK_SN_SYNC() __syncwarp()
#else
#define CK_SN_SYNC() ((void)0)
#endif

#define CK_SN_FRAME_HDR 16u          // magic (8) + version + compatible version (big-endian u32 each)
#define CK_SN_RATIO 22u              // no element emits more than 64 / 3 bytes per input byte: a longer declared length is refused

// one chunk of a fetch's snappy batches, as the host lists them for ck_rb_snappy_kernel: its raw block at buf[in_off,
// in_off + in_len), decoding to out_len bytes at out_off inside the slot of batch `batch`
struct ck_sn_chunk {
    long long in_off;
    u32 batch, in_len, out_off, out_len;
};

// the decoded length at the start of a raw block p[0, n): false when it is not a varint32 snappy reads (cut off by the end of
// the input, more than 5 bytes, or a 5th byte of 16 or more); *ip = the first element
CK_SN_HD bool ck_sn_varint(const u8* p, u32 n, u32* ip, u32* len) {
    u32 v = 0;
    for (u32 k = 0; k < 5; k++) {
        if (k >= n) return false;
        u32 b = p[k];
        if (k == 4 && b >= 16u) return false;
        v |= (b & 0x7fu) << (7 * k);
        if (b < 128u) { *ip = k + 1; *len = v; return true; }
    }
    return false;
}

// the section p[0, n) framed by snappy-java?
CK_SN_HD bool ck_sn_framed(const u8* p, unsigned long long n) {
    const u8 magic[8] = {0x82, 'S', 'N', 'A', 'P', 'P', 'Y', 0};
    if (n <= CK_SN_FRAME_HDR) return false;
    for (u32 i = 0; i < 8; i++) if (p[i] != magic[i]) return false;
    return true;
}

// The walk of a records section p[0, n): its shape, its chunk chain when framed, and every block's declared length, one
// block per ck_sn_next (a raw-block section is one).  A section cannot be walked when a chunk length is 0, runs past the
// end or leaves bytes that do not tile the section, when a block's varint is one snappy refuses, or when a block declares
// more than CK_SN_RATIO times its own size (snappy would refuse it: this keeps a corrupt block from reserving gigabytes)
struct ck_sn_walker {
    unsigned long long pos;            // the next chunk length (framed)
    bool framed, done;
};
CK_SN_HD void ck_sn_begin(const u8* p, unsigned long long n, ck_sn_walker& w) {
    w.framed = ck_sn_framed(p, n);
    w.pos = w.framed ? CK_SN_FRAME_HDR : 0;
    w.done = false;
}
// 1: the next raw block lies at p[*off, *off + *len) and declares *dl bytes; 0: the section ends; -1: it cannot be walked
CK_SN_HD int ck_sn_next(const u8* p, unsigned long long n, ck_sn_walker& w, unsigned long long* off, u32* len, u32* dl) {
    unsigned long long o, c;
    if (!w.framed) {
        if (w.done) return 0;
        if (n > 0xffffffffull) return -1;
        o = 0; c = n; w.done = true;
    } else {
        if (w.pos == n) return 0;                              // a framed section is longer than its header: one chunk at least
        if (n - w.pos < 4) return -1;
        c = ((u32)p[w.pos] << 24) | ((u32)p[w.pos + 1] << 16) | ((u32)p[w.pos + 2] << 8) | p[w.pos + 3];
        w.pos += 4;
        if (c == 0 || c > n - w.pos) return -1;
        o = w.pos; w.pos += c;
    }
    u32 ip, d;
    if (!ck_sn_varint(p + o, (u32)c, &ip, &d) || (unsigned long long)d > CK_SN_RATIO * c) return -1;
    *off = o; *len = (u32)c; *dl = d;
    return 1;
}

// One raw snappy block src[0, n) decoded by one warp into out[0, cap): cap is the block's declared length (the walk's),
// and the block is refused unless its varint says so.  Every lane parses the same elements; the warp copies each literal
// and match.  A match copies out[pos - off + (i mod off)]: bytes that lie before it, so overlapping matches need no
// ordering.  Returns the decoded size (= cap), or -1 for a block snappy refuses
CK_SN_DEV long long ck_sn_decode_block(const u8* __restrict__ src, u32 n, u8* __restrict__ out, u32 cap, u32 lane) {
    u32 ip, len;
    if (!ck_sn_varint(src, n, &ip, &len) || len != cap) return -1;
    u32 op = 0;
    while (ip < n) {
        u32 tag = src[ip++], kind = tag & 3u, l, off;
        if (kind == 0) {
            l = (tag >> 2) + 1u;
            if (l > 60u) {
                u32 k = l - 60u;
                if (k > n - ip) return -1;
                u32 v = 0;
                for (u32 j = 0; j < k; j++) v |= (u32)src[ip + j] << (8 * j);
                ip += k;
                l = v + 1u;                                    // 32-bit, as snappy: 0xffffffff + 1 is an empty literal
            }
            if (l > n - ip || l > cap - op) return -1;
            for (u32 i = lane; i < l; i += CK_SN_LANES) out[op + i] = src[ip + i];
            ip += l; op += l;
            continue;
        }
        if (kind == 1) {
            if (ip >= n) return -1;
            l = 4u + ((tag >> 2) & 7u);
            off = ((tag >> 5) << 8) | src[ip++];
        } else if (kind == 2) {
            if (n - ip < 2) return -1;
            l = (tag >> 2) + 1u;
            off = (u32)src[ip] | ((u32)src[ip + 1] << 8);
            ip += 2;
        } else {
            if (n - ip < 4) return -1;
            l = (tag >> 2) + 1u;
            off = (u32)src[ip] | ((u32)src[ip + 1] << 8) | ((u32)src[ip + 2] << 16) | ((u32)src[ip + 3] << 24);
            ip += 4;
        }
        if (off == 0 || off > op || l > cap - op) return -1;
        CK_SN_SYNC();                                          // the literals (and earlier matches) before they are read
        const u8* m = out + (op - off);
        if (off >= l) for (u32 i = lane; i < l; i += CK_SN_LANES) out[op + i] = m[i];
        else for (u32 i = lane; i < l; i += CK_SN_LANES) out[op + i] = m[i % off];
        op += l;
        CK_SN_SYNC();
    }
    CK_SN_SYNC();
    return op == cap ? (long long)op : -1;
}

#endif  // CK_SNAPPY_CUH
