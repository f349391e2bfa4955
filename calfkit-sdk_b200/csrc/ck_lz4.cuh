// LZ4 block compression by one warp (the format: lz4's doc/lz4_Block_format.md), used by the frame pass's LZ4 stage
// (ck_kafka.cuh).  Depends on nothing else of the device code, so that it can be compiled and tested on its own.
#ifndef CK_LZ4_CUH
#define CK_LZ4_CUH

#include <stdint.h>
typedef uint8_t u8;
typedef uint32_t u32;

#define CK_LZ_BLOCK 65536u
#define CK_LZ_HBITS 12u              // hash table: 4096 positions (u16: position + 1, 0 = empty) per warp in shared memory
#define CK_LZ_WARPS 4u               // warps (= blocks in flight) per CTA

// little-endian 4 bytes at any address (two aligned loads; buffers carry CK_PAD bytes of tail padding)
__device__ __forceinline__ u32 ck_ld32u(const u8* p) {
    uintptr_t a = (uintptr_t)p;
    const u32* w = (const u32*)(a & ~(uintptr_t)3);
    return __funnelshift_r(w[0], w[1], (u32)(a & 3u) * 8u);
}
__device__ __forceinline__ u32 ck_lz_hash(u32 v) { return (v * 2654435761u) >> (32u - CK_LZ_HBITS); }
__device__ __forceinline__ u32 ck_lz_len_bytes(u32 l) { return l >= 15u ? (l - 15u) / 255u + 1u : 0u; }
// length continuation of `rem` = length - 15: 255 ... 255, rem % 255
__device__ __forceinline__ void ck_lz_put_len(u8* __restrict__ d, u32 rem, u32 lane) {
    u32 nb = rem / 255u + 1u;
    for (u32 i = lane; i < nb; i += 32) d[i] = i + 1 < nb ? (u8)255 : (u8)(rem - 255u * (nb - 1));
}
// one sequence: token, literal length, literals, then (ml != 0) offset and match length.  Returns its size
__device__ __forceinline__ u32 ck_lz_put_seq(u8* __restrict__ d, const u8* __restrict__ lit, u32 ll, u32 off, u32 ml, u32 lane) {
    u32 mcode = ml ? ml - 4u : 0u;
    if (lane == 0) d[0] = (u8)((min(ll, 15u) << 4) | min(mcode, 15u));
    u32 pos = 1;
    if (ll >= 15u) { ck_lz_put_len(d + pos, ll - 15u, lane); pos += ck_lz_len_bytes(ll); }
    for (u32 i = lane; i < ll; i += 32) d[pos + i] = lit[i];
    pos += ll;
    if (!ml) return pos;
    if (lane == 0) { d[pos] = (u8)off; d[pos + 1] = (u8)(off >> 8); }
    pos += 2;
    if (mcode >= 15u) { ck_lz_put_len(d + pos, mcode - 15u, lane); pos += ck_lz_len_bytes(mcode); }
    return pos;
}

// The block rules a decoder enforces (both parses below keep them through the two helpers that follow): a match starts at
// most at len - 12 and ends at most at len - 5 (the last 5 bytes are literals), the last sequence holds literals only,
// offsets are 1 .. 65535 (a block holds at most 65536 positions).  ck_lz_room: the most a match at ms may run
__device__ __forceinline__ u32 ck_lz_room(u32 len, u32 ms) { return len - 5u - ms; }
// length of the match src[ms ..] = src[mc ..] of which ml bytes are known equal, extended by the warp 128 bytes per round
// and held to the block rules
__device__ __forceinline__ u32 ck_lz_extend(const u8* __restrict__ src, u32 len, u32 ms, u32 mc, u32 ml, u32 lane) {
    u32 maxlen = ck_lz_room(len, ms);
    while (ml < maxlen) {
        u32 o = ml + 4u * lane;
        bool in = o < maxlen;
        u32 x = in ? ck_ld32u(src + ms + o) ^ ck_ld32u(src + mc + o) : 0u;
        u32 stop = __ballot_sync(0xffffffffu, x != 0u || !in);
        if (stop) {
            u32 l = (u32)__ffs(stop) - 1u, xl = __shfl_sync(0xffffffffu, x, l);
            ml += 4u * l + (xl ? ((u32)__ffs(xl) - 1u) >> 3 : 0u);
            break;
        }
        ml += 128u;
    }
    return min(ml, maxlen);
}
// the sequence literals src[anchor, ms) + match (ms - off, ml; ml 0: the last sequence, literals only) appended at dst[op];
// false when the block would reach cap bytes (it is then stored raw)
__device__ __forceinline__ bool ck_lz_emit(u8* __restrict__ dst, u32& op, u32 cap, const u8* __restrict__ src, u32 anchor, u32 ms,
                                           u32 off, u32 ml, u32 lane) {
    u32 ll = ms - anchor;
    if (op + 1u + ck_lz_len_bytes(ll) + ll + (ml ? 2u + ck_lz_len_bytes(ml - 4u) : 0u) > cap) return false;
    op += ck_lz_put_seq(dst + op, src + anchor, ll, off, ml, lane);
    return true;
}

// One LZ4 block of src[0, len), len <= 64 KB, compressed by one warp into dst (at most len - 1 bytes are written).  Returns
// the compressed size, or 0 when it would not be smaller than len (the caller stores the block raw).
// Greedy parse: the warp looks at the 32 positions p .. p+31 at once; each lane hashes its 4 bytes and takes the table's
// last position with that hash (inserted by an earlier round, so it lies before p) as its candidate.  The first lane whose
// candidate matches starts the match; positions up to it enter the table (one writer per hash: the highest position),
// the match is extended 128 bytes per round, and the literals before it and the match are written.  Every step is a
// fixed function of the input: the output is deterministic.
__device__ __forceinline__ u32 ck_lz4_block(const u8* __restrict__ src, u32 len, u8* __restrict__ dst, uint16_t* __restrict__ tab, u32 lane) {
    if (len < 13u) return 0;                                   // no match can start: literals only, one byte longer
    for (u32 i = lane; i < (1u << CK_LZ_HBITS) / 2; i += 32) ((u32*)tab)[i] = 0u;
    __syncwarp();
    const u32 last = len - 12u, cap = len - 1u;
    u32 p = 0, anchor = 0, op = 0;
    while (p <= last) {
        u32 q = p + lane;
        bool valid = q <= last;
        u32 v = valid ? ck_ld32u(src + q) : 0u, h = ck_lz_hash(v), c = 0;
        bool hit = false;
        if (valid) { u32 t = tab[h]; if (t) { c = t - 1u; hit = ck_ld32u(src + c) == v; } }
        u32 hits = __ballot_sync(0xffffffffu, hit);
        u32 f = hits ? (u32)__ffs(hits) - 1u : 31u;
        u32 ins = __ballot_sync(0xffffffffu, valid && lane <= f);
        u32 same = __match_any_sync(0xffffffffu, h) & ins;
        __syncwarp();                                          // every lookup of this round before any insertion
        if (((ins >> lane) & 1u) && lane == 31u - (u32)__clz(same)) tab[h] = (uint16_t)(q + 1u);
        __syncwarp();
        if (!hits) { p += 32; continue; }
        u32 ms = p + f, mc = __shfl_sync(0xffffffffu, c, f);
        u32 ml = ck_lz_extend(src, len, ms, mc, 4u, lane);
        if (!ck_lz_emit(dst, op, cap, src, anchor, ms, ms - mc, ml, lane)) return 0;
        anchor = p = ms + ml;
    }
    return ck_lz_emit(dst, op, cap, src, anchor, len, 0, 0, lane) ? op : 0;
}

// ---- hash-chain parse (compression levels 3 and up) ----------------------------------------------------------------------
// Search depth by compression level (ck_set_option 4, Kafka's compression.lz4.level 1 .. 17): 0 = the greedy parse above
// (levels 1 and 2 are liblz4's fast compressor, so they stay the default parse).  From level 3 the depth doubles per level,
// as liblz4's HC levels 3 .. 9 search 4 .. 256 candidates, up to CK_LZ_HC_DEPTH_CAP at level 9; levels 10 .. 17 search as
// level 9 does (liblz4 runs its optimal parser there; this parse stays the chain walk with the lazy step)
#define CK_LZ_LEVEL_MAX 17u
#define CK_LZ_HC_DEPTH_CAP 256u
static const uint16_t ck_lz_hc_depth[CK_LZ_LEVEL_MAX + 1] = {0, 0, 0, 4, 8, 16, 32, 64, 128, 256, 256, 256, 256, 256, 256, 256, 256, 256};
// a lane stops probing a candidate at this many equal bytes, and stops its walk at such a candidate (the nearest one of
// that length): the chosen match is then extended by the warp (ck_lz_extend)
#define CK_LZ_HC_NICE 64u

// positions [from, to) (at most 32) enter the head table and the chain: chain[q] = q - the previous position with q's hash
// (an earlier lane of the same round, else the head), 0 = none.  Every lane reads the head before any lane writes it
__device__ __forceinline__ void ck_lz_hc_insert(const u8* __restrict__ src, u32 from, u32 to, uint16_t* __restrict__ tab,
                                                uint16_t* __restrict__ chain, u32 lane) {
    u32 q = from + lane;
    bool valid = q < to;
    u32 h = valid ? ck_lz_hash(ck_ld32u(src + q)) : ~0u;
    u32 same = __match_any_sync(0xffffffffu, h) & __ballot_sync(0xffffffffu, valid);
    u32 t = valid ? tab[h] : 0u, below = same & ((1u << lane) - 1u);
    u32 prev = below ? from + 31u - (u32)__clz(below) : t ? t - 1u : q;
    if (valid) chain[q] = (uint16_t)(q - prev);
    __syncwarp();
    if (valid && lane == 31u - (u32)__clz(same)) tab[h] = (uint16_t)(q + 1u);
    __syncwarp();
}

// The same block contract as ck_lz4_block (one warp, len <= 64 KB, 0 = store raw, deterministic, the block rules) with a
// hash-chain search: chain (CK_LZ_BLOCK entries, global memory of this warp alone) links each position to the previous one
// with its hash, tab holds the last position per hash.  The warp looks at 32 positions per round, after every position up
// to them has entered the chain; each lane walks its own position's chain through at most `depth` candidates and keeps the
// longest match (the nearest among equals).  The first lane with a match starts it, unless the lane after it has a longer
// one (the lazy step, taken again while it holds); the chosen match is extended by the warp and written.  Positions
// inside a match enter the chain too, so later positions find them.  depth >= 1
__device__ __forceinline__ u32 ck_lz4_block_hc(const u8* __restrict__ src, u32 len, u8* __restrict__ dst, uint16_t* __restrict__ tab,
                                               uint16_t* __restrict__ chain, u32 depth, u32 lane) {
    if (len < 13u) return 0;
    for (u32 i = lane; i < (1u << CK_LZ_HBITS) / 2; i += 32) ((u32*)tab)[i] = 0u;
    __syncwarp();
    const u32 last = len - 12u, cap = len - 1u;
    u32 p = 0, anchor = 0, op = 0, ins = 0;                    // positions below ins are in the chain
    while (p <= last) {
        for (u32 end = min(p + 32u, last + 1u); ins < end; ins = min(ins + 32u, end)) ck_lz_hc_insert(src, ins, min(ins + 32u, end), tab, chain, lane);
        u32 q = p + lane, ml = 0, off = 0;
        if (q <= last) {
            u32 v = ck_ld32u(src + q), nice = min(ck_lz_room(len, q), CK_LZ_HC_NICE), c = q, d = chain[q];
            for (u32 k = 0; k < depth && d; k++) {
                c -= d;
                if (ck_ld32u(src + c) == v) {
                    u32 l = 4;
                    while (l < nice) {
                        u32 x = ck_ld32u(src + q + l) ^ ck_ld32u(src + c + l);
                        if (x) { l += ((u32)__ffs(x) - 1u) >> 3; break; }
                        l += 4u;
                    }
                    l = min(l, nice);
                    if (l > ml) { ml = l; off = q - c; if (ml == nice) break; }
                }
                d = chain[c];
            }
        }
        u32 hits = __ballot_sync(0xffffffffu, ml != 0u);
        if (!hits) { p += 32; continue; }
        u32 longer = __ballot_sync(0xffffffffu, __shfl_down_sync(0xffffffffu, ml, 1) > ml && lane < 31u);
        u32 f = (u32)__ffs(hits) - 1u;
        f += (u32)__ffs(~(longer >> f)) - 1u;                  // the lazy step: on while the next position's match is longer
        u32 ms = p + f, mo = __shfl_sync(0xffffffffu, off, f);
        u32 mlen = ck_lz_extend(src, len, ms, ms - mo, __shfl_sync(0xffffffffu, ml, f), lane);
        if (!ck_lz_emit(dst, op, cap, src, anchor, ms, mo, mlen, lane)) return 0;
        anchor = p = ms + mlen;
    }
    return ck_lz_emit(dst, op, cap, src, anchor, len, 0, 0, lane) ? op : 0;
}

// ---- decoding (lz4's doc/lz4_Frame_format.md and doc/lz4_Block_format.md) ------------------------------------------------
// The one parse of the LZ4 frame format: the host walks a frame's block chain to size its output (ck_submit_recordbatch),
// the device parses it again and decodes it (ck_lz_decode_kernel, ck_kafka.cuh).  Every read is checked against the
// frame's end and every write against the output's capacity: the frames are outside input.
#define CK_HD __host__ __device__ __forceinline__
#define CK_LZ_MAGIC 0x184D2204u

CK_HD u32 ck_lz_le32(const u8* p) { return (u32)p[0] | ((u32)p[1] << 8) | ((u32)p[2] << 16) | ((u32)p[3] << 24); }
CK_HD u32 ck_xxh_rotl(u32 x, u32 r) { return (x << r) | (x >> (32u - r)); }
#define CK_XXH_P1 2654435761u
#define CK_XXH_P2 2246822519u
#define CK_XXH_P3 3266489917u
#define CK_XXH_P4 668265263u
#define CK_XXH_P5 374761393u
// the tail of XXH32: h = the merged accumulators (or seed + P5) + n, then the bytes past the last 16-byte stripe
CK_HD u32 ck_xxh32_tail(u32 h, const u8* p, u32 n) {
    u32 i = n & ~15u;
    for (; i + 4 <= n; i += 4) h = ck_xxh_rotl(h + ck_lz_le32(p + i) * CK_XXH_P3, 17) * CK_XXH_P4;
    for (; i < n; i++) h = ck_xxh_rotl(h + p[i] * CK_XXH_P5, 11) * CK_XXH_P1;
    h ^= h >> 15; h *= CK_XXH_P2; h ^= h >> 13; h *= CK_XXH_P3; h ^= h >> 16;
    return h;
}
CK_HD u32 ck_xxh32_acc0(u32 k, u32 seed) {
    return k == 0 ? seed + CK_XXH_P1 + CK_XXH_P2 : k == 1 ? seed + CK_XXH_P2 : k == 2 ? seed : seed - CK_XXH_P1;
}
// XXH32 of p[0, n) (the xxHash specification), one thread
CK_HD u32 ck_xxh32(const u8* p, u32 n, u32 seed) {
    u32 h = seed + CK_XXH_P5;
    if (n >= 16) {
        u32 v[4];
        for (u32 k = 0; k < 4; k++) v[k] = ck_xxh32_acc0(k, seed);
        for (u32 s = 0; s + 16 <= n; s += 16)
            for (u32 k = 0; k < 4; k++) v[k] = ck_xxh_rotl(v[k] + ck_lz_le32(p + s + 4 * k) * CK_XXH_P2, 13) * CK_XXH_P1;
        h = ck_xxh_rotl(v[0], 1) + ck_xxh_rotl(v[1], 7) + ck_xxh_rotl(v[2], 12) + ck_xxh_rotl(v[3], 18);
    }
    return ck_xxh32_tail(h + n, p, n);
}
// the same by one warp (every lane returns it): lanes 0-3 run the four accumulators over the stripes side by side
__device__ __forceinline__ u32 ck_xxh32_warp(const u8* p, u32 n, u32 seed, u32 lane) {
    u32 v = ck_xxh32_acc0(lane & 3u, seed);
    if (n >= 16 && lane < 4)
        for (u32 s = 0; s + 16 <= n; s += 16) v = ck_xxh_rotl(v + ck_lz_le32(p + s + 4 * lane) * CK_XXH_P2, 13) * CK_XXH_P1;
    u32 v0 = __shfl_sync(0xffffffffu, v, 0), v1 = __shfl_sync(0xffffffffu, v, 1), v2 = __shfl_sync(0xffffffffu, v, 2), v3 = __shfl_sync(0xffffffffu, v, 3);
    u32 h = n >= 16 ? ck_xxh_rotl(v0, 1) + ck_xxh_rotl(v1, 7) + ck_xxh_rotl(v2, 12) + ck_xxh_rotl(v3, 18) : seed + CK_XXH_P5;
    return ck_xxh32_tail(h + n, p, n);
}

// frame descriptor: magic | FLG | BD | [content size u64 LE] | [dictionary id u32 LE] | HC
struct ck_lz_desc {
    u32 hdr_len;                       // bytes up to and including HC
    u32 block_max;                     // BD's block maximum: 64 KB, 256 KB, 1 MB or 4 MB
    bool linked, block_sum, content_sum, has_size;
    unsigned long long content_size;
};
// the descriptor of the frame p[0, n): false when it is not one this decoder takes (bad magic, version, reserved bits,
// block maximum or HC, a dictionary id — Kafka never sets one — or a frame that ends inside its descriptor)
CK_HD bool ck_lz_parse_desc(const u8* p, unsigned long long n, ck_lz_desc& d) {
    if (n < 7 || ck_lz_le32(p) != CK_LZ_MAGIC) return false;
    u32 flg = p[4], bd = p[5];
    if ((flg >> 6) != 1u || (flg & 2u) || (flg & 1u) || (bd & 0x8Fu)) return false;
    u32 id = (bd >> 4) & 7u;
    if (id < 4) return false;
    d.block_max = 1u << (2 * id + 8);                          // 4: 64 KB, 5: 256 KB, 6: 1 MB, 7: 4 MB
    d.linked = !(flg & 0x20u); d.block_sum = (flg & 0x10u) != 0; d.has_size = (flg & 8u) != 0; d.content_sum = (flg & 4u) != 0;
    u32 pos = 6;
    d.content_size = 0;
    if (d.has_size) {
        if (n < 15) return false;
        d.content_size = (unsigned long long)ck_lz_le32(p + 6) | ((unsigned long long)ck_lz_le32(p + 10) << 32);
        pos += 8;
    }
    if (pos >= n || p[pos] != ((ck_xxh32(p + 4, pos - 4, 0) >> 8) & 0xFFu)) return false;
    d.hdr_len = pos + 1;
    return true;
}
// the block chain of the frame p[0, n) after its descriptor: every size word to the end mark, block checksums and the
// content checksum stepped over, and nothing after them.  *nblocks = blocks, *bound = the most the blocks decode to (the
// block maximum per compressed block, the size of a stored block; at most the content size when the frame states it).
// false: the chain leaves the frame, a block is larger than the block maximum, or bytes follow the frame
CK_HD bool ck_lz_walk(const u8* p, unsigned long long n, const ck_lz_desc& d, u32* nblocks, unsigned long long* bound) {
    unsigned long long pos = d.hdr_len, b = 0;
    u32 k = 0;
    for (;;) {
        if (pos + 4 > n) return false;
        u32 w = ck_lz_le32(p + pos);
        pos += 4;
        if (!w) break;
        u32 sz = w & 0x7FFFFFFFu;
        if (sz > d.block_max) return false;
        pos += sz + (d.block_sum ? 4u : 0u);
        if (pos > n) return false;
        b += (w >> 31) ? sz : d.block_max;
        k++;
    }
    if (d.content_sum) pos += 4;
    if (pos != n) return false;
    if (d.has_size && d.content_size < b) b = d.content_size;
    *nblocks = k; *bound = b;
    return true;
}

// LZ4 length continuation: 255 ... 255, last (< 255).  Every lane reads the same bytes; false when the block ends inside it
__device__ __forceinline__ bool ck_lz_get_len(const u8* __restrict__ src, u32& ip, u32 n, unsigned long long& len) {
    for (;;) {
        if (ip >= n) return false;
        u32 b = src[ip++];
        len += b;
        if (b != 255u) return true;
    }
}
// One LZ4 block src[0, n) decoded by one warp into out[op, ...): out holds the frame's output so far, and a match may
// reach back to out[lo] (lo = 0 for linked blocks, op for an independent block).  The block decodes to at most block_max
// bytes and out to at most cap.  Every lane parses the same sequences; the warp copies the literals and the match of each.
// A match copies out[pos - off + (i mod off)]: bytes that lie before it, so overlapping matches need no ordering.
// Returns the decoded size, or -1 for a malformed block: a missing literals-only last sequence, lengths or literals past
// the block, offset 0 or reaching before out[lo], output past block_max or cap, or a last match nearer than 12 bytes to
// the end of the block (or ending inside its last 5 bytes)
__device__ __forceinline__ long long ck_lz4_decode_block(const u8* __restrict__ src, u32 n, u8* __restrict__ out,
                                                         unsigned long long op, unsigned long long lo, unsigned long long cap,
                                                         u32 block_max, u32 lane) {
    const unsigned long long start = op, lim = min(cap, start + block_max);
    unsigned long long m_start = ~0ull, m_end = 0;             // the last match, relative to the block
    u32 ip = 0;
    for (;;) {
        if (ip >= n) return -1;
        u32 token = src[ip++];
        unsigned long long ll = token >> 4;
        if (ll == 15u && !ck_lz_get_len(src, ip, n, ll)) return -1;
        if (ll > n - ip || op + ll > lim) return -1;
        for (u32 i = lane; i < ll; i += 32) out[op + i] = src[ip + i];
        ip += (u32)ll; op += ll;
        if (ip == n) break;                                    // the last sequence: literals only
        if (ip + 2 > n) return -1;
        u32 off = src[ip] | ((u32)src[ip + 1] << 8);
        ip += 2;
        unsigned long long ml = token & 15u;
        if (ml == 15u && !ck_lz_get_len(src, ip, n, ml)) return -1;
        ml += 4;
        if (off == 0 || off > op - lo || op + ml > lim) return -1;
        __syncwarp();                                          // the literals (and earlier matches) before they are read
        const u8* m = out + (op - off);
        for (u32 i = lane; i < ml; i += 32) out[op + i] = m[i % off];
        m_start = op - start; op += ml; m_end = op - start;
        __syncwarp();
    }
    __syncwarp();
    unsigned long long len = op - start;
    if (m_start != ~0ull && (m_start + 12 > len || m_end + 5 > len)) return -1;
    return (long long)len;
}

#endif  // CK_LZ4_CUH
