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

// One LZ4 block of src[0, len), len <= 64 KB, compressed by one warp into dst (at most len - 1 bytes are written).  Returns
// the compressed size, or 0 when it would not be smaller than len (the caller stores the block raw).
// Greedy parse: the warp looks at the 32 positions p .. p+31 at once; each lane hashes its 4 bytes and takes the table's
// last position with that hash (inserted by an earlier round, so it lies before p) as its candidate.  The first lane whose
// candidate matches starts the match; positions up to it enter the table (one writer per hash: the highest position),
// the match is extended 128 bytes per round, and the literals before it and the match are written.  Every step is a
// fixed function of the input: the output is deterministic.
// Block rules a decoder enforces: a match starts at most len - 12, ends at most len - 5 (the last 5 bytes are literals),
// the last sequence holds literals only, offsets are 1 .. 65535 (a block holds at most 65536 positions)
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
        u32 maxlen = len - 5u - ms, ml = 4;
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
        ml = min(ml, maxlen);
        u32 ll = ms - anchor;
        if (op + 3u + ck_lz_len_bytes(ll) + ll + ck_lz_len_bytes(ml - 4u) > cap) return 0;
        op += ck_lz_put_seq(dst + op, src + anchor, ll, ms - mc, ml, lane);
        anchor = p = ms + ml;
    }
    u32 ll = len - anchor;
    if (op + 1u + ck_lz_len_bytes(ll) + ll > cap) return 0;
    op += ck_lz_put_seq(dst + op, src + anchor, ll, 0, 0, lane);
    return op;
}

#endif  // CK_LZ4_CUH
