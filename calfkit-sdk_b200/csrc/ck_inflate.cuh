// gzip members (RFC 1952) and DEFLATE (RFC 1951) inflated by one warp, for the gzip batches of fetch responses
// (ck_rb_gzip_kernel, ck_kafka.cuh).  The one parse of both formats.  Depends on nothing else of the device code, and
// compiles with g++ as well (one "lane", no warp): the header parse and the trailer read are __host__ __device__, because
// the host sizes each batch's slot from them (ck_submit_recordbatch), and the inflate core is the same source on both
// sides, so that the CPU suite holds it against zlib (tests/test_inflate_hostsim.py).  The only device-specific parts are
// the warp-strided loops and __syncwarp.
//
// What is accepted is exactly what zlib 1.3's inflate accepts for one gzip member, and nothing else: reserved FLG bits,
// a wrong FHCRC, BTYPE 3, stored LEN != ~NLEN, more than 286 litlen or 30 distance codes, over-subscribed code sets and
// incomplete ones (except one code of one bit, for litlen and distances, or no distance code at all), a repeat code 16
// with no length before it, repeats past HLIT + HDIST, no end-of-block code, litlen symbols 286 / 287, distance
// symbols 30 / 31, a distance reaching before the member's output and a stream that ends early are refused.  Every input
// read is checked against the stream's end and every output write against the output's capacity: the members are
// outside input.
#ifndef CK_INFLATE_CUH
#define CK_INFLATE_CUH

#include <stdint.h>
typedef uint8_t u8;
typedef uint32_t u32;

#ifdef __CUDACC__
#define CK_GZ_HD __host__ __device__ __forceinline__
#define CK_GZ_DEV __device__ __forceinline__
#define CK_GZ_LANES 32u
#else
#define CK_GZ_HD inline
#define CK_GZ_DEV inline
#define CK_GZ_LANES 1u
#endif
#ifdef __CUDA_ARCH__
#define CK_GZ_SYNC() __syncwarp()
#else
#define CK_GZ_SYNC() ((void)0)
#endif

// Huffman tables (zlib's `enough`: 852 entries for 286 litlen codes with a 9-bit root, 592 for 30 distance codes with a
// 6-bit root, both up to 15 bits), a root table then the second-level tables behind it.  An entry is
//   symbol << 16 | code length          a symbol (length 1 - 15: the bits it takes, root bits included)
//   offset << 16 | 0x100 | sub bits     a link to the second-level table at `offset` indexed by the next `sub bits` bits
//   0                                   no code: refused when read
#define CK_GZ_ENOUGH_L 852u
#define CK_GZ_ENOUGH_D 592u
#define CK_GZ_ROOT_L 9u
#define CK_GZ_ROOT_D 6u
#define CK_GZ_ROOT_C 7u              // the code-length code: 19 symbols of up to 7 bits, root only
// a warp's workspace in shared memory (7.0 KB)
struct ck_gz_ws {
    u32 lit[CK_GZ_ENOUGH_L];
    u32 dist[CK_GZ_ENOUGH_D];       // its first 128 entries hold the code-length code's table while the lengths are read
    u32 cnt[16], first[16], offs[16], glo[16], gn[16], gs[16];   // per code length, of the table being built
    uint16_t sorted[320];           // symbols by (code length, symbol)
    u8 lens[320];                   // HLIT litlen then HDIST distance code lengths
    u8 cll[20];                     // the code-length code's lengths
};

// the order the code-length code's lengths come in
#ifdef __CUDACC__
__constant__
#else
static const
#endif
u8 ck_gz_order[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};

CK_GZ_HD u32 ck_gz_le16(const u8* p) { return (u32)p[0] | ((u32)p[1] << 8); }
CK_GZ_HD u32 ck_gz_le32(const u8* p) { return (u32)p[0] | ((u32)p[1] << 8) | ((u32)p[2] << 16) | ((u32)p[3] << 24); }
// CRC32 (IEEE, reflected 0xEDB88320) of a few header bytes, bit by bit: the FHCRC check only
CK_GZ_HD u32 ck_gz_crc32_bytes(const u8* p, unsigned long long n) {
    u32 c = 0xffffffffu;
    for (unsigned long long i = 0; i < n; i++) {
        c ^= p[i];
        for (int k = 0; k < 8; k++) c = (c >> 1) ^ ((c & 1u) ? 0xEDB88320u : 0u);
    }
    return ~c;
}

// The gzip member p[0, n): ID1 ID2 = 1f 8b, CM = 8, no reserved FLG bit; FEXTRA, FNAME and FCOMMENT stepped over, FHCRC
// checked, every scan bounded by n.  *hdr = where the deflate stream starts, *isize = the trailer's ISIZE.  false: not a
// member this decoder takes, one shorter than its header + the 8-byte trailer, or an ISIZE that the deflate bytes between
// them cannot produce (at most 1032 bytes per byte: a 258-byte match in two bits)
CK_GZ_HD bool ck_gz_member(const u8* p, unsigned long long n, u32* hdr, u32* isize) {
    if (n < 18 || p[0] != 0x1f || p[1] != 0x8b || p[2] != 8 || (p[3] & 0xe0)) return false;
    u32 flg = p[3];
    unsigned long long pos = 10;
    if (flg & 4) {                                             // FEXTRA
        if (pos + 2 > n) return false;
        pos += 2 + ck_gz_le16(p + pos);
    }
    if (flg & 8) {                                             // FNAME
        while (pos < n && p[pos]) pos++;
        if (pos >= n) return false;
        pos++;
    }
    if (flg & 16) {                                            // FCOMMENT
        while (pos < n && p[pos]) pos++;
        if (pos >= n) return false;
        pos++;
    }
    if (flg & 2) {                                             // FHCRC: the low 16 bits of the CRC32 of the header so far
        if (pos + 2 > n || ck_gz_le16(p + pos) != (ck_gz_crc32_bytes(p, pos) & 0xffffu)) return false;
        pos += 2;
    }
    if (pos + 8 > n) return false;
    u32 sz = ck_gz_le32(p + n - 4);
    if ((unsigned long long)sz > 1032ull * (n - 8 - pos)) return false;
    *hdr = (u32)pos; *isize = sz;
    return true;
}

CK_GZ_DEV u32 ck_gz_rev(u32 x, u32 n) {                       // the low n (1 - 15) bits of x, reversed
#ifdef __CUDA_ARCH__
    return __brev(x) >> (32u - n);
#else
    u32 r = 0;
    for (u32 i = 0; i < n; i++) r |= ((x >> i) & 1u) << (n - 1u - i);
    return r;
#endif
}

// The canonical code of lens[0, n) as a table at tab (root bits `root`), built by the warp.  kind 0: the code-length code,
// 1: litlen, 2: distances — what zlib's inflate_table accepts for each: no over-subscribed set; an incomplete one only
// for litlen / distances with one code of one bit, or distances with no code at all (refused if a distance is read).
// Every lane returns the same verdict
CK_GZ_DEV bool ck_gz_build(ck_gz_ws& ws, const u8* lens, u32 n, u32* tab, u32 root, u32 cap, u32 kind, u32 lane) {
    for (u32 L = lane + 1; L < 16; L += CK_GZ_LANES) {
        u32 c = 0;
        for (u32 s = 0; s < n; s++) c += lens[s] == L;
        ws.cnt[L] = c;
    }
    CK_GZ_SYNC();
    int left = 1;
    u32 maxl = 0;
    for (u32 L = 1; L < 16; L++) {
        left = 2 * left - (int)ws.cnt[L];
        if (left < 0) return false;                            // over-subscribed
        if (ws.cnt[L]) maxl = L;
    }
    if (left > 0 && !(kind != 0 && maxl == 1) && !(kind == 2 && maxl == 0)) return false;
    // first code and first sorted slot of every length; for the lengths past the root, the root prefixes whose longest
    // code has that length: glo[L] .. glo[L] + gn[L], each a second-level table of 2^(L - root) entries from gs[L] on
    if (lane == 0) {
        u32 c = 0, o = 0;
        for (u32 L = 1; L < 16; L++) { ws.first[L] = c; ws.offs[L] = o; o += ws.cnt[L]; c = (c + ws.cnt[L]) << 1; }
        u32 S = 1u << root;
        for (u32 L = root + 1; L < 16; L++) {
            ws.glo[L] = 0; ws.gn[L] = 0; ws.gs[L] = S;
            if (!ws.cnt[L]) continue;
            u32 a = ws.first[L] >> (L - root), b = ((ws.first[L] + ws.cnt[L] - 1u) >> (L - root)) + 1u;
            for (u32 M = L + 1; M < 16; M++)                   // a longer code under the last prefix takes it over
                if (ws.cnt[M]) { if ((ws.first[M] >> (M - root)) + 1u == b) b--; break; }
            ws.glo[L] = a; ws.gn[L] = b > a ? b - a : 0u;
            S += ws.gn[L] << (L - root);
        }
        ws.gs[0] = S;                                          // the table's size
    }
    CK_GZ_SYNC();
    for (u32 L = lane + 1; L < 16; L += CK_GZ_LANES) {
        u32 o = ws.offs[L];
        for (u32 s = 0; s < n; s++) if (lens[s] == L) ws.sorted[o++] = (uint16_t)s;
    }
    const u32 total = ws.gs[0];
    CK_GZ_SYNC();
    if (total > cap) return false;                             // not for a set the checks above let through
    for (u32 k = lane; k < total; k += CK_GZ_LANES) {
        u32 e = 0;
        if (k < (1u << root)) {
            u32 c = ck_gz_rev(k, root);                        // the root bits as a code prefix, first bit highest
            for (u32 L = 1; L <= root && L < 16; L++) {
                u32 v = (c >> (root - L)) - ws.first[L];
                if (v < ws.cnt[L]) { e = ((u32)ws.sorted[ws.offs[L] + v] << 16) | L; break; }
            }
            if (!e)
                for (u32 L = root + 1; L < 16; L++)
                    if (c - ws.glo[L] < ws.gn[L]) { e = ((ws.gs[L] + ((c - ws.glo[L]) << (L - root))) << 16) | 0x100u | (L - root); break; }
        } else {
            u32 L = root + 1;
            while (L < 15 && k >= ws.gs[L] + (ws.gn[L] << (L - root))) L++;
            u32 sb = L - root, q = k - ws.gs[L];
            u32 c = ((ws.glo[L] + (q >> sb)) << sb) | ck_gz_rev(q & ((1u << sb) - 1u), sb);   // root + sb bits
            for (u32 M = root + 1; M <= L; M++) {
                u32 v = (c >> (L - M)) - ws.first[M];
                if (v < ws.cnt[M]) { e = ((u32)ws.sorted[ws.offs[M] + v] << 16) | M; break; }
            }
        }
        tab[k] = e;
    }
    CK_GZ_SYNC();
    return true;
}

// the bit stream: bits taken from the low end of bb, refilled a byte at a time up to the stream's end.  Bits past the end
// read as 0 and are never taken: a code or field that needs them is a stream that ends early
struct ck_gz_bits {
    const u8* p;
    unsigned long long ip, n, bb;
    u32 bn;
};
CK_GZ_DEV void ck_gz_fill(ck_gz_bits& s) {
    while (s.bn <= 56 && s.ip < s.n) { s.bb |= (unsigned long long)s.p[s.ip++] << s.bn; s.bn += 8; }
}
// take k (<= 32) bits; false when fewer are left
CK_GZ_DEV bool ck_gz_take(ck_gz_bits& s, u32 k, u32& v) {
    if (k > s.bn) return false;
    v = (u32)s.bb & ((1u << k) - 1u);
    s.bb >>= k; s.bn -= k;
    return true;
}
// one symbol of the table tab (root bits `root`); -1: no such code, or the stream ends inside it
CK_GZ_DEV int ck_gz_sym(ck_gz_bits& s, const u32* tab, u32 root) {
    u32 e = tab[(u32)s.bb & ((1u << root) - 1u)];
    if (e & 0x100u) e = tab[(e >> 16) + ((u32)(s.bb >> root) & ((1u << (e & 0xffu)) - 1u))];
    u32 len = e & 0xffu;
    if (!len || len > s.bn) return -1;
    s.bb >>= len; s.bn -= len;
    return (int)(e >> 16);
}

// The raw deflate stream src[0, n) inflated by one warp into out[0, cap): every lane parses the same bits; lane 0 writes
// literals, the warp copies stored blocks and matches (a match copies out[pos - dist + (i mod dist)], bytes that lie
// before it, so overlapping matches need no ordering).  *used = the bytes the stream took, through the final block's
// last byte.  Returns the inflated length, or -1 for a stream zlib refuses, that ends early, or that overruns cap
CK_GZ_DEV long long ck_inflate(const u8* src, unsigned long long n, u8* out, unsigned long long cap, ck_gz_ws& ws, u32 lane,
                               unsigned long long* used) {
    ck_gz_bits s = {src, 0, n, 0, 0};
    unsigned long long op = 0;
    u32 v, fin;
    do {
        ck_gz_fill(s);
        if (!ck_gz_take(s, 1, fin) || !ck_gz_take(s, 2, v)) return -1;
        if (v == 3) return -1;                                 // BTYPE 3
        if (v == 0) {                                          // stored: LEN, NLEN on the next byte boundary, then LEN bytes
            s.bb = 0; s.ip -= s.bn >> 3; s.bn = 0;
            if (s.ip + 4 > n) return -1;
            u32 len = ck_gz_le16(src + s.ip);
            if (len != (~ck_gz_le16(src + s.ip + 2) & 0xffffu)) return -1;
            s.ip += 4;
            if (len > n - s.ip || len > cap - op) return -1;
            for (u32 i = lane; i < len; i += CK_GZ_LANES) out[op + i] = src[s.ip + i];
            s.ip += len; op += len;
            continue;
        }
        CK_GZ_SYNC();                                          // every lane done with the tables of the block before
        u32 nlen = 288, ndist = 32;
        if (v == 1) {                                          // fixed codes: 0-143 8 bits, 144-255 9, 256-279 7, 280-287 8; 5-bit distances
            for (u32 i = lane; i < 320; i += CK_GZ_LANES)
                ws.lens[i] = i < 144 ? 8 : i < 256 ? 9 : i < 280 ? 7 : i < 288 ? 8 : 5;
        } else {                                               // dynamic: HLIT, HDIST, HCLEN, the code-length code, the lengths
            u32 hl, hd, hc;
            if (!ck_gz_take(s, 5, hl) || !ck_gz_take(s, 5, hd) || !ck_gz_take(s, 4, hc)) return -1;
            nlen = hl + 257; ndist = hd + 1;
            if (nlen > 286 || ndist > 30) return -1;
            if (lane == 0) for (u32 i = 0; i < 19; i++) ws.cll[i] = 0;
            CK_GZ_SYNC();
            for (u32 i = 0; i < hc + 4; i++) {
                if (!(i & 15)) ck_gz_fill(s);
                if (!ck_gz_take(s, 3, v)) return -1;
                if (lane == 0) ws.cll[ck_gz_order[i]] = (u8)v;
            }
            CK_GZ_SYNC();
            if (!ck_gz_build(ws, ws.cll, 19, ws.dist, CK_GZ_ROOT_C, 1u << CK_GZ_ROOT_C, 0, lane)) return -1;
            u32 have = 0, prev = 0;
            while (have < nlen + ndist) {
                ck_gz_fill(s);
                int sym = ck_gz_sym(s, ws.dist, CK_GZ_ROOT_C);
                if (sym < 0) return -1;
                u32 rep = 1, val = (u32)sym;
                if (sym == 16) {                               // the previous length 3 - 6 times
                    if (!have || !ck_gz_take(s, 2, rep)) return -1;
                    rep += 3; val = prev;
                } else if (sym == 17) {                        // 0, 3 - 10 times
                    if (!ck_gz_take(s, 3, rep)) return -1;
                    rep += 3; val = 0;
                } else if (sym == 18) {                        // 0, 11 - 138 times
                    if (!ck_gz_take(s, 7, rep)) return -1;
                    rep += 11; val = 0;
                }
                if (have + rep > nlen + ndist) return -1;
                if (lane == 0) for (u32 i = 0; i < rep; i++) ws.lens[have + i] = (u8)val;
                have += rep; prev = val;
            }
            CK_GZ_SYNC();
            if (!ws.lens[256]) return -1;                      // no end-of-block code
        }
        CK_GZ_SYNC();
        if (!ck_gz_build(ws, ws.lens, nlen, ws.lit, CK_GZ_ROOT_L, CK_GZ_ENOUGH_L, 1, lane) ||
            !ck_gz_build(ws, ws.lens + nlen, ndist, ws.dist, CK_GZ_ROOT_D, CK_GZ_ENOUGH_D, 2, lane)) return -1;
        for (;;) {                                             // 15 + 5 + 15 + 13 bits at most per symbol: one refill
            ck_gz_fill(s);
            int sym = ck_gz_sym(s, ws.lit, CK_GZ_ROOT_L);
            if (sym < 0) return -1;
            if (sym < 256) {
                if (op >= cap) return -1;
                if (lane == 0) out[op] = (u8)sym;
                op++;
                continue;
            }
            if (sym == 256) break;
            u32 ls = (u32)sym - 257u;
            if (ls > 28) return -1;                            // 286, 287
            u32 len, x, dist;
            if (ls < 8) len = 3 + ls;
            else if (ls == 28) len = 258;
            else {
                u32 eb = (ls >> 2) - 1u;
                if (!ck_gz_take(s, eb, x)) return -1;
                len = ((4u + (ls & 3u)) << eb) + 3u + x;
            }
            int ds = ck_gz_sym(s, ws.dist, CK_GZ_ROOT_D);
            if (ds < 0 || ds > 29) return -1;                  // no code, 30, 31
            if (ds < 4) dist = (u32)ds + 1u;
            else {
                u32 eb = ((u32)ds >> 1) - 1u;
                if (!ck_gz_take(s, eb, x)) return -1;
                dist = ((2u + ((u32)ds & 1u)) << eb) + 1u + x;
            }
            if (dist > op || len > cap - op) return -1;        // before the member's output / past the output
            CK_GZ_SYNC();                                      // the literals (and earlier matches) before they are read
            const u8* m = out + (op - dist);
            if (dist >= len) for (u32 i = lane; i < len; i += CK_GZ_LANES) out[op + i] = m[i];
            else for (u32 i = lane; i < len; i += CK_GZ_LANES) out[op + i] = m[i % dist];
            op += len;
            CK_GZ_SYNC();
        }
    } while (!fin);
    CK_GZ_SYNC();
    *used = s.ip - (s.bn >> 3);                                // the final block's partial byte counts, its spare bits are dropped
    return (long long)op;
}

// The gzip member z[0, zn) inflated into out[0, cap) with cap = its ISIZE: the header (ck_gz_member), the deflate stream,
// and its trailer, which must start right behind the stream's final block and end exactly at zn — anything after it,
// a second member included, is refused.  Returns the inflated length (= ISIZE), or -1.  The trailer's CRC32 of the
// output is the caller's to check (the device folds it over the warp, ck_kafka.cuh)
CK_GZ_DEV long long ck_gz_decode(const u8* z, unsigned long long zn, u8* out, unsigned long long cap, ck_gz_ws& ws, u32 lane) {
    u32 hdr, isize;
    if (!ck_gz_member(z, zn, &hdr, &isize) || isize != cap) return -1;
    unsigned long long m = zn - 8 - hdr, used = 0;
    long long r = ck_inflate(z + hdr, m, out, cap, ws, lane, &used);
    return r >= 0 && (unsigned long long)r == cap && used == m ? r : -1;
}

#endif  // CK_INFLATE_CUH
