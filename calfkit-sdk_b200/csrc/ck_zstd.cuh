// zstd frames (RFC 8878) decoded by one warp, for the zstd batches of fetch responses (ck_rb_zstd_kernel, ck_kafka.cuh).
// The one parse of the format.  Depends on nothing else of the device code, and compiles with g++ as well (one "lane", no
// warp): the frame header parse and the block walk are __host__ __device__, because the host sizes each batch's slot from
// them (ck_submit_recordbatch), and the decode core is the same source on both sides, so that the CPU suite holds it
// against libzstd (tests/test_zstd_hostsim.py).  The only device-specific parts are the warp-strided loops, __syncwarp and
// the lane broadcasts.
//
// What is accepted is exactly what libzstd 1.5.5 accepts for one frame through a DCtx with default parameters, with two
// declared exceptions, both refused: a section holding more than one frame (a second frame, or a skippable frame) and
// anything after the frame.  So, as libzstd's default windowLogMax does, a window above 2^27 + 1 bytes is refused; every
// block must fit Block_Maximum_Size = min(window, 128 KiB) (an RLE block counts its one input byte and its output);
// Dictionary_ID must be 0 (Kafka has no dictionaries); Frame_Content_Size and the XXH64 content checksum are checked when
// the frame carries them.  Inside compressed blocks, every entropy stage decides as libzstd 1.5.5 does: the normalized
// count reader, the Huffman weights (direct or FSE, tables up to 12 bits), the 1- and 4-stream Huffman literals, which must
// end exactly, and the backward bit container of the sequences, which libzstd reads as a 64-bit register that wraps when
// overread, and which passes when the stream is consumed at least to its start.  Repeat offsets, the Huffman table and the
// three sequence tables carry across the blocks of a frame; Treeless literals and Repeat modes need an earlier table.  A
// match may reach back to the frame's first byte and no further.  Every input read is checked against the section and
// every output write against the slot: the sections are outside input.
//
// Literals.  Raw literals are read where they lie in the section.  RLE and Huffman literals are decoded into the tail of
// the block's own reservation in the slot: block k reserves [R_k, R_k + B_k) where B_k is its walk bound (raw / RLE: its
// size, compressed: Block_Maximum_Size) and R_k the sum of the bounds before it, and its L literals go to
// [R_k + B_k - L, R_k + B_k), as libzstd decodes literals into dst.  The block's output starts at op <= R_k (no block
// outputs more than its bound).  When the sequences have consumed c literals and written m match bytes, the next write
// lands at op + c + m and the next unread literal lies at R_k + B_k - L + c: the write stays below it while m + L <= B_k.
// The decoder refuses a match before writing it unless (block output so far) + match + (literals not yet consumed) <= B_k,
// i.e. m + L <= B_k after it, which a block libzstd accepts satisfies (all its literals and matches are output, and its
// output is at most Block_Maximum_Size).  So a copy never overtakes an unread literal; a literal run that overlaps its
// own destination is read into registers before it is written.
#ifndef CK_ZSTD_CUH
#define CK_ZSTD_CUH

#include <stdint.h>
typedef uint8_t u8;
typedef uint32_t u32;
typedef unsigned long long ck_zu64;

#ifdef __CUDACC__
#define CK_ZS_HD __host__ __device__ __forceinline__
#define CK_ZS_DEV __device__ __forceinline__
#define CK_ZS_LANES 32u
#else
#define CK_ZS_HD inline
#define CK_ZS_DEV inline
#define CK_ZS_LANES 1u
#endif
#ifdef __CUDA_ARCH__
#define CK_ZS_SYNC() __syncwarp()
#define CK_ZS_BC(x) __shfl_sync(0xffffffffu, (x), 0)
#define CK_ZS_ALL(x) __all_sync(0xffffffffu, (x))
#else
#define CK_ZS_SYNC() ((void)0)
#define CK_ZS_BC(x) (x)
#define CK_ZS_ALL(x) (x)
#endif

#define CK_ZS_MAGIC 0xFD2FB528u
#define CK_ZS_BLOCK_MAX (128u << 10)
#define CK_ZS_WINDOW_MAX ((1ull << 27) + 1ull)   // libzstd's default maxWindowSize (ZSTD_d_windowLogMax 27)
#define CK_ZS_HUF_LOG 12u                        // the largest Huffman table libzstd builds (HUF_TABLELOG_MAX)

// a sequence table entry: the state's symbol (a code of its alphabet), the bits of its state update and the base of it
struct ck_zs_fse { uint16_t next; u8 nb; u8 sym; };

// a warp's workspace in shared memory (14.6 KB): the frame's Huffman table and its three sequence tables, which later
// blocks may repeat, and the scratch their descriptions are read into
struct ck_zs_ws {
    uint16_t huf[1u << CK_ZS_HUF_LOG];   // symbol | bits << 8, indexed by the next `hlog` bits of a stream
    ck_zs_fse ll[512], ml[512], of[256]; // literal length (log <= 9), match length (<= 9), offset (<= 8) codes
    ck_zs_fse wt[64];                    // the FSE table of the Huffman weights (log <= 6)
    short norm[256];                     // a normalized count
    uint16_t next[256];                  // per symbol: its next state while a table is built / its first Huffman entry
    u8 w[257];                           // Huffman weights, the implied last one included
    u32 rank[16];                        // symbols per Huffman weight
};

CK_ZS_HD u32 ck_zs_le16(const u8* p) { return (u32)p[0] | ((u32)p[1] << 8); }
CK_ZS_HD u32 ck_zs_le24(const u8* p) { return (u32)p[0] | ((u32)p[1] << 8) | ((u32)p[2] << 16); }
CK_ZS_HD u32 ck_zs_le32(const u8* p) { return ck_zs_le24(p) | ((u32)p[3] << 24); }
CK_ZS_HD ck_zu64 ck_zs_le64(const u8* p) { return (ck_zu64)ck_zs_le32(p) | ((ck_zu64)ck_zs_le32(p + 4) << 32); }
CK_ZS_HD u32 ck_zs_hb(u32 x) {                // index of the highest set bit (x > 0)
#ifdef __CUDA_ARCH__
    return 31u - (u32)__clz(x);
#else
    return 31u - (u32)__builtin_clz(x);
#endif
}

// ---- frame header and block walk (host and device) -----------------------------------------------------------------
struct ck_zs_frame {
    u32 hdr;              // header bytes (magic included)
    u32 bmax;             // Block_Maximum_Size
    u32 checksum;         // the frame ends with the low 32 bits of XXH64(content)
    u32 has_fcs;          // fcs is known
    ck_zu64 fcs;          // Frame_Content_Size
};

// The frame header at p[0, n): magic, no reserved descriptor bit, no Dictionary_ID but 0, a window libzstd's default
// limit takes (the Frame_Content_Size when Single_Segment is set).  false: not such a header, or one longer than n
CK_ZS_HD bool ck_zs_header(const u8* p, ck_zu64 n, ck_zs_frame& f) {
    if (n < 5 || ck_zs_le32(p) != CK_ZS_MAGIC) return false;
    u32 fhd = p[4];
    if (fhd & 8u) return false;                                      // reserved bit
    u32 did = fhd & 3u, ss = (fhd >> 5) & 1u, fid = fhd >> 6;
    const u32 dsz = did == 3 ? 4u : did, fsz = fid ? 1u << fid : 0u;
    u32 h = 5 + !ss + dsz + fsz + (ss && !fid);
    if (n < h) return false;
    u32 pos = 5;
    ck_zu64 win = 0;
    if (!ss) {
        u32 wb = p[pos++];
        win = 1ull << ((wb >> 3) + 10);
        win += (win >> 3) * (wb & 7u);
    }
    u32 id = did == 1 ? p[pos] : did == 2 ? ck_zs_le16(p + pos) : did == 3 ? ck_zs_le32(p + pos) : 0u;
    if (id) return false;                                            // a dictionary
    pos += dsz;
    ck_zu64 fcs = ~0ull;
    if (fid == 0 && ss) fcs = p[pos];
    else if (fid == 1) fcs = ck_zs_le16(p + pos) + 256ull;
    else if (fid == 2) fcs = ck_zs_le32(p + pos);
    else if (fid == 3) fcs = ck_zs_le64(p + pos);                    // all ones: libzstd's "unknown"
    if (ss) win = fcs;
    if ((win > 1024 ? win : 1024) > CK_ZS_WINDOW_MAX) return false;
    f.hdr = h;
    f.bmax = (u32)(win < CK_ZS_BLOCK_MAX ? win : CK_ZS_BLOCK_MAX);
    f.checksum = (fhd >> 2) & 1u;
    f.has_fcs = fcs != ~0ull;
    f.fcs = fcs;
    return true;
}

// The blocks of the frame p[0, n) with header f: every 3-byte block header stepped over, block type 3 refused, every
// block within Block_Maximum_Size and inside n, the checksum after the last block, and the frame ending exactly at n.
// *bound = what the frame decodes to at most (raw and RLE blocks their size, compressed ones Block_Maximum_Size).  false
// also when a Frame_Content_Size is larger than that bound
CK_ZS_HD bool ck_zs_walk(const u8* p, ck_zu64 n, const ck_zs_frame& f, ck_zu64* bound) {
    ck_zu64 pos = f.hdr, b = 0;
    for (;;) {
        if (n - pos < 3) return false;
        u32 bh = ck_zs_le24(p + pos), type = (bh >> 1) & 3u, size = bh >> 3;
        pos += 3;
        if (type == 3) return false;
        u32 in = type == 1 ? 1u : size;
        if (in > f.bmax || (type == 1 && size > f.bmax) || in > n - pos) return false;
        b += type == 2 ? f.bmax : size;
        pos += in;
        if (bh & 1u) break;
    }
    if (f.checksum) {
        if (n - pos < 4) return false;
        pos += 4;
    }
    if (pos != n || (f.has_fcs && f.fcs > b)) return false;
    *bound = b;
    return true;
}

// ---- tables ---------------------------------------------------------------------------------------------------------
#ifdef __CUDACC__
#define CK_ZS_CONST __constant__
#else
#define CK_ZS_CONST static const
#endif
CK_ZS_CONST u32 ck_zs_ll_base[36] = {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16, 18, 20, 22, 24, 28, 32, 40,
                                     48, 64, 0x80, 0x100, 0x200, 0x400, 0x800, 0x1000, 0x2000, 0x4000, 0x8000, 0x10000};
CK_ZS_CONST u8 ck_zs_ll_bits[36] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 3, 3,
                                    4, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16};
CK_ZS_CONST u32 ck_zs_ml_base[53] = {3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16, 17, 18, 19, 20, 21, 22, 23, 24, 25, 26,
                                     27, 28, 29, 30, 31, 32, 33, 34, 35, 37, 39, 41, 43, 47, 51, 59, 67, 83, 99, 0x83, 0x103,
                                     0x203, 0x403, 0x803, 0x1003, 0x2003, 0x4003, 0x8003, 0x10003};
CK_ZS_CONST u8 ck_zs_ml_bits[53] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0,
                                    0, 0, 0, 1, 1, 1, 1, 2, 2, 3, 3, 4, 4, 5, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16};
// the predefined distributions (RFC 8878 3.1.1.3.2.2)
CK_ZS_CONST short ck_zs_ll_def[36] = {4, 3, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 1, 1, 1, 2, 2, 2, 2, 2, 2, 2, 2,
                                      2, 3, 2, 1, 1, 1, 1, 1, -1, -1, -1, -1};
CK_ZS_CONST short ck_zs_ml_def[53] = {1, 4, 3, 2, 2, 2, 2, 2, 2, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1,
                                      1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, -1, -1, -1, -1, -1, -1, -1};
CK_ZS_CONST short ck_zs_of_def[29] = {1, 1, 1, 1, 1, 1, 2, 2, 2, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, -1, -1, -1, -1, -1};

// four little-endian bytes at i of p[0, n), zero past n
CK_ZS_DEV u32 ck_zs_rdz(const u8* p, u32 n, u32 i) {
    u32 v = 0;
    for (u32 k = 0; k < 4; k++) if (i + k < n) v |= (u32)p[i + k] << (8 * k);
    return v;
}

// A normalized count p[0, n) (RFC 8878 4.1.1), read as libzstd's FSE_readNCount reads it, buffer-end handling included:
// norm[0, maxsv] and the accuracy log; maxsv in = the largest symbol the alphabet has, out = the last one present.
// Returns the bytes it took, or -1
CK_ZS_DEV int ck_zs_ncount(const u8* p, u32 n, short* norm, u32& maxsv, u32& log) {
    const u32 iend = n < 8 ? 8u : n;                             // a short header is read as if zero-padded to 8 bytes
    const u32 msv1 = maxsv + 1;
    for (u32 s = 0; s < msv1; s++) norm[s] = 0;
    u32 ip = 0, bs = ck_zs_rdz(p, n, 0);
    int nb = (int)(bs & 15u) + 5;
    if (nb > 15) return -1;
    bs >>= 4;
    int bc = 4;
    log = (u32)nb;
    int remaining = (1 << nb) + 1, threshold = 1 << nb;
    nb++;
    u32 charnum = 0;
    bool prev0 = false;
    for (;;) {
        if (prev0) {                                             // runs of zero-probability symbols, 2 bits a repeat
            u32 rep;
#ifdef __CUDA_ARCH__
            rep = (u32)(__ffs(~bs | 0x80000000u) - 1) >> 1;
#else
            rep = (u32)__builtin_ctz(~bs | 0x80000000u) >> 1;
#endif
            while (rep >= 12) {
                charnum += 36;
                if (ip + 7 <= iend) ip += 3;
                else { bc -= 8 * (int)(iend - 7 - ip); bc &= 31; ip = iend - 4; }
                bs = ck_zs_rdz(p, n, ip) >> bc;
#ifdef __CUDA_ARCH__
                rep = (u32)(__ffs(~bs | 0x80000000u) - 1) >> 1;
#else
                rep = (u32)__builtin_ctz(~bs | 0x80000000u) >> 1;
#endif
            }
            charnum += 3 * rep;
            bs >>= 2 * rep;
            bc += 2 * (int)rep;
            charnum += bs & 3u;
            bc += 2;
            if (charnum >= msv1) break;
            if (ip + 7 <= iend || ip + (u32)(bc >> 3) + 4 <= iend) { ip += (u32)(bc >> 3); bc &= 7; }
            else { bc -= 8 * (int)(iend - 4 - ip); bc &= 31; ip = iend - 4; }
            bs = ck_zs_rdz(p, n, ip) >> bc;
        }
        int mx = (2 * threshold - 1) - remaining, count;
        if ((int)(bs & (u32)(threshold - 1)) < mx) { count = (int)(bs & (u32)(threshold - 1)); bc += nb - 1; }
        else {
            count = (int)(bs & (u32)(2 * threshold - 1));
            if (count >= threshold) count -= mx;
            bc += nb;
        }
        count--;
        remaining -= count < 0 ? -count : count;
        norm[charnum++] = (short)count;
        prev0 = !count;
        if (remaining < threshold) {
            if (remaining <= 1) break;
            nb = (int)ck_zs_hb((u32)remaining) + 1;
            threshold = 1 << (nb - 1);
        }
        if (charnum >= msv1) break;
        if (ip + 7 <= iend || ip + (u32)(bc >> 3) + 4 <= iend) { ip += (u32)(bc >> 3); bc &= 7; }
        else { bc -= 8 * (int)(iend - 4 - ip); bc &= 31; ip = iend - 4; }
        bs = ck_zs_rdz(p, n, ip) >> bc;
    }
    if (remaining != 1 || charnum > msv1 || bc > 32) return -1;
    maxsv = charnum - 1;
    ip += (u32)(bc + 7) >> 3;
    if (ip > n) return -1;                                       // (only a short header can end past n)
    return (int)ip;
}

// the decoding table of norm[0, maxsv] at accuracy `log` (each symbol's cells spread, low-probability ones from the top)
CK_ZS_DEV void ck_zs_fse_build(ck_zs_fse* t, const short* norm, u32 maxsv, u32 log, uint16_t* next) {
    const u32 size = 1u << log, mask = size - 1, step = (size >> 1) + (size >> 3) + 3;
    u32 high = size - 1;
    for (u32 s = 0; s <= maxsv; s++) {
        if (norm[s] == -1) { t[high--].sym = (u8)s; next[s] = 1; }
        else next[s] = (uint16_t)norm[s];
    }
    u32 pos = 0;
    for (u32 s = 0; s <= maxsv; s++)
        for (int i = 0; i < norm[s]; i++) {
            t[pos].sym = (u8)s;
            do pos = (pos + step) & mask; while (pos > high);
        }
    for (u32 u = 0; u < size; u++) {
        u32 nx = next[t[u].sym]++;
        u32 nb = log - ck_zs_hb(nx);
        t[u].nb = (u8)nb;
        t[u].next = (uint16_t)((nx << nb) - size);
    }
}

// ---- the backward bit container, as libzstd reads it ------------------------------------------------------------------
// A 64-bit register over p[0, n) loaded from the end: `used` bits of it are consumed from the top; reloads step back a
// whole number of bytes.  Reading past the stream's start is not checked here: the register wraps (as libzstd's does) and
// the callers decide from `used` and the reload status whether that is a refusal
struct ck_zs_br { const u8* p; u32 ptr; u32 used; ck_zu64 c; };
#define CK_ZS_UNFINISHED 0
#define CK_ZS_END_OF_BUFFER 1
#define CK_ZS_COMPLETED 2
#define CK_ZS_OVERFLOW 3
CK_ZS_DEV bool ck_zs_br_init(ck_zs_br& b, const u8* p, u32 n) {
    if (n < 1 || !p[n - 1]) return false;                         // empty, or no end mark
    b.p = p;
    u32 last = p[n - 1];
    if (n >= 8) { b.ptr = n - 8; b.c = ck_zs_le64(p + b.ptr); b.used = 8 - ck_zs_hb(last); }
    else {
        b.ptr = 0; b.c = 0;
        for (u32 k = 0; k < n; k++) b.c |= (ck_zu64)p[k] << (8 * k);
        b.used = 8 - ck_zs_hb(last) + (8 - n) * 8;
    }
    return true;
}
CK_ZS_DEV u32 ck_zs_look(const ck_zs_br& b, u32 nb) {           // BIT_lookBits (nb <= 31; 0 gives 0)
    return (u32)((b.c >> ((64u - b.used - nb) & 63u)) & ((1ull << nb) - 1ull));
}
CK_ZS_DEV u32 ck_zs_look_fast(const ck_zs_br& b, u32 nb) {      // BIT_lookBitsFast (nb >= 1)
    return (u32)((b.c << (b.used & 63u)) >> ((64u - nb) & 63u));
}
CK_ZS_DEV u32 ck_zs_read(ck_zs_br& b, u32 nb) { u32 v = ck_zs_look(b, nb); b.used += nb; return v; }
CK_ZS_DEV u32 ck_zs_read_fast(ck_zs_br& b, u32 nb) { u32 v = ck_zs_look_fast(b, nb); b.used += nb; return v; }
CK_ZS_DEV int ck_zs_reload(ck_zs_br& b) {
    if (b.used > 64) return CK_ZS_OVERFLOW;
    if (b.ptr >= 8) { b.ptr -= b.used >> 3; b.used &= 7; b.c = ck_zs_le64(b.p + b.ptr); return CK_ZS_UNFINISHED; }
    if (b.ptr == 0) return b.used < 64 ? CK_ZS_END_OF_BUFFER : CK_ZS_COMPLETED;
    u32 nbytes = b.used >> 3;
    int r = CK_ZS_UNFINISHED;
    if (nbytes > b.ptr) { nbytes = b.ptr; r = CK_ZS_END_OF_BUFFER; }
    b.ptr -= nbytes; b.used -= nbytes * 8;
    b.c = ck_zs_le64(b.p + b.ptr);
    return r;
}
CK_ZS_DEV bool ck_zs_br_end(const ck_zs_br& b) { return b.ptr == 0 && b.used == 64; }

// ---- Huffman literals -------------------------------------------------------------------------------------------------
// the FSE-compressed Huffman weights p[0, n) into ws.w: their number (at most 255), or -1.  Two interleaved states,
// libzstd's stopping rule: after the symbol that overreads the stream, one more from the other state
CK_ZS_DEV int ck_zs_fse_weights(const u8* p, u32 n, ck_zs_ws& ws) {
    u32 maxsv = 255, log = 0;
    int h = ck_zs_ncount(p, n, ws.norm, maxsv, log);
    if (h < 0 || log > 6) return -1;
    ck_zs_fse_build(ws.wt, ws.norm, maxsv, log, ws.next);
    bool fast = true;                                            // no state update of 0 bits: libzstd's fast reads
    for (u32 s = 0; s <= maxsv; s++) if (ws.norm[s] >= (short)(1 << (log - 1))) fast = false;
    ck_zs_br b;
    if (!ck_zs_br_init(b, p + h, n - (u32)h)) return -1;
    u32 s1 = ck_zs_read(b, log); ck_zs_reload(b);
    u32 s2 = ck_zs_read(b, log); ck_zs_reload(b);
    u32 op = 0;
#define CK_ZS_WSYM(st) do { ck_zs_fse e_ = ws.wt[st]; ws.w[op++] = e_.sym; \
                            st = e_.next + (fast ? (e_.nb ? ck_zs_read_fast(b, e_.nb) : 0u) : ck_zs_read(b, e_.nb)); } while (0)
    for (;;) {
        int r = ck_zs_reload(b);
        if (r != CK_ZS_UNFINISHED || op >= 252) break;
        CK_ZS_WSYM(s1); CK_ZS_WSYM(s2); CK_ZS_WSYM(s1); CK_ZS_WSYM(s2);
    }
    for (;;) {
        if (op > 253) return -1;
        CK_ZS_WSYM(s1);
        if (ck_zs_reload(b) == CK_ZS_OVERFLOW) { CK_ZS_WSYM(s2); break; }
        if (op > 253) return -1;
        CK_ZS_WSYM(s2);
        if (ck_zs_reload(b) == CK_ZS_OVERFLOW) { CK_ZS_WSYM(s1); break; }
    }
#undef CK_ZS_WSYM
    return (int)op;
}

// The Huffman tree description p[0, n) (RFC 8878 4.2.1): weights direct or FSE-compressed, the last one implied.
// Returns its bytes, or -1; *nsym symbols, table log *log (<= 12)
CK_ZS_DEV int ck_zs_huf_desc(const u8* p, u32 n, ck_zs_ws& ws, u32& nsym, u32& log) {
    if (!n) return -1;
    u32 isz = p[0], osz;
    if (isz >= 128) {
        osz = isz - 127; isz = (osz + 1) / 2;
        if (isz + 1 > n) return -1;
        for (u32 k = 0; k < osz; k += 2) { ws.w[k] = p[1 + k / 2] >> 4; ws.w[k + 1] = p[1 + k / 2] & 15u; }
    } else {
        if (isz + 1 > n) return -1;
        int r = ck_zs_fse_weights(p + 1, isz, ws);
        if (r < 0) return -1;
        osz = (u32)r;
    }
    for (u32 k = 0; k < 16; k++) ws.rank[k] = 0;
    u32 total = 0;
    for (u32 k = 0; k < osz; k++) {
        if (ws.w[k] > CK_ZS_HUF_LOG) return -1;
        ws.rank[ws.w[k]]++;
        total += (1u << ws.w[k]) >> 1;
    }
    if (!total) return -1;
    log = ck_zs_hb(total) + 1;
    if (log > CK_ZS_HUF_LOG) return -1;
    u32 rest = (1u << log) - total;
    if ((1u << ck_zs_hb(rest)) != rest) return -1;               // the implied weight must complete a power of 2
    u32 lw = ck_zs_hb(rest) + 1;
    ws.w[osz] = (u8)lw;
    ws.rank[lw]++;
    if (ws.rank[1] < 2 || (ws.rank[1] & 1u)) return -1;
    nsym = osz + 1;
    return (int)isz + 1;
}

// one Huffman stream p[0, n) into out[0, cnt): libzstd's X1 decode; true when it ends exactly at the stream's start
CK_ZS_DEV bool ck_zs_huf_stream(const u8* p, u32 n, u8* out, u32 cnt, const uint16_t* dt, u32 log) {
    ck_zs_br b;
    if (!ck_zs_br_init(b, p, n)) return false;
    u32 i = 0;
#define CK_ZS_HSYM() do { u32 e_ = dt[ck_zs_look_fast(b, log)]; out[i++] = (u8)e_; b.used += e_ >> 8; } while (0)
    if (cnt > 3) {
        for (;;) {
            int r = ck_zs_reload(b);
            if (r != CK_ZS_UNFINISHED || i >= cnt - 3) break;
            CK_ZS_HSYM(); CK_ZS_HSYM(); CK_ZS_HSYM(); CK_ZS_HSYM();
        }
    } else ck_zs_reload(b);
    while (i < cnt) CK_ZS_HSYM();
#undef CK_ZS_HSYM
    return ck_zs_br_end(b);
}

// ---- XXH64 ------------------------------------------------------------------------------------------------------------
#define CK_XXP1 0x9E3779B185EBCA87ull
#define CK_XXP2 0xC2B2AE3D27D4EB4Full
#define CK_XXP3 0x165667B19E3779F9ull
#define CK_XXP4 0x85EBCA77C2B2AE63ull
#define CK_XXP5 0x27D4EB2F165667C5ull
CK_ZS_HD ck_zu64 ck_xx_rotl(ck_zu64 x, u32 r) { return (x << r) | (x >> (64 - r)); }
CK_ZS_HD ck_zu64 ck_xx_round(ck_zu64 acc, ck_zu64 in) { acc += in * CK_XXP2; return ck_xx_rotl(acc, 31) * CK_XXP1; }
CK_ZS_HD ck_zu64 ck_xx_merge(ck_zu64 h, ck_zu64 v) { h ^= ck_xx_round(0, v); return h * CK_XXP1 + CK_XXP4; }
// accumulator k (0 - 3) of XXH64 (seed 0) over the whole 32-byte stripes of p[0, n)
CK_ZS_DEV ck_zu64 ck_xx_acc(const u8* p, ck_zu64 n, u32 k) {
    ck_zu64 v = k == 0 ? CK_XXP1 + CK_XXP2 : k == 1 ? CK_XXP2 : k == 2 ? 0ull : 0ull - CK_XXP1;
    for (ck_zu64 s = 0; s + 32 <= n; s += 32) v = ck_xx_round(v, ck_zs_le64(p + s + 8 * k));
    return v;
}
// XXH64 (seed 0) of p[0, n): lanes 0 - 3 run the four accumulators, every lane returns the digest
CK_ZS_DEV ck_zu64 ck_zs_xxh64(const u8* p, ck_zu64 n, u32 lane) {
    ck_zu64 h;
    if (n >= 32) {
#ifdef __CUDA_ARCH__
        ck_zu64 mine = lane < 4 ? ck_xx_acc(p, n, lane) : 0ull;
        ck_zu64 v1 = __shfl_sync(0xffffffffu, mine, 0), v2 = __shfl_sync(0xffffffffu, mine, 1);
        ck_zu64 v3 = __shfl_sync(0xffffffffu, mine, 2), v4 = __shfl_sync(0xffffffffu, mine, 3);
#else
        ck_zu64 v1 = ck_xx_acc(p, n, 0), v2 = ck_xx_acc(p, n, 1), v3 = ck_xx_acc(p, n, 2), v4 = ck_xx_acc(p, n, 3);
#endif
        h = ck_xx_rotl(v1, 1) + ck_xx_rotl(v2, 7) + ck_xx_rotl(v3, 12) + ck_xx_rotl(v4, 18);
        h = ck_xx_merge(h, v1); h = ck_xx_merge(h, v2); h = ck_xx_merge(h, v3); h = ck_xx_merge(h, v4);
    } else h = CK_XXP5;
    h += n;
    ck_zu64 i = n & ~31ull;
    for (; i + 8 <= n; i += 8) { h ^= ck_xx_round(0, ck_zs_le64(p + i)); h = ck_xx_rotl(h, 27) * CK_XXP1 + CK_XXP4; }
    if (i + 4 <= n) { h ^= (ck_zu64)ck_zs_le32(p + i) * CK_XXP1; h = ck_xx_rotl(h, 23) * CK_XXP2 + CK_XXP3; i += 4; }
    for (; i < n; i++) { h ^= p[i] * CK_XXP5; h = ck_xx_rotl(h, 11) * CK_XXP1; }
    h ^= h >> 33; h *= CK_XXP2; h ^= h >> 29; h *= CK_XXP3; h ^= h >> 32;
    return h;
}

// ---- the frame --------------------------------------------------------------------------------------------------------
// the sequence table of one code kind (0 literal lengths, 1 offsets, 2 match lengths) for mode `mode` at p[0, n) into t:
// the bytes its description took, or -1.  *log = its accuracy log; `have` = a table from an earlier block (Repeat)
CK_ZS_DEV int ck_zs_seq_table(u32 kind, u32 mode, const u8* p, u32 n, ck_zs_fse* t, u32& log, bool have, ck_zs_ws& ws) {
    const u32 maxs = kind == 0 ? 35u : kind == 1 ? 31u : 52u, maxlog = kind == 1 ? 8u : 9u;
    if (mode == 0) {                                             // predefined
        const short* d = kind == 0 ? ck_zs_ll_def : kind == 1 ? ck_zs_of_def : ck_zs_ml_def;
        u32 ms = kind == 0 ? 35u : kind == 1 ? 28u : 52u;
        for (u32 s = 0; s <= ms; s++) ws.norm[s] = d[s];
        log = kind == 1 ? 5u : 6u;
        ck_zs_fse_build(t, ws.norm, ms, log, ws.next);
        return 0;
    }
    if (mode == 1) {                                             // RLE: one code, no state bits
        if (!n || p[0] > maxs) return -1;
        t[0].sym = p[0]; t[0].nb = 0; t[0].next = 0;
        log = 0;
        return 1;
    }
    if (mode == 3) return have ? 0 : -1;                         // Repeat
    u32 ms = maxs, lg = 0;
    int h = ck_zs_ncount(p, n, ws.norm, ms, lg);
    if (h < 0 || lg > maxlog) return -1;
    ck_zs_fse_build(t, ws.norm, ms, lg, ws.next);
    log = lg;
    return h;
}

// The zstd frame z[0, zn) decoded by one warp into out[0, cap), where cap must be the frame's walk bound (ck_zs_walk):
// header, blocks, Frame_Content_Size and checksum as the notes on top of this file say.  Every lane returns the decoded
// length, or -1 for a frame libzstd refuses, one this decoder refuses (more than one frame, bytes after the frame) or one
// whose bound is not cap
CK_ZS_DEV long long ck_zs_decode(const u8* z, ck_zu64 zn, u8* out, ck_zu64 cap, ck_zs_ws& ws, u32 lane) {
    ck_zs_frame f;
    ck_zu64 bound = 0;
    if (!ck_zs_header(z, zn, f) || !ck_zs_walk(z, zn, f, &bound) || bound != cap) return -1;
    const u32 B = f.bmax;
    ck_zu64 pos = f.hdr, op = 0, res = 0;                        // res: where the block's reservation starts
    u32 rep0 = 1, rep1 = 4, rep2 = 8;
    bool lit_ent = false, fse_ent = false;                       // a Huffman table / sequence tables from an earlier block
    u32 hlog = 0, lllog = 0, oflog = 0, mllog = 0;
    for (;;) {
        u32 bh = ck_zs_le24(z + pos), type = (bh >> 1) & 3u, size = bh >> 3;
        pos += 3;
        const u8* src = z + pos;
        if (type == 0 || type == 1) {                            // raw / RLE: the walk checked their sizes
            for (u32 i = lane; i < size; i += CK_ZS_LANES) out[op + i] = type == 0 ? src[i] : src[0];
            op += size; res += size;
            pos += type == 0 ? size : 1u;
            CK_ZS_SYNC();
            if (bh & 1u) break;
            continue;
        }
        // compressed: the literals section (lane 0 parses, the warp builds the Huffman table, lanes 0 - 3 decode)
        int lt = 0;                                              // 0 raw (in the section), 1 RLE, 2 Huffman
        u32 L = 0, lh = 0, C = 0, ns = 1, used = 0, nsym = 0, hl = hlog;
        int hs = 0;
        bool ok = true;
        if (lane == 0) {
            do {
                if (size < 2) { ok = false; break; }
                u32 b0 = src[0], ty = b0 & 3u, sf = (b0 >> 2) & 3u;
                if (ty == 0 || ty == 1) {
                    if (sf == 1) { lh = 2; L = ck_zs_le16(src) >> 4; if (ty == 1 && size < 3) { ok = false; break; } }
                    else if (sf == 3) { lh = 3; if (size < (ty == 1 ? 4u : 3u)) { ok = false; break; } L = ck_zs_le24(src) >> 4; }
                    else { lh = 1; L = b0 >> 3; }
                    if (L > B) { ok = false; break; }
                    if (ty == 0) { if (lh + L > size) { ok = false; break; } used = lh + L; lt = 0; }
                    else { used = lh + 1; lt = 1; }
                    break;
                }
                if (ty == 3 && !lit_ent) { ok = false; break; }  // Treeless with no earlier table
                if (size < 5) { ok = false; break; }
                u32 lhc = ck_zs_le32(src);
                if (sf <= 1) { lh = 3; L = (lhc >> 4) & 0x3FFu; C = (lhc >> 14) & 0x3FFu; ns = sf ? 4u : 1u; }
                else if (sf == 2) { lh = 4; L = (lhc >> 4) & 0x3FFFu; C = lhc >> 18; ns = 4; }
                else { lh = 5; L = (lhc >> 4) & 0x3FFFFu; C = (lhc >> 22) + ((u32)src[4] << 10); ns = 4; }
                if (L > CK_ZS_BLOCK_MAX || (ns == 4 && L < 6) || C + lh > size || L > B) { ok = false; break; }
                lt = 2;
                used = lh + C;
                if (ty == 2) {
                    hs = ck_zs_huf_desc(src + lh, C, ws, nsym, hl);
                    if (hs < 0 || (u32)hs >= C) { ok = false; break; }
                }
            } while (0);
        }
        ok = CK_ZS_BC(ok);
        if (!ok) return -1;
        lt = CK_ZS_BC(lt); L = CK_ZS_BC(L); lh = CK_ZS_BC(lh); C = CK_ZS_BC(C); ns = CK_ZS_BC(ns); used = CK_ZS_BC(used);
        hs = CK_ZS_BC(hs); nsym = CK_ZS_BC(nsym); hl = CK_ZS_BC(hl);
        u8* lit = lt == 0 ? (u8*)(src + lh) : out + (res + B - L);
        if (lt == 1) {
            for (u32 i = lane; i < L; i += CK_ZS_LANES) lit[i] = src[lh];
        } else if (lt == 2) {
            if (hs > 0) {                                        // a new table: each lane fills the entries of its symbols
                CK_ZS_SYNC();
                if (lane == 0) {                                 // rank[w] becomes the first entry of weight w
                    u32 cur = 0;
                    for (u32 w = 1; w <= hl; w++) { u32 t = ws.rank[w] << (w - 1); ws.rank[w] = cur; cur += t; }
                    for (u32 s = 0; s < nsym; s++) {
                        u32 w = ws.w[s];
                        ws.next[s] = (uint16_t)(w ? ws.rank[w] : 0u);
                        if (w) ws.rank[w] += 1u << (w - 1);
                    }
                }
                CK_ZS_SYNC();
                for (u32 s = lane; s < nsym; s += CK_ZS_LANES) {
                    u32 w = ws.w[s];
                    if (!w) continue;
                    uint16_t e = (uint16_t)(s | ((hl + 1 - w) << 8));
                    for (u32 k = 0; k < (1u << (w - 1)); k++) ws.huf[ws.next[s] + k] = e;
                }
                hlog = hl;
                CK_ZS_SYNC();
            }
            const u8* st = src + lh + (u32)hs;
            u32 sn = C - (u32)hs;
            bool hok = true;
            if (ns == 1) {
                if (lane == 0) hok = ck_zs_huf_stream(st, sn, lit, L, ws.huf, hlog);
            } else {
                u32 l1 = 0, l2 = 0, l3 = 0, seg = (L + 3) / 4;
                if (sn < 10 || 3 * seg > L) hok = false;
                else {
                    l1 = ck_zs_le16(st); l2 = ck_zs_le16(st + 2); l3 = ck_zs_le16(st + 4);
                    if ((ck_zu64)l1 + l2 + l3 + 6 > sn) hok = false;
                }
                if (hok)
                    for (u32 k = lane; k < 4; k += CK_ZS_LANES) {
                        u32 o = k == 0 ? 6 : k == 1 ? 6 + l1 : k == 2 ? 6 + l1 + l2 : 6 + l1 + l2 + l3;
                        u32 sl = k == 0 ? l1 : k == 1 ? l2 : k == 2 ? l3 : sn - 6 - l1 - l2 - l3;
                        hok &= ck_zs_huf_stream(st + o, sl, lit + k * seg, k < 3 ? seg : L - 3 * seg, ws.huf, hlog);
                    }
            }
            hok = CK_ZS_ALL(hok);
            if (!hok) return -1;
            lit_ent = true;
        }
        CK_ZS_SYNC();
        // the sequences section: lane 0 parses the header and builds the tables
        const u8* q = src + used;
        u32 qn = size - used, nseq = 0, sh = 1;     // sh: the sequences header's bytes
        if (lane == 0) {
            do {
                if (qn < 1) { ok = false; break; }
                u32 k = 0, b0 = q[k++];
                if (!b0) { if (qn != 1) ok = false; break; }
                if (b0 < 128) nseq = b0;
                else if (b0 == 255) { if (qn < 3) { ok = false; break; } nseq = ck_zs_le16(q + 1) + 0x7F00u; k = 3; }
                else { if (qn < 2) { ok = false; break; } nseq = ((b0 - 128) << 8) + q[1]; k = 2; }
                if (qn < k + 1) { ok = false; break; }          // no modes byte (libzstd 1.5.5 ignores its reserved bits)
                u32 modes = q[k++];
                int r = ck_zs_seq_table(0, modes >> 6, q + k, qn - k, ws.ll, lllog, fse_ent, ws);
                if (r < 0) { ok = false; break; }
                k += (u32)r;
                r = ck_zs_seq_table(1, (modes >> 4) & 3u, q + k, qn - k, ws.of, oflog, fse_ent, ws);
                if (r < 0) { ok = false; break; }
                k += (u32)r;
                r = ck_zs_seq_table(2, (modes >> 2) & 3u, q + k, qn - k, ws.ml, mllog, fse_ent, ws);
                if (r < 0) { ok = false; break; }
                k += (u32)r;
                sh = k;
            } while (0);
        }
        ok = CK_ZS_BC(ok);
        if (!ok) return -1;
        nseq = CK_ZS_BC(nseq); sh = CK_ZS_BC(sh);
        lllog = CK_ZS_BC(lllog); oflog = CK_ZS_BC(oflog); mllog = CK_ZS_BC(mllog);
        CK_ZS_SYNC();
        // the sequences, every lane decoding the same bits; the warp copies
        ck_zu64 bo = 0;                                          // the block's output so far
        u32 c = 0;                                               // literals consumed
        const bool alias = lt != 0;
        if (nseq) {
            fse_ent = true;
            ck_zs_br b;
            if (!ck_zs_br_init(b, q + sh, qn - sh)) return -1;
            u32 sll = ck_zs_read(b, lllog); ck_zs_reload(b);
            u32 sof = ck_zs_read(b, oflog); ck_zs_reload(b);
            u32 sml = ck_zs_read(b, mllog); ck_zs_reload(b);
            for (u32 i = 0;;) {
                ck_zs_fse ell = ws.ll[sll], eml = ws.ml[sml], eof = ws.of[sof];
                u32 llb = ck_zs_ll_bits[ell.sym], mlb = ck_zs_ml_bits[eml.sym], ofb = eof.sym;
                u32 ll = ck_zs_ll_base[ell.sym], ml = ck_zs_ml_base[eml.sym], off;
                if (ofb > 1) {
                    off = ((1u << ofb) - 3u) + ck_zs_read_fast(b, ofb);
                    rep2 = rep1; rep1 = rep0; rep0 = off;
                } else {
                    u32 ll0 = ll == 0;
                    if (ofb == 0) {
                        off = ll0 ? rep1 : rep0;
                        rep1 = ll0 ? rep0 : rep1;
                        rep0 = off;
                    } else {
                        u32 ix = 1u + ll0 + ck_zs_read_fast(b, 1);   // repeat offset 1 - 3; 3 = the first one minus 1
                        u32 t = ix == 3 ? rep0 - 1u : ix == 1 ? rep1 : rep2;
                        t += !t;
                        if (ix != 1) rep2 = rep1;
                        rep1 = rep0; rep0 = off = t;
                    }
                }
                if (mlb) ml += ck_zs_read_fast(b, mlb);
                if (llb + mlb + ofb >= 31) ck_zs_reload(b);
                if (llb) ll += ck_zs_read_fast(b, llb);
                sll = ell.next + ck_zs_read(b, ell.nb);
                sml = eml.next + ck_zs_read(b, eml.nb);
                sof = eof.next + ck_zs_read(b, eof.nb);
                // execute: ll literals, then ml bytes from off back
                if (ll > L - c) return -1;                       // more literals than the section holds
                if (bo + ll + ml + (L - c - ll) > B) return -1;  // past the block's maximum (see the notes on top)
                if (off > op + bo + ll) return -1;               // before the frame's output
                u8* o = out + op + bo;
                for (u32 i0 = 0; i0 < ll; i0 += CK_ZS_LANES) {
                    u32 j = i0 + lane;
                    u8 v = j < ll ? lit[c + j] : (u8)0;
                    if (alias) CK_ZS_SYNC();
                    if (j < ll) o[j] = v;
                }
                c += ll; bo += ll; o += ll;
                CK_ZS_SYNC();
                const u8* m = o - off;
                if (off >= ml) for (u32 j = lane; j < ml; j += CK_ZS_LANES) o[j] = m[j];
                else for (u32 j = lane; j < ml; j += CK_ZS_LANES) o[j] = m[j % off];
                bo += ml;
                CK_ZS_SYNC();
                if (++i == nseq) break;
                ck_zs_reload(b);
            }
            if (ck_zs_reload(b) < CK_ZS_COMPLETED) return -1;    // bits left over
        }
        {                                                        // the last literals
            u32 ll = L - c;
            u8* o = out + op + bo;
            for (u32 i0 = 0; i0 < ll; i0 += CK_ZS_LANES) {
                u32 j = i0 + lane;
                u8 v = j < ll ? lit[c + j] : (u8)0;
                if (alias) CK_ZS_SYNC();
                if (j < ll) o[j] = v;
            }
            bo += ll;
        }
        CK_ZS_SYNC();
        op += bo; res += B;
        pos += size;
        if (bh & 1u) break;
    }
    if (f.has_fcs && op != f.fcs) return -1;
    if (f.checksum && (u32)ck_zs_xxh64(out, op, lane) != ck_zs_le32(z + pos)) return -1;
    return (long long)op;
}

#endif  // CK_ZSTD_CUH
