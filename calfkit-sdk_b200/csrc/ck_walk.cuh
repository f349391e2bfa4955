// Canonical-Envelope recogniser + field extractor: one sequential walker per record.
//
// Replaces, for records that are byte-wise fixed points of the reference codec, the work of
//   Envelope.model_validate_json          (reference calfkit/models/envelope.py:9-17, pydantic-core)
//   envelope.context.model_copy(deep=True) (reference calfkit/nodes/base.py:64-68)
// by proving "this byte string is exactly what model_dump_json() would emit for a valid Envelope"
// (key order, defaults present, compact separators, canonical scalars — SURVEY.md Appendix A) while
// recording the spans the routing / splice kernels need.  Anything it cannot prove gets
// CK_NOT_CANONICAL and is left to the canonicaliser; it never accepts a record the reference
// would reject or re-emit differently.
//
// Written as __host__ __device__ so tests/hostsim can fuzz the *same source* against pydantic on
// the CPU (test infrastructure only — the shipped library has no host entry point to it).
#ifndef CK_WALK_CUH
#define CK_WALK_CUH

#include "ck_common.h"

#if defined(__CUDACC__)
#define CK_HD __host__ __device__ __forceinline__
#define CK_HD_NOINLINE __host__ __device__ __noinline__
#else
#define CK_HD inline __attribute__((always_inline))
#define CK_HD_NOINLINE __attribute__((noinline))
#endif

typedef uint8_t u8;
typedef uint32_t u32;
typedef uint64_t u64;
#if !defined(__CUDACC__)
struct uint4 { u32 x, y, z, w; };        // host test build of the device sources
#endif

struct Span { u32 off, len; };

// -------------------------------------------------------------------------------------------------
// Long records (ck_walk_long.cuh): one WARP walks a record.  All lanes run the walker in lockstep on the same bytes (reader
// URd: kWarp); where the schema has a long list — the entries of tool_calls / tool_results, the messages of message_history,
// the parts of a message — the lanes take one element each and validate it with the unchanged recognisers through their
// own reader.  The element boundaries come from a data-parallel structural pre-scan of the record (string mask by prefix
// XOR of the quote bits, nesting depth by prefix sums of the bracket bits: positions of the commas and closers at depths 4
// and 6).  The pre-scan only PROPOSES boundaries: element e must start right after the opener / the previous comma and its
// walk must end exactly at the next proposed comma / the closer, so the element walks chain into exactly the cover the
// sequential walker would produce — a wrong proposal fails a walk and the record goes to the canonicaliser path.
// The helpers below have single-lane stand-ins so that the host (g++) build of this file parses the hooks.
// -------------------------------------------------------------------------------------------------
#if defined(__CUDA_ARCH__)
extern __shared__ uint4 ck_win_smem[];       // dynamic shared memory of the walk kernels (per-thread windows / per-warp indexes)
#endif
#define CK_LX_SEP 640u               // commas indexed per depth
#define CK_LX_CLOSE 320u             // closers indexed per depth
#define CK_LX_MIN 4u                 // lists shorter than this are walked sequentially
#define CK_LX_KEYS 128u              // = CK_DICT_KEYS
#define CK_DEFER_MAX 4096u           // = CK_ELEM_MAX: list elements longer than this are not handed to the one-thread-per-element pass
#define CK_LX_OPEN 8u                // depth-4 list openers remembered per record
struct ck_elem { u32 rec, start, end; };         // one deferred list element: bytes [start, end) of record `rec` must be exactly one message
struct ck_long_index {
    u32 n_sep[2], n_close[2], ok, rec, defer_cap, n_open;
    u32 open_sq[CK_LX_OPEN];                     // '[' that open a depth-4 list (message_history is one of them)
    ck_elem* defer_list; u32* defer_ctr;         // device-wide element list of the batch (ck_walk_elems_kernel); null: walk elements in the warp
    u32 sep[2][CK_LX_SEP];           // [0]: depth 4, [1]: depth 6 — record-relative positions of commas outside strings
    u32 close_[2][CK_LX_CLOSE];      // closers that end a container of that depth
    u32 kh[2][CK_LX_KEYS], koff[2][CK_LX_KEYS];      // key hash / offset of the entries of tool_calls [0], tool_results [1]
};
#if defined(__CUDA_ARCH__)
CK_HD u32 ck_lane() { return threadIdx.x & 31u; }
CK_HD bool ck_all(bool p) { return __all_sync(0xffffffffu, p); }
CK_HD u32 ck_bcast(u32 v, u32 src) { return __shfl_sync(0xffffffffu, v, src); }
CK_HD u32 ck_or_reduce(u32 v) { return __reduce_or_sync(0xffffffffu, v); }
CK_HD void ck_warp_sync() { __syncwarp(); }
CK_HD u32 ck_defer_reserve(u32* ctr, u32 n) { u32 b = 0; if ((threadIdx.x & 31u) == 0) b = atomicAdd(ctr, n); return __shfl_sync(0xffffffffu, b, 0); }
CK_HD u32 ck_max_reduce(u32 v) { return __reduce_max_sync(0xffffffffu, v); }
#else
CK_HD u32 ck_max_reduce(u32 v) { return v; }
CK_HD u32 ck_defer_reserve(u32*, u32) { return 0xffffffffu; }
CK_HD u32 ck_lane() { return 0; }
CK_HD bool ck_all(bool p) { return p; }
CK_HD u32 ck_bcast(u32 v, u32) { return v; }
CK_HD u32 ck_or_reduce(u32 v) { return v; }
CK_HD void ck_warp_sync() {}
#endif
// elements of the list whose content starts at `pos` (just after its opener) at depth index di (0: depth 4, 1: depth 6):
// closer position q, index of the first separator inside and the number of separators; false = no usable proposal
CK_HD bool ck_lx_range(const ck_long_index* lx, u32 di, u32 pos, u32& q, u32& s0, u32& k) {
    if (!lx || !lx->ok) return false;
    u32 lo = 0, hi = lx->n_close[di];
    while (lo < hi) { u32 mid = (lo + hi) >> 1; if (lx->close_[di][mid] < pos) lo = mid + 1; else hi = mid; }
    if (lo >= lx->n_close[di]) return false;
    q = lx->close_[di][lo];
    lo = 0; hi = lx->n_sep[di];
    while (lo < hi) { u32 mid = (lo + hi) >> 1; if (lx->sep[di][mid] < pos) lo = mid + 1; else hi = mid; }
    s0 = lo;
    u32 a = lo; hi = lx->n_sep[di];
    while (a < hi) { u32 mid = (a + hi) >> 1; if (lx->sep[di][mid] < q) a = mid + 1; else hi = mid; }
    k = a - s0;
    return true;
}

// -------------------------------------------------------------------------------------------------
// Reader: byte access to one record through aligned 8-byte global loads (one 32 B sector serves
// four consecutive loads of a lane; L1 keeps the line for the next three).  The input buffer is
// allocated with >= 16 bytes of tail padding and a 256 B aligned base, so aligned-down / +8 loads
// around a record never leave the allocation.
// -------------------------------------------------------------------------------------------------
struct GRd {
    static const bool kWindow = false;
    static const bool kWarp = false;          // see URd (ck_walk_long.cuh)
    static const bool kTrustFloats = false;   // see WRdT
    const u8* g;     // record start
    u32 n;           // record length
    const u64* wp;   // address of the cached aligned word
    u64 w;

    CK_HD static u64 ld64(const u64* p) {
#if defined(__CUDA_ARCH__)
        return __ldg((const unsigned long long*)p);
#else
        return *p;
#endif
    }
    CK_HD void init(const u8* base, u32 len, u32 st = 0) { (void)st; g = base; n = len; wp = nullptr; w = 0; }
    CK_HD u32 st() const { return 0; }           // reader state carried through out-of-line calls (none here)
    CK_HD void set_st(u32) {}
    CK_HD void invalidate() {}

    CK_HD u8 at(u32 pos) {           // caller guarantees pos < n
        const u8* a = g + pos;
        const u64* q = (const u64*)((uintptr_t)a & ~(uintptr_t)7);
        if (q != wp) { wp = q; w = ld64(q); }
        return (u8)(w >> (8 * ((uintptr_t)a & 7)));
    }
    // 8 bytes starting at pos, little endian; bytes at/after n are unspecified (but readable)
    CK_HD u64 load8(u32 pos) {
        const u8* a = g + pos;
        u32 s = (u32)((uintptr_t)a & 7);
        const u64* q = (const u64*)((uintptr_t)a - s);
        u64 lo = (q == wp) ? w : ld64(q);
        if (s == 0) { wp = q; w = lo; return lo; }
        u64 hi = ld64(q + 1);
        wp = q + 1; w = hi;
        return (lo >> (8 * s)) | (hi << (64 - 8 * s));
    }
    CK_HD void load16(u32 pos, u64& x0, u64& x1) {
        const u8* a = g + pos;
        u32 s = (u32)((uintptr_t)a & 7);
        const u64* q = (const u64*)((uintptr_t)a - s);
        u64 w0 = ld64(q), w1 = ld64(q + 1);
        x0 = w0; x1 = w1;
        if (s) {
            u64 w2 = ld64(q + 2);
            x0 = (w0 >> (8 * s)) | (w1 << (64 - 8 * s));
            x1 = (w1 >> (8 * s)) | (w2 << (64 - 8 * s));
        }
    }
};

typedef GRd Rd;        // the plan / fan-out kernels read a few scattered spots of a record: plain global loads

// the reader of a warp that walks ONE record: plain global loads (in lockstep every lane reads the same address: one
// transaction, broadcast), plus the record's structural index in shared memory.  The same type serves the lockstep walk and
// the per-lane element walks (one instantiation of the walker: the long kernel's code must fit the instruction cache); the
// reader state says which one it is — only a lockstep walk (state 2; bit 0 is used by the match cores) may fan a list out.
struct URd : GRd {
    static const bool kWarp = true;
    u32 lock;
    CK_HD void init(const u8* base, u32 len, u32 st = 0) { GRd::init(base, len); lock = st; }
    CK_HD u32 st() const { return lock; }
    CK_HD void set_st(u32 s) { lock = s; }
    CK_HD void invalidate() {}
    CK_HD const ck_long_index* lx() const {
#if defined(__CUDA_ARCH__)
        return lock ? (const ck_long_index*)ck_win_smem + (threadIdx.x >> 5) : nullptr;
#else
        return nullptr;
#endif
    }
    CK_HD ck_long_index* lxw() const {
#if defined(__CUDA_ARCH__)
        return (ck_long_index*)ck_win_smem + (threadIdx.x >> 5);
#else
        return nullptr;
#endif
    }
};

// -------------------------------------------------------------------------------------------------
// Window reader (the walker's): each thread stages CK_WIN_BYTES of its record in shared memory with
// 16-byte asynchronous copies (cp.async, no data registers, all chunks of a refill in flight at once)
// and reads bytes / unaligned words from there.  Thirty-two lanes walking thirty-two different records
// cost one L1 tag lookup per lane per *load instruction* through global memory (what bounds the GRd
// walker); through shared memory a warp-wide access is one wavefront unless banks
// collide, and the global side shrinks to len/16 chunk copies per record.  Every access checks the
// window and refills on demand (re-centred CK_WIN_BACK bytes behind the position), so correctness does not
// depend on access order.  The window base is the reader's state; it travels through out-of-line
// calls by value (cores return it next to their result).
// -------------------------------------------------------------------------------------------------
// 224 bytes: a 1.15 KB record takes about six refills, each a full round trip on the thread's critical path.  The 240-byte
// slot (15 x 16 B) x 128 threads x CK_WALK_MINB (6) blocks is 180 KB of shared memory per SM
#ifndef CK_WIN_BYTES
#define CK_WIN_BYTES 224
#endif
#define CK_WIN_BACK 16
#define CK_WIN_STRIDE (CK_WIN_BYTES + 16)     // per-thread slot; the pad spreads the slots over the banks
#define CK_WIN_NONE 0x80000000u     // o = ap - wbase is then >= 2^31 for every position: always refills
#if defined(__CUDA_ARCH__)
extern __shared__ uint4 ck_win_smem[];       // blockDim.x * CK_WIN_STRIDE bytes (dynamic shared memory of the walk kernel)
#else
static thread_local uint8_t ck_win_host[CK_WIN_STRIDE];
#endif

// (re)load the window so that it holds [wb, wb + CK_WIN_BYTES) of the 16-byte aligned stream gb[]; chunks at or
// beyond `lim` (the record end rounded up to 16) are not touched.  Returns wb.
CK_HD_NOINLINE u32 ck_win_refill(const u8* gb, u32 ap, u32 lim) {
    u32 wb = ap & ~15u;
    wb = wb >= CK_WIN_BACK ? wb - CK_WIN_BACK : 0u;
#if defined(__CUDA_ARCH__)
    u32 dst = (u32)__cvta_generic_to_shared((const u8*)ck_win_smem + threadIdx.x * CK_WIN_STRIDE);
    const u8* src = gb + wb;
#pragma unroll
    for (u32 k = 0; k < CK_WIN_BYTES; k += 16)
        if (wb + k < lim) asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" :: "r"(dst + k), "l"(src + k) : "memory");
    asm volatile("cp.async.wait_all;" ::: "memory");
#else
    for (u32 k = 0; k < CK_WIN_BYTES; k += 16) if (wb + k < lim) for (u32 j = 0; j < 16; j++) ck_win_host[k + j] = gb[wb + k + j];
#endif
    return wb;
}

struct WRd {
    static const bool kWindow = true;
    static const bool kWarp = false;
    static const bool kTrustFloats = false;
    const u8* g;     // record start
    u32 n;           // record length
    u32 wbase;       // window base in the aligned stream (multiple of 16), CK_WIN_NONE = nothing staged
    u32 m;           // g & 15: position p of the record is byte p + m of the 16-byte aligned stream
    const u8* wp;    // this thread's window slot

    CK_HD void init(const u8* base, u32 len, u32 st = CK_WIN_NONE) {
        g = base; n = len; wbase = st; m = (u32)((uintptr_t)base & 15);
#if defined(__CUDA_ARCH__)
        wp = (const u8*)ck_win_smem + threadIdx.x * CK_WIN_STRIDE;
#else
        wp = ck_win_host;
#endif
    }
    CK_HD u32 st() const { return wbase; }
    CK_HD void set_st(u32 s) { wbase = s; }
    CK_HD void invalidate() { wbase = CK_WIN_NONE; }
    CK_HD u32 mis() const { return m; }
    CK_HD const u8* win() const { return wp; }
    CK_HD void refill(u32 ap) { wbase = ck_win_refill(g - m, ap, (m + n + 15u) & ~15u); }
    CK_HD u8 at(u32 pos) {           // caller guarantees pos < n
        u32 ap = pos + mis();
        u32 o = ap - wbase;
        if (o >= (u32)CK_WIN_BYTES) { refill(ap); o = ap - wbase; }
        return win()[o];
    }
    // 8 bytes starting at pos, little endian; bytes at/after n are unspecified
    CK_HD u64 load8(u32 pos) {
        u32 ap = pos + mis();
        u32 o = ap - wbase;
        if (o > (u32)(CK_WIN_BYTES - 12)) { refill(ap); o = ap - wbase; }
        const u32* w = (const u32*)(win() + (o & ~3u));
        u32 a = w[0], b = w[1], c = w[2], sh = (o & 3u) * 8u;
#if defined(__CUDA_ARCH__)
        u32 lo = __funnelshift_r(a, b, sh), hi = __funnelshift_r(b, c, sh);
#else
        u32 lo = sh ? (u32)((((u64)b << 32) | a) >> sh) : a, hi = sh ? (u32)((((u64)c << 32) | b) >> sh) : b;
#endif
        return ((u64)hi << 32) | lo;
    }
    // 16 bytes starting at pos (literal compare): two words of 8
    CK_HD void load16(u32 pos, u64& x0, u64& x1) {
        u32 ap = pos + mis();
        u32 o = ap - wbase;
        if (o > (u32)(CK_WIN_BYTES - 20)) { refill(ap); o = ap - wbase; }
        const u32* w = (const u32*)(win() + (o & ~3u));
        u32 a = w[0], b = w[1], c = w[2], d = w[3], e = w[4], sh = (o & 3u) * 8u;
#if defined(__CUDA_ARCH__)
        u32 q0 = __funnelshift_r(a, b, sh), q1 = __funnelshift_r(b, c, sh), q2 = __funnelshift_r(c, d, sh), q3 = __funnelshift_r(d, e, sh);
#else
        u32 q0 = sh ? (u32)((((u64)b << 32) | a) >> sh) : a, q1 = sh ? (u32)((((u64)c << 32) | b) >> sh) : b;
        u32 q2 = sh ? (u32)((((u64)d << 32) | c) >> sh) : c, q3 = sh ? (u32)((((u64)e << 32) | d) >> sh) : d;
#endif
        x0 = ((u64)q1 << 32) | q0; x1 = ((u64)q3 << 32) | q2;
    }
};

// Readers for the second walk of the decode pass, over records the canonicaliser has just re-emitted: float literals
// with 16-17 significant digits are taken on trust there, because ck_canon.cuh only emits such a literal after the
// exact "is repr() of its double" test of ck_float.cuh.  The first walk (WRd / GRd) leaves them to the canonicaliser,
// which keeps that arithmetic (bignums, 128-bit division) out of the hot kernel.
struct WRdT : WRd { static const bool kTrustFloats = true; };
struct GRdT : GRd { static const bool kTrustFloats = true; };

#define CK_REP8(b) ((u64)(b) * 0x0101010101010101ull)

// 0x80 in every byte of x that is zero; false positives only ABOVE a true hit (callers use ctz)
CK_HD u64 ck_haszero(u64 x) { return (x - CK_REP8(0x01)) & ~x & CK_REP8(0x80); }
// 0x80 in every byte < 0x20 (same caveat); bytes >= 0x80 are never flagged here
CK_HD u64 ck_lt20(u64 x) { return (x - CK_REP8(0x20)) & ~x & CK_REP8(0x80); }

CK_HD u32 ck_ctz64(u64 x) {
#if defined(__CUDA_ARCH__)
    return (u32)(__ffsll((long long)x) - 1);
#else
    return (u32)__builtin_ctzll(x);
#endif
}

// literal compare.  The literal is folded at compile time into 64-bit immediates; the unaligned
// fetch + compare lives in two small out-of-line functions (8 and 16 bytes per call) so that the
// ~150 literal sites of the schema cost a handful of instructions each instead of an inlined
// unaligned-load sequence (instruction-cache footprint, DESIGN.md §walker).
// Out-of-line cores return the reader state next to their result (see WRd): match cores as
// (state & ~1) | ok, the others as state << 32 | result with result 0 = failure (state then unspecified:
// the caller invalidates its reader).
#define CK_RET(res) (((u64)r.st() << 32) | (u64)(u32)(res))
#define CK_CALL(e, call) u64 e##64 = (call); u32 e = (u32)e##64; if (!e) { r.invalidate(); return false; } r.set_st((u32)(e##64 >> 32))

template <class R>
CK_HD_NOINLINE u32 ck_match8_core(const u8* g, u32 n, u32 pos, u32 st, u64 want, u32 nb) {
    R r; r.init(g, n, st);
    u64 got = r.load8(pos);
    u64 mask = ~0ull >> (8 * (8 - nb));
    return (r.st() & ~1u) | (u32)(((got ^ want) & mask) == 0);
}
template <class R>
CK_HD_NOINLINE u32 ck_match16_core(const u8* g, u32 n, u32 pos, u32 st, u64 want0, u64 want1, u32 nb1) {
    R r; r.init(g, n, st);
    u64 g0, g1;
    r.load16(pos, g0, g1);
    u64 mask1 = ~0ull >> (8 * (8 - nb1));
    return (r.st() & ~1u) | (u32)((g0 == want0) & (((g1 ^ want1) & mask1) == 0));
}
CK_HD u64 ck_lit_word(const char* lit, u32 L, u32 k) {      // bytes [k, k+8) of the literal, zero padded
    u64 w = 0;
#pragma unroll
    for (u32 j = 0; j < 8; j++) if (k + j < L) w |= (u64)(u8)lit[k + j] << (8 * j);
    return w;
}
CK_HD u32 ck_lit_nb(u32 L, u32 k) { return (L - k >= 8) ? 8u : (L - k); }      // valid bytes of the word at k
template <class R>
CK_HD bool ck_match(R& r, u32& pos, const char* lit, u32 L) {
    if (pos + L > r.n) return false;
    u32 k = 0;
    if (R::kWindow) {          // shared-memory reads are short enough to inline: no call, no parameter traffic
#pragma unroll
        for (; k + 8 < L; k += 16) {
            u64 g0, g1;
            r.load16(pos + k, g0, g1);
            if (!((g0 == ck_lit_word(lit, L, k)) & (((g1 ^ ck_lit_word(lit, L, k + 8)) & (~0ull >> (8 * (8 - ck_lit_nb(L, k + 8))))) == 0))) return false;
        }
        if (k < L) { if (((r.load8(pos + k) ^ ck_lit_word(lit, L, k)) & (~0ull >> (8 * (8 - ck_lit_nb(L, k))))) != 0) return false; }
        pos += L;
        return true;
    }
#pragma unroll
    for (; k + 8 < L; k += 16) {
        u32 s = ck_match16_core<R>(r.g, r.n, pos + k, r.st(), ck_lit_word(lit, L, k), ck_lit_word(lit, L, k + 8), ck_lit_nb(L, k + 8));
        r.set_st(s & ~1u);
        if (!(s & 1u)) return false;
    }
    if (k < L) {
        u32 s = ck_match8_core<R>(r.g, r.n, pos + k, r.st(), ck_lit_word(lit, L, k), ck_lit_nb(L, k));
        r.set_st(s & ~1u);
        if (!(s & 1u)) return false;
    }
    pos += L;
    return true;
}
#define M(lit) ck_match(r, pos, lit, (u32)(sizeof(lit) - 1))
#define PEEK(c) (pos < r.n && r.at(pos) == (u8)(c))
// Speculative fused literals: pydantic emits every optional field, and in practice most of them are `null`, so
// long runs of `"key":null` pairs are tried as ONE literal first; a miss costs one 16-byte compare and falls back to
// the field-by-field path, which accepts exactly the same bytes (the fused literal is one of its spellings).

// -------------------------------------------------------------------------------------------------
// Strings.  pos is AT the opening quote; on success pos is just after the closing quote and
// `out` is the content span.  Accepts exactly the canonical spelling pydantic-core emits:
// raw bytes >= 0x20 except " and \, valid UTF-8 (no surrogates / overlongs / > U+10FFFF),
// escapes \" \\ \n \t \r \b \f, and \u00XX (lower-case hex) only for the other controls.
// -------------------------------------------------------------------------------------------------
template <class R>
CK_HD bool ck_utf8_seq(R& r, u32& pos) {       // pos at a byte >= 0x80
    u8 c = r.at(pos);
    u32 need; u8 lo = 0x80, hi = 0xBF;
    if (c >= 0xC2 && c <= 0xDF) need = 1;
    else if (c == 0xE0) { need = 2; lo = 0xA0; }
    else if (c >= 0xE1 && c <= 0xEC) need = 2;
    else if (c == 0xED) { need = 2; hi = 0x9F; }
    else if (c >= 0xEE && c <= 0xEF) need = 2;
    else if (c == 0xF0) { need = 3; lo = 0x90; }
    else if (c >= 0xF1 && c <= 0xF3) need = 3;
    else if (c == 0xF4) { need = 3; hi = 0x8F; }
    else return false;
    if (pos + need >= r.n) return false;
    u8 c1 = r.at(pos + 1);
    if (c1 < lo || c1 > hi) return false;
    for (u32 k = 2; k <= need; k++) { u8 ck = r.at(pos + k); if (ck < 0x80 || ck > 0xBF) return false; }
    pos += need + 1;
    return true;
}

// returns the position just after the closing quote, 0 on failure.  One out-of-line copy: the
// walker calls it ~100 times per record and the code must stay inside the instruction cache.
template <class R>
CK_HD_NOINLINE u64 ck_string_core(const u8* g, u32 n, u32 pos, u32 st) {
    R r; r.init(g, n, st);
    if (!(pos < r.n) || r.at(pos) != '"') return 0;
    pos++;
    for (;;) {
        if (pos >= r.n) return false;
        u64 x = r.load8(pos);
        u64 special = (x & CK_REP8(0x80)) | ck_haszero(x ^ CK_REP8('"')) | ck_haszero(x ^ CK_REP8('\\')) | ck_lt20(x);
        if (special == 0) { pos += 8; continue; }
        u32 bi = ck_ctz64(special) >> 3;
        pos += bi;
        if (pos >= r.n) return false;
        // the special byte and what follows it in the word already loaded: multi-byte sequences and the two-character
        // escapes that lie inside it are checked from the register (text in other scripts has one every few bytes)
        u64 y = x >> (8 * bi);
        u32 avail = 8 - bi;
        u8 c = (u8)y;
        if (c == '"') return CK_RET(pos + 1);
        if (c >= 0x80) {
            u32 need; u32 lo = 0x80, hi = 0xBF;
            if (c >= 0xC2 && c <= 0xDF) need = 1;
            else if (c >= 0xE0 && c <= 0xEF) { need = 2; if (c == 0xE0) lo = 0xA0; if (c == 0xED) hi = 0x9F; }
            else if (c >= 0xF0 && c <= 0xF4) { need = 3; if (c == 0xF0) lo = 0x90; if (c == 0xF4) hi = 0x8F; }
            else return false;
            if (need < avail) {
                if (pos + need >= r.n) return false;
                u32 c1 = (u32)(y >> 8) & 0xFFu;
                if (c1 < lo || c1 > hi) return false;
                if (need >= 2) { u32 c2 = (u32)(y >> 16) & 0xFFu; if (c2 < 0x80 || c2 > 0xBF) return false; }
                if (need == 3) { u32 c3 = (u32)(y >> 24) & 0xFFu; if (c3 < 0x80 || c3 > 0xBF) return false; }
                pos += need + 1;
                continue;
            }
            if (!ck_utf8_seq(r, pos)) return false;         // the sequence crosses the word: byte by byte
            continue;
        }
        if (c == '\\' && avail >= 2) {
            u8 e = (u8)(y >> 8);
            if (e == '"' || e == '\\' || e == 'n' || e == 't' || e == 'r' || e == 'b' || e == 'f') { if (pos + 1 >= r.n) return false; pos += 2; continue; }
        }
        if (c == '\\') {
            if (pos + 1 >= r.n) return false;
            u8 e = r.at(pos + 1);
            if (e == '"' || e == '\\' || e == 'n' || e == 't' || e == 'r' || e == 'b' || e == 'f') { pos += 2; continue; }
            if (e != 'u' || pos + 5 >= r.n) return false;
            if (r.at(pos + 2) != '0' || r.at(pos + 3) != '0') return false;
            u8 h1 = r.at(pos + 4), h2 = r.at(pos + 5);
            if (h1 != '0' && h1 != '1') return false;
            u32 v;
            if (h2 >= '0' && h2 <= '9') v = h2 - '0';
            else if (h2 >= 'a' && h2 <= 'f') v = h2 - 'a' + 10;
            else return false;
            v |= (u32)(h1 - '0') << 4;
            if (v == 8 || v == 9 || v == 10 || v == 12 || v == 13) return false;   // have short forms
            pos += 6;
            continue;
        }
        if (c < 0x20) return false;
        if (!ck_utf8_seq(r, pos)) return false;
    }
}

template <class R>
CK_HD bool ck_string(R& r, u32& pos, Span& out) {
    CK_CALL(e, ck_string_core<R>(r.g, r.n, pos, r.st()));
    out.off = pos + 1; out.len = e - pos - 2; pos = e;
    return true;
}

template <class R>
CK_HD bool ck_null(R& r, u32& pos) { return M("null"); }

template <class R>
CK_HD bool ck_string_or_null(R& r, u32& pos, Span& out) {
    if (PEEK('n')) { out.off = pos; out.len = 0; return ck_null(r, pos); }
    return ck_string(r, pos, out);
}

// -------------------------------------------------------------------------------------------------
// Numbers.  Canonical ints: -?(0|[1-9][0-9]*) except "-0".  Floats are accepted only in the
// positional spelling whose round trip is provable without a shortest-digits printer:
// -?INT.FRAC with <= 15 significant digits, no trailing fractional zero (except the single ".0"),
// magnitude in [1e-5, 1e16)  (DBL_DIG argument, DESIGN.md §canonical numbers); with 16 or 17 digits the literal
// is left to the canonicaliser, which applies the exact "is repr of its double" test of ck_float.cuh.
// -------------------------------------------------------------------------------------------------
template <class R>
CK_HD_NOINLINE u64 ck_number_core(const u8* g, u32 n, u32 pos, u32 st, bool allow_int, bool allow_float) {
    R r; r.init(g, n, st);
    u32 p = pos;
    bool neg = false;
    if (p < r.n && r.at(p) == '-') { neg = true; p++; }
    if (p >= r.n) return false;
    u8 c = r.at(p);
    if (c < '0' || c > '9') return false;
    u32 int_start = p;
    bool int_zero = (c == '0');
    p++;
    if (!int_zero) { while (p < r.n) { u8 d = r.at(p); if (d < '0' || d > '9') break; p++; } }
    else if (p < r.n) { u8 d = r.at(p); if (d >= '0' && d <= '9') return false; }   // leading zero
    u32 int_len = p - int_start;
    bool is_float = false;
    u32 frac_start = 0, frac_len = 0;
    if (p < r.n && r.at(p) == '.') {
        is_float = true;
        p++;
        frac_start = p;
        while (p < r.n) { u8 d = r.at(p); if (d < '0' || d > '9') break; p++; }
        frac_len = p - frac_start;
        if (frac_len == 0) return false;
    }
    if (p < r.n && r.at(p) == 'e') {
        // canonical scientific spelling d[.ddd]e[+-]X: what the reference prints outside [1e-5, 1e16).  A fixed
        // point when it has <= 15 significant digits, no trailing fractional zero, the exponent is in the range
        // that is printed this way, and the value is far from overflow / subnormals (DBL_DIG argument).
        if (!allow_float || int_zero || int_len != 1) return false;
        if (is_float && r.at(frac_start + frac_len - 1) == '0') return false;
        if (1 + frac_len > (R::kTrustFloats ? 17u : 15u)) return false;     // 16-17 digits: the canonicaliser decides (WRdT)
        p++;
        if (p >= r.n) return false;
        u8 sg = r.at(p);
        if (sg != '+' && sg != '-') return false;
        p++;
        if (p >= r.n) return false;
        u8 d0 = r.at(p);
        if (d0 < '1' || d0 > '9') return false;
        u32 x = 0, xl = 0;
        while (p < r.n) { u8 d = r.at(p); if (d < '0' || d > '9') break; x = x * 10 + (u32)(d - '0'); p++; if (++xl > 3) return false; }
        // (second walk, over the canonicaliser's own output: it has decided the extremes exactly, e-324 .. e+308)
        if (x > (R::kTrustFloats ? (sg == '-' ? 324u : 308u) : 290u) || (sg == '-' ? x < 6 : x < 16)) return false;
        return CK_RET(p);
    }
    if (p < r.n && r.at(p) == 'E') return false;
    if (!is_float) {
        if (!allow_int) return false;
        if (neg && int_zero) return false;          // "-0" re-emits as "0"
        if (int_len > 4000) return false;           // CPython int<->str digit limit is 4300
        return CK_RET(p);
    }
    if (!allow_float) return false;
    if (int_len > 16) return false;
    u8 last = r.at(frac_start + frac_len - 1);
    if (last == '0' && frac_len != 1) return false;
    // significant digits: from the first non-zero digit to the last non-zero digit
    u32 sig;
    if (!int_zero) {
        if (frac_len == 1 && last == '0') {         // INT.0 : trailing integer zeros are not significant
            u32 q = int_start + int_len;
            u32 tz = 0;
            while (tz < int_len && r.at(q - 1 - tz) == '0') tz++;
            sig = int_len - tz;
        } else sig = int_len + frac_len;
    } else {
        u32 lz = 0;
        while (lz < frac_len && r.at(frac_start + lz) == '0') lz++;
        if (lz == frac_len) { if (frac_len != 1) return false; sig = 1; }   // 0.0 / -0.0 only
        else { if (lz > 4) return false; sig = frac_len - lz; }             // < 1e-5 prints as 1e-6 ...
    }
    // 16-17 significant digits (computed values such as 0.30000000000000004) are a fixed point iff the literal is
    // exactly what the shortest-round-trip printer emits for its double: decided by the canonicaliser in exact
    // integer arithmetic (ck_float.cuh); this walk accepts them only on its say-so (WRdT)
    if (sig > (R::kTrustFloats ? 17u : 15u)) return false;
    return CK_RET(p);
}
template <class R>
CK_HD bool ck_number(R& r, u32& pos, bool allow_int, bool allow_float) {
    CK_CALL(e, ck_number_core<R>(r.g, r.n, pos, r.st(), allow_int, allow_float));
    pos = e;
    return true;
}


// -------------------------------------------------------------------------------------------------
// Generic canonical JSON value ("Any" subtrees: provided_deps, args, metadata, return_value ...).
// Iterative (explicit container bit-stack); duplicate keys make a value non-canonical because the
// reference re-emits a Python dict, so each open object keeps 32-bit key hashes in a small stack.
// -------------------------------------------------------------------------------------------------
#define CK_MAX_DEPTH 208         // array sizes; the rule itself: a value enclosed by more than 200 containers is json_invalid
#define CK_KEYSTACK 64
#define CK_DICT_KEYS 128     // tool_calls / tool_results entries handled on the fast path

struct AnyCtx {
    u32 kind[(CK_MAX_DEPTH + 31) / 32]; // bit = 1: object, 0: array
    u32 khash[CK_KEYSTACK];
    u8  kbase[CK_MAX_DEPTH];            // khash fill level when the object at this depth was opened
    u32 kfill;
};

// hash of a key span, eight bytes a step (equal spans -> equal hashes is all the duplicate checks and the key tables
// need; every hit is confirmed by a byte compare or sends the record to the canonicaliser)
template <class R>
CK_HD u32 ck_hash_span(R& r, u32 off, u32 len) {
    u32 h = 2166136261u ^ len;
    u32 i = 0;
    for (; i + 8 <= len; i += 8) {
        u64 w = r.load8(off + i);
        h = (h ^ (u32)w) * 16777619u;
        h = (h ^ (u32)(w >> 32)) * 16777619u;
    }
    if (i < len) {
        u64 w = r.load8(off + i) & (~0ull >> (8 * (8 - (len - i))));
        h = (h ^ (u32)w) * 16777619u;
        h = (h ^ (u32)(w >> 32)) * 16777619u;
    }
    return h ^ (h >> 15);
}

// two spans of the same length, byte-equal?  Eight bytes a step through two readers (each keeps its own cached word)
template <class RA, class RB>
CK_HD bool ck_spans_equal(RA& ra, u32 a, RB& rb, u32 b, u32 len) {
    u64 diff = 0;
    u32 i = 0;
    for (; i + 8 <= len; i += 8) diff |= ra.load8(a + i) ^ rb.load8(b + i);
    if (i < len) diff |= (ra.load8(a + i) ^ rb.load8(b + i)) & (~0ull >> (8 * (8 - (len - i))));
    return diff == 0;
}

// base_depth: nesting level of the value inside the document (root object = depth 1)
template <class R>
CK_HD_NOINLINE u64 ck_any_core(const u8* g, u32 n, u32 pos, u32 st, u32 base_depth, AnyCtx* cxp) {
    R r; r.init(g, n, st);
    AnyCtx& cx = *cxp;
    u32 depth = 0;
    cx.kfill = 0;
    Span s;
    for (;;) {
        // ---- parse a value (nesting index = base_depth - 1 + depth must not exceed jiter's 200)
        if (pos >= r.n) return false;
        if (base_depth + depth > 201) return false;
        u8 c = r.at(pos);
        bool opened = false;
        if (c == '{' || c == '[') {
            bool is_obj = (c == '{');
            if (is_obj) cx.kind[depth >> 5] |= (1u << (depth & 31)); else cx.kind[depth >> 5] &= ~(1u << (depth & 31));
            cx.kbase[depth] = (u8)cx.kfill;
            depth++; pos++;
            if (pos >= r.n) return false;
            u8 d = r.at(pos);
            if (d == (is_obj ? '}' : ']')) { pos++; depth--; cx.kfill = cx.kbase[depth]; }
            else opened = true;
        } else if (c == '"') { if (!ck_string(r, pos, s)) return false; }
        else if (c == 't') { if (!M("true")) return false; }
        else if (c == 'f') { if (!M("false")) return false; }
        else if (c == 'n') { if (!M("null")) return false; }
        else { if (!ck_number(r, pos, true, true)) return false; }

        // ---- what follows
        for (;;) {
            bool in_obj;
            if (opened) { in_obj = (cx.kind[(depth - 1) >> 5] >> ((depth - 1) & 31)) & 1; opened = false;
                          if (!in_obj) break; /* array: first element */ }
            else {
                if (depth == 0) return CK_RET(pos);
                in_obj = (cx.kind[(depth - 1) >> 5] >> ((depth - 1) & 31)) & 1;
                if (pos >= r.n) return false;
                u8 d = r.at(pos);
                if (d == (in_obj ? '}' : ']')) { pos++; depth--; cx.kfill = cx.kbase[depth]; continue; }
                if (d != ',') return false;
                pos++;
                if (!in_obj) break;                 // next array element
            }
            // object member: key, duplicate check, colon
            if (!ck_string(r, pos, s)) return false;
            u32 h = ck_hash_span(r, s.off, s.len);
            for (u32 k = cx.kbase[depth - 1]; k < cx.kfill; k++) if (cx.khash[k] == h) return false;
            if (cx.kfill >= CK_KEYSTACK) return false;
            cx.khash[cx.kfill++] = h;
            if (!(pos < r.n) || r.at(pos) != ':') return false;
            pos++;
            break;
        }
    }
}

template <class R>
CK_HD bool ck_any(R& r, u32& pos, u32 base_depth, AnyCtx& cx) {
    CK_CALL(e, ck_any_core<R>(r.g, r.n, pos, r.st(), base_depth, &cx));
    pos = e;
    return true;
}
template <class R>
CK_HD bool ck_any_obj(R& r, u32& pos, u32 d, AnyCtx& cx) { return PEEK('{') && ck_any(r, pos, d, cx); }
template <class R>
CK_HD bool ck_any_obj_or_null(R& r, u32& pos, u32 d, AnyCtx& cx) { return PEEK('n') ? ck_null(r, pos) : ck_any_obj(r, pos, d, cx); }

// -------------------------------------------------------------------------------------------------
// datetime: the spellings pydantic re-emits unchanged:
//   YYYY-MM-DDTHH:MM:SS[.ffffff](Z | +HH:MM | -HH:MM | <naive>)   fraction: 6 digits, not 000000;
//   offset != 00:00 (that prints as Z); calendar-valid date; year >= 1.
// -------------------------------------------------------------------------------------------------
template <class R>
CK_HD bool ck_2d(R& r, u32 p, u32& v) {
    u8 a = r.at(p), b = r.at(p + 1);
    if (a < '0' || a > '9' || b < '0' || b > '9') return false;
    v = (u32)(a - '0') * 10 + (u32)(b - '0');
    return true;
}
template <class R>
CK_HD_NOINLINE u64 ck_datetime_core(const u8* g, u32 n, u32 pos, u32 st) {
    R r; r.init(g, n, st);
    u32 p = pos;
    if (p + 21 > r.n) return false;                 // "YYYY-MM-DDTHH:MM:SS" + quotes
    if (r.at(p) != '"') return false;
    p++;
    u32 y1, y2, mo, d, h, mi, s;
    if (!ck_2d(r, p, y1) || !ck_2d(r, p + 2, y2) || r.at(p + 4) != '-' || !ck_2d(r, p + 5, mo) || r.at(p + 7) != '-' ||
        !ck_2d(r, p + 8, d) || r.at(p + 10) != 'T' || !ck_2d(r, p + 11, h) || r.at(p + 13) != ':' ||
        !ck_2d(r, p + 14, mi) || r.at(p + 16) != ':' || !ck_2d(r, p + 17, s)) return false;
    u32 y = y1 * 100 + y2;
    if (y < 1 || mo < 1 || mo > 12 || d < 1 || h > 23 || mi > 59 || s > 59) return false;
    u32 dim = (mo == 2) ? (((y % 4 == 0 && y % 100 != 0) || y % 400 == 0) ? 29 : 28)
                        : ((mo == 4 || mo == 6 || mo == 9 || mo == 11) ? 30 : 31);
    if (d > dim) return false;
    p += 19;
    if (p >= r.n) return false;
    u8 c = r.at(p);
    if (c == '.') {
        if (p + 7 >= r.n) return false;
        bool nz = false;
        for (u32 k = 1; k <= 6; k++) { u8 f = r.at(p + k); if (f < '0' || f > '9') return false; nz |= (f != '0'); }
        if (!nz) return false;
        p += 7;
        c = r.at(p);
    }
    if (c == 'Z') { p++; if (p >= r.n) return false; c = r.at(p); }
    else if (c == '+' || c == '-') {
        if (p + 6 >= r.n) return false;
        u32 oh, om;
        if (!ck_2d(r, p + 1, oh) || r.at(p + 3) != ':' || !ck_2d(r, p + 4, om)) return false;
        if (oh > 23 || om > 59 || (oh == 0 && om == 0)) return false;
        p += 6;
        c = r.at(p);
    }
    if (c != '"') return false;
    return CK_RET(p + 1);
}
template <class R>
CK_HD bool ck_datetime(R& r, u32& pos) {
    CK_CALL(e, ck_datetime_core<R>(r.g, r.n, pos, r.st()));
    pos = e;
    return true;
}
template <class R>
CK_HD bool ck_datetime_or_null(R& r, u32& pos) { return PEEK('n') ? ck_null(r, pos) : ck_datetime(r, pos); }

template <class R>
CK_HD bool ck_bool(R& r, u32& pos) { return PEEK('t') ? M("true") : M("false"); }

// -------------------------------------------------------------------------------------------------
// Typed pieces of the Envelope schema, in canonical key order (SURVEY.md Appendix A).
// `d` = nesting depth of the value being recognised.
// -------------------------------------------------------------------------------------------------
struct ToolCallSpans { Span tool_name, args, tool_call_id; };

// ToolCallPart / BuiltinToolCallPart (reference _vendor/pydantic_ai/messages.py:1187-1283)
// returns 1 = tool-call, 2 = builtin-tool-call, 0 = no match
template <class R>
CK_HD u32 ck_tool_call_part(R& r, u32& pos, u32 d, AnyCtx& cx, ToolCallSpans& o) {
    Span t;
    if (!M("{\"tool_name\":") || !ck_string(r, pos, o.tool_name) || !M(",\"args\":")) return 0;
    o.args.off = pos;
    if (PEEK('"')) { if (!ck_string(r, pos, t)) return 0; }
    else if (!ck_any_obj_or_null(r, pos, d + 1, cx)) return 0;
    o.args.len = pos - o.args.off;
    if (!M(",\"tool_call_id\":") || !ck_string(r, pos, o.tool_call_id)) return 0;
    if (M(",\"id\":null,\"provider_name\":null,\"provider_details\":null,\"part_kind\":\"tool-call\"}")) return 1;
    if (!M(",\"id\":") || !ck_string_or_null(r, pos, t) ||
        !M(",\"provider_name\":") || !ck_string_or_null(r, pos, t) || !M(",\"provider_details\":") ||
        !ck_any_obj_or_null(r, pos, d + 1, cx) || !M(",\"part_kind\":\"")) return 0;
    if (M("tool-call\"}")) return 1;
    if (M("builtin-tool-call\"}")) return 2;
    return 0;
}

// message parts.  Returns 1 for a request-side part, 2 for a response-side part, 0 = no match.
// (request: system-prompt / user-prompt / tool-return / retry-prompt, messages.py:112,739,883,918;
//  response: text / tool-call / builtin-tool-call / builtin-tool-return / thinking, :1059-1283)
template <class R>
CK_HD u32 ck_message_part(R& r, u32& pos, u32 d, AnyCtx& cx) {
    Span t;
    if (M("{\"content\":")) {
        // content-first parts: system-prompt, user-prompt, retry-prompt (request) | text, thinking (response)
        bool content_is_str = PEEK('"');
        bool content_is_strlist = false;
        if (content_is_str) { if (!ck_string(r, pos, t)) return 0; }
        else {                                         // user-prompt may carry list[str]
            if (!M("[")) return 0;
            if (!PEEK(']')) { for (;;) { if (!ck_string(r, pos, t)) return 0; if (PEEK(',')) { pos++; continue; } break; } }
            if (!M("]")) return 0;
            content_is_strlist = true;
        }
        if (M(",\"timestamp\":")) {
            if (!ck_datetime(r, pos)) return 0;
            if (M(",\"dynamic_ref\":")) {
                if (content_is_strlist) return 0;
                if (!ck_string_or_null(r, pos, t) || !M(",\"name\":") || !ck_string_or_null(r, pos, t) ||
                    !M(",\"part_kind\":\"system-prompt\"}")) return 0;
                return 1;
            }
            if (M(",\"name\":null,\"part_kind\":\"user-prompt\"}")) return 1;
            if (!M(",\"name\":") || !ck_string_or_null(r, pos, t) || !M(",\"part_kind\":\"user-prompt\"}")) return 0;
            return 1;
        }
        if (content_is_strlist) return 0;
        if (M(",\"tool_name\":")) {                   // retry-prompt (str content only on the fast path)
            if (!ck_string_or_null(r, pos, t) || !M(",\"tool_call_id\":") || !ck_string(r, pos, t) ||
                !M(",\"timestamp\":") || !ck_datetime(r, pos) || !M(",\"part_kind\":\"retry-prompt\"}")) return 0;
            return 1;
        }
        if (!M(",\"id\":") || !ck_string_or_null(r, pos, t)) return 0;
        bool thinking = false;
        if (M(",\"signature\":")) { thinking = true; if (!ck_string_or_null(r, pos, t)) return 0; }
        if (!M(",\"provider_name\":") || !ck_string_or_null(r, pos, t) || !M(",\"provider_details\":") ||
            !ck_any_obj_or_null(r, pos, d + 1, cx)) return 0;
        if (thinking) return M(",\"part_kind\":\"thinking\"}") ? 2 : 0;
        return M(",\"part_kind\":\"text\"}") ? 2 : 0;
    }
    // tool_name-first parts: tool-return (request) | tool-call, builtin-tool-call, builtin-tool-return (response)
    u32 save = pos;
    if (!M("{\"tool_name\":") || !ck_string(r, pos, t)) return 0;
    if (M(",\"content\":")) {
        if (!ck_any(r, pos, d + 1, cx) || !M(",\"tool_call_id\":") || !ck_string(r, pos, t) || !M(",\"metadata\":") ||
            !ck_any(r, pos, d + 1, cx) || !M(",\"timestamp\":") || !ck_datetime(r, pos)) return 0;
        if (M(",\"part_kind\":\"tool-return\"}")) return 1;
        if (!M(",\"provider_name\":") || !ck_string_or_null(r, pos, t) || !M(",\"provider_details\":") ||
            !ck_any_obj_or_null(r, pos, d + 1, cx) || !M(",\"part_kind\":\"builtin-tool-return\"}")) return 0;
        return 2;
    }
    pos = save;
    ToolCallSpans tc;
    return ck_tool_call_part(r, pos, d, cx, tc) ? 2 : 0;
}

// RequestUsage (reference _vendor/pydantic_ai/usage.py)
template <class R>
CK_HD bool ck_usage(R& r, u32& pos, AnyCtx& cx) {
    Span t;
    if (!M("{\"input_tokens\":") || !ck_number(r, pos, true, false) || !M(",\"cache_write_tokens\":") || !ck_number(r, pos, true, false) ||
        !M(",\"cache_read_tokens\":") || !ck_number(r, pos, true, false) || !M(",\"output_tokens\":") || !ck_number(r, pos, true, false) ||
        !M(",\"input_audio_tokens\":") || !ck_number(r, pos, true, false) || !M(",\"cache_audio_read_tokens\":") ||
        !ck_number(r, pos, true, false) || !M(",\"output_audio_tokens\":") || !ck_number(r, pos, true, false) || !M(",\"details\":{")) return false;
    if (!PEEK('}')) {
        cx.kfill = 0;
        for (;;) {
            if (!ck_string(r, pos, t)) return false;
            u32 h = ck_hash_span(r, t.off, t.len);
            for (u32 k = 0; k < cx.kfill; k++) if (cx.khash[k] == h) return false;
            if (cx.kfill >= CK_KEYSTACK) return false;
            cx.khash[cx.kfill++] = h;
            if (!M(":") || !ck_number(r, pos, true, false)) return false;
            if (PEEK(',')) { pos++; continue; }
            break;
        }
    }
    return M("}}");
}

// ModelMessage = ModelRequest | ModelResponse (messages.py:1014-1041, :1292-1345, :1554).
// returns 1 = request, 2 = response, 0 = no match
template <class R>
CK_HD_NOINLINE u64 ck_message_core(const u8* g, u32 n, u32 pos, u32 st, u32 d, AnyCtx* cxp) {   // -> end | kind << 30
    R r; r.init(g, n, st);
    AnyCtx& cx = *cxp;
    Span t;
    if (!M("{\"parts\":[")) return 0;
    u32 seen = 0;
    if (!PEEK(']')) {
        bool par = false;
        if constexpr (R::kWarp) {
            // a message of message_history (d == 5): its parts are list elements at depth 6 — one lane each
            u32 q, s0, k;
            if (d == 5 && ck_lx_range(r.lx(), 1, pos, q, s0, k) && k + 1 >= CK_LX_MIN) {
                par = true;
                const ck_long_index* lx = r.lx();
                bool good = true;
                for (u32 base = 0; base <= k; base += 32) {
                    u32 e = base + ck_lane(), kind = 0;
                    bool ok = true;
                    if (e <= k) {
                        u32 p = e ? lx->sep[1][s0 + e - 1] + 1 : pos, tend = e == k ? q : lx->sep[1][s0 + e];
                        R lr; lr.init(r.g, r.n, 0);
                        kind = ck_message_part(lr, p, d + 2, cx);
                        ok = kind != 0 && p == tend;
                    }
                    good = ck_all(ok) && good;
                    seen |= ck_or_reduce(kind);
                }
                if (!good) return 0;
                pos = q;
            }
        }
        if (!par) {
        for (;;) {
            u32 k = ck_message_part(r, pos, d + 2, cx);
            if (!k) return 0;
            seen |= k;
            if (PEEK(',')) { pos++; continue; }
            break;
        }
        }
    }
    if (!M("]")) return 0;
    u32 kind;
    if (M(",\"timestamp\":")) {
        if (seen & 2) return 0;
        if (!ck_datetime_or_null(r, pos)) return 0;
        if (M(",\"instructions\":null,\"kind\":\"request\",\"run_id\":null,\"metadata\":null}")) return CK_RET(pos | (1u << 30));
        if (!M(",\"instructions\":") || !ck_string_or_null(r, pos, t) ||
            !M(",\"kind\":\"request\",\"run_id\":") || !ck_string_or_null(r, pos, t) || !M(",\"metadata\":") ||
            !ck_any_obj_or_null(r, pos, d + 1, cx) || !M("}")) return 0;
        kind = 1;
    } else {
        if (seen & 1) return 0;
        if (!M(",\"usage\":") || !ck_usage(r, pos, cx) || !M(",\"model_name\":") || !ck_string_or_null(r, pos, t) ||
            !M(",\"name\":") || !ck_string_or_null(r, pos, t) || !M(",\"timestamp\":") || !ck_datetime(r, pos) ||
            !M(",\"kind\":\"response\",\"provider_name\":") || !ck_string_or_null(r, pos, t) || !M(",\"provider_url\":") ||
            !ck_string_or_null(r, pos, t) || !M(",\"provider_details\":") || !ck_any_obj_or_null(r, pos, d + 1, cx) ||
            !M(",\"provider_response_id\":") || !ck_string_or_null(r, pos, t) || !M(",\"finish_reason\":")) return 0;
        if (!PEEK('n')) {
            if (!(M("\"stop\"") || M("\"length\"") || M("\"content_filter\"") || M("\"tool_call\"") || M("\"error\""))) return 0;
        } else if (!ck_null(r, pos)) return 0;
        if (!M(",\"run_id\":") || !ck_string_or_null(r, pos, t) || !M(",\"metadata\":") ||
            !ck_any_obj_or_null(r, pos, d + 1, cx) || !M("}")) return 0;
        kind = 2;
    }
    return CK_RET(pos | (kind << 30));
}
template <class R>
CK_HD u32 ck_message(R& r, u32& pos, u32 d, AnyCtx& cx) {
    CK_CALL(e, ck_message_core<R>(r.g, r.n, pos, r.st(), d, &cx));
    pos = e & 0x3fffffffu;
    return e >> 30;
}

// ToolDefinition (reference _vendor/pydantic_ai/tools.py:474-540)
template <class R>
CK_HD bool ck_tool_definition(R& r, u32& pos, u32 d, AnyCtx& cx) {
    Span t;
    if (!M("{\"name\":") || !ck_string(r, pos, t) || !M(",\"parameters_json_schema\":") || !ck_any_obj(r, pos, d + 1, cx) ||
        !M(",\"description\":") || !ck_string_or_null(r, pos, t) || !M(",\"outer_typed_dict_key\":") || !ck_string_or_null(r, pos, t) ||
        !M(",\"strict\":")) return false;
    if (PEEK('n')) { if (!ck_null(r, pos)) return false; } else if (!ck_bool(r, pos)) return false;
    if (!M(",\"sequential\":") || !ck_bool(r, pos) || !M(",\"kind\":\"")) return false;
    if (!(M("function\"") || M("output\"") || M("external\"") || M("unapproved\""))) return false;
    if (!M(",\"metadata\":") || !ck_any_obj_or_null(r, pos, d + 1, cx) || !M(",\"timeout\":")) return false;
    if (PEEK('n')) { if (!ck_null(r, pos)) return false; } else if (!ck_number(r, pos, false, true)) return false;
    return M("}");
}

// OverridesState | null (reference calfkit/models/state.py:22-26, node_schema.py:6-21)
template <class R>
CK_HD_NOINLINE u64 ck_overrides_core(const u8* g, u32 n, u32 pos, u32 st, u32 d, AnyCtx* cxp) {
    R r; r.init(g, n, st);
    AnyCtx& cx = *cxp;
    Span t;
    if (PEEK('n')) { if (!ck_null(r, pos)) return 0; return CK_RET(pos); }
    if (!M("{\"override_agent_tools\":")) return false;
    if (PEEK('n')) { if (!ck_null(r, pos)) return false; }
    else {
        if (!M("[")) return false;
        if (!PEEK(']')) {
            for (;;) {
                if (!M("{\"node_id\":") || !ck_string(r, pos, t) || !M(",\"subscribe_topics\":[")) return false;
                if (!PEEK(']')) { for (;;) { if (!ck_string(r, pos, t)) return false; if (PEEK(',')) { pos++; continue; } break; } }
                if (!M("],\"publish_topic\":") || !ck_string_or_null(r, pos, t) || !M(",\"tool_schema\":") ||
                    !ck_tool_definition(r, pos, d + 3, cx) || !M("}")) return false;
                if (PEEK(',')) { pos++; continue; }
                break;
            }
        }
        if (!M("]")) return false;
    }
    if (!M("}")) return 0;
    return CK_RET(pos);
}
template <class R>
CK_HD bool ck_overrides_or_null(R& r, u32& pos, u32 d, AnyCtx& cx) {
    CK_CALL(e, ck_overrides_core<R>(r.g, r.n, pos, r.st(), d, &cx));
    pos = e;
    return true;
}

// final_output_parts element (reference calfkit/models/payload.py:6-35): `kind` comes first.
// returns 0 = no match, 1 = text (val = the `text` JSON string, quotes included), 2 = data (val = the `data` value),
// 3 = file / tool part
template <class R>
CK_HD u32 ck_content_part(R& r, u32& pos, u32 d, AnyCtx& cx, Span& val) {
    Span t;
    if (!M("{\"kind\":\"")) return 0;
    if (M("text\",\"text\":")) {
        val.off = pos;
        bool ok = ck_string(r, pos, t);
        val.len = pos - val.off;
        return (ok && M(",\"metadata\":") && ck_any_obj_or_null(r, pos, d + 1, cx) && M("}")) ? 1u : 0u;
    }
    if (M("data\",\"data\":")) {
        // the field's alias is "schema": a "schema_" key is ignored on validation and re-emitted as null
        // (SURVEY.md Appendix C item 2), so only null is a fixed point
        val.off = pos;
        bool ok = ck_any(r, pos, d + 1, cx);
        val.len = pos - val.off;
        if (!ok) return 0;
        if (!M(",\"schema_\":null,\"metadata\":")) {
            // a non-null schema_ is what the reference dumps when the value came in through the alias; it is not a fixed point
            // (validation ignores the key), so only the canonicaliser's own output is taken at its word
            if (!R::kTrustFloats || !M(",\"schema_\":") || !ck_any(r, pos, d + 1, cx) || !M(",\"metadata\":")) return 0;
        }
        return (ck_any_obj_or_null(r, pos, d + 1, cx) && M("}")) ? 2u : 0u;
    }
    if (M("file\",\"media_type\":")) {
        return (ck_string(r, pos, t) && M(",\"uri\":") && ck_string_or_null(r, pos, t) && M(",\"data\":") &&
                ck_string_or_null(r, pos, t) && M(",\"metadata\":") && ck_any_obj_or_null(r, pos, d + 1, cx) && M("}")) ? 3u : 0u;
    }
    if (M("tool\",\"tool_call_id\":")) {
        return (ck_string(r, pos, t) && M(",\"kwargs\":") && ck_any_obj(r, pos, d + 1, cx) && M(",\"tool_name\":") &&
                ck_string(r, pos, t) && M(",\"metadata\":") && ck_any_obj_or_null(r, pos, d + 1, cx) && M("}")) ? 3u : 0u;
    }
    return 0;
}

// skip one already-validated canonical value (used for second looks at spans proven canonical)
template <class R>
CK_HD void ck_skip_value(R& r, u32& pos) {
    u32 depth = 0;
    for (;;) {
        if (pos >= r.n) return;
        u8 c = r.at(pos);
        if (c == '"') {
            pos++;
            for (;;) {
                if (pos >= r.n) return;
                u8 s = r.at(pos);
                if (s == '\\') { pos += 2; continue; }
                pos++;
                if (s == '"') break;
            }
        } else if (c == '{' || c == '[') { depth++; pos++; continue; }
        else if (c == '}' || c == ']') { depth--; pos++; }
        else if (c == ',' || c == ':') { if (depth == 0) return; pos++; continue; }
        else { pos++; while (pos < r.n) { u8 s = r.at(pos); if (s == ',' || s == '}' || s == ']' || s == ':') break; pos++; } }
        if (depth == 0) return;
    }
}

// tool_results value: ToolReturn | ModelRetry | RetryPromptPart (callable discriminator on
// `kind`, then `part_kind`) with an `| Any` fallback (reference models/state.py:70,
// _vendor/pydantic_ai/tools.py:189-210).  A value is a fixed point if it is the canonical form of
// its tagged model, or if it carries no such tag and is generically canonical.
template <class R>
CK_HD_NOINLINE u64 ck_tool_result_core(const u8* g, u32 n, u32 pos, u32 st, u32 d, AnyCtx* cxp) {
    R r; r.init(g, n, st);
    AnyCtx& cx = *cxp;
    Span t;
    u32 start = pos;
    if (PEEK('{')) {
        if (M("{\"return_value\":")) {
            if (ck_any(r, pos, d + 1, cx) && M(",\"content\":") && ck_string_or_null(r, pos, t) && M(",\"metadata\":") &&
                ck_any(r, pos, d + 1, cx) && M(",\"kind\":\"tool-return\"}")) return CK_RET(pos);
        } else if (M("{\"message\":")) {
            if (ck_string(r, pos, t) && M(",\"kind\":\"model-retry\"}")) return CK_RET(pos);
        } else if (M("{\"content\":")) {
            if (ck_string(r, pos, t) && M(",\"tool_name\":") && ck_string_or_null(r, pos, t) && M(",\"tool_call_id\":") &&
                ck_string(r, pos, t) && M(",\"timestamp\":") && ck_datetime(r, pos) && M(",\"part_kind\":\"retry-prompt\"}")) {
                return CK_RET(pos);
            }
        }
        // not the canonical form of a tagged model: generic value, provided it carries no tag
        pos = start;
        if (!ck_any(r, pos, d, cx)) return false;
        u32 end = pos;
        u32 p = start + 1;
        bool have_kind = false, tagged = false, part_tagged = false;
        while (p < end && r.at(p) != '}') {
            Span k;
            if (!ck_string(r, p, k)) return false;
            p++;                                       // ':'
            u32 v = p;
            ck_skip_value(r, p);
            bool is_kind = (k.len == 4 && r.at(k.off) == 'k' && r.at(k.off + 1) == 'i' && r.at(k.off + 2) == 'n' && r.at(k.off + 3) == 'd');
            u32 q = k.off;
            bool is_pk = (k.len == 9) && ck_match(r, q, "part_kind", 9);
            if (is_kind || is_pk) {
                u32 vv = v;
                bool tag = ck_match(r, vv, "\"tool-return\"", 13) || ck_match(r, vv, "\"model-retry\"", 13) ||
                           ck_match(r, vv, "\"retry-prompt\"", 14);
                tag = tag && (vv == p);
                if (is_kind) { have_kind = true; tagged = tag; } else part_tagged = tag;
            }
            if (p < end && r.at(p) == ',') p++;
        }
        // tagged: it would be validated as the model — not proven here; the canonicaliser emits such a value only after the
        // tagged model failed to validate (smart union -> plain data), so its own output is taken at its word
        if ((have_kind ? tagged : part_tagged) && !R::kTrustFloats) return false;
        return CK_RET(end);
    }
    if (!ck_any(r, pos, d, cx)) return 0;
    return CK_RET(pos);
}
template <class R>
CK_HD bool ck_tool_result_value(R& r, u32& pos, u32 d, AnyCtx& cx) {
    CK_CALL(e, ck_tool_result_core<R>(r.g, r.n, pos, r.st(), d, &cx));
    pos = e;
    return true;
}

// -------------------------------------------------------------------------------------------------
// Whole Envelope.  On success fills cols[] (spans relative to the record start).
// -------------------------------------------------------------------------------------------------
// column sink: device = the SoA table in HBM (lane i of a warp owns element i of every column, so
// a convergent warp writes 128 contiguous bytes per column); host tests = a plain array (stride 1)
struct WalkOut {
    u32* base; size_t stride; bool active = true;       // a warp walking one record: only lane 0 stores
    // message_history of this record, if the pre-scan pass (ck_hist_prescan_kernel) has listed its messages for
    // ck_walk_elems_kernel: position of its '[' and of the matching ']' (0 / 0: walk the list here)
    u32 skip_open = 0, skip_close = 0;
    CK_HD void set(u32 col, u32 v) { if (active) base[(size_t)col * stride] = v; }
};

#define SETSPAN(COL, a, b) do { o.set(COL, (a)); o.set(COL + 1, (b) - (a)); } while (0)

// key `ko` (content offset) of the record equal to bytes [a, a + len): the closing quote, then the bytes (plain global
// loads: two far-apart spans)
CK_HD bool ck_key_is(const u8* g, u32 n, u32 ko, u32 a, u32 len) {
    GRd gr, gq; gr.init(g, n); gq.init(g, n);
    if (ko + len >= n || gr.at(ko + len) != '"') return false;
    return ck_spans_equal(gr, ko, gq, a, len);
}

// keys of one id-keyed dict (tool_calls / tool_results): 32-bit hash (uniqueness check: the reference holds Python
// dicts) + content offset, so that dict[input_args[0]] can be resolved at the end of the walk.  Up to CK_DICT_KEYS
// entries.  A thread walking its record keeps the first CK_DICT_REG keys in registers (statically indexed: no local
// memory) and finds the later ones again by re-scanning the dict from key CK_DICT_REG (values already validated:
// ck_skip_value) — quadratic, but only dicts of more than CK_DICT_REG entries pay it.  A warp walking one record keeps
// the whole table in shared memory (ck_long_index), where its lanes fill it in parallel.
#ifndef CK_DICT_REG
#define CK_DICT_REG 2
#endif
template <class R, bool kShared = R::kWarp>
struct DictKeys {
    u32 kh[CK_DICT_REG], koff[CK_DICT_REG];
    u32 n;           // entries so far
    u32 more;        // opening quote of key CK_DICT_REG
    CK_HD void init(u32*, u32*) { n = 0; more = 0; }
    // does key k (k >= CK_DICT_REG) hash to h?  Calls fn(k, content offset) for each such key until it returns true
    template <class F>
    CK_HD bool scan_more(R& r, u32 h, F fn) {
        u32 p = more;
        for (u32 k = CK_DICT_REG; k < n; k++) {
            u32 q = p;
            ck_skip_value(r, p);                               // the key string
            if (ck_hash_span(r, q + 1, p - q - 2) == h && fn(q + 1)) return true;
            p++;                                               // ':'
            ck_skip_value(r, p);                               // the value
            p++;                                               // ','
        }
        return false;
    }
    // record key `off` with hash h; false: a duplicate (or a hash collision) or too many entries
    CK_HD bool add(R& r, u32 h, u32 off) {
        bool dup = false;
#pragma unroll
        for (u32 k = 0; k < CK_DICT_REG; k++) dup |= (k < n) & (kh[k] == h);
        if (dup || n >= CK_DICT_KEYS) return false;
        if (n > CK_DICT_REG && scan_more(r, h, [](u32) { return true; })) return false;
#pragma unroll
        for (u32 k = 0; k < CK_DICT_REG; k++) if (k == n) { kh[k] = h; koff[k] = off; }
        if (n == CK_DICT_REG) more = off - 1;
        n++;
        return true;
    }
    // index of the first key equal to bytes [a, a + len) (hash h), ~0u if none; ko = its content offset
    CK_HD u32 find(R& r, u32 h, u32 a, u32 len, u32& ko) {
#pragma unroll
        for (u32 k = 0; k < CK_DICT_REG; k++)
            if (k < n && kh[k] == h && ck_key_is(r.g, r.n, koff[k], a, len)) { ko = koff[k]; return k; }
        u32 hit = ~0u;
        if (n > CK_DICT_REG) scan_more(r, h, [&](u32 off) { if (!ck_key_is(r.g, r.n, off, a, len)) return false; ko = off; hit = CK_DICT_REG; return true; });
        return hit;
    }
};
template <class R>
struct DictKeys<R, true> {
    u32 *kh, *koff;
    u32 n;
    CK_HD void init(u32* h, u32* off) { kh = h; koff = off; n = 0; }
    CK_HD bool add(R&, u32 h, u32 off) {
        for (u32 k = 0; k < n; k++) if (kh[k] == h) return false;
        if (n >= CK_DICT_KEYS) return false;
        kh[n] = h; koff[n] = off; n++;
        return true;
    }
    CK_HD u32 find(R& r, u32 h, u32 a, u32 len, u32& ko) {
        for (u32 k = 0; k < n; k++)
            if (kh[k] == h && ck_key_is(r.g, r.n, koff[k], a, len)) { ko = koff[k]; return k; }
        return ~0u;
    }
};

template <class R>
CK_HD bool ck_walk_envelope(R& r, WalkOut& o, AnyCtx& cx, u32& stop) {
    u32 pos = 0;
    Span t;
    stop = 0;
    // keys of the two id-keyed dicts (DictKeys), so that tool_calls[input_args[0]] / tool_results[...] can be resolved
    // at the end of the walk; the key length is re-derived from the closing quote
    DictKeys<R> tck, trk;
    if constexpr (R::kWarp) {          // a warp on one record: the lanes share the key tables (shared memory)
        ck_long_index* lw = r.lxw();
        tck.init(lw->kh[0], lw->koff[0]); trk.init(lw->kh[1], lw->koff[1]);
    } else { tck.init(nullptr, nullptr); trk.init(nullptr, nullptr); }
    ToolCallSpans first_tc = {{0, 0}, {0, 0}, {0, 0}};
    u32 first_tc0 = 0, first_tc1 = 0, first_tr0 = 0, first_tr1 = 0;
#define FAIL do { stop = pos; return false; } while (0)
    // ---- context.state ---------------------------------------------------------------------
    if (!M("{\"context\":{\"state\":{\"tool_calls\":{")) FAIL;
    u32 a = pos - 1;
    if (!PEEK('}')) {
        bool par = false;
        if constexpr (R::kWarp) {
            u32 q, s0, k;
            if (ck_lx_range(r.lx(), 0, pos, q, s0, k) && k + 1 >= CK_LX_MIN) {
                par = true;
                if (k + 1 > CK_DICT_KEYS) FAIL;
                const ck_long_index* lx = r.lx();
                bool good = true;
                for (u32 base = 0; base <= k; base += 32) {
                    u32 e = base + ck_lane(), v0 = 0, v1 = 0;
                    bool ok = true;
                    ToolCallSpans tc = {{0, 0}, {0, 0}, {0, 0}};
                    if (e <= k) {
                        u32 p = e ? lx->sep[0][s0 + e - 1] + 1 : pos, tend = e == k ? q : lx->sep[0][s0 + e];
                        R lr; lr.init(r.g, r.n, 0);
                        Span key;
                        ok = ck_string(lr, p, key) && ck_match(lr, p, ":", 1);
                        v0 = p;
                        ok = ok && ck_tool_call_part(lr, p, 5, cx, tc) == 1 && p == tend;
                        v1 = p;
                        if (ok) { tck.kh[e] = ck_hash_span(lr, key.off, key.len); tck.koff[e] = key.off; }
                    }
                    good = ck_all(ok) && good;
                    if (base == 0) {       // entry 0 (lane 0 of the first round): the common single-call case needs no second look
                        first_tc.tool_name.off = ck_bcast(tc.tool_name.off, 0); first_tc.tool_name.len = ck_bcast(tc.tool_name.len, 0);
                        first_tc.args.off = ck_bcast(tc.args.off, 0); first_tc.args.len = ck_bcast(tc.args.len, 0);
                        first_tc.tool_call_id.off = ck_bcast(tc.tool_call_id.off, 0); first_tc.tool_call_id.len = ck_bcast(tc.tool_call_id.len, 0);
                        first_tc0 = ck_bcast(v0, 0); first_tc1 = ck_bcast(v1, 0);
                    }
                }
                if (!good) FAIL;
                ck_warp_sync();
                bool dup = false;
                for (u32 e = ck_lane(); e <= k; e += 32) for (u32 j = 0; j < e; j++) dup |= (tck.kh[j] == tck.kh[e]);
                if (!ck_all(!dup)) FAIL;
                tck.n = k + 1; pos = q;
            }
        }
        if (!par) {
        // dict[str, ToolCallPart]; keys must be unique (a Python dict on the reference side):
        // 32-bit hashes of the raw key bytes, a (vanishingly rare) collision only costs the fast path
        for (;;) {
            if (!ck_string(r, pos, t)) FAIL;
            if (!tck.add(r, ck_hash_span(r, t.off, t.len), t.off)) FAIL;
            ToolCallSpans tc;
            if (!M(":")) FAIL;
            u32 v0 = pos;
            if (ck_tool_call_part(r, pos, 5, cx, tc) != 1) FAIL;
            if (tck.n == 1) { first_tc = tc; first_tc0 = v0; first_tc1 = pos; }      // the common single-call case needs no second look
            if (PEEK(',')) { pos++; continue; }
            break;
        }
        }
    }
    if (!M("}")) FAIL;
    SETSPAN(CK_COL_TC_OFF, a, pos);

    bool spec_tr = M(",\"tool_results\":{},\"uncommitted_message\":null,\"message_history\":[");
    if (spec_tr) {
        // ,"tool_results":{}  ,"uncommitted_message":null  ,"message_history":[      (lengths 18 / 27 / 20)
        u32 e = pos;
        o.set(CK_COL_TR_OFF, e - 20 - 27 - 2); o.set(CK_COL_TR_LEN, 2);
        o.set(CK_COL_UNC_OFF, e - 20 - 4); o.set(CK_COL_UNC_LEN, 4);
    } else {
    if (!M(",\"tool_results\":{")) FAIL;
    a = pos - 1;
    if (!PEEK('}')) {
        bool par = false;
        if constexpr (R::kWarp) {
            u32 q, s0, k;
            if (ck_lx_range(r.lx(), 0, pos, q, s0, k) && k + 1 >= CK_LX_MIN) {
                par = true;
                if (k + 1 > CK_DICT_KEYS) FAIL;
                const ck_long_index* lx = r.lx();
                bool good = true;
                for (u32 base = 0; base <= k; base += 32) {
                    u32 e = base + ck_lane(), v0 = 0, v1 = 0;
                    bool ok = true;
                    if (e <= k) {
                        u32 p = e ? lx->sep[0][s0 + e - 1] + 1 : pos, tend = e == k ? q : lx->sep[0][s0 + e];
                        R lr; lr.init(r.g, r.n, 0);
                        Span key;
                        ok = ck_string(lr, p, key) && ck_match(lr, p, ":", 1);
                        v0 = p;
                        ok = ok && ck_tool_result_value(lr, p, 5, cx) && p == tend;
                        v1 = p;
                        if (ok) { trk.kh[e] = ck_hash_span(lr, key.off, key.len); trk.koff[e] = key.off; }
                    }
                    good = ck_all(ok) && good;
                    if (base == 0) { first_tr0 = ck_bcast(v0, 0); first_tr1 = ck_bcast(v1, 0); }
                }
                if (!good) FAIL;
                ck_warp_sync();
                bool dup = false;
                for (u32 e = ck_lane(); e <= k; e += 32) for (u32 j = 0; j < e; j++) dup |= (trk.kh[j] == trk.kh[e]);
                if (!ck_all(!dup)) FAIL;
                trk.n = k + 1; pos = q;
            }
        }
        if (!par) {
        for (;;) {
            if (!ck_string(r, pos, t)) FAIL;
            if (!trk.add(r, ck_hash_span(r, t.off, t.len), t.off)) FAIL;
            if (!M(":")) FAIL;
            u32 v0 = pos;
            if (!ck_tool_result_value(r, pos, 5, cx)) FAIL;
            if (trk.n == 1) { first_tr0 = v0; first_tr1 = pos; }
            if (PEEK(',')) { pos++; continue; }
            break;
        }
        }
    }
    if (!M("}")) FAIL;
    SETSPAN(CK_COL_TR_OFF, a, pos);

    if (!M(",\"uncommitted_message\":")) FAIL;
    a = pos;
    if (PEEK('n')) { if (!ck_null(r, pos)) FAIL; } else if (!ck_message(r, pos, 4, cx)) FAIL;
    SETSPAN(CK_COL_UNC_OFF, a, pos);

    if (!M(",\"message_history\":[")) FAIL;
    }
    a = pos - 1;
    if (o.skip_close && o.skip_open == a) pos = o.skip_close;      // the messages are validated one thread each, batch-wide
    else if (!PEEK(']')) {
        bool par = false;
        if constexpr (R::kWarp) {
            u32 q, s0, k;
            if (ck_lx_range(r.lx(), 0, pos, q, s0, k)) {
                const ck_long_index* lx = r.lx();
                // the messages are pure validation (no columns come out of them): hand them to the batch-wide element list —
                // one THREAD per message through the window reader, all long records' messages side by side
                // (ck_walk_elems_kernel; a message that fails there sends its record to the canonicaliser) ...
                bool deferred = false;
                u32 longest = 0;
                for (u32 e = ck_lane(); e <= k; e += 32) { u32 a0 = e ? lx->sep[0][s0 + e - 1] + 1 : pos, a1 = e == k ? q : lx->sep[0][s0 + e]; if (a1 - a0 > longest) longest = a1 - a0; }
                if (lx->defer_list && ck_max_reduce(longest) <= CK_DEFER_MAX) {      // long messages: here, their parts lane-parallel
                    u32 slot = ck_defer_reserve(lx->defer_ctr, k + 1);
                    bool fits = slot <= lx->defer_cap && k + 1 <= lx->defer_cap - slot;
                    for (u32 e = ck_lane(); e <= k; e += 32) {
                        if (slot >= lx->defer_cap || e >= lx->defer_cap - slot) break;
                        ck_elem el;
                        el.rec = fits ? lx->rec : 0xffffffffu;       // a reservation that does not fit is voided
                        el.start = e ? lx->sep[0][s0 + e - 1] + 1 : pos; el.end = e == k ? q : lx->sep[0][s0 + e];
                        lx->defer_list[slot + e] = el;
                    }
                    deferred = fits;
                }
                // ... or, without a list (or with a full one), walk them here, one lane each (short lists: sequentially, below)
                par = deferred || k + 1 >= CK_LX_MIN;
                bool good = true;
                for (u32 base = 0; par && !deferred && base <= k; base += 32) {
                    u32 e = base + ck_lane();
                    bool ok = true;
                    if (e <= k) {
                        u32 p = e ? lx->sep[0][s0 + e - 1] + 1 : pos, tend = e == k ? q : lx->sep[0][s0 + e];
                        R lr; lr.init(r.g, r.n, 0);
                        ok = ck_message(lr, p, 5, cx) != 0 && p == tend;
                    }
                    good = ck_all(ok) && good;
                }
                if (!good) FAIL;
                if (par) pos = q;
            }
        }
        if (!par) {
        for (;;) {
            if (!ck_message(r, pos, 5, cx)) FAIL;
            if (PEEK(',')) { pos++; continue; }
            break;
        }
        }
    }
    if (!M("]")) FAIL;
    SETSPAN(CK_COL_HIST_OFF, a, pos);

    if (M(",\"final_output_parts\":[],\"temp_instructions\":null,\"metadata\":null,\"overrides\":null},\"deps\":{\"correlation_id\":")) {
        // ,"final_output_parts":[]  ,"temp_instructions":null  ,"metadata":null  ,"overrides":null  },"deps":{"correlation_id":
        //  lengths                24                        25               16                17                          27
        u32 e = pos;
        o.set(CK_COL_FOP_OFF, e - 27 - 17 - 16 - 25 - 2); o.set(CK_COL_FOP_LEN, 2);
        o.set(CK_COL_ODATA_OFF, 0); o.set(CK_COL_ODATA_LEN, 0); o.set(CK_COL_OTEXT_OFF, 0); o.set(CK_COL_OTEXT_LEN, 0);
        o.set(CK_COL_TI_OFF, e - 27 - 17 - 16 - 4); o.set(CK_COL_TI_LEN, 4);
        o.set(CK_COL_SMETA_OFF, e - 27 - 17 - 4); o.set(CK_COL_SMETA_LEN, 4);
        o.set(CK_COL_SOV_OFF, e - 27 - 4); o.set(CK_COL_SOV_LEN, 4);
    } else {
    if (!M(",\"final_output_parts\":[")) FAIL;
    a = pos - 1;
    Span odata = {0, 0}, otext = {0, 0};
    if (!PEEK(']')) {
        for (;;) {
            Span val = {0, 0};
            u32 pk = ck_content_part(r, pos, 5, cx, val);
            if (!pk) FAIL;
            if (pk == 1 && otext.len == 0) otext = val;            // first TextPart / first DataPart (client/deserialize.py:63-70)
            if (pk == 2 && odata.len == 0) odata = val;
            if (PEEK(',')) { pos++; continue; }
            break;
        }
    }
    if (!M("]")) FAIL;
    SETSPAN(CK_COL_FOP_OFF, a, pos);
    o.set(CK_COL_ODATA_OFF, odata.off); o.set(CK_COL_ODATA_LEN, odata.len);
    o.set(CK_COL_OTEXT_OFF, otext.off); o.set(CK_COL_OTEXT_LEN, otext.len);

    if (!M(",\"temp_instructions\":")) FAIL;
    a = pos;
    if (!ck_string_or_null(r, pos, t)) FAIL;
    SETSPAN(CK_COL_TI_OFF, a, pos);

    if (!M(",\"metadata\":")) FAIL;
    a = pos;
    if (!ck_any(r, pos, 4, cx)) FAIL;
    SETSPAN(CK_COL_SMETA_OFF, a, pos);

    if (!M(",\"overrides\":")) FAIL;
    a = pos;
    if (!ck_overrides_or_null(r, pos, 4, cx)) FAIL;
    SETSPAN(CK_COL_SOV_OFF, a, pos);

    // ---- context.deps ----------------------------------------------------------------------
    if (!M("},\"deps\":{\"correlation_id\":")) FAIL;
    }
    if (!ck_string(r, pos, t)) FAIL;
    o.set(CK_COL_CORR_OFF, t.off); o.set(CK_COL_CORR_LEN, t.len);
    if (!M(",\"provided_deps\":")) FAIL;
    a = pos;
    if (!ck_any_obj(r, pos, 4, cx)) FAIL;
    SETSPAN(CK_COL_PD_OFF, a, pos);

    // ---- internal_workflow_state -----------------------------------------------------------
    if (!M("}},\"internal_workflow_state\":{\"call_stack\":{\"_internal_list\":[")) FAIL;
    a = pos - 1;
    u32 nframes = 0;
    // the LAST frame is the current one (Stack.peek, reference models/session_context.py:26-30)
    u32 top0 = 0, top1 = 0, fov0 = 0, fov1 = 0, top_nargs = CK_NARGS_NULL, top_kinds = 0;
    Span top_tgt = {0, 0}, top_cb = {0, 0}, top_a0 = {0, 0}, top_a1 = {0, 0};
    if (!PEEK(']')) {
        for (;;) {
            u32 f0 = pos;
            Span tgt, cb;
            if (!M("{\"target_topic\":") || !ck_string(r, pos, tgt) || !M(",\"callback_topic\":") || !ck_string(r, pos, cb)) FAIL;
            u32 nargs = CK_NARGS_NULL, kinds = 0;
            Span a0 = {0, 0}, a1 = {0, 0};
            if (!M(",\"input_args\":null,\"frame_id\":")) {
            if (!M(",\"input_args\":")) FAIL;
            if (PEEK('n')) { if (!ck_null(r, pos)) FAIL; }
            else {
                if (!M("[")) FAIL;
                nargs = 0;
                if (!PEEK(']')) {
                    for (;;) {
                        u32 v0 = pos;
                        Span sv;
                        bool is_str = PEEK('"');
                        if (is_str) { if (!ck_string(r, pos, sv)) FAIL; }
                        else { if (!ck_any(r, pos, 6, cx)) FAIL; sv.off = v0; sv.len = pos - v0; }
                        if (nargs == 0) { a0 = sv; kinds |= is_str ? 1u : 0u; }
                        if (nargs == 1) { a1 = sv; kinds |= is_str ? 2u : 0u; }
                        nargs++;
                        if (PEEK(',')) { pos++; continue; }
                        break;
                    }
                }
                if (!M("]")) FAIL;
            }
            if (!M(",\"frame_id\":")) FAIL;
            }
            if (!ck_string(r, pos, t)) FAIL;
            u32 ov0, ov1;
            if (M(",\"overrides\":null}")) { ov1 = pos - 1; ov0 = ov1 - 4; } else
            {
                if (!M(",\"overrides\":")) FAIL;
                ov0 = pos;
                if (!ck_overrides_or_null(r, pos, 6, cx)) FAIL;
                ov1 = pos;
                if (!M("}")) FAIL;
            }
            nframes++;
            top0 = f0; top1 = pos; fov0 = ov0; fov1 = ov1; top_nargs = nargs; top_kinds = kinds;
            top_tgt = tgt; top_cb = cb; top_a0 = a0; top_a1 = a1;
            if (PEEK(',')) { pos++; continue; }
            break;
        }
    }
    SETSPAN(CK_COL_TOP_OFF, top0, top1);
    o.set(CK_COL_TGT_OFF, top_tgt.off); o.set(CK_COL_TGT_LEN, top_tgt.len);
    o.set(CK_COL_CB_OFF, top_cb.off); o.set(CK_COL_CB_LEN, top_cb.len);
    o.set(CK_COL_NARGS, top_nargs); o.set(CK_COL_ARGKINDS, top_kinds);
    o.set(CK_COL_ARG0_OFF, top_a0.off); o.set(CK_COL_ARG0_LEN, top_a0.len);
    o.set(CK_COL_ARG1_OFF, top_a1.off); o.set(CK_COL_ARG1_LEN, top_a1.len);
    SETSPAN(CK_COL_FOV_OFF, fov0, fov1);
    if (M("]},\"metadata\":null}}")) {             // ]  },"metadata":  null  }}     (lengths 1 / 13 / 4 / 2)
        u32 e = pos;
        o.set(CK_COL_FRAMES_OFF, a); o.set(CK_COL_FRAMES_LEN, e - 19 - a);
        o.set(CK_COL_NFRAMES, nframes);
        o.set(CK_COL_WFMETA_OFF, e - 6); o.set(CK_COL_WFMETA_LEN, 4);
    } else {
    if (!M("]")) FAIL;
    SETSPAN(CK_COL_FRAMES_OFF, a, pos);
    o.set(CK_COL_NFRAMES, nframes);
    if (!M("},\"metadata\":")) FAIL;
    a = pos;
    if (!ck_any(r, pos, 3, cx)) FAIL;
    SETSPAN(CK_COL_WFMETA_OFF, a, pos);
    if (!M("}}")) FAIL;
    }
    if (pos != r.n) FAIL;                 // trailing bytes (even whitespace) are not a fixed point
    // resolve tool_calls[input_args[0]] and tool_results[input_args[0]] (what ToolNodeDef.run looks up,
    // reference nodes/tool.py:45, models/state.py:78-79) from the recorded key spans
    u32 call0 = 0, call1 = 0, res0 = 0, res1 = 0;
    Span tn = {0, 0}, ar = {0, 0};
    if (nframes > 0 && top_nargs == 2 && (top_kinds & 1u)) {
        u32 h = ck_hash_span(r, top_a0.off, top_a0.len);
        // the hash covers the length, so a hit is (almost surely) the key: find() verifies bytes + closing quote
        u32 ko = 0;
        u32 k = tck.find(r, h, top_a0.off, top_a0.len, ko);
        if (k == 0) { call0 = first_tc0; call1 = first_tc1; tn = first_tc.tool_name; ar = first_tc.args; }
        else if (k != ~0u) {
            u32 p2 = ko + top_a0.len + 2;
            call0 = p2;
            ToolCallSpans tcs;
            ck_tool_call_part(r, p2, 5, cx, tcs);
            call1 = p2; tn = tcs.tool_name; ar = tcs.args;
        }
        k = trk.find(r, h, top_a0.off, top_a0.len, ko);
        if (k == 0) { res0 = first_tr0; res1 = first_tr1; }
        else if (k != ~0u) {
            u32 p2 = ko + top_a0.len + 2;
            res0 = p2;
            ck_tool_result_value(r, p2, 5, cx);
            res1 = p2;
        }
    }
    SETSPAN(CK_COL_CALL_VAL_OFF, call0, call1);
    o.set(CK_COL_TNAME_OFF, tn.off); o.set(CK_COL_TNAME_LEN, tn.len);
    o.set(CK_COL_ARGS_OFF, ar.off); o.set(CK_COL_ARGS_LEN, ar.len);
    SETSPAN(CK_COL_RES_OFF, res0, res1);
    return true;
#undef FAIL
}

#endif  // CK_WALK_CUH
