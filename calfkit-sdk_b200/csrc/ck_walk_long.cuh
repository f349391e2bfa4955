// Long records: one warp per record, intra-record parallelism (see the block comment in ck_walk.cuh above ck_long_index).
//
// Why: a schema walk is sequential per record, so one thread per record takes (record length) x (~100-200 cycles per byte)
// no matter how idle the machine is: milliseconds for a 20 KB fan-out record or a 64 KB history, a few percent of the HBM
// roofline for configs 3 and 5.  Long records are long because of LISTS (64 tool calls, 64 parts, dozens of
// messages): their elements are independent given the boundaries.
//   ck_lx_build          warp-parallel structural pre-scan, 512 bytes per iteration (16 per lane): byte-class bit masks by
//                        SIMD-in-word compares, escaped quotes from the backslash runs, string mask by prefix XOR (within
//                        the lane by shifts, across lanes by shuffles), nesting depth by prefix sums of the bracket bits;
//                        the positions of commas and closers at depths 4 and 6 go to shared memory in order
//   ck_walk_long_kernel  the walker in lockstep over the record (URd); at the long lists the lanes take one element each
// The thread-per-record kernel hands every record of CK_LONG_MIN bytes or more to this one through a device-side list.
#ifndef CK_WALK_LONG_CUH
#define CK_WALK_LONG_CUH

#ifndef CK_LONG_MIN
#define CK_LONG_MIN 16384u
#endif
#define CK_LONG_WARPS 4

// bytes of a word equal to a character -> 4 bits.  Exact zero-byte test of x = word ^ cccc (no borrow between bytes):
// bit 7 of a byte of ~(((x & 0x7f..) + 0x7f..) | x) is set iff the byte is 0; the multiply gathers the four flags.
__device__ __forceinline__ u32 ck_nib_eq(u32 x) {
    u32 t = ~(((x & 0x7F7F7F7Fu) + 0x7F7F7F7Fu) | x) & 0x80808080u;
    return ((t >> 7) * 0x01020408u) >> 24;
}
__device__ __forceinline__ u32 ck_mask16(const uint4& w, u32 c) {
    u32 cc = c * 0x01010101u;
    return ck_nib_eq(w.x ^ cc) | (ck_nib_eq(w.y ^ cc) << 4) | (ck_nib_eq(w.z ^ cc) << 8) | (ck_nib_eq(w.w ^ cc) << 12);
}
__device__ __forceinline__ u32 ck_mask16_or20(const uint4& w, u32 c) {          // bytes equal to c once bit 5 is set: '{' / '[' and '}' / ']'
    const u32 b = 0x20202020u;
    u32 cc = c * 0x01010101u;
    return ck_nib_eq((w.x | b) ^ cc) | (ck_nib_eq((w.y | b) ^ cc) << 4) | (ck_nib_eq((w.z | b) ^ cc) << 8) | (ck_nib_eq((w.w | b) ^ cc) << 12);
}

// [from, to): the bytes to scan (the whole record, or one container that starts at a structural character outside any
// string); depth0: containers open before `from`
// DEEP: also index depth 6 (the parts of a message); the history pre-scan needs depth 4 only
template <bool DEEP = true>
__device__ __forceinline__ void ck_lx_build(const u8* __restrict__ g, u32 n, ck_long_index* __restrict__ lx, u32 from = 0, u32 to = 0xffffffffu, int depth0 = 0) {
    u32 lane = threadIdx.x & 31;
    u32 m0 = (u32)((uintptr_t)g & 15);
    const uint4* stream = (const uint4*)(g - m0);                   // 16-byte aligned; the buffers are padded on both sides of a record
    if (to > n) to = n;
    u32 m = m0 + from, total = m0 + to;                             // valid stream positions: [m, total)
    u32 n_sep[2] = {0, 0}, n_close[2] = {0, 0};
    u32 prev_bs = 0, str_carry = 0; int depth_carry = depth0;
    bool overflow = false;
    u32 n_open = 0;
    uint4 wn = make_uint4(0, 0, 0, 0);                               // the next tile's bytes are in flight while this one is scanned
    { u32 pf = (m & ~511u) + 16 * lane; if (pf < total) wn = __ldg(stream + (pf >> 4)); }
    for (u32 t0 = m & ~511u; t0 < total; t0 += 512) {
        u32 p0 = t0 + 16 * lane;                                    // stream position of this lane's first byte
        uint4 w = wn;
        wn = make_uint4(0, 0, 0, 0);
        if (p0 + 512 < total) wn = __ldg(stream + ((p0 + 512) >> 4));
        // valid bytes: [m, total)
        u32 V = 0xFFFFu;
        if (p0 < m) V &= (m - p0 >= 16) ? 0u : (0xFFFFu << (m - p0));
        if (p0 + 16 > total) V &= (p0 >= total) ? 0u : (0xFFFFu >> (p0 + 16 - total));
        u32 Q = ck_mask16(w, '"') & V, B = ck_mask16(w, '\\') & V;
        // escaped quotes: preceded by a backslash run of length 1 or 3 (longer runs: the proposal may be wrong, the walk decides)
        u32 up = __shfl_up_sync(0xffffffffu, B >> 12, 1);
        u32 prev4 = lane ? up : prev_bs;
        prev_bs = __shfl_sync(0xffffffffu, B >> 12, 31);
        u32 B20 = (B << 4) | prev4;
        u32 e1 = B20 << 1, r2 = e1 & (B20 << 2), r3 = r2 & (B20 << 3), r4 = r3 & (B20 << 4);
        Q &= ~(((e1 & ~r2) | (r3 & ~r4)) >> 4);
        // string mask: exclusive prefix parity of the quote bits
        u32 S = Q; S ^= S << 1; S ^= S << 2; S ^= S << 4; S ^= S << 8; S &= 0xFFFFu;
        u32 par = __popc(Q) & 1u;
        u32 odd = __ballot_sync(0xffffffffu, par != 0);             // lanes with an odd number of quotes
        u32 carry = (__popc(odd & ((1u << lane) - 1u)) & 1u) ^ str_carry;   // parity before this lane's first byte
        str_carry ^= __popc(odd) & 1u;
        u32 E = ((S << 1) & 0xFFFFu) ^ (carry ? 0xFFFFu : 0u);      // bit b: byte b lies inside a string
        // commas and brackets matter outside strings only: a lane whose 16 bytes all lie inside one (most lanes of a
        // conversation's text) skips their masks
        u32 K = 0, O = 0, C = 0;
        u32 outside = ~E & V;
        if (outside) { K = ck_mask16(w, ',') & outside; O = ck_mask16_or20(w, '{') & outside; C = ck_mask16_or20(w, '}') & outside; }
        // nesting depth before each byte
        int dbase = depth_carry;
        if (__any_sync(0xffffffffu, (O | C) != 0)) {                // (tiles inside one long string have no bracket at all)
            int delta = (int)__popc(O) - (int)__popc(C), dinc = delta;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) { int y = __shfl_up_sync(0xffffffffu, dinc, o); if (lane >= (u32)o) dinc += y; }
            dbase = depth_carry + dinc - delta;
            depth_carry += __shfl_sync(0xffffffffu, dinc, 31);
        }
        // '[' that opens a depth-4 list (rare: a handful per record) — remembered for the message_history look-up
        {
            u32 SQ = O ? ck_mask16(w, '[') & O : 0u;
            u32 mine = 0, firstpos = 0;
            for (u32 x = SQ; x; x &= x - 1) {
                u32 b = __ffs(x) - 1, below = (1u << b) - 1u;
                int d = dbase + (int)__popc(O & below) - (int)__popc(C & below);
                if (d == 3) { if (!mine) firstpos = p0 + b - m0; mine++; }
            }
            u32 any = __ballot_sync(0xffffffffu, mine != 0);
            while (any) {                                           // in stream order; a lane with two such openers in 16 bytes cannot
                u32 src = __ffs(any) - 1; any &= any - 1;           // be canonical JSON ("[[": depth 3 then 4), the second is dropped
                u32 pp = __shfl_sync(0xffffffffu, firstpos, src);
                if (n_open < CK_LX_OPEN) { if (lane == 0) lx->open_sq[n_open] = pp; }
                n_open++;
            }
        }
        // this lane's entries for the four lists (sep / close at depth 4, sep / close at depth 6); scalars, not an indexed
        // array: a dynamically indexed local array lives in local memory
        u32 c_s0 = 0, c_s1 = 0, c_c0 = 0, c_c1 = 0;
        u32 pend = K | C;
        {   // the depths this lane's bytes can be at: nothing to list if neither 4 nor (DEEP) 6 is among them
            int dlo = dbase - (int)__popc(C), dhi = dbase + (int)__popc(O);
            if (!((dlo <= 4 && dhi >= 4) || (DEEP && dlo <= 6 && dhi >= 6))) pend = 0;
        }
        for (u32 x = pend; x; x &= x - 1) {
            u32 b = __ffs(x) - 1, below = (1u << b) - 1u;
            int d = dbase + (int)__popc(O & below) - (int)__popc(C & below);
            bool cl = ((C >> b) & 1u) != 0;
            if (d == 4) { if (cl) c_c0++; else c_s0++; }
            else if (DEEP && d == 6) { if (cl) c_c1++; else c_s1++; }
        }
        if (!__any_sync(0xffffffffu, (c_s0 | c_s1 | c_c0 | c_c1) != 0)) continue;      // nothing to list in this tile
        u32 o_s0, o_s1 = 0, o_c0, o_c1 = 0;
        {
            auto scan = [&](u32 c, u32& total) { u32 sc = c;
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) { u32 y = __shfl_up_sync(0xffffffffu, sc, o); if (lane >= (u32)o) sc += y; }
                total = __shfl_sync(0xffffffffu, sc, 31); return sc - c; };
            u32 tot;
            o_s0 = n_sep[0] + scan(c_s0, tot); if (n_sep[0] + tot > CK_LX_SEP) overflow = true; n_sep[0] += tot;
            o_c0 = n_close[0] + scan(c_c0, tot); if (n_close[0] + tot > CK_LX_CLOSE) overflow = true; n_close[0] += tot;
            if (DEEP) {
                o_s1 = n_sep[1] + scan(c_s1, tot); if (n_sep[1] + tot > CK_LX_SEP) overflow = true; n_sep[1] += tot;
                o_c1 = n_close[1] + scan(c_c1, tot); if (n_close[1] + tot > CK_LX_CLOSE) overflow = true; n_close[1] += tot;
            }
        }
        if (!overflow) {
            for (u32 x = pend; x; x &= x - 1) {
                u32 b = __ffs(x) - 1, below = (1u << b) - 1u;
                int d = dbase + (int)__popc(O & below) - (int)__popc(C & below);
                bool cl = ((C >> b) & 1u) != 0;
                u32 pos = p0 + b - m0;
                if (d == 4) { if (cl) lx->close_[0][o_c0++] = pos; else lx->sep[0][o_s0++] = pos; }
                else if (DEEP && d == 6) { if (cl) lx->close_[1][o_c1++] = pos; else lx->sep[1][o_s1++] = pos; }
            }
        }
    }
    if (lane == 0) {
        lx->n_sep[0] = n_sep[0]; lx->n_sep[1] = n_sep[1]; lx->n_close[0] = n_close[0]; lx->n_close[1] = n_close[1];
        lx->ok = overflow ? 0u : 1u;                                // too many entries: plain lockstep walk, no element parallelism
        lx->n_open = n_open <= CK_LX_OPEN ? n_open : 0u;            // too many to remember: no look-up
    }
    __syncwarp();
}

// ---- the warp-per-record pass over the records of CK_HIST_MIN bytes or more (listed by ck_classify_kernel) ---------------------
// A warp builds the structural index of its record and looks for the '[' of message_history among the depth-4 list openers
// (the 18 bytes before it spell the key).
//  (a) The history is the bulk of the record and its messages are short: the messages between the '[' and its closer go on the
//      batch-wide element list (ck_walk_elems_kernel: one thread per message) and (open, close) is left in hist_skip[i].  The
//      thread-per-record walker then jumps over the list — it verifies that `open` is where message_history really starts and
//      that a ']' stands at `close` — so what a thread walks of such a record is the kilobyte around the history.
//  (b) Otherwise, a record of CK_LONG_MIN bytes or more is walked right here by the warp (lockstep walker; its long dicts and
//      lists fan out over the lanes, ck_walk.cuh) and hist_skip[i] = (~0, ~0) tells the thread-per-record kernel to leave it.
//  (c) Otherwise (0, 0): the thread-per-record kernel walks it whole.
// Everything the index says is a proposal: a wrong one fails in the element walk or in the record walk and costs a trip
// through the canonicaliser.
#ifndef CK_ELEM_MAX
#define CK_ELEM_MAX 4096u           // longer messages stay with their record's warp (their parts are walked lane-parallel there)
#endif
#ifndef CK_LONG_MINB
#define CK_LONG_MINB 6          // <= 80 registers: 24 warps per SM (the warp walk is latency bound: more warps hide more of it than 16 do)
#endif
__global__ void __launch_bounds__(32 * CK_LONG_WARPS, CK_LONG_MINB)
ck_walk_long_kernel(ck_view v, u32* __restrict__ cols, u32 stride, const u32* __restrict__ cand, uint2* __restrict__ hist_skip) {
    u32 lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    u32 count = v.canon_ctl->cand;
    ck_long_index* lx = (ck_long_index*)ck_win_smem + w;
    if (lane == 0) { lx->defer_list = v.elems; lx->defer_ctr = &v.canon_ctl->elems; lx->defer_cap = v.elem_cap; }
    // a warp takes the next record when it is done with its own: the tail of the kernel is one record, not a static share
    for (;;) {
        u32 kq = 0;
        if (lane == 0) kq = atomicAdd(&v.canon_ctl->cand_next, 1u);
        kq = __shfl_sync(0xffffffffu, kq, 0);
        if (kq >= count) break;
        u32 i = cand[kq];
        u32 len; const u8* rec = ck_rec_in(v, i, len);
        bool longrec = len >= CK_LONG_MIN;
        if (longrec) ck_lx_build<true>(rec, len, lx); else ck_lx_build<false>(rec, len, lx);
        uint2 res = make_uint2(0u, 0u);
        u32 open = 0xffffffffu;
        if (lx->ok) {
            const char key[] = "\"message_history\":";                // 18 bytes
            for (u32 j = 0; j < lx->n_open && open == 0xffffffffu; j++) {
                u32 pp = lx->open_sq[j];
                bool eq = pp >= 18;
                if (eq && lane < 18) eq = rec[pp - 18 + lane] == (u8)key[lane];
                if (__all_sync(0xffffffffu, eq)) open = pp;
            }
        }
        u32 q, s0, k;
        bool take = open != 0xffffffffu && ck_lx_range(lx, 0, open + 1, q, s0, k) && q > open + 1 && (unsigned long long)(q - open) * 2 >= len;
        if (take) {                                                 // a thread per message pays only while the messages are short
            u32 mx = 0;
            for (u32 e = lane; e <= k; e += 32) { u32 a0 = e ? lx->sep[0][s0 + e - 1] + 1 : open + 1, a1 = e == k ? q : lx->sep[0][s0 + e]; mx = max(mx, a1 - a0); }
            take = __reduce_max_sync(0xffffffffu, mx) <= CK_ELEM_MAX;
        }
        if (take) {
            u32 slot = ck_defer_reserve(&v.canon_ctl->elems, k + 1);
            take = slot <= v.elem_cap && k + 1 <= v.elem_cap - slot;
            for (u32 e = lane; e <= k; e += 32) {
                if (!take && (slot >= v.elem_cap || e >= v.elem_cap - slot)) break;
                ck_elem el; el.rec = take ? i : 0xffffffffu;        // a reservation that does not fit is voided
                el.start = e ? lx->sep[0][s0 + e - 1] + 1 : open + 1; el.end = e == k ? q : lx->sep[0][s0 + e];
                // requests and responses alternate in a conversation and differ in shape and length: even messages first,
                // then the odd ones, so that the lanes of a warp of the element pass walk alike messages
                v.elems[slot + (take ? (e >> 1) + ((e & 1u) ? (k >> 1) + 1u : 0u) : e)] = el;
            }
            if (take) res = make_uint2(open, q);
        }
        if (!take && longrec) {
            if (lane == 0) lx->rec = i;
            __syncwarp();
            WalkOut o; o.base = cols + i; o.stride = stride; o.active = (lane == 0);
            URd r; r.init(rec, len, 2);                             // state 2 (bit 0 belongs to the match cores): lockstep, lists may fan out
            AnyCtx cx; cx.kfill = 0;
            u32 stop = 0;
            u32 status = ck_walk_envelope(r, o, cx, stop) ? CK_OK : CK_NOT_CANONICAL;
            o.set(CK_COL_STATUS, status);
            o.set(CK_COL_ERR, stop);
            if (lane == 0 && status == CK_NOT_CANONICAL && v.canon_ctl) {
                u32 kk = atomicAdd(&v.canon_ctl->count, 1u);
                v.canon_list[kk] = i;
            }
            res = make_uint2(0xffffffffu, 0xffffffffu);
        }
        if (lane == 0) hist_skip[i] = res;
        __syncwarp();
    }
}

// the messages the long walker deferred: one thread each through the window reader (the same code and the same per-thread
// efficiency as the thread-per-record walk).  The long walker has already taken the element boundaries on trust and
// finished its record as CK_OK; an element that is not exactly one canonical message turns its record into
// CK_NOT_CANONICAL here and lists it for the canonicaliser pass (once: the exchange on the status column decides).
__global__ void __launch_bounds__(CK_WALK_THREADS, CK_WALK_MINB)
ck_walk_elems_kernel(ck_view v, u32* __restrict__ cols, u32 stride) {
    u32 cnt = v.canon_ctl->elems;
    if (cnt > v.elem_cap) cnt = v.elem_cap;
    for (u32 k = blockIdx.x * blockDim.x + threadIdx.x; k < cnt; k += gridDim.x * blockDim.x) {
        ck_elem el = v.elems[k];
        if (el.rec == 0xffffffffu) continue;
        u32 len; const u8* rec = ck_rec_in(v, el.rec, len);
        WRd r; r.init(rec, len);
        AnyCtx cx; cx.kfill = 0;
        u32 p = el.start;
        bool ok = el.end <= len && ck_message(r, p, 5, cx) != 0 && p == el.end;
        if (!ok && atomicExch(&cols[(size_t)CK_COL_STATUS * stride + el.rec], (u32)CK_NOT_CANONICAL) == CK_OK) {
            u32 kk = atomicAdd(&v.canon_ctl->count, 1u);
            v.canon_list[kk] = el.rec;
        }
    }
}

#endif  // CK_WALK_LONG_CUH
