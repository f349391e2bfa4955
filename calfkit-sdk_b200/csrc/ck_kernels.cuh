// sm_90a (H100) kernels of the calfkit-b200 hot path.  No tensor cores: the path has no dense
// contraction; everything here is HBM-bound byte/integer work (DESIGN.md §kernels).
//
//   ck_walk_kernel        decode: prove each record is a canonical Envelope + extract spans   (a2,a3,a4)
//   ck_plan_tool_kernel   ToolNodeDef.run + _publish_action(ReturnCall|Silent) as a splice plan, routed  (a5,a6,a8)
//                         (ck_plan.cuh)
//   ck_fanout2_*_kernel   Agent fan-out: one Call envelope per pending tool call (ck_fanout2.cuh)   (a9,a6)
//   ck_scan_*             exclusive prefix sum of payload lengths -> output offsets
//   ck_emit_kernel        encode: gather segments into contiguous output payloads               (a7)
//   ck_route_kernel       topic string -> registered topic id, Kafka partition of the key        (a8)
#ifndef CK_KERNELS_CUH
#define CK_KERNELS_CUH

#include <cuda_runtime.h>
#include "ck_walk.cuh"
#include "ck_canon.cuh"

#if !defined(__CUDA_ARCH__)
extern __shared__ uint4 ck_win_smem[];   // nvcc's host pass parses the device code too; ck_walk.cuh declares it for the device pass
#endif

// ------------------------------------------------------------------------------------------------
// A batch as the kernels see it: the submitted records (concatenated bytes + offsets) plus an overlay —
// the canonical re-emission of the records that arrived in a non-canonical spelling (ck_canon.cuh).
// Every stage after decode reads a record through ck_rec(), i.e. its canonical bytes.
// ------------------------------------------------------------------------------------------------
#ifndef CK_HIST_MIN
#define CK_HIST_MIN 2048u        // records at least this long get the message_history pre-scan (ck_walk_long.cuh)
#endif
#ifndef CK_LONG_MIN
#define CK_LONG_MIN 16384u       // records at least this long are walked one per warp (ck_walk_long.cuh)
#endif
// per-batch counters (zeroed by launch_decode): overlay bytes handed out; records listed for the canonicaliser; list elements
// deferred to ck_walk_elems_kernel (may exceed the capacity: clamp); records listed for the warp-per-record pass / handed out
struct ck_canon_ctl { unsigned long long cursor; u32 count; u32 elems; u32 cand; u32 cand_next; };
struct ck_view {
    const u8* in; const long long* off;
    const u8* ovl; const long long* ovl_off; const u32* ovl_len;     // ovl_off[i] < 0: record i has no overlay
    ck_canon_ctl* canon_ctl; u32* canon_list;                        // records the walker left to the canonicaliser
    const u32* perm;                                                 // NULL, or thread t of the walk takes record perm[t] (length-bucketed batch)
    const uint2* hist_skip;                                          // per record: (open, close) of a message_history whose messages are on the element list
    ck_elem* elems; u32 elem_cap;                                    // deferred list elements of long records (ck_walk_elems_kernel)
    const u32* len;                                                  // NULL: record i = [off[i], off[i+1]); else off[i] .. + len[i]
};                                                                   //       (values inside raw Kafka record batches are not contiguous)
__device__ __forceinline__ const u8* ck_rec_in(const ck_view& v, u32 i, u32& len) {     // the submitted bytes of record i
    long long a = v.off[i];
    len = v.len ? v.len[i] : (u32)(v.off[i + 1] - a);
    return v.in + a;
}
__device__ __forceinline__ const u8* ck_rec(const ck_view& v, u32 i, u32& len) {
    long long o = v.ovl_off[i];
    if (o >= 0) { len = v.ovl_len[i]; return v.ovl + o; }
    return ck_rec_in(v, i, len);
}

// ------------------------------------------------------------------------------------------------
// node configuration living in device memory
// ------------------------------------------------------------------------------------------------
// Pieces of a tool splice besides the template's, in the worst case (no existing result, frame overrides): 4 before
// the return value (prefix, `,"` or `"`, id, `":{"return_value":`), 3 after it (lit_mid, id, lit_close), 2 for the
// overrides rule and 2 for the unwind.  With the template's parts on top they must fit one descriptor.
#define CK_TOOL_FIXED_PIECES 11
#define CK_TPL_MAX_PARTS 5
static_assert(CK_TOOL_FIXED_PIECES + CK_TPL_MAX_PARTS <= CK_MAX_SEGS, "a tool splice must fit one descriptor");
struct ck_tool_cfg {
    int32_t  publish_topic_id;          // registered id of node.publish_topic, -1 = none
    uint32_t tpl_nparts;                // 0 = results come from the host (aux blob)
    uint32_t tpl_kind[CK_TPL_MAX_PARTS];   // 0: literal (lit pool span)  1: string argument (lit pool span = key name)
    uint32_t tpl_off[CK_TPL_MAX_PARTS];
    uint32_t tpl_len[CK_TPL_MAX_PARTS];
    // fixed literals in the pool (offset, length)
    uint32_t lit_comma_q[2];            // ,"
    uint32_t lit_q[2];                  // "
    uint32_t lit_open[2];               // ":{"return_value":
    uint32_t lit_mid[2];                // ,"content":null,"metadata":{"tool_call_id":"
    uint32_t lit_close[2];              // "},"kind":"tool-return"}
    uint32_t lit_value_open[2];         // {"return_value":
};

struct ck_pub {                          // one publish (nodes/base.py:82-87; worker/worker.py:52-53)
    uint32_t payload;                    // index of the payload descriptor, 0xffffffff = no publish
    int32_t  topic_id;                   // >= 0 resolved; -1: unresolved, see topic_off/len
    uint32_t topic_off, topic_len;       // topic string span inside the input record
    uint32_t record;                     // source record
    uint32_t has_key;                    // key = correlation id bytes
    int32_t  partition;                  // murmur2(key) % num_partitions, -1 if unkeyed
    uint32_t pad;
};

struct ck_topic_table {                  // open addressing, power-of-two capacity
    uint32_t cap;
    const uint32_t* hash;                // 0 = empty slot
    const int32_t*  id;
    const uint32_t* name_off;            // into names
    const uint32_t* name_len;
    const uint8_t*  names;
};

// ------------------------------------------------------------------------------------------------
// decode
// ------------------------------------------------------------------------------------------------
#define CK_WALK_THREADS 128
// 6 blocks of 128 threads per SM: <= 80 registers (at 64 the walker spills about twice as much) and room for the
// CK_WIN_BYTES = 224 windows.  Measured on H100 against 8 blocks with 160-byte windows: config-2 walk 1.30 -> 1.14 ms
// (DESIGN.md §7)
#ifndef CK_WALK_MINB
#define CK_WALK_MINB 6
#endif
// records long enough for the history pre-scan (ck_hist_prescan_kernel), listed with one atomic per warp
__global__ void __launch_bounds__(256)
ck_classify_kernel(ck_view v, u32 n, u32* __restrict__ cand) {
    u32 j = blockIdx.x * blockDim.x + threadIdx.x;
    bool take = false; u32 i = 0;
    if (j < n) { i = v.perm ? v.perm[j] : j; u32 len; ck_rec_in(v, i, len); take = len >= CK_HIST_MIN; }
    u32 m = __ballot_sync(0xffffffffu, take);
    if (!m) return;
    u32 lane = threadIdx.x & 31, base = 0;
    if (lane == (u32)(__ffs(m) - 1)) base = atomicAdd(&v.canon_ctl->cand, (u32)__popc(m));
    base = __shfl_sync(0xffffffffu, base, __ffs(m) - 1);
    if (take) cand[base + __popc(m & ((1u << lane) - 1u))] = i;
}
// recursive-descent walker (csrc/ck_walk.cuh), one thread per submitted record, read through a per-thread
// shared-memory window (WRd; dynamic shared memory: blockDim.x * CK_WIN_STRIDE bytes).  Records it cannot prove
// canonical are listed for the canonicaliser pass.
__global__ void __launch_bounds__(CK_WALK_THREADS, CK_WALK_MINB)
ck_walk_kernel(ck_view v, u32 n, u32* __restrict__ cols, u32 stride) {
    u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    if (v.perm) i = v.perm[i];                                                                       // bucketed batch: neighbours in a warp are of one size class
    u32 len; const u8* rec = ck_rec_in(v, i, len);
    uint2 skip = make_uint2(0u, 0u);
    if (len >= CK_HIST_MIN && v.hist_skip) {
        skip = v.hist_skip[i];                                       // written by ck_hist_prescan_kernel for every such record
        if (skip.x == 0xffffffffu) return;                           // long record, not history-dominated: a whole warp has walked it (ck_walk_long_kernel)
    }
    WalkOut o; o.base = cols + i; o.stride = stride; o.skip_open = skip.x; o.skip_close = skip.y;
    u32 stop = 0;
    bool ok = true;
    if (len) {
        WRd r; r.init(rec, len);
        AnyCtx cx;
        cx.kfill = 0;
        ok = ck_walk_envelope(r, o, cx, stop);
    }
    o.set(CK_COL_STATUS, len == 0 ? CK_EMPTY : ok ? CK_OK : CK_NOT_CANONICAL);
    o.set(CK_COL_ERR, stop);
    if (!ok && v.canon_ctl) {      // rare: hand the record to the canonicaliser pass
        u32 k = atomicAdd(&v.canon_ctl->count, 1u);
        v.canon_list[k] = i;
    }
}

// ------------------------------------------------------------------------------------------------
// canonicaliser kernels (ck_canon.cuh): one thread per record that the walker left as CK_NOT_CANONICAL.
//   count: verdict + canonical length (the emitter runs with a zero-capacity sink)
//   write: after the exclusive scan of the lengths, emit into the overlay buffer
// ------------------------------------------------------------------------------------------------
// One launch for the whole pass: the walker listed the records it could not prove canonical (usually none: the kernel
// then exits at once); every listed record is re-emitted canonically into the overlay — counting pass, space handed out
// by one atomic on a byte cursor (overlay order is irrelevant: ovl_off[i] says where), writing pass; ck_rewalk_list_kernel
// then walks them again in that spelling with the trusting reader.
__global__ void __launch_bounds__(64)
ck_canon_kernel(ck_view v, u32 n, u32* __restrict__ cols, u32 stride, u8* __restrict__ ovl, long long ovl_cap,
                long long* __restrict__ ovl_off, u32* __restrict__ ovl_len) {
    u32 cnt = v.canon_ctl->count;
    for (u32 k = blockIdx.x * blockDim.x + threadIdx.x; k < cnt; k += gridDim.x * blockDim.x) {
        u32 i = v.canon_list[k];
        u32 len, out_len = 0;
        const u8* src = ck_rec_in(v, i, len);
        u32 st = ck_canonicalise(src, len, nullptr, 0, out_len);
        if (st != CK_OK) { cols[(size_t)CK_COL_STATUS * stride + i] = st; continue; }
        u32 need = (out_len + 15u) & ~15u;
        long long o0 = (long long)atomicAdd(&v.canon_ctl->cursor, (unsigned long long)need);
        if (o0 + need > ovl_cap) { cols[(size_t)CK_COL_STATUS * stride + i] = CK_UNSUPPORTED; continue; }   // overlay buffer full
        st = ck_canonicalise(src, len, ovl + o0, need, out_len);
        if (st != CK_OK) { cols[(size_t)CK_COL_STATUS * stride + i] = CK_UNSUPPORTED; continue; }
        for (u32 b = out_len; b < need; b++) ovl[o0 + b] = 0;
        ovl_len[i] = out_len;
        ovl_off[i] = o0;
    }
}

// second walk of the listed records, over the canonical bytes the kernel above wrote (a separate launch: the walker
// reads through the non-coherent path)
__global__ void __launch_bounds__(64)
ck_rewalk_list_kernel(ck_view v, u32 n, u32* __restrict__ cols, u32 stride) {
    u32 cnt = v.canon_ctl->count;
    for (u32 k = blockIdx.x * blockDim.x + threadIdx.x; k < cnt; k += gridDim.x * blockDim.x) {
        u32 i = v.canon_list[k];
        if (v.ovl_off[i] < 0) continue;
        u32 len; const u8* rec = ck_rec(v, i, len);
        WalkOut o; o.base = cols + i; o.stride = stride;
        u32 stop = 0;
        GRdT r; r.init(rec, len);
        AnyCtx cx; cx.kfill = 0;
        u32 status = ck_walk_envelope(r, o, cx, stop) ? CK_OK : CK_UNSUPPORTED;   // never happens by construction (hostsim fuzz)
        o.set(CK_COL_STATUS, status);
        o.set(CK_COL_ERR, stop);
    }
}

// ------------------------------------------------------------------------------------------------
// helpers on validated canonical spans
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ bool ck_span_eq(Rd& r, u32 a, u32 b, u32 len) {
    for (u32 k = 0; k < len; k++) if (r.at(a + k) != r.at(b + k)) return false;
    return true;
}

// look `key` (content span) up in the canonical dict object starting at `obj` ('{'); returns the
// value span, len 0 if absent
__device__ __forceinline__ Span ck_dict_find(Rd& r, u32 obj, u32 key_off, u32 key_len) {
    u32 pos = obj + 1;
    Span none = {0, 0};
    while (pos < r.n && r.at(pos) != '}') {
        Span k;
        if (!ck_string(r, pos, k)) return none;
        pos++;                                   // ':'
        u32 v = pos;
        ck_skip_value(r, pos);
        if (k.len == key_len && ck_span_eq(r, k.off, key_off, key_len)) { Span s = {v, pos - v}; return s; }
        if (pos < r.n && r.at(pos) == ',') pos++;
    }
    return none;
}

// ------------------------------------------------------------------------------------------------
// Output layout planner for the producers that generate text (uuid7 frame ids, merged values): the fan-out,
// tail-call, reply and gate plans.  The emit kernel accepts segments at any byte boundary (ck_out_desc); this
// writer keeps the stricter aligned layout — every segment starts at a 16-byte aligned offset of the output
// payload and every segment but the last is a multiple of 16 bytes long — so each output vector it describes
// comes from exactly one segment and takes the emitter's single-gather path.
// Pieces arrive in output order.  Long input / aux pieces become DIRECT segments (copied from where
// they lie); everything short — literals, generated ids, and the <= 15 bytes on either side of a splice
// point that do not fill a vector — is packed by this thread, 8 aligned bytes per store, into the
// payload's glue slot and becomes a GLUE segment.
// ------------------------------------------------------------------------------------------------
#define CK_DIRECT_MIN 48u
struct SegWriter {
    ck_out_desc* d;
    Rd* r; const u8* lit; const u8* aux; u8* slot;         // byte sources and this payload's glue slot
    u32 n, total;                                          // segments so far, output offset
    bool in_glue, overflow;
    u32 gfill, grun;                                       // bytes of the slot used, start of the open run
    unsigned long long acc; u32 cnt;

    __device__ __forceinline__ void init(ck_out_desc* dd, Rd* rr, const u8* l, const u8* a, u8* s) {
        d = dd; r = rr; lit = l; aux = a; slot = s; n = 0; total = 0; in_glue = false; overflow = false; gfill = 0; grun = 0; acc = 0; cnt = 0;
    }
    __device__ __forceinline__ void seg(u32 src, u32 off, u32 len) {
        if (n < CK_MAX_SEGS) { d->seg[n][0] = off; d->seg[n][1] = (len << 2) | src; n++; } else overflow = true;
    }
    // append the low `nb` (1..8) bytes of `chunk` to the open run: 8 aligned bytes per store
    __device__ __forceinline__ void put8(unsigned long long chunk, u32 nb) {
        if (gfill + nb > CK_GLUE_STRIDE) { overflow = true; return; }
        if (nb < 8) chunk &= (~0ull >> (8 * (8 - nb)));
        acc |= chunk << (8 * cnt);
        u32 c2 = cnt + nb;
        gfill += nb;
        if (c2 >= 8) {
            *(unsigned long long*)(slot + ((gfill - (c2 - 8)) - 8)) = acc;
            acc = cnt ? (chunk >> (8 * (8 - cnt))) : 0ull;
            c2 -= 8;
        }
        cnt = c2;
    }
    __device__ __forceinline__ void put(u8 b) { put8((unsigned long long)b, 1); }
    __device__ __forceinline__ static unsigned long long load8_g(const u8* p) {    // unaligned 8 bytes from global memory
        u32 s = (u32)((uintptr_t)p & 7);
        const unsigned long long* q = (const unsigned long long*)((uintptr_t)p - s);
        unsigned long long lo = q[0];
        if (s == 0) return lo;
        unsigned long long hi = q[1];
        return (lo >> (8 * s)) | (hi << (64 - 8 * s));
    }
    __device__ __forceinline__ unsigned long long fetch8(u32 src, u32 off) {
        return src == CK_SRC_INPUT ? r->load8(off) : load8_g((src == CK_SRC_LIT ? lit : aux) + off);
    }
    __device__ __forceinline__ void close_run() {          // the open glue run becomes a segment
        if (cnt) { *(unsigned long long*)(slot + (gfill & ~7u)) = acc; acc = 0; cnt = 0; }
        seg(CK_SRC_GLUE, grun, gfill - grun);
        gfill = (gfill + 15u) & ~15u;                      // next run starts 16-aligned inside the slot
        in_glue = false;
    }
    __device__ __forceinline__ void glue_bytes(u32 src, u32 off, u32 len) {
        if (!in_glue) { in_glue = true; grun = gfill; }
        for (u32 k = 0; k < len; k += 8) put8(fetch8(src, off + k), len - k < 8 ? len - k : 8);
        total += len;
    }
    __device__ __forceinline__ void add(u32 src, u32 off, u32 len) {
        if (len == 0) return;
        bool direct_ok = (src == CK_SRC_INPUT || src == CK_SRC_AUX) && len >= CK_DIRECT_MIN;
        if (!direct_ok) { glue_bytes(src, off, len); return; }
        if (in_glue || (total & 15u)) {                    // bring the output offset to a vector boundary first
            u32 need = (16u - (total & 15u)) & 15u;
            glue_bytes(src, off, need);
            off += need; len -= need;
            close_run();
        }
        u32 body = len & ~15u;
        seg(src, off, body);
        total += body;
        if (len - body) glue_bytes(src, off + body, len - body);   // the ragged end opens the next glue run
    }
    __device__ __forceinline__ void hex_uuid7(unsigned long long unix_ms, unsigned long long seed, unsigned long long idx);
    __device__ __forceinline__ bool finish(u32 record) {
        if (in_glue) close_run();
        d->nseg = n; d->record = record; d->total_len = total;
        return !overflow;
    }
};

// ------------------------------------------------------------------------------------------------
// agent fan-out: Agent.run's list[Call] branch (reference nodes/agent.py:177-211) followed by
// _publish_action's fan-out branch (nodes/base.py:73-88): every pending tool call (in tool_calls,
// not yet in tool_results) becomes one envelope = input state + one pushed CallFrame
//   {target_topic: registry[tool_name].subscribe_topics[0], callback_topic: self.subscribe_topics[0],
//    input_args: [tool_call_id, agent_name], frame_id: fresh uuid7, overrides: null}
// (models/session_context.py:33-39,62-70).  One pending call -> a single Call whose envelope is
// also the handler's return value; >1 -> list[Call] and the handler returns the ORIGINAL envelope.
// ------------------------------------------------------------------------------------------------
struct ck_agent_cfg {
    int32_t  publish_topic_id;
    uint32_t lit_comma[2];             // ,
    uint32_t lit_mid[2];               // ","<agent_name>"],"frame_id":"
    uint32_t lit_tail[2];              // ","overrides":null}
    uint32_t lit_tc_head[2];           // {"target_topic":"<self topic>","callback_topic":"      (TailCall to self)
    uint32_t lit_tc_mid[2];            // ","input_args":null,"frame_id":"
    int32_t  self_topic_id;            // registered id of subscribe_topics[0] (or -1)
    uint32_t ntools;
    // per tool k (device arrays): name span + frame-prefix literal span in the pool:
    //   {"target_topic":"<topic_k>","callback_topic":"<callback>","input_args":["
    const uint32_t* tool_name_off; const uint32_t* tool_name_len;
    const uint32_t* tool_lit_off;  const uint32_t* tool_lit_len;
    const uint32_t* tool_topic_id;     // registered id of the tool's subscribe topic (or 0xffffffff)
};

__device__ __forceinline__ unsigned long long ck_splitmix64(unsigned long long x) {
    x += 0x9E3779B97F4A7C15ull;
    x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
    x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
    return x ^ (x >> 31);
}

// uuid7 hex (RFC 9562): 48-bit unix ms | 0x7 | 12 random | 0b10 | 62 random, from (seed, index)
__device__ __forceinline__ void ck_uuid7_hex(unsigned long long unix_ms, unsigned long long seed, unsigned long long idx, u8* out32) {
    unsigned long long r0 = ck_splitmix64(seed + 2 * idx), r1 = ck_splitmix64(seed + 2 * idx + 1);
    unsigned long long hi = ((unix_ms & 0xFFFFFFFFFFFFull) << 16) | 0x7000ull | (r0 & 0xFFFull);
    unsigned long long lo = (0x2ull << 62) | (r1 & 0x3FFFFFFFFFFFFFFFull);
    const char* hx = "0123456789abcdef";
#pragma unroll
    for (int k = 0; k < 16; k++) { out32[k] = hx[(hi >> (60 - 4 * k)) & 15]; out32[16 + k] = hx[(lo >> (60 - 4 * k)) & 15]; }
}

__device__ __forceinline__ void SegWriter::hex_uuid7(unsigned long long unix_ms, unsigned long long seed, unsigned long long idx) {
    u8 tmp[32];
    ck_uuid7_hex(unix_ms, seed, idx, tmp);
    if (!in_glue) { in_glue = true; grun = gfill; }
#pragma unroll
    for (int k = 0; k < 32; k++) put(tmp[k]);
    total += 32;
}

// (the count / plan kernels of the fan-out are in ck_fanout2.cuh: one warp per record)

// TailCall to self (reference nodes/agent.py:171-175 -> nodes/base.py:120-136): the current frame is
// replaced by {target_topic: self.subscribe_topics[0], callback_topic: <popped frame's callback>,
// input_args: null, frame_id: fresh uuid7, overrides: null}; one payload, published keyed to the
// target and, as the handler's return value, unkeyed to publish_topic.
__global__ void __launch_bounds__(128)
ck_tailcall_plan_kernel(ck_view v, u32 n, u32* __restrict__ cols, u32 stride, const ck_agent_cfg* __restrict__ cfgp,
                        const u8* __restrict__ lit, unsigned long long unix_ms, unsigned long long seed,
                        const u8* __restrict__ aux, u8* __restrict__ glue,
                        ck_out_desc* __restrict__ descs, u32* __restrict__ pay_len, ck_pub* __restrict__ pubs) {
    u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
#define COL(k) cols[(size_t)(k) * stride + i]
    const ck_agent_cfg& cfg = *cfgp;
    ck_pub none; none.payload = 0xffffffffu; none.topic_id = -1; none.topic_off = none.topic_len = 0; none.record = i;
    none.has_key = 0; none.partition = -1; none.pad = 0;
    pubs[2 * i] = none; pubs[2 * i + 1] = none;
    pay_len[i] = 0;
    COL(CK_COL_NOUT) = 0;
    u32 rlen; const u8* rec = ck_rec(v, i, rlen);
    Rd r; r.init(rec, rlen);
    SegWriter w; w.init(descs + i, &r, lit, aux, glue + (size_t)i * CK_GLUE_STRIDE);
    if (COL(CK_COL_STATUS) != CK_OK) { COL(CK_COL_ACTION) = CK_ACT_NONE; w.finish(i); return; }
    if (COL(CK_COL_NFRAMES) == 0) { COL(CK_COL_ACTION) = CK_ACT_RAISES; w.finish(i); return; }   // unwind_frame on an empty stack
    u32 top_off = COL(CK_COL_TOP_OFF), top_len = COL(CK_COL_TOP_LEN);
    u32 cur = 0, fo = COL(CK_COL_FOV_OFF);
    if (r.at(fo) != 'n') {                                   // overrides rule (nodes/base.py:66-67)
        u32 so = COL(CK_COL_SOV_OFF);
        w.add(CK_SRC_INPUT, 0, so); w.add(CK_SRC_INPUT, fo, COL(CK_COL_FOV_LEN)); cur = so + COL(CK_COL_SOV_LEN);
    }
    w.add(CK_SRC_INPUT, cur, top_off - cur);
    w.add(CK_SRC_LIT, cfg.lit_tc_head[0], cfg.lit_tc_head[1]);
    w.add(CK_SRC_INPUT, COL(CK_COL_CB_OFF), COL(CK_COL_CB_LEN));
    w.add(CK_SRC_LIT, cfg.lit_tc_mid[0], cfg.lit_tc_mid[1]);
    w.hex_uuid7(unix_ms, seed, (unsigned long long)i);
    w.add(CK_SRC_LIT, cfg.lit_tail[0], cfg.lit_tail[1]);
    w.add(CK_SRC_INPUT, top_off + top_len, r.n - (top_off + top_len));
    w.finish(i);
    pay_len[i] = w.total;
    COL(CK_COL_ACTION) = CK_ACT_TAILCALL;
    ck_pub p = none; p.payload = i; p.topic_id = cfg.self_topic_id; p.has_key = 1; pubs[2 * i] = p;
    u32 nout = 1;
    if (cfg.publish_topic_id >= 0) { ck_pub q = none; q.payload = i; q.topic_id = cfg.publish_topic_id; pubs[2 * i + 1] = q; nout = 2; }
    COL(CK_COL_NOUT) = nout;
#undef COL
}

// ------------------------------------------------------------------------------------------------
// client reply path (reference client/deserialize.py:55-89, SURVEY.md section 8f row 3): the output of a final reply
// envelope is the first DataPart.data of final_output_parts, else the first TextPart.text (mode 0, auto);
// only the TextPart (mode 1, output_type=str); only the DataPart (mode 2, a typed output: the host validates
// the value).  Payload i = that value's JSON bytes; no publishes.  A reply without the wanted part is the
// reference's DeserializationError: CK_ACT_RAISES.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128)
ck_reply_plan_kernel(ck_view v, u32 n, u32* __restrict__ cols, u32 stride, u32 mode, u8* __restrict__ glue,
                     ck_out_desc* __restrict__ descs, u32* __restrict__ pay_len) {
    u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
#define COL(k) cols[(size_t)(k) * stride + i]
    ck_out_desc* d = descs + i;
    pay_len[i] = 0; d->nseg = 0; d->total_len = 0; d->record = i;
    COL(CK_COL_NOUT) = 0;
    if (COL(CK_COL_STATUS) != CK_OK) { COL(CK_COL_ACTION) = CK_ACT_NONE; return; }
    u32 doff = COL(CK_COL_ODATA_OFF), dlen = COL(CK_COL_ODATA_LEN), toff = COL(CK_COL_OTEXT_OFF), tlen = COL(CK_COL_OTEXT_LEN);
    u32 off, len;
    if (mode != 1 && dlen) { off = doff; len = dlen; }
    else if (mode != 2 && tlen) { off = toff; len = tlen; }
    else { COL(CK_COL_ACTION) = CK_ACT_RAISES; return; }
    u32 rlen; const u8* rec = ck_rec(v, i, rlen);
    Rd r; r.init(rec, rlen);
    SegWriter w; w.init(d, &r, nullptr, nullptr, glue + (size_t)i * CK_GLUE_STRIDE);
    w.add(CK_SRC_INPUT, off, len);
    if (!w.finish(i)) { COL(CK_COL_ACTION) = CK_ACT_RAISES; COL(CK_COL_STATUS) = CK_UNSUPPORTED; d->nseg = 0; d->total_len = 0; return; }
    pay_len[i] = w.total;
    COL(CK_COL_ACTION) = CK_ACT_REPLY;
#undef COL
}

// ------------------------------------------------------------------------------------------------
// multi-GPU exchange planning (SURVEY.md section 8e): the keyed publishes whose partition is owned by another
// rank (partition % world != rank) are selected and ordered by destination rank, stably, so that one
// variable-size all-to-all can forward them.  Two passes over the publish table around one scan:
//   count   : per block, a histogram of destinations (shared-memory atomics) -> hist[dest][block],
//             and the bytes per destination (one global atomic per destination per block)
//   (scan)  : exclusive scan of hist[] flattened destination-major = first output slot of every (dest, block)
//   scatter : every selected publish finds its rank among the block's publishes for the same destination
//             (__match_any_sync inside the warp + warp totals in shared memory) and writes its span
// ------------------------------------------------------------------------------------------------
#define CK_X_MAXWORLD 16
#define CK_X_BLOCK 256
__device__ __forceinline__ bool ck_x_foreign(const ck_pub& p, u32 rank, u32 world, u32& dest) {
    if (p.payload == 0xffffffffu || p.has_key != 1 || p.partition < 0) return false;
    dest = (u32)p.partition % world;
    return dest != rank;
}

__global__ void __launch_bounds__(CK_X_BLOCK)
ck_xplan_count_kernel(const ck_pub* __restrict__ pubs, u32 npubs, const u32* __restrict__ pay_len, u32 rank, u32 world,
                      u32* __restrict__ hist /* [world][gridDim.x] */, unsigned long long* __restrict__ nbytes /* [world] */) {
    __shared__ u32 s_cnt[CK_X_MAXWORLD];
    __shared__ unsigned long long s_bytes[CK_X_MAXWORLD];
    if (threadIdx.x < CK_X_MAXWORLD) { s_cnt[threadIdx.x] = 0; s_bytes[threadIdx.x] = 0; }
    __syncthreads();
    u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    u32 dest = 0;
    if (i < npubs) {
        ck_pub p = pubs[i];
        if (ck_x_foreign(p, rank, world, dest)) { atomicAdd(&s_cnt[dest], 1u); atomicAdd(&s_bytes[dest], (unsigned long long)pay_len[p.payload]); }
    }
    __syncthreads();
    if (threadIdx.x < world) {
        hist[(size_t)threadIdx.x * gridDim.x + blockIdx.x] = s_cnt[threadIdx.x];
        if (s_bytes[threadIdx.x]) atomicAdd(&nbytes[threadIdx.x], s_bytes[threadIdx.x]);
    }
}

__global__ void __launch_bounds__(CK_X_BLOCK)
ck_xplan_scatter_kernel(const ck_pub* __restrict__ pubs, u32 npubs, const u32* __restrict__ pay_len, const long long* __restrict__ out_off,
                        u32 rank, u32 world, const long long* __restrict__ base /* scan of hist */,
                        long long* __restrict__ x_src_off, long long* __restrict__ x_len, u32* __restrict__ x_len32, u32* __restrict__ x_pub) {
    __shared__ u32 s_w[CK_X_BLOCK / 32][CK_X_MAXWORLD];
    u32 lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x < (CK_X_BLOCK / 32) * CK_X_MAXWORLD) (&s_w[0][0])[threadIdx.x] = 0;
    __syncthreads();
    u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    u32 dest = 0, rank_in_warp = 0;
    bool sel = false;
    ck_pub p;
    if (i < npubs) { p = pubs[i]; sel = ck_x_foreign(p, rank, world, dest); }
    u32 act = __ballot_sync(0xffffffffu, sel);
    if (sel) {
        u32 same = __match_any_sync(act, dest);
        rank_in_warp = __popc(same & ((1u << lane) - 1u));
        if (rank_in_warp == 0) s_w[warp][dest] = __popc(same);
    }
    __syncthreads();
    if (sel) {
        u32 before = 0;
        for (u32 w = 0; w < warp; w++) before += s_w[w][dest];
        long long slot = base[(size_t)dest * gridDim.x + blockIdx.x] + before + rank_in_warp;
        u32 len = pay_len[p.payload];
        x_src_off[slot] = out_off[p.payload]; x_len[slot] = (long long)len; x_len32[slot] = len; x_pub[slot] = i;
    }
}

// ------------------------------------------------------------------------------------------------
// exclusive scan u32 -> int64 (three small kernels; lengths are tiny next to the payload bytes)
// ------------------------------------------------------------------------------------------------
#define CK_SCAN_BLOCK 256
#define CK_SCAN_ITEMS 8
#define CK_SCAN_TILE (CK_SCAN_BLOCK * CK_SCAN_ITEMS)

__device__ __forceinline__ unsigned long long ck_block_scan_excl(unsigned long long v, unsigned long long* total) {
    __shared__ unsigned long long wsum[CK_SCAN_BLOCK / 32];
    u32 lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    unsigned long long x = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) { unsigned long long y = __shfl_up_sync(0xffffffffu, x, d); if (lane >= d) x += y; }
    if (lane == 31) wsum[wid] = x;
    __syncthreads();
    if (wid == 0) {
        unsigned long long s = lane < CK_SCAN_BLOCK / 32 ? wsum[lane] : 0;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) { unsigned long long y = __shfl_up_sync(0xffffffffu, s, d); if (lane >= d) s += y; }
        if (lane < CK_SCAN_BLOCK / 32) wsum[lane] = s;
    }
    __syncthreads();
    unsigned long long base = wid ? wsum[wid - 1] : 0;
    *total = wsum[CK_SCAN_BLOCK / 32 - 1];
    __syncthreads();
    return base + x - v;
}

// pad = 15: every length is rounded up to a multiple of 16 so that payloads start 16-byte aligned
__global__ void __launch_bounds__(CK_SCAN_BLOCK)
ck_scan_tiles_kernel(const u32* __restrict__ len, u32 n, unsigned long long* __restrict__ tile_sum, u32 pad) {
    u32 base = blockIdx.x * CK_SCAN_TILE + threadIdx.x * CK_SCAN_ITEMS;
    unsigned long long s = 0;
#pragma unroll
    for (int k = 0; k < CK_SCAN_ITEMS; k++) if (base + k < n) s += (len[base + k] + pad) & ~pad;
    unsigned long long total;
    ck_block_scan_excl(s, &total);
    if (threadIdx.x == 0) tile_sum[blockIdx.x] = total;
}

__global__ void __launch_bounds__(CK_SCAN_BLOCK)
ck_scan_sums_kernel(unsigned long long* __restrict__ tile_sum, u32 ntiles, unsigned long long* __restrict__ grand) {
    unsigned long long carry = 0;
    for (u32 base = 0; base < ntiles; base += CK_SCAN_BLOCK) {
        u32 i = base + threadIdx.x;
        unsigned long long v = i < ntiles ? tile_sum[i] : 0, total;
        unsigned long long e = ck_block_scan_excl(v, &total);
        if (i < ntiles) tile_sum[i] = carry + e;
        carry += total;
    }
    if (threadIdx.x == 0) *grand = carry;
}

__global__ void __launch_bounds__(CK_SCAN_BLOCK)
ck_scan_apply_kernel(const u32* __restrict__ len, u32 n, const unsigned long long* __restrict__ tile_sum,
                     long long* __restrict__ out_off /* n+1 */, u32 pad) {
    u32 base = blockIdx.x * CK_SCAN_TILE + threadIdx.x * CK_SCAN_ITEMS;
    u32 v[CK_SCAN_ITEMS];
    unsigned long long s = 0;
#pragma unroll
    for (int k = 0; k < CK_SCAN_ITEMS; k++) { v[k] = (base + k < n) ? ((len[base + k] + pad) & ~pad) : 0; s += v[k]; }
    unsigned long long total;
    unsigned long long e = ck_block_scan_excl(s, &total) + tile_sum[blockIdx.x];
#pragma unroll
    for (int k = 0; k < CK_SCAN_ITEMS; k++) { if (base + k < n) out_off[base + k] = (long long)e; e += v[k]; }
    if (blockIdx.x == gridDim.x - 1 && threadIdx.x == CK_SCAN_BLOCK - 1) out_off[n] = (long long)e;
}

// ------------------------------------------------------------------------------------------------
// encode: one warp per payload gathers its segments into out[out_off[i] ...)
// ------------------------------------------------------------------------------------------------
// warp-cooperative byte copy.  Short pieces (the literal / id segments of a splice, <= 128 B) go one
// byte per lane; long pieces go as 16-byte destination-aligned vector stores, each assembled from two
// source-aligned 16-byte loads with a warp-uniform byte shift (src and dst are generally misaligned
// relative to each other: JSON spans start anywhere).
__device__ __forceinline__ u32 ck_fsr(u32 lo, u32 hi, u32 bits) { return __funnelshift_r(lo, hi, bits); }

__device__ __forceinline__ void ck_warp_copy(u8* __restrict__ dst, const u8* __restrict__ src, u32 len, u32 lane) {
    if (len <= 128) {
#pragma unroll
        for (u32 k = 0; k < 4; k++) { u32 idx = lane + 32 * k; if (idx < len) dst[idx] = src[idx]; }
        return;
    }
    u32 head = (u32)((16 - ((uintptr_t)dst & 15)) & 15);
    if (lane < head) dst[lane] = src[lane];
    dst += head; src += head; len -= head;
    u32 nvec = len >> 4;
    u32 sh = (u32)((uintptr_t)src & 15);
    const uint4* s16 = (const uint4*)((uintptr_t)src - sh);
    uint4* d16 = (uint4*)dst;
    u32 q = sh >> 2, bits = (sh & 3) * 8;
    for (u32 v = lane; v < nvec; v += 32) {
        uint4 a = __ldg(s16 + v);
        uint4 o;
        if (sh == 0) o = a;
        else {
            uint4 b = __ldg(s16 + v + 1);       // may touch <= 31 bytes past the span: inside the padded buffers
            u32 w0, w1, w2, w3, w4;
            switch (q) {                        // warp-uniform
                case 0: w0 = a.x; w1 = a.y; w2 = a.z; w3 = a.w; w4 = b.x; break;
                case 1: w0 = a.y; w1 = a.z; w2 = a.w; w3 = b.x; w4 = b.y; break;
                case 2: w0 = a.z; w1 = a.w; w2 = b.x; w3 = b.y; w4 = b.z; break;
                default: w0 = a.w; w1 = b.x; w2 = b.y; w3 = b.z; w4 = b.w; break;
            }
            o.x = ck_fsr(w0, w1, bits); o.y = ck_fsr(w1, w2, bits); o.z = ck_fsr(w2, w3, bits); o.w = ck_fsr(w3, w4, bits);
        }
        d16[v] = o;
    }
    u32 done = nvec << 4, tail = len - done;
    if (lane < tail) dst[done + lane] = src[done + lane];
}

// ------------------------------------------------------------------------------------------------
// encode: one warp per payload.  The payload is a sequence of aligned 16-byte output vectors; lane l of
// iteration k produces vector 32k + l with one aligned 16-byte store.  Segments may start and end at any
// byte (ck_out_desc), so a vector either lies inside one segment — one unaligned 16-byte gather from that
// segment's source, the common case — or crosses segment boundaries and is assembled from the masked,
// shifted bytes of every segment it overlaps.  The segment holding a vector's first byte is found by a
// 4-step binary search over the prefix-summed segment starts (lanes 0..15 hold the table); the boundary
// lanes, which diverge, read the table from shared memory instead.  Descriptors in the aligned layout
// (SegWriter) take the single-gather path throughout (a warp-uniform choice per payload, below).
// ------------------------------------------------------------------------------------------------
#define CK_EMIT_THREADS 256
#define CK_EMIT_MINB 8         // 64 warps per SM: <= 32 registers, as the single-gather emitter used (no spills)
// 16 bytes from an arbitrary address: 5 aligned words (may touch <= 19 bytes past the 16: all sources are padded)
__device__ __forceinline__ uint4 ck_gather16(const u8* src) {
    u32 sh = (u32)((uintptr_t)src & 3u) * 8u;
    const u32* a = (const u32*)((uintptr_t)src & ~(uintptr_t)3);
    u32 w0 = __ldg(a), w1 = __ldg(a + 1), w2 = __ldg(a + 2), w3 = __ldg(a + 3), w4 = __ldg(a + 4);
    uint4 o;
    o.x = __funnelshift_r(w0, w1, sh); o.y = __funnelshift_r(w1, w2, sh);
    o.z = __funnelshift_r(w2, w3, sh); o.w = __funnelshift_r(w3, w4, sh);
    return o;
}
struct ck_emit_segs { const u8* ptr[CK_MAX_SEGS]; u32 start[CK_MAX_SEGS]; u32 end[CK_MAX_SEGS]; };   // one per warp
// ORs the bytes of x that land in output bytes [b0, b1) of the vector at pos into (lo, hi); x holds output bytes b0..b0+15
__device__ __forceinline__ void ck_emit_part(uint4 x, u32 b0, u32 b1, u32 pos, unsigned long long& lo, unsigned long long& hi) {
    unsigned long long xl = ((unsigned long long)x.y << 32) | x.x, xh = ((unsigned long long)x.w << 32) | x.z;
    u32 nb = b1 - b0, sh = b0 - pos;                               // nb + sh <= 16
    if (nb < 8) { xl &= (1ull << (8 * nb)) - 1ull; xh = 0; }
    else if (nb < 16) xh &= (1ull << (8 * (nb - 8))) - 1ull;
    if (sh >= 8) { xh = xl << (8 * (sh - 8)); xl = 0; }
    else if (sh) { xh = (xh << (8 * sh)) | (xl >> (64 - 8 * sh)); xl <<= 8 * sh; }
    lo |= xl; hi |= xh;
}
// output bytes [pos, lim) (lim - pos <= 16) of a vector that crosses segment boundaries: segment s holds bytes
// [pos, s_end), already gathered in x0 (the same gather as the single-segment path); the later segments start inside the
// vector and are gathered one after the other.  (Issuing two of them at a time needs 38 registers, i.e. 6 blocks per SM:
// config-2 emit 1.22 ms against 1.05 ms for this loop at 8 blocks, H100 at 400 W.)
__device__ __forceinline__ uint4 ck_emit_boundary(const ck_emit_segs* t, u32 s, u32 pos, u32 lim, uint4 x0, u32 s_end) {
    unsigned long long lo = 0, hi = 0;
    ck_emit_part(x0, pos, s_end, pos, lo, hi);
    for (u32 k = s + 1; k < CK_MAX_SEGS; k++) {
        u32 a1 = t->start[k];
        if (a1 >= lim) break;
        u32 e1 = t->end[k]; e1 = e1 < lim ? e1 : lim;
        if (e1 > a1) ck_emit_part(ck_gather16(t->ptr[k]), a1, e1, pos, lo, hi);
    }
    return make_uint4((u32)lo, (u32)(lo >> 32), (u32)hi, (u32)(hi >> 32));
}
__global__ void __launch_bounds__(CK_EMIT_THREADS, CK_EMIT_MINB)
ck_emit_kernel(ck_view vw, const u8* __restrict__ lit,
               const u8* __restrict__ aux, const u8* __restrict__ glue, const ck_out_desc* __restrict__ descs,
               const long long* __restrict__ out_off, u32 n, u8* __restrict__ out, long long out_cap) {
    __shared__ ck_emit_segs s_tab[CK_EMIT_THREADS / 32];
    u32 warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (warp >= n) return;
    long long o0 = out_off[warp], o1 = out_off[warp + 1];
    if (o1 == o0 || o1 > out_cap) return;    // overflow is reported by ck_fetch_output, never written
    const ck_out_desc* d = descs + warp;
    u32 nseg = d->nseg;
    if (nseg == 0 || nseg > CK_MAX_SEGS) return;
    u32 total = d->total_len;
    u32 rec_len; const u8* rec = ck_rec(vw, d->record, rec_len);
    // segment table: lane s holds segment s (source address, output start, length); lanes past nseg hold empty
    // segments starting at the payload's end, so the search below never picks them
    u32 my_len = 0;
    const u8* my_ptr = rec;
    if (lane < nseg) {
        uint2 sg = *(const uint2*)d->seg[lane]; u32 so = sg.x, ls = sg.y;
        u32 src = ls & 3u;
        my_len = ls >> 2;
        my_ptr = (src == CK_SRC_INPUT) ? rec + so : (src == CK_SRC_LIT ? lit + so : (src == CK_SRC_AUX ? aux + so
                 : glue + (size_t)warp * CK_GLUE_STRIDE + so));
    }
    u32 start = my_len;                      // exclusive prefix sum of the segment lengths = output offset (lanes 0..15)
#pragma unroll
    for (int k = 1; k < CK_MAX_SEGS; k <<= 1) { u32 y = __shfl_up_sync(0xffffffffu, start, k); if (lane >= k) start += y; }
    start -= my_len;
    u32 end = start + my_len;
    unsigned long long pbits = (unsigned long long)(uintptr_t)my_ptr;
    u32 plo = (u32)pbits, phi = (u32)(pbits >> 32);
    uint4* dst = (uint4*)(out + o0);
    u32 nvec = (total + 15u) >> 4;
    // warp-uniform choice per payload: in the aligned layout (SegWriter: every segment starts on a vector, all but the
    // last are whole vectors) no vector crosses a segment, and the segment of a vector is found without a search — the
    // lanes holding the table mark the vectors where a segment starts, one warp-wide OR gives the mask, a popcount the index.
    // The popcount counts non-empty segments only, so it is a lane index only if no empty segment comes before the last one:
    // an empty segment is not a whole vector, and a payload with one before its last segment takes the search below
    u32 part = my_len ? (my_len & 15u) : 1u;         // 0: the segment is one or more whole vectors
    bool aligned = __all_sync(0xffffffffu, lane >= nseg || ((start & 15u) == 0 && (lane + 1 == nseg || part == 0)));
    ck_emit_segs* tab = &s_tab[threadIdx.x >> 5];
    if (!aligned) {                          // the table for the boundary lanes
        if (lane < CK_MAX_SEGS) { tab->ptr[lane] = my_ptr; tab->start[lane] = start; tab->end[lane] = end; }
        __syncwarp();
    }
    u32 start_vec = start >> 4, segs_before = 0;
    for (u32 v0 = 0; v0 < nvec; v0 += 32) {
        u32 v = v0 + lane, pos = v << 4;
        u32 seg = 0;                         // last segment starting at or before pos
        if (aligned) {
            u32 bit = (lane < nseg && my_len && start_vec >= v0 && start_vec < v0 + 32) ? (1u << (start_vec - v0)) : 0u;
            u32 mask = __reduce_or_sync(0xffffffffu, bit);
            seg = (segs_before + __popc(mask & (0xffffffffu >> (31 - lane))) - 1) & 31;
            segs_before += __popc(mask);
        } else {
#pragma unroll
            for (u32 step = CK_MAX_SEGS / 2; step; step >>= 1)
                if (__shfl_sync(0xffffffffu, start, seg + step) <= pos) seg += step;
        }
        u32 s_start = __shfl_sync(0xffffffffu, start, seg);
        u32 s_lo = __shfl_sync(0xffffffffu, plo, seg), s_hi = __shfl_sync(0xffffffffu, phi, seg);
        u32 s_end = aligned ? 0u : __shfl_sync(0xffffffffu, end, seg);
        if (v < nvec) {
            uint4 o = ck_gather16((const u8*)(uintptr_t)(((unsigned long long)s_hi << 32) | s_lo) + (pos - s_start));
            if (!aligned) {
                u32 lim = total - pos < 16u ? total : pos + 16u;
                if (s_end < lim) o = ck_emit_boundary(tab, seg, pos, lim, o, s_end);
            }
            dst[v] = o;
        }
    }
}

// ------------------------------------------------------------------------------------------------
// route: destination topic string -> registered topic id (hash probe + byte compare), Kafka
// partition of the key (murmur2, the default partitioner's hash), and a per-topic histogram
// aggregated inside the warp (match_any + popc: one atomic per distinct topic per warp).
// ------------------------------------------------------------------------------------------------
// Kafka's default partitioner hashes the KEY bytes = correlation_id.encode() (nodes/base.py:86): the JSON string
// content unescaped.  Raw content without a backslash is its own unescaped form (the common case: ids are hex /
// uuid text); otherwise the escapes pydantic emits (\" \\ \n \t \r \b \f \u00xx) are decoded on the fly.
template <class R>
__device__ __forceinline__ u32 ck_key_byte(R& r, u32& p) {
    u8 c = r.at(p++);
    if (c != '\\') return c;
    u8 e = r.at(p++);
    switch (e) {
        case 'n': return '\n'; case 't': return '\t'; case 'r': return '\r'; case 'b': return '\b'; case 'f': return '\f';
        case 'u': {
            u32 v = 0;
            for (int k = 0; k < 4; k++) { u8 h = r.at(p++); v = (v << 4) | (u32)(h <= '9' ? h - '0' : (h | 0x20) - 'a' + 10); }
            return v & 0xffu;                       // canonical \u00xx only (controls); wider code points are emitted raw
        }
        default: return e;                           // \" and \\ (and \/ which pydantic never emits)
    }
}
template <class R>
__device__ __forceinline__ u32 ck_murmur2_key(R& r, u32 off, u32 len) {
    const u32 m = 0x5bd1e995u;
    // one pass over the raw content, 8 bytes per read: its hash, and whether it holds a backslash at all
    u32 h = 0x9747b28cu ^ len, len4 = len >> 2, tail = len & 3u;
    u64 esc = 0;
    for (u32 i = 0; i < len4; i += 2) {
        u64 x = r.load8(off + 4 * i);
        if (i + 1 == len4) x &= 0xffffffffull;          // the last 4-byte block: the bytes after it are not the key's
        esc |= ck_haszero(x ^ CK_REP8('\\'));
        u32 k = (u32)x;
        k *= m; k ^= k >> 24; k *= m; h *= m; h ^= k;
        if (i + 1 < len4) { k = (u32)(x >> 32); k *= m; k ^= k >> 24; k *= m; h *= m; h ^= k; }
    }
    if (tail) {
        u32 t = (u32)r.load8(off + (len4 << 2)) & (0xffffffu >> (8 * (3 - tail)));
        esc |= ck_haszero((u64)t ^ CK_REP8('\\'));
        h ^= t; h *= m;
    }
    if (!esc) { h ^= h >> 13; h *= m; h ^= h >> 15; return h; }
    u32 ulen = 0;
    for (u32 p = off; p < off + len; ulen++) ck_key_byte(r, p);
    h = 0x9747b28cu ^ ulen;
    u32 p = off, k = 0, nb = 0, left = ulen;
    while (left >= 4) {
        k = ck_key_byte(r, p); k |= ck_key_byte(r, p) << 8; k |= ck_key_byte(r, p) << 16; k |= ck_key_byte(r, p) << 24;
        k *= m; k ^= k >> 24; k *= m; h *= m; h ^= k;
        left -= 4;
    }
    u32 t0 = 0, t1 = 0, t2 = 0;
    nb = left;
    if (nb >= 1) t0 = ck_key_byte(r, p);
    if (nb >= 2) t1 = ck_key_byte(r, p);
    if (nb >= 3) t2 = ck_key_byte(r, p);
    if (nb == 3) h ^= t2 << 16;
    if (nb >= 2) h ^= t1 << 8;
    if (nb >= 1) { h ^= t0; h *= m; }
    h ^= h >> 13; h *= m; h ^= h >> 15;
    return h;
}

// topic string (raw JSON content at [off, off+len) of the record) -> registered id, -1 if not registered
template <class R>
__device__ __forceinline__ int ck_topic_lookup(R& r, u32 off, u32 len, const ck_topic_table& tab, u32* hash_out = nullptr) {
    u32 h = 2166136261u;
    for (u32 i = 0; i < len; i++) h = (h ^ r.at(off + i)) * 16777619u;
    if (!h) h = 1u;
    if (hash_out) *hash_out = h;          // unregistered topics (a client's reply topic): the host groups them by this hash
    if (!len || !tab.cap) return -1;
    u32 slot = h & (tab.cap - 1);
    for (u32 probe = 0; probe < tab.cap; probe++) {
        u32 th = tab.hash[slot];
        if (th == 0) return -1;
        if (th == h && tab.name_len[slot] == len) {
            const u8* nm = tab.names + tab.name_off[slot];
            bool eq = true;
            for (u32 b = 0; b < len; b++) if (nm[b] != r.at(off + b)) { eq = false; break; }
            if (eq) return tab.id[slot];
        }
        slot = (slot + 1) & (tab.cap - 1);
    }
    return -1;
}

__global__ void __launch_bounds__(256)
ck_route_kernel(ck_view vw, const u32* __restrict__ cols, u32 stride,
                ck_pub* __restrict__ pubs, u32 npubs, ck_topic_table tab, u32 num_partitions, u32* __restrict__ topic_hist, u32 hist_cap) {
    u32 j = blockIdx.x * blockDim.x + threadIdx.x;
    bool live = j < npubs;
    ck_pub p;
    if (live) { p = pubs[j]; live = (p.payload != 0xffffffffu); }
    int tid = -1;
    if (live) {
        u32 rec_len; const u8* rec = ck_rec(vw, p.record, rec_len);
        GRd r; r.init(rec, rec_len);
        tid = p.topic_id;
        if (tid < 0 && p.topic_len && tab.cap) tid = ck_topic_lookup(r, p.topic_off, p.topic_len, tab, &pubs[j].pad);
        int part = -1;
        if (p.has_key && num_partitions) {
            u32 co = cols[(size_t)CK_COL_CORR_OFF * stride + p.record], cl = cols[(size_t)CK_COL_CORR_LEN * stride + p.record];
            part = (int)((ck_murmur2_key(r, co, cl) & 0x7fffffffu) % num_partitions);
        }
        pubs[j].topic_id = tid;
        pubs[j].partition = part;
    }
    // warp-aggregated histogram of destination topics
    u32 active = __ballot_sync(0xffffffffu, live && tid >= 0 && (u32)tid < hist_cap);
    if (live && tid >= 0 && (u32)tid < hist_cap) {
        u32 peers = __match_any_sync(active, tid);
        if ((threadIdx.x & 31) == (u32)(__ffs(peers) - 1)) atomicAdd(topic_hist + tid, __popc(peers));
    }
}

#include "ck_walk_long.cuh"
#include "ck_plan.cuh"
#include "ck_fanout2.cuh"
#include "ck_gate.cuh"
#include "ck_kafka.cuh"
#include "ck_group.cuh"
#include "ck_xsend.cuh"

#endif  // CK_KERNELS_CUH
