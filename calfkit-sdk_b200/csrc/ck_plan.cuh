// Tool-node plan (ToolNodeDef.run, all three modes), thread per record, staged through shared memory, with the route
// step of its publishes folded in.
//
// Why: a thread-per-record planner that reads and writes global memory directly issued ~150 dependent, lane-divergent
// global loads per warp (byte / 8-byte reads of ten far-apart spots of each record) and 80 lane-divergent store
// instructions (the 144 B descriptor, the 512 B-stride glue slot and the two 32 B publishes written array-of-structs
// by one thread each, so most sectors of every store request were partial) — latency bound, moving several times the
// algorithmic DRAM traffic.  Here
//   * the splice is written as it is: one segment per piece (input spans from the walker's columns, literals from the
//     pool, a host result from the aux blob) at whatever byte it falls on — the emitter assembles the vectors that
//     cross a piece boundary (ck_emit_kernel) — so no glue text is built and no record byte is read for the splice,
//   * the record is read only where a decision needs it (the args object for the template, a non-string
//     input_args[0], the callback topic, the correlation id), through a 64-byte per-thread window in shared memory
//     filled by 16-byte cp.async copies (no data registers; one memory round trip per 48 fresh bytes),
//   * the descriptor and the two publishes are assembled in shared memory and written to HBM by the whole warp,
//     16 bytes per lane, two records per store instruction (full sectors),
//   * the route step (topic table probe, murmur2 partition of the key, per-topic histogram) runs in the same thread.
// Every splice fits one descriptor: at most CK_TOOL_FIXED_PIECES + CK_TPL_MAX_PARTS <= CK_MAX_SEGS pieces.
#ifndef CK_PLAN_CUH
#define CK_PLAN_CUH

#define CK_P2_THREADS 128
#define CK_P2_WIN 64u                 // window bytes per thread
#define CK_P2_WSTRIDE 80u             // slot stride (the pad spreads the slots over the banks)
// 7 blocks per SM: 28,672 B of shared memory per block (windows + descriptors) and <= 72 registers both allow 7
#ifndef CK_P2_MINB
#define CK_P2_MINB 7
#endif

__device__ __forceinline__ void ck_prefetch_l2(const u8* p) { asm volatile("prefetch.global.L2 [%0];" :: "l"(p)); }

// out of line and by value: a member function taking `this` would pin the reader (and everything that points to it) in
// local memory — the first version of this kernel made 307 local-memory loads per warp that way
__device__ __noinline__ u32 ck_p2_refill(const u8* gb, u32 ap, u32 lim) {
    u32 wb = ap & ~15u;
    wb = wb >= 16u ? wb - 16u : 0u;
    u32 dst = (u32)__cvta_generic_to_shared((const u8*)ck_win_smem + threadIdx.x * CK_P2_WSTRIDE);
    const u8* src = gb + wb;
#pragma unroll
    for (u32 k = 0; k < CK_P2_WIN; k += 16)
        if (wb + k < lim) asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" :: "r"(dst + k), "l"(src + k) : "memory");
    asm volatile("cp.async.wait_all;" ::: "memory");
    return wb;
}

struct PRd {
    static const bool kWindow = true;
    static const bool kTrustFloats = false;
    const u8* g; u32 n; u32 wbase; u32 m; const u8* wp;
    __device__ __forceinline__ void init(const u8* base, u32 len, u32 st = CK_WIN_NONE) {
        g = base; n = len; wbase = st; m = (u32)((uintptr_t)base & 15);
        wp = (const u8*)ck_win_smem + threadIdx.x * CK_P2_WSTRIDE;
    }
    __device__ __forceinline__ u32 st() const { return wbase; }
    __device__ __forceinline__ void set_st(u32 s) { wbase = s; }
    __device__ __forceinline__ void invalidate() { wbase = CK_WIN_NONE; }
    __device__ __forceinline__ void refill(u32 ap) { wbase = ck_p2_refill(g - m, ap, (m + n + 15u) & ~15u); }
    __device__ __forceinline__ u8 at(u32 pos) {
        u32 ap = pos + m, o = ap - wbase;
        if (o >= CK_P2_WIN) { refill(ap); o = ap - wbase; }
        return wp[o];
    }
    __device__ __forceinline__ u64 load8(u32 pos) {
        u32 ap = pos + m, o = ap - wbase;
        if (o > CK_P2_WIN - 12u) { refill(ap); o = ap - wbase; }
        const u32* w = (const u32*)(wp + (o & ~3u));
        u32 a = w[0], b = w[1], c = w[2], sh = (o & 3u) * 8u;
        return ((u64)__funnelshift_r(b, c, sh) << 32) | __funnelshift_r(a, b, sh);
    }
    __device__ __forceinline__ void load16(u32 pos, u64& x0, u64& x1) { x0 = load8(pos); x1 = load8(pos + 8); }
};

struct ck_p2_stage { ck_out_desc desc[32]; };   // one per warp
#define CK_P2_SMEM (CK_P2_THREADS * CK_P2_WSTRIDE + (CK_P2_THREADS / 32) * sizeof(ck_p2_stage))

// the splice as a list of pieces, one segment each, at any byte boundary of the output (ck_out_desc)
struct SpliceWriter {
    ck_out_desc* d; u32 n, total;
    __device__ __forceinline__ void init(ck_out_desc* dd) { d = dd; n = 0; total = 0; }
    __device__ __forceinline__ void add(u32 src, u32 off, u32 len) {
        if (len == 0) return;
        *(uint2*)d->seg[n] = make_uint2(off, (len << 2) | src); n++;
        total += len;
    }
    __device__ __forceinline__ void finish(u32 record) { d->nseg = n; d->record = record; d->total_len = total; d->pad = 0; }
};

struct ck_p2_res { u32 action, nout, status, pay_len, desc_len; };

// the plan proper: ToolNodeDef.run + handler dispatch + _publish_action(ReturnCall | Silent) + overrides rule
// (nodes/tool.py:37-86, nodes/base.py:66-67,105-118,137-145,157-160), into shared memory
//   mode 0: classify; a host tool gets the record's args JSON as its payload (one segment), no publishes
//   mode 1: classify + the final payload from the device template or the host's results (aux)
//   mode 2: plain ReturnCall(state) of a node whose run() left the state as it is on the wire (the Agent's final output)
__device__ __forceinline__ void
ck_plan_tool_one(ck_view v, u32 i, const u32* __restrict__ cols, u32 stride, const ck_tool_cfg& cfg, const u8* __restrict__ lit,
                 const long long* __restrict__ aux_off, int mode,
                 ck_out_desc* d, ck_pub* pb /* [2] */, const ck_topic_table& tab, u32 num_partitions, ck_p2_res& out) {
#define COL(k) cols[(size_t)(k) * stride + i]
    ck_pub none; none.payload = 0xffffffffu; none.topic_id = -1; none.topic_off = none.topic_len = 0; none.record = i;
    none.has_key = 0; none.partition = -1; none.pad = 0;
    pb[0] = none; pb[1] = none;
    d->nseg = 0; d->record = i; d->total_len = 0; d->pad = 0;
    out.action = CK_ACT_NONE; out.nout = 0; out.pay_len = 0; out.desc_len = 16;
    u32 status = COL(CK_COL_STATUS);
    out.status = status;
    if (status != CK_OK) return;
    u32 rlen; const u8* rec = ck_rec(v, i, rlen);
    u32 nframes = COL(CK_COL_NFRAMES), nargs = COL(CK_COL_NARGS), kinds = COL(CK_COL_ARGKINDS);
    u32 tr_off = COL(CK_COL_TR_OFF), tr_len = COL(CK_COL_TR_LEN), top_off = COL(CK_COL_TOP_OFF), top_len = COL(CK_COL_TOP_LEN);
    u32 fov_off = COL(CK_COL_FOV_OFF), fov_len = COL(CK_COL_FOV_LEN), sov_off = COL(CK_COL_SOV_OFF), sov_len = COL(CK_COL_SOV_LEN);
    u32 cb_off = COL(CK_COL_CB_OFF), cb_len = COL(CK_COL_CB_LEN), corr_off = COL(CK_COL_CORR_OFF), corr_len = COL(CK_COL_CORR_LEN);
    u32 id_off = COL(CK_COL_ARG0_OFF), id_len = COL(CK_COL_ARG0_LEN);
    if (nframes > 0) {
        // the spots this thread will read, far apart in the record: start all of them towards L2 now so that the
        // window refills below find them there instead of queueing one DRAM miss behind the other
        ck_prefetch_l2(rec + COL(CK_COL_ARGS_OFF)); ck_prefetch_l2(rec + cb_off); ck_prefetch_l2(rec + corr_off);
    }
    PRd r; r.init(rec, rlen);
    SpliceWriter w; w.init(d);
    // a canonical OverridesState is an object, never 4 bytes long: "null" <=> length 4 (no read needed)
    bool fov_set = nframes > 0 && fov_len != 4;
    u32 cur = 0;
    if (mode == 2) {
        if (nframes == 0) { out.action = CK_ACT_RAISES; return; }
    } else {
        u32 action;
        if (nframes == 0 || nargs != 2) action = CK_ACT_RAISES;
        else if (!(kinds & 1u)) { u8 c0 = r.at(id_off); action = (c0 == '[' || c0 == '{') ? CK_ACT_RAISES : CK_ACT_SILENT; }
        else action = COL(CK_COL_CALL_VAL_LEN) ? CK_ACT_RETURN : CK_ACT_SILENT;
        if (action == CK_ACT_RAISES) { out.action = action; return; }
        if (mode == 0) {
            if (action == CK_ACT_SILENT) { out.action = action; return; }
            w.add(CK_SRC_INPUT, COL(CK_COL_ARGS_OFF), COL(CK_COL_ARGS_LEN));
            w.finish(i);
            out.action = CK_ACT_HOST_TOOL; out.pay_len = w.total; out.desc_len = 16 + 8 * w.n;
            return;
        }
        if (action == CK_ACT_SILENT) {
            // only the handler-return publish: the input envelope, unchanged (nodes/base.py:142, worker.py:52-53)
            w.add(CK_SRC_INPUT, 0, r.n);
            w.finish(i);
            out.action = action;
            if (cfg.publish_topic_id >= 0) {
                out.pay_len = r.n; out.nout = 1;
                ck_pub p = none; p.payload = i; p.topic_id = cfg.publish_topic_id; pb[1] = p;
            }
            out.desc_len = 16 + 8 * w.n;
            return;
        }
        Span args = {COL(CK_COL_ARGS_OFF), COL(CK_COL_ARGS_LEN)};
        Span existing = {COL(CK_COL_RES_OFF), COL(CK_COL_RES_LEN)};
        bool host = cfg.tpl_nparts == 0 || aux_off != nullptr;   // host results, when supplied, win over the template
        if (host && aux_off == nullptr) { out.action = CK_ACT_HOST_TOOL; return; }
        if (!host && r.at(args.off) != '{') { out.action = CK_ACT_RAISES; out.status = CK_UNSUPPORTED; return; }
        if (existing.len == 0) {
            w.add(CK_SRC_INPUT, 0, tr_off + tr_len - 1);
            if (tr_len > 2) w.add(CK_SRC_LIT, cfg.lit_comma_q[0], cfg.lit_comma_q[1]); else w.add(CK_SRC_LIT, cfg.lit_q[0], cfg.lit_q[1]);
            w.add(CK_SRC_INPUT, id_off, id_len);
            w.add(CK_SRC_LIT, cfg.lit_open[0], cfg.lit_open[1]);
            cur = tr_off + tr_len - 1;
        } else {
            w.add(CK_SRC_INPUT, 0, existing.off);
            w.add(CK_SRC_LIT, cfg.lit_value_open[0], cfg.lit_value_open[1]);
            cur = existing.off + existing.len;
        }
        // the tool's return value as JSON: the host's result, or the template's literals and raw string arguments
        if (host) {
            long long r0 = aux_off[i], r1 = aux_off[i + 1];
            w.add(CK_SRC_AUX, (u32)r0, (u32)(r1 - r0));
        } else {
            for (u32 k = 0; k < cfg.tpl_nparts; k++) {
                if (cfg.tpl_kind[k] == 0) { w.add(CK_SRC_LIT, cfg.tpl_off[k], cfg.tpl_len[k]); continue; }
                u32 p = args.off + 1; bool found = false;
                while (p < args.off + args.len && r.at(p) != '}') {
                    Span k2; ck_string(r, p, k2); p++;
                    u32 vv = p; ck_skip_value(r, p);
                    bool eq = (k2.len == cfg.tpl_len[k]);
                    for (u32 b = 0; eq && b < k2.len; b++) eq = (r.at(k2.off + b) == lit[cfg.tpl_off[k] + b]);
                    if (eq) {
                        if (r.at(vv) != '"') break;                      // non-string argument: host formats it
                        w.add(CK_SRC_INPUT, vv + 1, p - vv - 2);
                        found = true; break;
                    }
                    if (p < r.n && r.at(p) == ',') p++;
                }
                // the segments written so far are not published: nseg stays 0 and only the header is written out
                if (!found) { out.action = CK_ACT_RAISES; out.status = CK_UNSUPPORTED; return; }
            }
        }
        w.add(CK_SRC_LIT, cfg.lit_mid[0], cfg.lit_mid[1]);
        w.add(CK_SRC_INPUT, id_off, id_len);
        w.add(CK_SRC_LIT, cfg.lit_close[0], cfg.lit_close[1]);
    }
    if (fov_set) { w.add(CK_SRC_INPUT, cur, sov_off - cur); w.add(CK_SRC_INPUT, fov_off, fov_len); cur = sov_off + sov_len; }
    u32 cut0 = nframes > 1 ? top_off - 1 : top_off;
    w.add(CK_SRC_INPUT, cur, cut0 - cur);
    w.add(CK_SRC_INPUT, top_off + top_len, r.n - (top_off + top_len));
    w.finish(i);
    out.pay_len = w.total; out.desc_len = 16 + 8 * w.n;
    out.action = CK_ACT_RETURN;
    // publishes: callback (keyed by correlation id), then the handler return value to publish_topic; routed here
    ck_pub p = none; p.payload = i; p.topic_off = cb_off; p.topic_len = cb_len; p.has_key = 1;
    p.topic_id = ck_topic_lookup(r, cb_off, cb_len, tab, &p.pad);
    if (num_partitions) p.partition = (int)((ck_murmur2_key(r, corr_off, corr_len) & 0x7fffffffu) % num_partitions);
    pb[0] = p;
    out.nout = 1;
    if (cfg.publish_topic_id >= 0) { ck_pub q = none; q.payload = i; q.topic_id = cfg.publish_topic_id; pb[1] = q; out.nout = 2; }
#undef COL
}

__global__ void __launch_bounds__(CK_P2_THREADS, CK_P2_MINB)
ck_plan_tool_kernel(ck_view v, u32 n, u32* __restrict__ cols, u32 stride,
                    const ck_tool_cfg* __restrict__ cfgp, const u8* __restrict__ lit, const long long* __restrict__ aux_off,
                    int mode, ck_out_desc* __restrict__ descs, u32* __restrict__ pay_len, ck_pub* __restrict__ pubs,
                    ck_topic_table tab, u32 num_partitions, u32* __restrict__ topic_hist, u32 hist_cap) {
    u32 lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    ck_p2_stage* st = (ck_p2_stage*)((u8*)ck_win_smem + CK_P2_THREADS * CK_P2_WSTRIDE) + warp;
    u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    u32 i0 = i - lane;                                   // first record of this warp
    ck_p2_res res; res.action = CK_ACT_NONE; res.nout = 0; res.status = CK_OK; res.pay_len = 0; res.desc_len = 0;
    bool live = i < n;
    ck_pub pb[2];
    pb[0].payload = pb[1].payload = 0xffffffffu; pb[0].topic_id = pb[1].topic_id = -1;
    if (live) {
        ck_plan_tool_one(v, i, cols, stride, *cfgp, lit, aux_off, mode, &st->desc[lane], pb, tab, num_partitions, res);
        pay_len[i] = res.pay_len;
        cols[(size_t)CK_COL_ACTION * stride + i] = res.action;
        cols[(size_t)CK_COL_NOUT * stride + i] = res.nout;
        if (res.status != CK_OK) cols[(size_t)CK_COL_STATUS * stride + i] = res.status;
        // the two publishes: 64 contiguous bytes per record, four 16-byte stores (adjacent lanes fill adjacent sectors)
        uint4* gp = (uint4*)(pubs + 2 * (size_t)i);
        const uint4* sp = (const uint4*)pb;
        gp[0] = sp[0]; gp[1] = sp[1]; gp[2] = sp[2]; gp[3] = sp[3];
    }
    __syncwarp();
    // ---- coalesced write-out of the descriptors: two records per store instruction, 16 bytes per lane
    u32 half = lane >> 4, hl = lane & 15;
#pragma unroll 1
    for (u32 it = 0; it < 16; it++) {
        u32 rr = 2 * it + half;
        u32 dl = __shfl_sync(0xffffffffu, res.desc_len, rr);
        if (hl * 16 < dl) *(uint4*)((u8*)(descs + i0 + rr) + hl * 16) = *(const uint4*)((const u8*)&st->desc[rr] + hl * 16);
    }
    // ---- per-topic histogram, aggregated inside the warp (one atomic per distinct topic)
#pragma unroll
    for (u32 k = 0; k < 2; k++) {
        bool cnt = live && pb[k].payload != 0xffffffffu && pb[k].topic_id >= 0 && (u32)pb[k].topic_id < hist_cap;
        u32 active = __ballot_sync(0xffffffffu, cnt);
        if (cnt) {
            u32 peers = __match_any_sync(active, pb[k].topic_id);
            if (lane == (u32)(__ffs(peers) - 1)) atomicAdd(topic_hist + pb[k].topic_id, __popc(peers));
        }
    }
}

#endif  // CK_PLAN_CUH
