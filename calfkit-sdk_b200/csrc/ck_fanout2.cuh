// Agent fan-out, one WARP per record (replaces the thread-per-record ck_fanout_count / ck_fanout_plan kernels).
//
// Reference: Agent.run's list[Call] branch (calfkit/nodes/agent.py:177-211) + _publish_action (nodes/base.py:73-88).
// Round 1 ran one thread per record: with 64 pending calls per 20 KB record that thread walked tool_calls once per pass,
// looked every key up in tool_results by walking that dict again (O(F^2) bytes) and searched the tool registry linearly
// per call — most of the config-3 step, on only 128 warps.  Here a warp owns a record: lane 0
// indexes the two dicts once into shared memory (key span, value span, 32-bit key hash), then the lanes take one tool
// call each: pending test against the hashed tool_results keys, registry lookup by name hash, and the splice descriptor
// of their own Call envelope (same SegWriter, same bytes as before).
// The index itself is built by the whole warp too: the structural pre-scan of ck_walk_long.cuh proposes the entry
// boundaries of both dicts, every lane parses its own entry and checks that it ends exactly where the next one starts and
// that the dict closes where the walker's column says; only if that chain does not hold does lane 0 index sequentially
// (milliseconds for a 20 KB record).
#ifndef CK_FANOUT2_CUH
#define CK_FANOUT2_CUH

#define CK_F2_WARPS 4
#define CK_F2_MAX 256u              // tool calls / results indexed per record (more: CK_UNSUPPORTED, as before beyond max_fanout)
#define CK_F2_SMEM (CK_F2_WARPS * (sizeof(ck_long_index) + sizeof(ck_f2_index)))

struct ck_f2_index {                // per warp, shared memory
    u32 k_off[CK_F2_MAX], k_len[CK_F2_MAX], v_off[CK_F2_MAX], k_hash[CK_F2_MAX];     // tool_calls entries (v_off = the ToolCallPart)
    u32 r_off[CK_F2_MAX], r_len[CK_F2_MAX], r_hash[CK_F2_MAX];                       // tool_results keys
    u32 n_calls, n_results, overflow;
};

// lane 0: one pass over each dict
__device__ __forceinline__ void ck_f2_build(ck_f2_index* ix, Rd& r, u32 tc, u32 tr) {
    u32 n = 0, m = 0, ovf = 0;
    u32 pos = tc + 1;
    while (pos < r.n && r.at(pos) != '}') {
        Span k; ck_string(r, pos, k); pos++;
        u32 v = pos; ck_skip_value(r, pos);
        if (n < CK_F2_MAX) { ix->k_off[n] = k.off; ix->k_len[n] = k.len; ix->v_off[n] = v; ix->k_hash[n] = ck_hash_span(r, k.off, k.len); n++; } else ovf = 1;
        if (pos < r.n && r.at(pos) == ',') pos++;
    }
    pos = tr + 1;
    while (pos < r.n && r.at(pos) != '}') {
        Span k; ck_string(r, pos, k); pos++;
        ck_skip_value(r, pos);
        if (m < CK_F2_MAX) { ix->r_off[m] = k.off; ix->r_len[m] = k.len; ix->r_hash[m] = ck_hash_span(r, k.off, k.len); m++; } else ovf = 1;
        if (pos < r.n && r.at(pos) == ',') pos++;
    }
    ix->n_calls = n; ix->n_results = m; ix->overflow = ovf;
}
__device__ __forceinline__ bool ck_f2_pending(const ck_f2_index* ix, Rd& r, u32 j) {
    u32 h = ix->k_hash[j], len = ix->k_len[j], off = ix->k_off[j];
    for (u32 q = 0; q < ix->n_results; q++)
        if (ix->r_hash[q] == h && ix->r_len[q] == len && ck_span_eq(r, ix->r_off[q], off, len)) return false;
    return true;
}

// warp-parallel index of one dict (entries at nesting depth 4) from the pre-scan's proposals; false = chain broken
__device__ __forceinline__ bool ck_f2_index_dict(const ck_long_index* lx, Rd& r, u32 dict_off, u32 dict_len, u32* k_off, u32* k_len, u32* v_off, u32* k_hash, u32& n_out) {
    u32 lane = threadIdx.x & 31;
    u32 pos = dict_off + 1;
    if (dict_len == 2) { n_out = 0; return true; }
    u32 q, s0, k;
    if (!ck_lx_range(lx, 0, pos, q, s0, k) || q != dict_off + dict_len - 1 || k + 1 > CK_F2_MAX) return false;
    bool good = true;
    for (u32 base = 0; base <= k; base += 32) {
        u32 e = base + lane;
        bool ok = true;
        if (e <= k) {
            u32 p = e ? lx->sep[0][s0 + e - 1] + 1 : pos, tend = e == k ? q : lx->sep[0][s0 + e];
            Span key;
            ok = r.at(p) == '"' && ck_string(r, p, key) && r.at(p) == ':';
            u32 v = p + 1, p2 = v;
            if (ok) { ck_skip_value(r, p2); ok = (p2 == tend); }
            if (ok) { k_off[e] = key.off; k_len[e] = key.len; if (v_off) v_off[e] = v; k_hash[e] = ck_hash_span(r, key.off, key.len); }
        }
        good = __all_sync(0xffffffffu, ok) && good;
    }
    n_out = k + 1;
    return good;
}
// all lanes call it; the record is a validated canonical envelope (STATUS == CK_OK)
__device__ __forceinline__ void ck_f2_build_warp(ck_f2_index* ix, ck_long_index* lx, const u8* rec, u32 rlen, Rd& r, u32 tc, u32 tcl, u32 tr, u32 trl) {
    u32 lane = threadIdx.x & 31;
    u32 n = 0, m = 0;
    bool ok = true;
    if (tcl > 2) { ck_lx_build(rec, rlen, lx, tc, tc + tcl, 3); ok = ck_f2_index_dict(lx, r, tc, tcl, ix->k_off, ix->k_len, ix->v_off, ix->k_hash, n); }
    if (ok && trl > 2) { __syncwarp(); ck_lx_build(rec, rlen, lx, tr, tr + trl, 3); ok = ck_f2_index_dict(lx, r, tr, trl, ix->r_off, ix->r_len, nullptr, ix->r_hash, m); }
    if (ok) { if (lane == 0) { ix->n_calls = n; ix->n_results = m; ix->overflow = 0; } }
    else if (lane == 0) ck_f2_build(ix, r, tc, tr);
    __syncwarp();
}

// pass 1: payload slots per record (pending + 1 for the handler return of a list[Call])
__global__ void __launch_bounds__(32 * CK_F2_WARPS)
ck_fanout2_count_kernel(ck_view v, u32 n, u32* __restrict__ cols, u32 stride, const ck_agent_cfg* __restrict__ cfgp, u32 max_fanout, u32 sequential,
                        u32* __restrict__ counts) {
    u32 lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    u32 i = blockIdx.x * CK_F2_WARPS + w;
    if (i >= n) return;
    ck_long_index* lx = (ck_long_index*)ck_win_smem + w;
    ck_f2_index* ix = (ck_f2_index*)((ck_long_index*)ck_win_smem + CK_F2_WARPS) + w;
#define COL(k) cols[(size_t)(k) * stride + i]
    u32 status = COL(CK_COL_STATUS), nframes = COL(CK_COL_NFRAMES);
    if (status != CK_OK || nframes == 0) {
        if (lane == 0) { counts[i] = 0; COL(CK_COL_NOUT) = 0; COL(CK_COL_ACTION) = status != CK_OK ? CK_ACT_NONE : CK_ACT_RAISES; }
        return;
    }
    u32 rlen; const u8* rec = ck_rec(v, i, rlen);
    Rd r; r.init(rec, rlen);
    ck_f2_build_warp(ix, lx, rec, rlen, r, COL(CK_COL_TC_OFF), COL(CK_COL_TC_LEN), COL(CK_COL_TR_OFF), COL(CK_COL_TR_LEN));
    u32 pending = 0;
    for (u32 j = lane; j < ix->n_calls; j += 32) pending += ck_f2_pending(ix, r, j) ? 1u : 0u;
    for (int o = 16; o; o >>= 1) pending += __shfl_xor_sync(0xffffffffu, pending, o);
    if (lane == 0) {
        if (sequential && pending > 1) pending = 1;       // sequential_only_mode (agent.py:94-108,179-192): first pending call only, as a single Call
        if (ix->overflow || pending == 0 || pending > max_fanout) { counts[i] = 0; COL(CK_COL_NOUT) = 0; COL(CK_COL_ACTION) = CK_ACT_RAISES; COL(CK_COL_STATUS) = CK_UNSUPPORTED; }
        else {
            u32 extra = (cfgp->publish_topic_id >= 0 && pending > 1) ? 1u : 0u;      // list[Call]: the input envelope is the handler's return value
            counts[i] = pending + extra;
            COL(CK_COL_ACTION) = pending == 1 ? CK_ACT_CALL : CK_ACT_FANOUT;
            COL(CK_COL_NOUT) = pending + ((cfgp->publish_topic_id >= 0) ? 1u : 0u);
        }
    }
#undef COL
}

// pass 2: descriptors; slot_base = exclusive scan of counts
__global__ void __launch_bounds__(32 * CK_F2_WARPS)
ck_fanout2_plan_kernel(ck_view v, u32 n, u32* __restrict__ cols, u32 stride, const ck_agent_cfg* __restrict__ cfgp, const u8* __restrict__ lit,
                       const u32* __restrict__ tool_name_hash, const long long* __restrict__ slot_base, unsigned long long unix_ms, unsigned long long seed,
                       const u8* __restrict__ aux, u8* __restrict__ glue, ck_out_desc* __restrict__ descs, u32* __restrict__ pay_len, ck_pub* __restrict__ pubs) {
    u32 lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    u32 i = blockIdx.x * CK_F2_WARPS + w;
    if (i >= n) return;
    ck_long_index* lx = (ck_long_index*)ck_win_smem + w;
    ck_f2_index* ix = (ck_f2_index*)((ck_long_index*)ck_win_smem + CK_F2_WARPS) + w;
#define COL(k) cols[(size_t)(k) * stride + i]
    u32 action = COL(CK_COL_ACTION);
    if (COL(CK_COL_STATUS) != CK_OK || (action != CK_ACT_CALL && action != CK_ACT_FANOUT)) return;
    const ck_agent_cfg& cfg = *cfgp;
    u32 rlen; const u8* rec = ck_rec(v, i, rlen);
    Rd r; r.init(rec, rlen);
    ck_f2_build_warp(ix, lx, rec, rlen, r, COL(CK_COL_TC_OFF), COL(CK_COL_TC_LEN), COL(CK_COL_TR_OFF), COL(CK_COL_TR_LEN));
    u32 slot0 = (u32)slot_base[i];
    u32 frames_off = COL(CK_COL_FRAMES_OFF), frames_len = COL(CK_COL_FRAMES_LEN), nframes = COL(CK_COL_NFRAMES);
    u32 fov_off = COL(CK_COL_FOV_OFF), fov_len = COL(CK_COL_FOV_LEN), sov_off = COL(CK_COL_SOV_OFF), sov_len = COL(CK_COL_SOV_LEN);
    bool ov = fov_len != 4;                                    // a canonical OverridesState is never 4 bytes: "null" <=> 4
    u32 list_end = frames_off + frames_len - 1;
    ck_pub none; none.payload = 0xffffffffu; none.topic_id = -1; none.topic_off = none.topic_len = 0; none.record = i;
    none.has_key = 0; none.partition = -1; none.pad = 0;
    u32 before = 0;                                            // pending calls in earlier rounds of 32
    bool bad = false;
    for (u32 base = 0; base < ix->n_calls; base += 32) {
        u32 j = base + lane;
        bool pend = j < ix->n_calls && ck_f2_pending(ix, r, j);
        u32 mask = __ballot_sync(0xffffffffu, pend);
        u32 my = before + __popc(mask & ((1u << lane) - 1u));  // rank among the pending calls, in tool_calls order
        if (action == CK_ACT_CALL) pend = pend && my == 0;     // single Call: the first pending only
        if (pend) {
            // tool_name of this ToolCallPart -> registry (name hash, then bytes)
            u32 p2 = ix->v_off[j] + 13; Span tn; ck_string(r, p2, tn);
            u32 th = ck_hash_span(r, tn.off, tn.len);
            u32 tool = 0xffffffffu;
            for (u32 t = 0; t < cfg.ntools; t++) {
                if (tool_name_hash[t] != th || cfg.tool_name_len[t] != tn.len) continue;
                bool eq = true;
                for (u32 b = 0; b < tn.len; b++) if (lit[cfg.tool_name_off[t] + b] != r.at(tn.off + b)) { eq = false; break; }
                if (eq) { tool = t; break; }
            }
            u32 s = slot0 + my;
            ck_out_desc* d = descs + s;
            SegWriter wr; wr.init(d, &r, lit, aux, glue + (size_t)s * CK_GLUE_STRIDE);
            if (tool == 0xffffffffu) { bad = true; wr.finish(i); pay_len[s] = 0; pubs[2 * s] = none; pubs[2 * s + 1] = none; }
            else {
                u32 cur = 0;
                if (ov) { wr.add(CK_SRC_INPUT, 0, sov_off); wr.add(CK_SRC_INPUT, fov_off, fov_len); cur = sov_off + sov_len; }
                wr.add(CK_SRC_INPUT, cur, list_end - cur);
                if (nframes > 0) wr.add(CK_SRC_LIT, cfg.lit_comma[0], cfg.lit_comma[1]);
                wr.add(CK_SRC_LIT, cfg.tool_lit_off[tool], cfg.tool_lit_len[tool]);
                wr.add(CK_SRC_INPUT, ix->k_off[j], ix->k_len[j]);          // tool_call_id (raw JSON string content)
                wr.add(CK_SRC_LIT, cfg.lit_mid[0], cfg.lit_mid[1]);
                wr.hex_uuid7(unix_ms, seed, (unsigned long long)s);
                wr.add(CK_SRC_LIT, cfg.lit_tail[0], cfg.lit_tail[1]);
                wr.add(CK_SRC_INPUT, list_end, r.n - list_end);
                wr.finish(i);
                pay_len[s] = wr.total;
                ck_pub p = none; p.payload = s; p.topic_id = (int32_t)cfg.tool_topic_id[tool]; p.has_key = 1;
                pubs[2 * s] = p; pubs[2 * s + 1] = none;
                if (action == CK_ACT_CALL && cfg.publish_topic_id >= 0) { ck_pub q = none; q.payload = s; q.topic_id = cfg.publish_topic_id; pubs[2 * s + 1] = q; }
            }
        }
        before += __popc(mask);
        if (action == CK_ACT_CALL && before) break;
    }
    bad = __any_sync(0xffffffffu, bad);
    if (lane == 0) {
        if (action == CK_ACT_FANOUT && cfg.publish_topic_id >= 0) {
            // handler return value of the list[Call] branch: the original envelope (nodes/base.py:88)
            u32 s = slot0 + before;
            SegWriter wr; wr.init(descs + s, &r, lit, aux, glue + (size_t)s * CK_GLUE_STRIDE);
            wr.add(CK_SRC_INPUT, 0, r.n); wr.finish(i);
            pay_len[s] = r.n;
            ck_pub q = none; q.payload = s; q.topic_id = cfg.publish_topic_id; pubs[2 * s] = q; pubs[2 * s + 1] = none;
        }
        if (bad) COL(CK_COL_STATUS) = CK_UNSUPPORTED;
    }
#undef COL
}

#endif  // CK_FANOUT2_CUH
