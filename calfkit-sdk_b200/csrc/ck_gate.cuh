// Aggregation gate on the device (SURVEY.md section 8 rows a10 / f4).
//
// Reference: Agent._parallel_state_aggregation (calfkit/nodes/agent.py:57-68) with PendingToolBatch
// (calfkit/models/state.py:127-141): when an agent fans N tool calls out it remembers, per correlation id, the state it
// fanned out from (`base_state`) and the N expected tool_call_ids; every tool return that comes back carries that state
// plus its own entry in `tool_results`; the gate copies, for each expected id it has not collected yet, that entry out
// of the arriving state; N-1 of the N arrivals end in Silent, the one that completes the set continues with
// `base_state` + the collected results (dict insertion order = order of collection) and the entry is deleted.
//
// Here the pending table lives in HBM: an open-addressing hash table over the 64-bit FNV-1a of the correlation id, one
// 64-bit word per key slot that holds the hash's high 32 bits and the entry index together (bytes verified on a hit), one
// entry per pending fan-out (base-state blob + expected-id slots) and a bump-allocated byte arena for the blobs.
// Entries, slots and arena bytes are only ever appended; ck_gate_compact moves the live ones to a second set of buffers
// and rebuilds the key table, which gives back everything finished fan-outs used.  A whole batch of arrivals is processed at once and still reproduces the reference's
// one-at-a-time semantics exactly, through arrival stamps (stamp = records consumed before this batch + index in it):
//   probe    every arrival finds its entry and does atomicMin(slot.stamp, own stamp) on the slots of the expected ids
//            it carries: after the kernel each slot holds the stamp of the FIRST arrival that carried it — the one the
//            reference would have collected from;
//   resolve  a slot's winner copies its value into the arena; with every slot filled, T = max slot stamp is the arrival
//            that completed the set: stamp < T -> Silent, stamp == T -> completes (continues with the merge),
//            stamp > T -> the entry was already gone when the reference would have seen it (passes through); while
//            some slot is still empty every arrival is Silent;
//   merge    (warp per completing record) the collected `"id":value` pairs are laid out in stamp order — the order the
//            reference collected them in — and the merged envelope is described as a splice:
//            inbound[..."state":] + base_state up to the end of tool_results + pairs + rest of base_state + inbound[after state...].
// The N-1 Silent arrivals never leave the device.
#ifndef CK_GATE_CUH
#define CK_GATE_CUH

#define CK_GATE_INF 0xffffffffffffffffull
#define CK_STATE_OFF 20u            // {"context":{"state":  — the state object starts here in every canonical envelope

struct ck_gate_slot {               // one expected tool_call_id of a pending fan-out
    u32 id_hash, id_off, id_len;    // the id: span inside the entry's base-state blob (string content)
    u32 val_len;                    // collected value (its JSON text in the arena), 0 = not collected yet
    unsigned long long val_off;
    unsigned long long stamp;       // stamp of the first arrival that carried this id
};
struct ck_gate_entry {
    unsigned long long base_off;    // base-state blob in the arena
    unsigned long long corr_off;    // correlation id bytes in the arena
    unsigned long long reg;         // registration order (records registered before its batch + index in it): the later wins
    u32 base_len, corr_len;
    u32 tr_close;                   // offset inside the blob of the closing '}' of tool_results
    u32 tr_empty;                   // tool_results was {} at fan-out
    u32 n_expected, first_slot;
    u32 live, pad;
};
struct ck_gate {
    unsigned long long* keys;       // [cap] (hash >> 32) << 32 | (entry index + 1), 0 = empty
    u32 cap;                        // power of two
    ck_gate_entry* entries; u32 max_entries;
    ck_gate_slot* slots; u32 max_slots;
    u8* arena; unsigned long long arena_cap;
    // counters: [0] entries used, [1] slots used, [2] arena bytes used, [3] live entries,
    // [4] capacity failures of the last register / arrive call
    unsigned long long* ctr;
};

#define CK_GATE_TAG(h) ((h) >> 32)
__device__ __forceinline__ unsigned long long ck_fnv64(Rd& r, u32 off, u32 len) {
    unsigned long long h = 14695981039346656037ull;
    for (u32 i = 0; i < len; i++) h = (h ^ r.at(off + i)) * 1099511628211ull;
    return h < 2 ? h + 2 : h;
}
__device__ __forceinline__ bool ck_bytes_eq(Rd& r, u32 off, const u8* __restrict__ q, u32 len) {
    for (u32 i = 0; i < len; i++) if (r.at(off + i) != q[i]) return false;
    return true;
}
// the entry a key word names holds this correlation id; L2 reads: in the register kernel another SM may have published
// the entry a moment ago
__device__ __forceinline__ bool ck_gate_same_corr(const ck_gate& g, u32 e, Rd& r, u32 coff, u32 clen) {
    const ck_gate_entry* en = g.entries + e;
    if (__ldcg(&en->corr_len) != clen) return false;
    const u8* q = g.arena + __ldcg(&en->corr_off);
    for (u32 i = 0; i < clen; i++) if (r.at(coff + i) != __ldcg(q + i)) return false;
    return true;
}
__device__ __forceinline__ int ck_gate_find(const ck_gate& g, Rd& r, u32 coff, u32 clen, unsigned long long h) {
    u32 s = (u32)h & (g.cap - 1);
    for (u32 p = 0; p < g.cap; p++) {
        unsigned long long k = g.keys[s];
        if (k == 0) return -1;
        if (CK_GATE_TAG(k) == CK_GATE_TAG(h)) {
            u32 e = (u32)k - 1;
            const ck_gate_entry& en = g.entries[e];
            if (en.corr_len == clen && ck_bytes_eq(r, coff, g.arena + en.corr_off, clen)) return en.live ? (int)e : -1;   // one key per id
        }
        s = (s + 1) & (g.cap - 1);
    }
    return -1;
}
__device__ __forceinline__ unsigned long long ck_pad16(unsigned long long x) { return (x + 15u) & ~15ull; }

// ---- registration: after the fan-out plan of a batch of post-LLM envelopes, every record that went out as list[Call]
// (ACTION == FANOUT) becomes a pending entry: base_state = its `state` object, expected ids = its pending tool calls.
// (a) thread per record: allocate entry, slots and arena space, insert into the table, fill the slots
__global__ void __launch_bounds__(128)
ck_gate_register_kernel(ck_view v, u32 n, const u32* __restrict__ cols, u32 stride, ck_gate g, u32 min_pending,
                        unsigned long long reg_base, u32* __restrict__ rec_entry) {
    u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
#define COL(k) cols[(size_t)(k) * stride + i]
    rec_entry[i] = 0xffffffffu;
    // the reference registers a PendingToolBatch only for list[Call] (more than one pending call, agent.py:178,194-209);
    // min_pending = 1 also takes single Calls (tests of the gate itself: the golden cases include a one-id batch)
    u32 act = COL(CK_COL_ACTION);
    if (COL(CK_COL_STATUS) != CK_OK || !(act == CK_ACT_FANOUT || (min_pending <= 1 && act == CK_ACT_CALL))) return;
    u32 rlen; const u8* rec = ck_rec(v, i, rlen);
    Rd r; r.init(rec, rlen);
    u32 tc = COL(CK_COL_TC_OFF), tr = COL(CK_COL_TR_OFF), trl = COL(CK_COL_TR_LEN);
    u32 state_end = COL(CK_COL_SOV_OFF) + COL(CK_COL_SOV_LEN) + 1;            // one past the '}' that closes the state object
    u32 base_len = state_end - CK_STATE_OFF;
    u32 coff = COL(CK_COL_CORR_OFF), clen = COL(CK_COL_CORR_LEN);
    // pending ids = keys of tool_calls that have no entry in tool_results
    u32 pending = 0;
    { u32 pos = tc + 1; while (pos < r.n && r.at(pos) != '}') { Span k; ck_string(r, pos, k); pos++; ck_skip_value(r, pos);
        if (ck_dict_find(r, tr, k.off, k.len).len == 0) pending++; if (pos < r.n && r.at(pos) == ',') pos++; } }
    if (pending < min_pending || pending == 0) return;
    u32 e = (u32)atomicAdd(&g.ctr[0], 1ull);
    u32 s0 = (u32)atomicAdd(&g.ctr[1], (unsigned long long)pending);
    unsigned long long need = ck_pad16(base_len) + ck_pad16(clen);
    unsigned long long a0 = atomicAdd(&g.ctr[2], need);
    if (e >= g.max_entries || (unsigned long long)s0 + pending > g.max_slots || a0 + need > g.arena_cap) {
        if (e < g.max_entries) g.entries[e].live = 0;       // allocated but never filled: compaction must not read it as live
        atomicAdd(&g.ctr[4], 1ull);
        return;
    }
    ck_gate_entry en;
    en.base_off = a0; en.base_len = base_len; en.corr_off = a0 + ck_pad16(base_len); en.corr_len = clen; en.reg = reg_base + i;
    en.tr_close = tr + trl - 1 - CK_STATE_OFF; en.tr_empty = (trl == 2); en.n_expected = pending; en.first_slot = s0; en.live = 1; en.pad = 0;
    for (u32 b = 0; b < clen; b++) g.arena[en.corr_off + b] = r.at(coff + b);
    u32 pos = tc + 1, j = 0;
    while (pos < r.n && r.at(pos) != '}') {
        Span k; ck_string(r, pos, k); pos++; ck_skip_value(r, pos);
        if (ck_dict_find(r, tr, k.off, k.len).len == 0) {
            ck_gate_slot sl; sl.id_hash = ck_hash_span(r, k.off, k.len); sl.id_off = k.off - CK_STATE_OFF; sl.id_len = k.len;
            sl.val_len = 0; sl.val_off = 0; sl.stamp = CK_GATE_INF;
            g.slots[s0 + j++] = sl;
        }
        if (pos < r.n && r.at(pos) == ',') pos++;
    }
    g.entries[e] = en;
    __threadfence();
    // insert: claim an empty key slot, or take over the key slot of the same correlation id from an earlier registration
    // (dict assignment in the reference: a new PendingToolBatch replaces the old one; within a batch the highest record
    // index is the later one).  A key word names its entry in the same 64-bit store, so whoever reads the word finds the
    // entry already written.  An id keeps its key slot for good, and the key table is only rebuilt by ck_gate_compact.
    unsigned long long h = ck_fnv64(r, coff, clen);
    unsigned long long mine = (CK_GATE_TAG(h) << 32) | (e + 1ull);
    u32 s = (u32)h & (g.cap - 1);
    int won = -1;                                            // -1 still probing, 0 a later registration holds the id, 1 inserted
    for (u32 p = 0; p < g.cap && won < 0; p++, s = (s + 1) & (g.cap - 1)) {
        unsigned long long cur = atomicCAS(&g.keys[s], 0ull, mine);
        if (cur == 0) { won = 1; break; }
        // the word of a key slot only ever changes to the word of an entry with the same correlation id
        if (CK_GATE_TAG(cur) != CK_GATE_TAG(h) || !ck_gate_same_corr(g, (u32)cur - 1, r, coff, clen)) continue;
        while (won < 0) {
            u32 old = (u32)cur - 1;
            if (__ldcg(&g.entries[old].reg) > en.reg) { won = 0; break; }
            unsigned long long prev = atomicCAS(&g.keys[s], cur, mine);
            if (prev == cur) {
                won = 1;
                if (atomicExch(&g.entries[old].live, 0u)) atomicAdd(&g.ctr[3], (unsigned long long)-1ll);
            } else {
                cur = prev;
            }
        }
    }
    if (won != 1) {                                          // replaced by a later record of this batch (or no key slot left)
        g.entries[e].live = 0;
        if (won < 0) atomicAdd(&g.ctr[4], 1ull);
        return;
    }
    atomicAdd(&g.ctr[3], 1ull);
    rec_entry[i] = e;
#undef COL
}
// (b) warp per record: copy the base-state blob into the arena
__global__ void __launch_bounds__(256)
ck_gate_copy_base_kernel(ck_view v, u32 n, ck_gate g, const u32* __restrict__ rec_entry) {
    u32 w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (w >= n) return;
    u32 e = rec_entry[w];
    if (e == 0xffffffffu) return;
    u32 rlen; const u8* rec = ck_rec(v, w, rlen);
    const ck_gate_entry& en = g.entries[e];
    ck_warp_copy(g.arena + en.base_off, rec + CK_STATE_OFF, en.base_len, lane);
}

// ---- arrivals ----------------------------------------------------------------------------------------------------
template <class F>
__device__ __forceinline__ void ck_gate_each_match(const ck_gate& g, const ck_gate_entry& en, Rd& r, u32 tr_off, F f) {
    // every key of the arriving record's tool_results that is one of the entry's expected ids
    u32 pos = tr_off + 1;
    while (pos < r.n && r.at(pos) != '}') {
        Span k; ck_string(r, pos, k); pos++;
        u32 v0 = pos; ck_skip_value(r, pos);
        u32 hk = ck_hash_span(r, k.off, k.len);
        for (u32 q = 0; q < en.n_expected; q++) {
            ck_gate_slot& sl = g.slots[en.first_slot + q];
            if (sl.id_hash == hk && sl.id_len == k.len && ck_bytes_eq(r, k.off, g.arena + en.base_off + sl.id_off, k.len)) { f(sl, v0, pos - v0); break; }
        }
        if (pos < r.n && r.at(pos) == ',') pos++;
    }
}

__global__ void __launch_bounds__(128)
ck_gate_probe_kernel(ck_view v, u32 n, const u32* __restrict__ cols, u32 stride, ck_gate g, unsigned long long stamp_base, u32* __restrict__ rec_entry) {
    u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    rec_entry[i] = 0xffffffffu;
    if (cols[(size_t)CK_COL_STATUS * stride + i] != CK_OK) return;
    u32 rlen; const u8* rec = ck_rec(v, i, rlen);
    Rd r; r.init(rec, rlen);
    u32 coff = cols[(size_t)CK_COL_CORR_OFF * stride + i], clen = cols[(size_t)CK_COL_CORR_LEN * stride + i];
    int e = ck_gate_find(g, r, coff, clen, ck_fnv64(r, coff, clen));
    if (e < 0) return;
    rec_entry[i] = (u32)e;
    unsigned long long my = stamp_base + i;
    ck_gate_each_match(g, g.entries[e], r, cols[(size_t)CK_COL_TR_OFF * stride + i], [&](ck_gate_slot& sl, u32, u32) { atomicMin(&sl.stamp, my); });
}

__global__ void __launch_bounds__(128)
ck_gate_resolve_kernel(ck_view v, u32 n, u32* __restrict__ cols, u32 stride, ck_gate g, unsigned long long stamp_base,
                       const u32* __restrict__ rec_entry, int32_t publish_topic_id, u8* __restrict__ glue,
                       ck_out_desc* __restrict__ descs, u32* __restrict__ pay_len, ck_pub* __restrict__ pubs) {
    u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
#define COL(k) cols[(size_t)(k) * stride + i]
    ck_pub none; none.payload = 0xffffffffu; none.topic_id = -1; none.topic_off = none.topic_len = 0; none.record = i;
    none.has_key = 0; none.partition = -1; none.pad = 0;
    pubs[2 * i] = none; pubs[2 * i + 1] = none;
    pay_len[i] = 0;
    ck_out_desc* d = descs + i;
    d->nseg = 0; d->record = i; d->total_len = 0; d->pad = 0;
    COL(CK_COL_NOUT) = 0;
    if (COL(CK_COL_STATUS) != CK_OK) { COL(CK_COL_ACTION) = CK_ACT_NONE; return; }
    u32 e = rec_entry[i];
    if (e == 0xffffffffu) { COL(CK_COL_ACTION) = CK_ACT_GATE_PASS; return; }
    u32 rlen; const u8* rec = ck_rec(v, i, rlen);
    Rd r; r.init(rec, rlen);
    const ck_gate_entry& en = g.entries[e];
    unsigned long long my = stamp_base + i;
    // the first arrival that carried an id is the one the reference collects from: it copies the value into the arena
    ck_gate_each_match(g, en, r, COL(CK_COL_TR_OFF), [&](ck_gate_slot& sl, u32 v0, u32 vl) {
        if (sl.stamp != my) return;
        unsigned long long need = ck_pad16(vl);
        unsigned long long a0 = atomicAdd(&g.ctr[2], need);
        if (a0 + need > g.arena_cap) { atomicAdd(&g.ctr[4], 1ull); return; }     // val_len stays 0: the merge declines
        for (u32 b = 0; b < vl; b++) g.arena[a0 + b] = r.at(v0 + b);
        sl.val_off = a0; sl.val_len = vl;
    });
    bool filled = true; unsigned long long T = 0;
    for (u32 q = 0; q < en.n_expected; q++) { unsigned long long s = g.slots[en.first_slot + q].stamp; if (s == CK_GATE_INF) filled = false; else if (s > T) T = s; }
    u32 action;
    if (!filled || my < T) action = CK_ACT_SILENT;
    else if (my == T) action = CK_ACT_GATE_COMPLETE;
    else action = CK_ACT_GATE_PASS;
    COL(CK_COL_ACTION) = action;
    if (action == CK_ACT_SILENT && publish_topic_id >= 0) {
        // Silent: the handler returns the inbound envelope and the worker publishes that to publish_topic
        // (nodes/base.py:137-145, worker/worker.py:52-53)
        SegWriter w; w.init(d, &r, nullptr, nullptr, glue + (size_t)i * CK_GLUE_STRIDE);
        w.add(CK_SRC_INPUT, 0, r.n); w.finish(i);
        pay_len[i] = r.n;
        ck_pub p = none; p.payload = i; p.topic_id = publish_topic_id; pubs[2 * i + 1] = p;
        COL(CK_COL_NOUT) = 1;
    }
#undef COL
}

// warp per completing record: lay the collected "id":value pairs out in stamp order, describe the merged envelope
__global__ void __launch_bounds__(128)
ck_gate_merge_kernel(ck_view v, u32 n, u32* __restrict__ cols, u32 stride, ck_gate g, const u32* __restrict__ rec_entry, u8* __restrict__ glue,
                     ck_out_desc* __restrict__ descs, u32* __restrict__ pay_len) {
    u32 w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (w >= n) return;
    if (cols[(size_t)CK_COL_ACTION * stride + w] != CK_ACT_GATE_COMPLETE || cols[(size_t)CK_COL_STATUS * stride + w] != CK_OK) return;
    u32 e = rec_entry[w];
    ck_gate_entry& en = g.entries[e];
    u32 nexp = en.n_expected;
    const ck_gate_slot* sl = g.slots + en.first_slot;
    // piece q = ["," if not first] "id":value ; its rank = number of slots with a smaller stamp; offsets by rank
    // pass 1: every lane handles slots lane, lane+32, ...: rank + length
    u32 total = 0;
    bool lead_comma = !en.tr_empty, missing = false;
    for (u32 base = 0; base < nexp; base += 32) {
        u32 q = base + lane;
        u32 len = 0;
        if (q < nexp) len = 1 + sl[q].id_len + 2 + sl[q].val_len;          // "id": value
        missing |= __any_sync(0xffffffffu, q < nexp && sl[q].val_len == 0);  // a JSON value is never empty: its copy found no room
        // sum of lengths is order independent
        for (int o = 16; o; o >>= 1) len += __shfl_xor_sync(0xffffffffu, len, o);
        total += len;
    }
    total += nexp - 1 + (lead_comma ? 1u : 0u);                            // commas
    unsigned long long blob = CK_GATE_INF;
    if (lane == 0 && !missing) {
        unsigned long long need = ck_pad16(total);
        blob = atomicAdd(&g.ctr[2], need);
        if (blob + need > g.arena_cap) blob = CK_GATE_INF;
    }
    blob = __shfl_sync(0xffffffffu, blob, 0);
    if (blob == CK_GATE_INF) {
        // the arena could not hold a collected value or the merged pieces: the record is declined and the fan-out is
        // given up, so no envelope with a hole in it ever leaves the device
        if (lane == 0) {
            if (!missing) atomicAdd(&g.ctr[4], 1ull);                       // a missing value was counted by its copy
            cols[(size_t)CK_COL_STATUS * stride + w] = CK_UNSUPPORTED; cols[(size_t)CK_COL_ACTION * stride + w] = CK_ACT_RAISES;
            en.live = 0;
            atomicAdd(&g.ctr[3], (unsigned long long)-1ll);
        }
        return;
    }
    // pass 2: for every slot, its start = sum of the lengths of all pieces with a smaller stamp (+ commas)
    for (u32 q = 0; q < nexp; q++) {
        unsigned long long sq = sl[q].stamp;
        u32 before = 0, cnt = 0;
        // order of collection = (stamp, position among the expected ids): an arrival that carries several expected results is
        // collected in tool_calls order (the reference iterates a frozenset there: its own order is unspecified)
        for (u32 p = lane; p < nexp; p += 32) if (sl[p].stamp < sq || (sl[p].stamp == sq && p < q)) { before += 1 + sl[p].id_len + 2 + sl[p].val_len; cnt++; }
        for (int o = 16; o; o >>= 1) { before += __shfl_xor_sync(0xffffffffu, before, o); cnt += __shfl_xor_sync(0xffffffffu, cnt, o); }
        u32 start = before + cnt + (lead_comma ? 1u : 0u);                  // one comma before every piece but the very first
        u8* dst = g.arena + blob + start;
        if (lane == 0) {
            if (cnt || lead_comma) dst[-1] = ',';
            dst[0] = '"'; dst[1 + sl[q].id_len] = '"'; dst[2 + sl[q].id_len] = ':';
        }
        const u8* idp = g.arena + en.base_off + sl[q].id_off;
        for (u32 b = lane; b < sl[q].id_len; b += 32) dst[1 + b] = idp[b];
        ck_warp_copy(dst + 3 + sl[q].id_len, g.arena + sl[q].val_off, sl[q].val_len, lane);
    }
    __syncwarp();
    __threadfence();
    if (lane == 0) {
        u32 rlen; const u8* rec = ck_rec(v, w, rlen);
        Rd r; r.init(rec, rlen);
        u32 state_end = cols[(size_t)CK_COL_SOV_OFF * stride + w] + cols[(size_t)CK_COL_SOV_LEN * stride + w] + 1;
        ck_out_desc* d = descs + w;
        SegWriter sw; sw.init(d, &r, nullptr, g.arena, glue + (size_t)w * CK_GLUE_STRIDE);
        sw.add(CK_SRC_INPUT, 0, CK_STATE_OFF);
        sw.add(CK_SRC_AUX, (u32)en.base_off, en.tr_close);
        sw.add(CK_SRC_AUX, (u32)blob, total);
        sw.add(CK_SRC_AUX, (u32)en.base_off + en.tr_close, en.base_len - en.tr_close);
        sw.add(CK_SRC_INPUT, state_end, r.n - state_end);
        if (!sw.finish(w)) { cols[(size_t)CK_COL_STATUS * stride + w] = CK_UNSUPPORTED; cols[(size_t)CK_COL_ACTION * stride + w] = CK_ACT_RAISES; d->nseg = 0; d->total_len = 0; }
        else pay_len[w] = sw.total;
        en.live = 0;                                                          // del self._pending_batches[correlation_id]
        atomicAdd(&g.ctr[3], (unsigned long long)-1ll);
    }
}

// ---- compaction: the live entries, their slots, base blobs, correlation bytes and collected values move to the other
// set of buffers `d` (same capacities, same counters and key table), in index order; stamps and values are unchanged.
// The host clears the key table first and swaps the buffers afterwards.
__device__ __forceinline__ unsigned long long ck_gate_live_bytes(const ck_gate& g, const ck_gate_entry& en) {
    unsigned long long b = ck_pad16(en.base_len) + ck_pad16(en.corr_len);
    for (u32 q = 0; q < en.n_expected; q++) { u32 vl = g.slots[en.first_slot + q].val_len; if (vl) b += ck_pad16(vl); }
    return b;
}
// (a) one block: new entry index, first slot and arena offset of every live entry (block scan); src[new] = old index
__global__ void __launch_bounds__(1024)
ck_gate_compact_plan_kernel(ck_gate g, ck_gate d, u32* __restrict__ src) {
    __shared__ u32 s_e[32], s_s[32];
    __shared__ unsigned long long s_a[32];
    u32 t = threadIdx.x, lane = t & 31, wid = t >> 5;
    unsigned long long used = g.ctr[0];
    u32 ne = used < g.max_entries ? (u32)used : g.max_entries;
    u32 per = (ne + blockDim.x - 1) / blockDim.x, lo = min(t * per, ne), hi = min(lo + per, ne);
    u32 ce = 0, cs = 0; unsigned long long ca = 0;
    for (u32 e = lo; e < hi; e++) {
        const ck_gate_entry& en = g.entries[e];
        if (!en.live) continue;
        ce++; cs += en.n_expected; ca += ck_gate_live_bytes(g, en);
    }
    u32 ie = ce, is = cs; unsigned long long ia = ca;                      // inclusive scan in the warp
    for (int o = 1; o < 32; o <<= 1) {
        u32 x = __shfl_up_sync(0xffffffffu, ie, o), y = __shfl_up_sync(0xffffffffu, is, o);
        unsigned long long z = __shfl_up_sync(0xffffffffu, ia, o);
        if (lane >= (u32)o) { ie += x; is += y; ia += z; }
    }
    if (lane == 31) { s_e[wid] = ie; s_s[wid] = is; s_a[wid] = ia; }
    __syncthreads();                                                       // every thread has read ctr[0] by now
    if (wid == 0) {
        u32 nw = blockDim.x >> 5;
        u32 x = lane < nw ? s_e[lane] : 0, y = lane < nw ? s_s[lane] : 0; unsigned long long z = lane < nw ? s_a[lane] : 0;
        for (int o = 1; o < 32; o <<= 1) {
            u32 x2 = __shfl_up_sync(0xffffffffu, x, o), y2 = __shfl_up_sync(0xffffffffu, y, o);
            unsigned long long z2 = __shfl_up_sync(0xffffffffu, z, o);
            if (lane >= (u32)o) { x += x2; y += y2; z += z2; }
        }
        if (lane < nw) { s_e[lane] = x; s_s[lane] = y; s_a[lane] = z; }
    }
    __syncthreads();
    u32 oe = ie - ce + (wid ? s_e[wid - 1] : 0u), os = is - cs + (wid ? s_s[wid - 1] : 0u);
    unsigned long long oa = ia - ca + (wid ? s_a[wid - 1] : 0ull);
    for (u32 e = lo; e < hi; e++) {
        const ck_gate_entry& en = g.entries[e];
        if (!en.live) continue;
        ck_gate_entry m = en;
        m.first_slot = os; m.base_off = oa; m.corr_off = oa + ck_pad16(en.base_len);
        d.entries[oe] = m; src[oe] = e;
        oe++; os += en.n_expected; oa += ck_gate_live_bytes(g, en);
    }
    if (t == blockDim.x - 1) { g.ctr[0] = oe; g.ctr[1] = os; g.ctr[2] = oa; g.ctr[3] = oe; }
}
// (b) warp per live entry: copy blobs, slots and collected values (laid out after the correlation bytes in slot order),
// then insert its key into the cleared table
__global__ void __launch_bounds__(256)
ck_gate_compact_move_kernel(ck_gate g, ck_gate d, const u32* __restrict__ src) {
    u32 w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (w >= d.ctr[0]) return;
    const ck_gate_entry& ne = d.entries[w];
    const ck_gate_entry& oe = g.entries[src[w]];
    ck_warp_copy(d.arena + ne.base_off, g.arena + oe.base_off, ne.base_len, lane);
    ck_warp_copy(d.arena + ne.corr_off, g.arena + oe.corr_off, ne.corr_len, lane);
    unsigned long long vo = ne.corr_off + ck_pad16(ne.corr_len);
    for (u32 q = 0; q < ne.n_expected; q++) {
        ck_gate_slot sl = g.slots[oe.first_slot + q];
        if (sl.val_len) { ck_warp_copy(d.arena + vo, g.arena + sl.val_off, sl.val_len, lane); sl.val_off = vo; vo += ck_pad16(sl.val_len); }
        if (lane == 0) d.slots[ne.first_slot + q] = sl;
    }
    if (lane == 0) {
        Rd r; r.init(g.arena + oe.corr_off, oe.corr_len);
        unsigned long long h = ck_fnv64(r, 0, oe.corr_len);
        unsigned long long word = (CK_GATE_TAG(h) << 32) | (w + 1ull);
        u32 s = (u32)h & (d.cap - 1);
        for (u32 p = 0; p < d.cap; p++, s = (s + 1) & (d.cap - 1))
            if (atomicCAS(&d.keys[s], 0ull, word) == 0ull) break;
    }
}

#endif  // CK_GATE_CUH
