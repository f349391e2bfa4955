// C-ABI of libcalfkit_b200.so: handle, device buffers, stream, kernel launches.
// See include/calfkit_b200.h for the contract and the reference call sites each entry replaces.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/calfkit_b200.h"
#include "ck_buf.h"
#include "ck_kernels.cuh"
#include "ck_txn.h"

static_assert(sizeof(ck_publish) == sizeof(ck_pub), "ck_publish must mirror ck_pub");
static_assert(sizeof(ck_frame) == sizeof(ck_frame_ent), "ck_frame must mirror ck_frame_ent");

#define CK_LIT_CAP (256 * 1024)
#define CK_PAD 256   // tail padding of every byte buffer (readers may touch a few bytes past a span)

static thread_local std::string g_create_error;

// what ck_gate_create allocates: the key table and the counters, two sets of entries, slots and arena (ck_gate_compact
// moves the live fan-outs from the set the gate uses into the other), the compaction's old index of every new entry and
// each record's entry
struct ck_gate_bufs {
    ck_buf<unsigned long long> keys, ctr;
    ck_buf<ck_gate_entry> entries[2]; ck_buf<ck_gate_slot> slots[2]; ck_buf<u8> arena[2];
    ck_buf<u32> src, rec_entry;
};

struct ck_handle {
    int device = 0;
    u32 num_sms = 0;                 // grid size of the grid-stride kernels: a fixed number of blocks per SM
    cudaStream_t stream = nullptr;
    cudaStream_t xstream = nullptr; cudaEvent_t x_ev0 = nullptr, x_ev1 = nullptr;   // high-priority side stream of the exchange
    std::string err;
    uint64_t max_in = 0, max_out = 0, max_aux = 0;
    uint32_t max_records = 0, max_payloads = 0, max_pubs = 0;
    // device buffers
    ck_buf<u8> d_in; ck_buf<long long> d_in_off;
    ck_buf<u8> d_out; ck_buf<long long> d_out_off;
    ck_buf<u8> d_aux; ck_buf<long long> d_aux_off; ck_buf<u8> d_glue;
    ck_buf<u8> d_ovl; ck_buf<long long> d_ovl_off; ck_buf<u32> d_ovl_len; ck_buf<ck_canon_ctl> d_canon_ctl; ck_buf<u32> d_canon_list; ck_buf<ck_elem> d_elems; u32 elem_cap = 0; ck_buf<u32> d_cand; ck_buf<uint2> d_hist_skip;
    uint64_t max_ovl = 0;
    ck_buf<u32> d_cols; ck_buf<ck_out_desc> d_descs; ck_buf<u32> d_pay_len; ck_buf<ck_pub> d_pubs;
    ck_buf<unsigned long long> d_tile_sum, d_grand;
    ck_buf<u8> d_lit; ck_buf<ck_tool_cfg> d_tool_cfg; ck_buf<ck_agent_cfg> d_agent_cfg;
    ck_buf<u32> d_counts; ck_buf<long long> d_slot_base; ck_buf<u32> d_agent_tables;
    bool agent_set = false; ck_agent_cfg h_agent_cfg{};
    ck_buf<u32> d_topic_hist;
    // aggregation gate (ck_gate_create): the views the kernels take, over the buffers in gate_bufs
    ck_gate gate{}; bool gate_set = false;
    ck_gate gate_spare{};               // the entries, slots and arena ck_gate_compact moves the live fan-outs into
    ck_gate_bufs gate_bufs;
    unsigned long long gate_reg_seq = 0;    // records registered so far: registration order of the entries
    // peer exchange (ck_comm_create)
    ck_buf<u8> d_recv; ck_xpeers peers{}; void* peer_opened[CK_X_MAXWORLD] = {nullptr}; u32 comm_rank = 0, comm_world = 0, max_fwd = 0, x_nb = 0;
    unsigned long long region_stride = 0, region_data_cap = 0; ck_buf<u32> d_x_overflow; bool comm_ready = false;
    // publish grouping (allocated on first use)
    ck_buf<u32> d_g_hist, d_g_o1, d_g_o2, d_g_keys; ck_buf<long long> d_g_base; ck_buf<unsigned long long> d_g_tile, d_g_grand;
    bool grouped = false; bool opt_bucket = false; const u32* cur_perm = nullptr;
    // Kafka record-batch framing (allocated on first use)
    ck_buf<long long> d_rb_batch_off, d_rb_rec_pos, d_rb_key_off, d_rb_corr_off;
    ck_buf<u32> d_rb_rec_base, d_rb_batch_bad, d_rb_rec_batch, d_rb_val_len, d_rb_rec_bad;
    ck_buf<int> d_rb_key_len, d_rb_corr_len; uint32_t rb_n = 0;
    ck_pinned<long long> h_rb_boff; ck_pinned<u32> h_rb_rbase; cudaEvent_t rb_ev = nullptr;   // frame index staging
    // fetches holding compressed batches (gzip, snappy, LZ4, zstd; allocated on the first one): the raw bytes, then every
    // such batch's decoded records section in its slot; per batch its slot (dec_off, n + 1 long, staging h_rb_dec_off) and
    // its decoded length
    ck_buf<u8> d_rb_fetch; ck_buf<long long> d_rb_dec_off; ck_pinned<long long> h_rb_dec_off; ck_buf<u32> d_rb_dec_len;
    uint64_t rb_dec_base = 0, rb_dec_bytes = 0;      // the decoded region of the last fetch (0 bytes: no compressed batch)
    // the chunk table of fetches holding snappy batches (ck_snappy.cuh; allocated on the first one, grown as needed): every
    // raw snappy block of the fetch and its place in its batch's slot, staged in page-locked memory
    ck_buf<ck_sn_chunk> d_rb_sn; ck_pinned<ck_sn_chunk> h_rb_sn;
    // per batch the host's flag (ck_txn.h: bad / skipped), uploaded for a fetch that flags any (allocated on the first one);
    // rb_hide: the read_committed mask ck_set_fetch_hidden gave for the next fetch
    ck_buf<u32> d_rb_flag; ck_pinned<u32> h_rb_flag; std::vector<uint8_t> rb_hide; bool rb_hide_set = false;
    // frame pass (allocated on first use): per slot, then per record in group order; the frames and their table
    ck_buf<ck_fitem> d_fr_items; ck_buf<u32> d_fr_gkey, d_fr_idx, d_fr_head, d_fr_fstart, d_fr_gfirst;
    ck_buf<u32> d_fr_ffirst, d_fr_size, d_fr_nlive, d_fr_partial;
    ck_buf<long long> d_fr_gscan, d_fr_S, d_fr_F, d_fr_R; ck_buf<unsigned long long> d_fr_tile, d_fr_grand;
    ck_buf<u32> d_fr_o1, d_fr_o2;      // its own sort buffers: the per-topic order of ck_group_publishes stays intact
    // fr_cap: the frames d_fr_frames (and d_fr_partial) have room for, 0 until fr_grow has reserved both
    ck_buf<ck_frame_ent> d_fr_table; ck_buf<u8> d_fr_frames; uint64_t fr_cap = 0; u32 fr_max = 0, fr_n = 0; bool fr_info = false, fr_sized = false;
    const u32* fr_order = nullptr; long long fr_base = 0, fr_ts = 0;   // what the write half of the last pass needs to run again
    ck_buf<u8> d_fr_blob; ck_buf<long long> d_fr_desc; ck_pinned<long long> h_fr_info;   // h_fr_info: {frames, bytes}
    ck_buf<int32_t> d_fr_slot; u32 fr_nslots = 0, fr_ntopics = 0;
    // idempotent / transactional produce: the producer fields the passes write (ck_set_producer; fr_prod: those of the last
    // pass, which a rewrite into a grown buffer uses again) and, by topic id, the sticky partition of the topic's unkeyed
    // publishes (ck_set_sticky_partitions; host copy for the record form, device copy for the plan's publishes)
    ck_producer prod{-1, -1, 0}, fr_prod{-1, -1, 0};
    std::vector<int32_t> fr_sticky; ck_buf<int32_t> d_fr_sticky;
    uint64_t fr_window = 1ull << 20;                 // frame_bytes (ck_set_option 2)
    // LZ4 frames (ck_set_option 3; allocated on the first compressed pass): the uncompressed frames, then the block slots,
    // each fr_raw_cap bytes (0 until lz_grow has reserved every buffer); per block slot its size and their scan; the
    // offsets of the compressed frames
    u32 fr_codec = 0, fr_pass_codec = 0;             // option 3, and the codec of the last pass
    // compression level (option 4; 0 = the default parse) and the level of the last pass; the chains of the hash-chain
    // parse (ck_lz4_block_hc), one per warp of its fixed grid (allocated on the first pass at a level that uses it)
    u32 fr_level = 0, fr_pass_level = 0; ck_buf<uint16_t> d_fr_chain;
    ck_buf<u8> d_fr_raw; uint64_t fr_raw_cap = 0; u32 fr_bmax = 0; ck_buf<u32> d_fr_bsize;
    ck_buf<long long> d_fr_bscan, d_fr_zoff; ck_buf<unsigned long long> d_fr_btile;
    // exchange planning (allocated on first use)
    ck_buf<u32> d_x_hist; ck_buf<long long> d_x_base; ck_buf<unsigned long long> d_x_nbytes;
    ck_buf<long long> d_x_src_off, d_x_len, d_x_dst_off; ck_buf<u32> d_x_len32, d_x_pub;
    ck_buf<unsigned long long> d_x_tile, d_x_grand, d_x_grand2; ck_pinned<long long> h_x;
    // topic table
    ck_topic_table tab{}; ck_buf<u32> d_tab_hash, d_tab_off, d_tab_len; ck_buf<int32_t> d_tab_id; ck_buf<u8> d_tab_names;
    uint32_t num_partitions = 0, hist_cap = 0;
    // current batch
    const u8* cur_in = nullptr; const long long* cur_in_off = nullptr; const u32* cur_len = nullptr;
    uint32_t n = 0, n_payloads = 0, n_pubs = 0;
    bool tool_set = false; ck_tool_cfg h_tool_cfg{};
    unsigned long long n_launch = 0;
    ck_pinned<unsigned long long> h_grand;
    // profiling: asynchronous event pairs around every kernel, read back (and summed) on demand so
    // that timing the kernels does not serialise the stream during a timed region
    bool profile = false;
    std::vector<cudaEvent_t> ev_pool;                    // 2 events per recorded launch
    std::vector<int> ev_kernel;                          // kernel id of each recorded pair
    size_t ev_used = 0;
    float k_ms[CK_NUM_KERNELS] = {0}; uint32_t k_n[CK_NUM_KERNELS] = {0};
};

#define CUDA_TRY(h, call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) { \
    char b_[512]; snprintf(b_, sizeof b_, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e_), __FILE__, __LINE__); \
    (h)->err = b_; return 1; } } while (0)

#define CKL(h) (h)->n_launch++,          // every kernel launch is counted (ck_launch_count: bench.py's gpu_launches)
static int fail(ck_handle* h, const char* msg) { h->err = msg; return 1; }

struct KTimer {
    ck_handle* h; int k; size_t slot;
    KTimer(ck_handle* hh, int kk) : h(hh), k(kk), slot(0) {
        if (!h->profile) return;
        if (h->ev_used + 2 > h->ev_pool.size()) {
            for (int j = 0; j < 64; j++) { cudaEvent_t e; cudaEventCreate(&e); h->ev_pool.push_back(e); }
        }
        slot = h->ev_used; h->ev_used += 2; h->ev_kernel.push_back(k);
        cudaEventRecord(h->ev_pool[slot], h->stream);
    }
    ~KTimer() { if (h->profile) cudaEventRecord(h->ev_pool[slot + 1], h->stream); }
};
static void profile_collect(ck_handle* h) {
    cudaStreamSynchronize(h->stream);
    for (size_t p = 0; p * 2 < h->ev_used; p++) {
        float ms = 0;
        if (cudaEventElapsedTime(&ms, h->ev_pool[2 * p], h->ev_pool[2 * p + 1]) == cudaSuccess) { h->k_ms[h->ev_kernel[p]] += ms; h->k_n[h->ev_kernel[p]]++; }
    }
    h->ev_used = 0; h->ev_kernel.clear();
}

extern "C" int ck_version(void) { return 1; }

extern "C" const char* ck_last_error(ck_handle* h) { return h ? h->err.c_str() : g_create_error.c_str(); }

extern "C" int ck_create(int device, uint64_t max_in_bytes, uint64_t max_out_bytes, uint32_t max_records,
                         uint32_t max_payloads, uint64_t max_aux_bytes, ck_handle** out) {
    *out = nullptr;
    ck_handle* h = new ck_handle();
    auto bail = [&](const char* what, cudaError_t e) {
        char b[512]; snprintf(b, sizeof b, "ck_create: %s: %s", what, cudaGetErrorString(e));
        g_create_error = b; ck_destroy(h); return 1;
    };
    cudaError_t e;
    h->device = device;
    if ((e = cudaSetDevice(device)) != cudaSuccess) return bail("cudaSetDevice", e);
    cudaDeviceProp prop;
    if ((e = cudaGetDeviceProperties(&prop, device)) != cudaSuccess) return bail("cudaGetDeviceProperties", e);
    if (prop.major != 9 || prop.minor != 0) { g_create_error = "ck_create: this library is built for sm_90a (H100) only"; ck_destroy(h); return 1; }
    h->num_sms = (u32)prop.multiProcessorCount;
    if ((e = cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking)) != cudaSuccess) return bail("cudaStreamCreate", e);
    {   // the canonicaliser is (boundedly) recursive: give device threads room for its frames
        size_t cur = 0; cudaDeviceGetLimit(&cur, cudaLimitStackSize);
        if (cur < 12 * 1024 && (e = cudaDeviceSetLimit(cudaLimitStackSize, 12 * 1024)) != cudaSuccess) return bail("cudaDeviceSetLimit(stack)", e);
    }
    h->max_in = max_in_bytes; h->max_out = max_out_bytes; h->max_aux = max_aux_bytes; h->max_records = max_records;
    h->max_payloads = max_payloads > max_records ? max_payloads : max_records; h->max_pubs = 2 * h->max_payloads;
#define ALLOC(b, n) if ((e = (b).reserve((n), h->stream)) != cudaSuccess) return bail("allocating " #b, e)
    ALLOC(h->d_in, max_in_bytes + CK_PAD);
    ALLOC(h->d_in_off, (size_t)max_records + 1);
    ALLOC(h->d_out, max_out_bytes + CK_PAD);
    ALLOC(h->d_out_off, (size_t)h->max_payloads + 1);
    ALLOC(h->d_aux, max_aux_bytes + CK_PAD);
    ALLOC(h->d_aux_off, (size_t)max_records + 1);
    ALLOC(h->d_glue, (size_t)CK_GLUE_STRIDE * h->max_payloads + CK_PAD);
    h->max_ovl = max_in_bytes;
    ALLOC(h->d_ovl, h->max_ovl + CK_PAD);
    ALLOC(h->d_ovl_off, (size_t)max_records + 1);
    ALLOC(h->d_ovl_len, (size_t)max_records);
    ALLOC(h->d_canon_ctl, 1);
    ALLOC(h->d_canon_list, (size_t)max_records);
    // list elements of long records walked one per thread: a message of a history is rarely shorter than a few hundred bytes
    // (a full list only means the remaining ones are walked inside their record's warp)
    { unsigned long long cap = max_in_bytes / 256 + 1024; if (cap > 0x7fffffffull) cap = 0x7fffffffull; h->elem_cap = (u32)cap; }
    ALLOC(h->d_elems, (size_t)h->elem_cap);
    ALLOC(h->d_cand, (size_t)max_records);
    ALLOC(h->d_hist_skip, (size_t)max_records);
    ALLOC(h->d_cols, (size_t)CK_NUM_COLS * max_records);
    ALLOC(h->d_descs, (size_t)h->max_payloads);
    ALLOC(h->d_pay_len, (size_t)h->max_payloads);
    ALLOC(h->d_pubs, (size_t)h->max_pubs);
    ALLOC(h->d_tile_sum, (size_t)h->max_payloads / CK_SCAN_TILE + 2);
    ALLOC(h->d_grand, 1);
    ALLOC(h->d_lit, CK_LIT_CAP + CK_PAD);
    ALLOC(h->d_tool_cfg, 1);
    ALLOC(h->d_agent_cfg, 1);
    ALLOC(h->d_counts, (size_t)max_records);
    ALLOC(h->d_slot_base, (size_t)max_records + 1);
    h->hist_cap = 4096;
    ALLOC(h->d_topic_hist, h->hist_cap);
    ALLOC(h->h_grand, 1);
#undef ALLOC
    cudaMemsetAsync(h->d_in.p + max_in_bytes, 0, CK_PAD, h->stream);
    cudaMemsetAsync(h->d_topic_hist.p, 0, sizeof(u32) * h->hist_cap, h->stream);
    if ((e = cudaStreamSynchronize(h->stream)) != cudaSuccess) return bail("init sync", e);
    *out = h;
    return 0;
}

extern "C" void ck_destroy(ck_handle* h) {
    if (!h) return;
    cudaSetDevice(h->device);
    if (h->stream) cudaStreamSynchronize(h->stream);
    if (h->xstream) cudaStreamSynchronize(h->xstream);
    for (u32 d = 0; d < CK_X_MAXWORLD; d++) if (h->peer_opened[d]) cudaIpcCloseMemHandle(h->peer_opened[d]);
    if (h->rb_ev) cudaEventDestroy(h->rb_ev);
    for (cudaEvent_t e : h->ev_pool) cudaEventDestroy(e);
    if (h->x_ev0) cudaEventDestroy(h->x_ev0);
    if (h->x_ev1) cudaEventDestroy(h->x_ev1);
    if (h->xstream) cudaStreamDestroy(h->xstream);
    if (h->stream) cudaStreamDestroy(h->stream);
    delete h;                                          // the buffers free themselves
}

static u32 host_fnv1a(const u8* p, u32 n) { u32 h = 2166136261u; for (u32 i = 0; i < n; i++) h = (h ^ p[i]) * 16777619u; return h ? h : 1u; }

extern "C" int ck_register_topics(ck_handle* h, const uint8_t* names, const uint32_t* offsets, uint32_t n,
                                  const int32_t* ids, uint32_t num_partitions) {
    cudaSetDevice(h->device);
    u32 cap = 64;
    while (cap < 4 * n) cap <<= 1;
    std::vector<u32> th(cap, 0), toff(cap, 0), tlen(cap, 0);
    std::vector<int32_t> tid(cap, -1);
    for (u32 i = 0; i < n; i++) {
        if (ids[i] < 0) return fail(h, "ck_register_topics: ids must be >= 0");
        u32 len = offsets[i + 1] - offsets[i];
        u32 hh = host_fnv1a(names + offsets[i], len);
        u32 slot = hh & (cap - 1);
        while (th[slot] != 0) {
            if (th[slot] == hh && tlen[slot] == len && memcmp(names + toff[slot], names + offsets[i], len) == 0) break;   // duplicate name: last wins
            slot = (slot + 1) & (cap - 1);
        }
        th[slot] = hh; toff[slot] = offsets[i]; tlen[slot] = len; tid[slot] = ids[i];
    }
    CUDA_TRY(h, cudaStreamSynchronize(h->stream));    // the kernels queued so far may read the old table
    u32 total = n ? offsets[n] : 0;
    ck_buf<u32> d_hash, d_off, d_len; ck_buf<int32_t> d_id; ck_buf<u8> d_names;
    CUDA_TRY(h, d_hash.reserve(cap, h->stream));
    CUDA_TRY(h, d_off.reserve(cap, h->stream));
    CUDA_TRY(h, d_len.reserve(cap, h->stream));
    CUDA_TRY(h, d_id.reserve(cap, h->stream));
    CUDA_TRY(h, d_names.reserve((size_t)total + CK_PAD, h->stream));
    CUDA_TRY(h, cudaMemcpy(d_hash.p, th.data(), sizeof(u32) * cap, cudaMemcpyHostToDevice));
    CUDA_TRY(h, cudaMemcpy(d_off.p, toff.data(), sizeof(u32) * cap, cudaMemcpyHostToDevice));
    CUDA_TRY(h, cudaMemcpy(d_len.p, tlen.data(), sizeof(u32) * cap, cudaMemcpyHostToDevice));
    CUDA_TRY(h, cudaMemcpy(d_id.p, tid.data(), sizeof(int32_t) * cap, cudaMemcpyHostToDevice));
    if (total) CUDA_TRY(h, cudaMemcpy(d_names.p, names, total, cudaMemcpyHostToDevice));
    h->tab.cap = cap; h->tab.hash = d_hash.p; h->tab.id = d_id.p; h->tab.name_off = d_off.p; h->tab.name_len = d_len.p; h->tab.names = d_names.p;
    h->d_tab_hash = std::move(d_hash); h->d_tab_off = std::move(d_off); h->d_tab_len = std::move(d_len);
    h->d_tab_id = std::move(d_id); h->d_tab_names = std::move(d_names);
    h->num_partitions = num_partitions;
    return 0;
}

extern "C" int ck_set_tool_node(ck_handle* h, int32_t publish_topic_id, uint32_t nparts, const uint32_t* kinds,
                                const uint8_t* blob, const uint32_t* part_offsets) {
    cudaSetDevice(h->device);
    if (nparts > CK_TPL_MAX_PARTS) return fail(h, "ck_set_tool_node: too many template parts");
    std::vector<u8> pool;
    auto put = [&](const char* s, uint32_t out[2]) { out[0] = (u32)pool.size(); out[1] = (u32)strlen(s); pool.insert(pool.end(), s, s + strlen(s)); };
    ck_tool_cfg c{};
    c.publish_topic_id = publish_topic_id;
    put(",\"", c.lit_comma_q); put("\"", c.lit_q); put("\":{\"return_value\":", c.lit_open);
    put(",\"content\":null,\"metadata\":{\"tool_call_id\":\"", c.lit_mid); put("\"},\"kind\":\"tool-return\"}", c.lit_close);
    put("{\"return_value\":", c.lit_value_open);
    c.tpl_nparts = nparts;
    for (u32 k = 0; k < nparts; k++) {
        c.tpl_kind[k] = kinds[k]; c.tpl_off[k] = (u32)pool.size(); c.tpl_len[k] = part_offsets[k + 1] - part_offsets[k];
        pool.insert(pool.end(), blob + part_offsets[k], blob + part_offsets[k + 1]);
    }
    if (pool.size() > CK_LIT_CAP) return fail(h, "ck_set_tool_node: literal pool overflow");
    CUDA_TRY(h, cudaStreamSynchronize(h->stream));
    CUDA_TRY(h, cudaMemcpy(h->d_lit.p, pool.data(), pool.size(), cudaMemcpyHostToDevice));
    CUDA_TRY(h, cudaMemcpy(h->d_tool_cfg.p, &c, sizeof c, cudaMemcpyHostToDevice));
    h->h_tool_cfg = c; h->tool_set = true;
    return 0;
}

static ck_view view_of(ck_handle* h) {
    ck_view v; v.in = h->cur_in; v.off = h->cur_in_off; v.ovl = h->d_ovl.p; v.ovl_off = h->d_ovl_off.p; v.ovl_len = h->d_ovl_len.p;
    v.canon_ctl = h->d_canon_ctl.p; v.canon_list = h->d_canon_list.p; v.len = h->cur_len; v.perm = h->cur_perm; v.elems = h->d_elems.p; v.elem_cap = h->elem_cap; v.hist_skip = h->d_hist_skip.p;
    return v;
}

static int run_scan(ck_handle* h, const u32* len, u32 n, long long* out_off, u32 pad,
                    unsigned long long* tile_sum = nullptr, unsigned long long* grand = nullptr, int timer = CK_K_SCAN);

static int group_alloc(ck_handle* h) {
    size_t nh = 64 * (size_t)((h->max_pubs + CK_G_BLOCK - 1) / CK_G_BLOCK);
    CUDA_TRY(h, h->d_g_hist.reserve(nh, h->stream));
    CUDA_TRY(h, h->d_g_base.reserve(nh + 1, h->stream));
    CUDA_TRY(h, h->d_g_o1.reserve((size_t)h->max_pubs + 1, h->stream));
    CUDA_TRY(h, h->d_g_o2.reserve((size_t)h->max_pubs + 1, h->stream));
    CUDA_TRY(h, h->d_g_keys.reserve(CK_G_KEYS, h->stream));
    CUDA_TRY(h, h->d_g_tile.reserve(nh / CK_SCAN_TILE + 2, h->stream));
    CUDA_TRY(h, h->d_g_grand.reserve(1, h->stream));
    return 0;
}

// stable LSD radix sort of indices 0..n-1 by a key of 6 * passes bits (6 bits per pass, passes 1..5), ping-ponging between
// o1 and o2 (default d_g_o1 / d_g_o2; two passes: the result is in o2) -> *result.  key_hist (CK_G_KEYS entries, zeroed here): per-key
// counts, for keys below CK_G_KEYS
template <int SHIFT, class KeyFn>
static void group_pass(ck_handle* h, KeyFn keyf, const u32* in, u32 n, u32 nb, u32* key_hist, bool count, u32* dst) {
    if (count) CKL(h) ck_group_count_kernel<SHIFT, KeyFn><<<nb, CK_G_BLOCK, 0, h->stream>>>(keyf, in, n, h->d_g_hist.p, key_hist);
    else CKL(h) ck_group_scatter_kernel<SHIFT, KeyFn><<<nb, CK_G_BLOCK, 0, h->stream>>>(keyf, in, n, h->d_g_base.p, dst);
}
template <class KeyFn>
static void group_launch(ck_handle* h, KeyFn keyf, u32 p, const u32* in, u32 n, u32 nb, u32* key_hist, bool count, u32* dst) {
    switch (p) {
        case 0: group_pass<0>(h, keyf, in, n, nb, key_hist, count, dst); break;
        case 1: group_pass<6>(h, keyf, in, n, nb, key_hist, count, dst); break;
        case 2: group_pass<12>(h, keyf, in, n, nb, key_hist, count, dst); break;
        case 3: group_pass<18>(h, keyf, in, n, nb, key_hist, count, dst); break;
        default: group_pass<24>(h, keyf, in, n, nb, key_hist, count, dst); break;
    }
}
template <class KeyFn>
static int group_sort(ck_handle* h, KeyFn keyf, u32 n, int timer, u32 passes = 2, u32* key_hist = nullptr, const u32** result = nullptr,
                      u32* o1 = nullptr, u32* o2 = nullptr) {
    if (!o1) { o1 = h->d_g_o1.p; o2 = h->d_g_o2.p; }
    if (key_hist) CUDA_TRY(h, cudaMemsetAsync(key_hist, 0, sizeof(u32) * CK_G_KEYS, h->stream));
    if (result) *result = (passes & 1) ? o1 : o2;
    if (!n) return 0;
    if (passes < 1 || passes > 5) return fail(h, "group_sort: 1 to 5 passes");
    u32 nb = (n + CK_G_BLOCK - 1) / CK_G_BLOCK;
    auto out_of = [&](u32 p) -> u32* { return (p & 1) ? o2 : o1; };    // pass p scatters here
    for (u32 p = 0; p < passes; p++) {
        {   // the scatter of the previous pass, then the histogram of this one
            KTimer t(h, timer);
            if (p) group_launch(h, keyf, p - 1, p > 1 ? out_of(p - 2) : nullptr, n, nb, key_hist, false, out_of(p - 1));
            group_launch(h, keyf, p, p ? out_of(p - 1) : nullptr, n, nb, key_hist, true, nullptr);
            CUDA_TRY(h, cudaGetLastError());
        }
        if (run_scan(h, h->d_g_hist.p, 64 * nb, h->d_g_base.p, 0, h->d_g_tile.p, h->d_g_grand.p)) return 1;
    }
    {
        KTimer t(h, timer);
        group_launch(h, keyf, passes - 1, passes > 1 ? out_of(passes - 2) : nullptr, n, nb, key_hist, false, out_of(passes - 1));
        CUDA_TRY(h, cudaGetLastError());
    }
    return 0;
}

// decode = walk every submitted record; re-emit the ones that are valid but not canonical into the overlay
// (count -> scan -> write) and walk those again in their canonical spelling
static int launch_decode(ck_handle* h) {
    u32 n = h->n;
    if (!n) return 0;
    ck_view v = view_of(h);
    CUDA_TRY(h, cudaMemsetAsync(h->d_ovl_off.p, 0xff, sizeof(long long) * (size_t)n, h->stream));      // no overlays yet
    CUDA_TRY(h, cudaMemsetAsync(h->d_canon_ctl.p, 0, sizeof(ck_canon_ctl), h->stream));
    h->cur_perm = nullptr;
    if (h->opt_bucket && n > 64) {
        if (group_alloc(h)) return 1;
        ck_key_len kf; kf.v = v;
        if (group_sort(h, kf, n, CK_K_WALK, 2, h->d_g_keys.p)) return 1;
        h->cur_perm = h->d_g_o2.p;
        v = view_of(h);
    }
    {
        // records of CK_HIST_MIN bytes or more, one warp each: structural pre-scan; message_history listed message by message
        // for the element pass, or (long records that are long for another reason) the whole record walked by the warp.
        // Both kernels exit at once when there are no such records.
        KTimer t(h, CK_K_WALK_LONG);
        CKL(h) ck_classify_kernel<<<(n + 255) / 256, 256, 0, h->stream>>>(v, n, h->d_cand.p);
        u32 lblocks = (n + CK_LONG_WARPS - 1) / CK_LONG_WARPS; if (lblocks > h->num_sms * CK_LONG_MINB) lblocks = h->num_sms * CK_LONG_MINB;
        CKL(h) ck_walk_long_kernel<<<lblocks, 32 * CK_LONG_WARPS, CK_LONG_WARPS * sizeof(ck_long_index), h->stream>>>(v, h->d_cols.p, n, h->d_cand.p, h->d_hist_skip.p);
        CUDA_TRY(h, cudaGetLastError());
    }
    {
        KTimer t(h, CK_K_WALK);
        CKL(h) ck_walk_kernel<<<(n + 127) / 128, 128, CK_WALK_THREADS * CK_WIN_STRIDE, h->stream>>>(v, n, h->d_cols.p, n);
        CUDA_TRY(h, cudaGetLastError());
    }
    {
        // the history messages listed by the pre-scan or deferred by the long walker, one thread each (exits at once when
        // there are none)
        KTimer t(h, CK_K_WALK_ELEMS);
        CKL(h) ck_walk_elems_kernel<<<h->num_sms * CK_WALK_MINB, CK_WALK_THREADS, CK_WALK_THREADS * CK_WIN_STRIDE, h->stream>>>(v, h->d_cols.p, n);
        CUDA_TRY(h, cudaGetLastError());
    }
    {
        // the records the walker listed (usually none: both kernels exit at once) are re-emitted canonically into the
        // overlay and walked again in that spelling
        KTimer t(h, CK_K_CANON);
        u32 blocks = (n + 63) / 64; if (blocks > h->num_sms * 8) blocks = h->num_sms * 8;
        CKL(h) ck_canon_kernel<<<blocks, 64, 0, h->stream>>>(v, n, h->d_cols.p, n, h->d_ovl.p, (long long)h->max_ovl, h->d_ovl_off.p, h->d_ovl_len.p);
        CKL(h) ck_rewalk_list_kernel<<<blocks, 64, 0, h->stream>>>(v, n, h->d_cols.p, n);
        CUDA_TRY(h, cudaGetLastError());
    }
    return 0;
}

extern "C" int ck_submit(ck_handle* h, const uint8_t* host_in, const int64_t* host_off, uint32_t n) {
    cudaSetDevice(h->device);
    if (n > h->max_records) return fail(h, "ck_submit: batch has more records than max_records");
    uint64_t nbytes = n ? (uint64_t)(host_off[n] - host_off[0]) : 0;
    if (n && host_off[0] != 0) return fail(h, "ck_submit: offsets must start at 0");
    if (nbytes > h->max_in) return fail(h, "ck_submit: batch larger than max_in_bytes");
    CUDA_TRY(h, cudaMemcpyAsync(h->d_in.p, host_in, nbytes, cudaMemcpyHostToDevice, h->stream));
    CUDA_TRY(h, cudaMemcpyAsync(h->d_in_off.p, host_off, sizeof(long long) * ((size_t)n + 1), cudaMemcpyHostToDevice, h->stream));
    CUDA_TRY(h, cudaMemsetAsync(h->d_in.p + nbytes, 0, 16, h->stream));
    h->cur_in = h->d_in.p; h->cur_in_off = h->d_in_off.p; h->cur_len = nullptr; h->n = n; h->n_payloads = 0; h->n_pubs = 0;
    return launch_decode(h);
}

extern "C" int ck_submit_device(ck_handle* h, const uint8_t* dev_in, const int64_t* dev_off, uint32_t n) {
    cudaSetDevice(h->device);
    if (n > h->max_records) return fail(h, "ck_submit_device: batch has more records than max_records");
    h->cur_in = dev_in; h->cur_in_off = (const long long*)dev_off; h->cur_len = nullptr; h->n = n; h->n_payloads = 0; h->n_pubs = 0;
    return launch_decode(h);
}

static int run_scan(ck_handle* h, const u32* len, u32 n, long long* out_off, u32 pad,
                    unsigned long long* tile_sum, unsigned long long* grand, int timer) {
    KTimer t(h, timer);
    if (!tile_sum) { tile_sum = h->d_tile_sum.p; grand = h->d_grand.p; }
    u32 ntiles = (n + CK_SCAN_TILE - 1) / CK_SCAN_TILE;
    if (n) {
        CKL(h) ck_scan_tiles_kernel<<<ntiles, CK_SCAN_BLOCK, 0, h->stream>>>(len, n, tile_sum, pad);
        CKL(h) ck_scan_sums_kernel<<<1, CK_SCAN_BLOCK, 0, h->stream>>>(tile_sum, ntiles, grand);
        CKL(h) ck_scan_apply_kernel<<<ntiles, CK_SCAN_BLOCK, 0, h->stream>>>(len, n, tile_sum, out_off, pad);
    }
    CUDA_TRY(h, cudaGetLastError());
    return 0;
}

static int scan_emit(ck_handle* h, u32 npay, const u8* aux) {
    if (run_scan(h, h->d_pay_len.p, npay, h->d_out_off.p, 15)) return 1;   // payloads start 16-byte aligned
    {
        KTimer t(h, CK_K_EMIT);
        if (npay) {
            u32 warps_per_block = 256 / 32;
            CKL(h) ck_emit_kernel<<<(npay + warps_per_block - 1) / warps_per_block, 256, 0, h->stream>>>(
                view_of(h), h->d_lit.p, aux, h->d_glue.p, h->d_descs.p, h->d_out_off.p, npay, h->d_out.p, (long long)h->max_out);
        }
        CUDA_TRY(h, cudaGetLastError());
    }
    h->n_payloads = npay;
    return 0;
}

// tool plan (modes 0 / 1 / 2) staged through shared memory, publishes routed in the same kernel (ck_plan.cuh)
static int launch_plan(ck_handle* h, const long long* aux_off, int mode) {
    static bool attr_set = false;
    if (!attr_set) {
        CUDA_TRY(h, cudaFuncSetAttribute(ck_plan_tool_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)CK_P2_SMEM));
        attr_set = true;
    }
    KTimer t(h, CK_K_PLAN);
    if (h->n) CKL(h) ck_plan_tool_kernel<<<(h->n + CK_P2_THREADS - 1) / CK_P2_THREADS, CK_P2_THREADS, CK_P2_SMEM, h->stream>>>(
        view_of(h), h->n, h->d_cols.p, h->n, h->d_tool_cfg.p, h->d_lit.p, aux_off, mode, h->d_descs.p, h->d_pay_len.p, h->d_pubs.p,
        h->tab, h->num_partitions, h->d_topic_hist.p, h->hist_cap);
    CUDA_TRY(h, cudaGetLastError());
    return 0;
}

extern "C" int ck_tool_args(ck_handle* h) {
    cudaSetDevice(h->device);
    if (!h->tool_set) return fail(h, "ck_tool_args: call ck_set_tool_node first");
    if (launch_plan(h, nullptr, 0)) return 1;
    h->n_pubs = 0;
    return scan_emit(h, h->n, nullptr);
}

static int tool_plan_common(ck_handle* h, const u8* aux, const long long* aux_off) {
    if (!h->tool_set) return fail(h, "ck_tool_plan: call ck_set_tool_node first");
    if (h->h_tool_cfg.tpl_nparts == 0 && aux_off == nullptr) return fail(h, "ck_tool_plan: node has no device template, host results required");
    if (launch_plan(h, aux_off, 1)) return 1;
    // NOTE: payload sizes are bounded by in + per-record constant; the caller sizes max_out accordingly
    if (scan_emit(h, h->n, aux)) return 1;
    h->n_pubs = 2 * h->n;
    return 0;
}

extern "C" int ck_tool_plan(ck_handle* h, const uint8_t* host_aux, const int64_t* host_aux_off) {
    cudaSetDevice(h->device);
    if (host_aux_off) {
        uint64_t nb = (uint64_t)host_aux_off[h->n];
        if (nb > h->max_aux) return fail(h, "ck_tool_plan: results larger than max_aux_bytes");
        CUDA_TRY(h, cudaMemcpyAsync(h->d_aux.p, host_aux, nb, cudaMemcpyHostToDevice, h->stream));
        CUDA_TRY(h, cudaMemcpyAsync(h->d_aux_off.p, host_aux_off, sizeof(long long) * ((size_t)h->n + 1), cudaMemcpyHostToDevice, h->stream));
        return tool_plan_common(h, h->d_aux.p, h->d_aux_off.p);
    }
    return tool_plan_common(h, nullptr, nullptr);
}

// ReturnCall of the state as it is on the wire (Agent final output): pop the frame, publish to the
// callback topic and to publish_topic (nodes/base.py:105-118, worker/worker.py:52-53)
extern "C" int ck_return_plan(ck_handle* h) {
    cudaSetDevice(h->device);
    if (!h->tool_set) return fail(h, "ck_return_plan: call ck_set_tool_node (publish topic) first");
    if (launch_plan(h, nullptr, 2)) return 1;
    if (scan_emit(h, h->n, nullptr)) return 1;
    h->n_pubs = 2 * h->n;
    return 0;
}

// client reply decode: payload i = the output value of reply i (see ck_reply_plan_kernel)
extern "C" int ck_reply_plan(ck_handle* h, uint32_t mode) {
    cudaSetDevice(h->device);
    if (mode > 2) return fail(h, "ck_reply_plan: mode must be 0 (auto), 1 (text) or 2 (data)");
    {
        KTimer t(h, CK_K_PLAN);
        if (h->n) CKL(h) ck_reply_plan_kernel<<<(h->n + 127) / 128, 128, 0, h->stream>>>(view_of(h), h->n, h->d_cols.p, h->n, mode, h->d_glue.p,
                                                                               h->d_descs.p, h->d_pay_len.p);
        CUDA_TRY(h, cudaGetLastError());
    }
    if (scan_emit(h, h->n, nullptr)) return 1;
    h->n_pubs = 0;
    return 0;
}

extern "C" int ck_tool_plan_device(ck_handle* h, const uint8_t* dev_aux, const int64_t* dev_aux_off) {
    cudaSetDevice(h->device);
    return tool_plan_common(h, dev_aux, (const long long*)dev_aux_off);
}

extern "C" int ck_set_agent_node(ck_handle* h, int32_t publish_topic_id, const uint8_t* agent_name, uint32_t agent_name_len,
                                 const uint8_t* callback_topic, uint32_t callback_len,
                                 const uint8_t* tool_names, const uint32_t* tool_name_off,
                                 const uint8_t* tool_topics, const uint32_t* tool_topic_off, uint32_t ntools) {
    // agent_name / callback_topic / tool topics are spliced into JSON strings: the caller passes them
    // already JSON-escaped (the Python binding does); tool_names are compared against raw JSON bytes.
    cudaSetDevice(h->device);
    std::vector<u8> pool;
    auto puts = [&](const std::string& s, uint32_t out[2]) { out[0] = (u32)pool.size(); out[1] = (u32)s.size(); pool.insert(pool.end(), s.begin(), s.end()); };
    ck_agent_cfg c{};
    c.publish_topic_id = publish_topic_id;
    c.ntools = ntools;
    std::string an((const char*)agent_name, agent_name_len), cb((const char*)callback_topic, callback_len);
    puts(",", c.lit_comma);
    puts("\",\"" + an + "\"],\"frame_id\":\"", c.lit_mid);
    puts("\",\"overrides\":null}", c.lit_tail);
    puts("{\"target_topic\":\"" + cb + "\",\"callback_topic\":\"", c.lit_tc_head);
    puts("\",\"input_args\":null,\"frame_id\":\"", c.lit_tc_mid);
    c.self_topic_id = -1;
    std::vector<u32> tab(6 * (size_t)ntools);
    for (u32 k = 0; k < ntools; k++) {
        std::string nm((const char*)tool_names + tool_name_off[k], tool_name_off[k + 1] - tool_name_off[k]);
        std::string tp((const char*)tool_topics + tool_topic_off[k], tool_topic_off[k + 1] - tool_topic_off[k]);
        uint32_t sp[2];
        puts(nm, sp); tab[k] = sp[0]; tab[ntools + k] = sp[1];
        puts("{\"target_topic\":\"" + tp + "\",\"callback_topic\":\"" + cb + "\",\"input_args\":[\"", sp);
        tab[2 * ntools + k] = sp[0]; tab[3 * ntools + k] = sp[1];
        // registered id of the tool's topic, if any (host-side probe of the same table the device uses is
        // not needed: ids are resolved by the route kernel when this is 0xffffffff)
        tab[4 * ntools + k] = 0xffffffffu;
        { std::vector<u64> pad(nm.size() / 8 + 4, 0ull);          // 8-byte aligned, padded: the reader loads whole aligned words
          memcpy((u8*)pad.data() + 8, nm.data(), nm.size());
          GRd hr; hr.init((const u8*)pad.data() + 8, (u32)nm.size());
          tab[5 * ntools + k] = ck_hash_span(hr, 0, (u32)nm.size()); }    // the device compares it with ck_hash_span of the name in the record
    }
    if (pool.size() > CK_LIT_CAP) return fail(h, "ck_set_agent_node: literal pool overflow");
    CUDA_TRY(h, cudaStreamSynchronize(h->stream));    // the kernels queued so far may read the old tables
    ck_buf<u32> tables;
    CUDA_TRY(h, tables.reserve(tab.size() + 1, h->stream));
    CUDA_TRY(h, cudaMemcpy(tables.p, tab.data(), sizeof(u32) * tab.size(), cudaMemcpyHostToDevice));
    c.tool_name_off = tables.p; c.tool_name_len = tables.p + ntools;
    c.tool_lit_off = tables.p + 2 * ntools; c.tool_lit_len = tables.p + 3 * ntools;
    c.tool_topic_id = tables.p + 4 * ntools;
    CUDA_TRY(h, cudaMemcpy(h->d_lit.p, pool.data(), pool.size(), cudaMemcpyHostToDevice));
    CUDA_TRY(h, cudaMemcpy(h->d_agent_cfg.p, &c, sizeof c, cudaMemcpyHostToDevice));
    h->d_agent_tables = std::move(tables);
    h->h_agent_cfg = c; h->agent_set = true;
    return 0;
}

extern "C" int ck_set_agent_tool_topic_ids(ck_handle* h, int32_t self_topic_id, const uint32_t* ids, uint32_t ntools) {
    cudaSetDevice(h->device);
    if (!h->agent_set || ntools != h->h_agent_cfg.ntools) return fail(h, "ck_set_agent_tool_topic_ids: agent node not set / size mismatch");
    CUDA_TRY(h, cudaStreamSynchronize(h->stream));
    if (ntools) CUDA_TRY(h, cudaMemcpy(h->d_agent_tables.p + 4 * (size_t)ntools, ids, sizeof(u32) * ntools, cudaMemcpyHostToDevice));
    h->h_agent_cfg.self_topic_id = self_topic_id;
    CUDA_TRY(h, cudaMemcpy(h->d_agent_cfg.p, &h->h_agent_cfg, sizeof h->h_agent_cfg, cudaMemcpyHostToDevice));
    return 0;
}

extern "C" int ck_tailcall_plan(ck_handle* h, uint64_t unix_ms, uint64_t seed) {
    cudaSetDevice(h->device);
    if (!h->agent_set) return fail(h, "ck_tailcall_plan: call ck_set_agent_node first");
    if (h->h_agent_cfg.self_topic_id < 0) return fail(h, "ck_tailcall_plan: the agent's own topic is not registered");
    u32 n = h->n;
    if (n > h->max_payloads) return fail(h, "ck_tailcall_plan: more payloads than max_payloads");
    {
        KTimer t(h, CK_K_FANOUT);
        if (n) CKL(h) ck_tailcall_plan_kernel<<<(n + 127) / 128, 128, 0, h->stream>>>(view_of(h), n, h->d_cols.p, n, h->d_agent_cfg.p, h->d_lit.p,
            unix_ms, seed, h->d_aux.p, h->d_glue.p, h->d_descs.p, h->d_pay_len.p, h->d_pubs.p);
        CUDA_TRY(h, cudaGetLastError());
    }
    if (scan_emit(h, n, h->d_aux.p)) return 1;
    {
        KTimer t(h, CK_K_ROUTE);
        u32 npubs = 2 * n;
        if (npubs) CKL(h) ck_route_kernel<<<(npubs + 255) / 256, 256, 0, h->stream>>>(view_of(h), h->d_cols.p, n, h->d_pubs.p, npubs,
            h->tab, h->num_partitions, h->d_topic_hist.p, h->hist_cap);
        CUDA_TRY(h, cudaGetLastError());
        h->n_pubs = npubs;
    }
    return 0;
}

extern "C" int ck_fanout_plan(ck_handle* h, uint64_t unix_ms, uint64_t seed, uint32_t max_fanout, uint32_t sequential) {
    cudaSetDevice(h->device);
    if (!h->agent_set) return fail(h, "ck_fanout_plan: call ck_set_agent_node first");
    u32 n = h->n;
    {
        KTimer t(h, CK_K_FANOUT);
        static bool f2_attr = false;
        if (!f2_attr) {
            CUDA_TRY(h, cudaFuncSetAttribute(ck_fanout2_count_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)CK_F2_SMEM));
            CUDA_TRY(h, cudaFuncSetAttribute(ck_fanout2_plan_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)CK_F2_SMEM));
            f2_attr = true;
        }
        if (n) CKL(h) ck_fanout2_count_kernel<<<(n + CK_F2_WARPS - 1) / CK_F2_WARPS, 32 * CK_F2_WARPS, CK_F2_SMEM, h->stream>>>(view_of(h), n, h->d_cols.p, n, h->d_agent_cfg.p,
                                                                                                             max_fanout, sequential, h->d_counts.p);
        CUDA_TRY(h, cudaGetLastError());
    }
    if (run_scan(h, h->d_counts.p, n, h->d_slot_base.p, 0)) return 1;
    *h->h_grand.p = 0;
    if (n) CUDA_TRY(h, cudaMemcpyAsync(h->h_grand.p, h->d_grand.p, sizeof(unsigned long long), cudaMemcpyDeviceToHost, h->stream));
    CUDA_TRY(h, cudaStreamSynchronize(h->stream));
    unsigned long long slots = *h->h_grand.p;
    if (slots > h->max_payloads) return fail(h, "ck_fanout_plan: more payloads than max_payloads");
    {
        KTimer t(h, CK_K_FANOUT);
        if (n) CKL(h) ck_fanout2_plan_kernel<<<(n + CK_F2_WARPS - 1) / CK_F2_WARPS, 32 * CK_F2_WARPS, CK_F2_SMEM, h->stream>>>(view_of(h), n, h->d_cols.p, n, h->d_agent_cfg.p, h->d_lit.p,
            h->d_agent_tables.p + 5 * (size_t)h->h_agent_cfg.ntools, h->d_slot_base.p, unix_ms, seed, h->d_aux.p, h->d_glue.p, h->d_descs.p, h->d_pay_len.p, h->d_pubs.p);
        CUDA_TRY(h, cudaGetLastError());
    }
    if (scan_emit(h, (u32)slots, h->d_aux.p)) return 1;
    {
        KTimer t(h, CK_K_ROUTE);
        u32 npubs = 2 * (u32)slots;
        if (npubs) CKL(h) ck_route_kernel<<<(npubs + 255) / 256, 256, 0, h->stream>>>(view_of(h), h->d_cols.p, n, h->d_pubs.p, npubs,
            h->tab, h->num_partitions, h->d_topic_hist.p, h->hist_cap);
        CUDA_TRY(h, cudaGetLastError());
        h->n_pubs = npubs;
    }
    return 0;
}

// ---- grouping the publish table by topic (csrc/ck_group.cuh) ---------------------------------------------------------------
extern "C" int ck_group_publishes(ck_handle* h) {
    cudaSetDevice(h->device);
    if (group_alloc(h)) return 1;
    h->grouped = true;
    ck_key_pub kf; kf.pubs = h->d_pubs.p; kf.rank = h->comm_rank; kf.world = h->comm_ready ? h->comm_world : 1;
    return group_sort(h, kf, h->n_pubs, CK_K_ROUTE, 2, h->d_g_keys.p);
}

// engine options.  CK_OPT_BUCKET (1): bucket every submitted batch by record length before the thread-per-record walk —
// for topics that carry records of mixed sizes / shapes (a warp takes as long as its longest record, and lanes on
// different schema branches run one after the other); homogeneous batches do not need it (it costs six small launches).
extern "C" int ck_set_option(ck_handle* h, uint32_t option, uint64_t value) {
    if (option == 1) { h->opt_bucket = value != 0; return 0; }
    if (option == 2) { if (value < 1) return fail(h, "ck_set_option: frame_bytes must be at least 1"); h->fr_window = value; return 0; }
    if (option == 3) {
        if (value != 0 && value != 3) return fail(h, "ck_set_option: frame codec must be 0 (none) or 3 (lz4)");
        h->fr_codec = (u32)value; return 0;
    }
    if (option == 4) {
        if (value > CK_LZ_LEVEL_MAX) {
            char b[128];
            snprintf(b, sizeof b, "ck_set_option: compression level %llu is outside 0 (default) .. %u", (unsigned long long)value, CK_LZ_LEVEL_MAX);
            return fail(h, b);
        }
        h->fr_level = (u32)value; return 0;
    }
    return fail(h, "ck_set_option: unknown option");
}

// order[n_publishes]: publish indices grouped by key (0 = unregistered topic, 1 + id = registered topic id, 4095 = unused
// slot), send order kept inside a group; key_counts[4096].  wait = 0: copies queued only (page-locked destinations).
extern "C" int ck_fetch_groups(ck_handle* h, uint32_t* host_order, uint32_t* host_key_counts, int wait) {
    cudaSetDevice(h->device);
    if (!h->grouped) return fail(h, "ck_fetch_groups: call ck_group_publishes first");
    if (h->n_pubs) CUDA_TRY(h, cudaMemcpyAsync(host_order, h->d_g_o2.p, sizeof(u32) * (size_t)h->n_pubs, cudaMemcpyDeviceToHost, h->stream));
    CUDA_TRY(h, cudaMemcpyAsync(host_key_counts, h->d_g_keys.p, sizeof(u32) * CK_G_KEYS, cudaMemcpyDeviceToHost, h->stream));
    if (wait) CUDA_TRY(h, cudaStreamSynchronize(h->stream));
    return 0;
}

// ---- Kafka RecordBatch v2 framing (csrc/ck_kafka.cuh) -------------------------------------------------------------------
static inline uint32_t host_be32(const uint8_t* p) { return ((uint32_t)p[0] << 24) | ((uint32_t)p[1] << 16) | ((uint32_t)p[2] << 8) | p[3]; }

// room for n entries in the chunk table's staging, at least doubling it, its first `used` entries kept
static int rb_sn_reserve(ck_handle* h, u32 n, u32 used) {
    if (n <= h->h_rb_sn.cap) return 0;
    CUDA_TRY(h, h->h_rb_sn.reserve(std::max<size_t>(n, std::max<size_t>(1024, 2 * h->h_rb_sn.cap)), h->stream, used));
    return 0;
}

// A fetch response's record set (concatenated RecordBatch v2 frames, as it came off the socket) goes to HBM in one copy;
// CRC32C check, record split and varint field decode run on the device and the walker reads every value where it lies.
// The host only chains through the frame headers (12 + batchLength bytes each) to index the frames, through the LZ4 block
// chain of an LZ4 batch (ck_lz_walk) to bound what it decodes to, through the member header of a gzip batch to read its
// ISIZE (ck_gz_member), through the frame header and block headers of a zstd batch to bound what it decodes to
// (ck_zs_header, ck_zs_walk), and through the chunk chain of a snappy batch to read every block's declared length
// (ck_sn_next), listing each block in the chunk table.  A fetch holding a gzip, snappy, LZ4 or zstd batch goes to the
// fetch buffer instead of d_in, with a slot per such batch behind the raw bytes that the decode kernel of its codec fills
// (one launch per codec present); a fetch without one takes the path it always took.  The host also reads every control
// batch (ck_txn_control: its CRC32C, its one record's key) and flags it skipped, or bad when malformed; a read_committed
// mask (ck_set_fetch_hidden) flags the aborted transactions' batches skipped.  A flagged batch gets no slot: it is never
// sized or decoded
extern "C" int ck_set_fetch_hidden(ck_handle* h, const uint8_t* mask, uint32_t nbatches) {
    h->rb_hide.assign(mask, mask + nbatches);
    h->rb_hide_set = true;
    return 0;
}
extern "C" int ck_submit_recordbatch(ck_handle* h, const uint8_t* host_buf, uint64_t nbytes, uint32_t* n_records) {
    cudaSetDevice(h->device);
    bool hide = h->rb_hide_set;                        // the mask given for this fetch, consumed by it whatever happens
    h->rb_hide_set = false;
    if (nbytes > h->max_in) return fail(h, "ck_submit_recordbatch: buffer larger than max_in_bytes");
    size_t mr = (size_t)h->max_records + 1;
    CUDA_TRY(h, h->d_rb_batch_off.reserve(mr, h->stream)); CUDA_TRY(h, h->d_rb_rec_base.reserve(mr, h->stream));
    CUDA_TRY(h, h->d_rb_batch_bad.reserve(mr, h->stream)); CUDA_TRY(h, h->d_rb_rec_pos.reserve(mr, h->stream));
    CUDA_TRY(h, h->d_rb_rec_batch.reserve(mr, h->stream)); CUDA_TRY(h, h->d_rb_val_len.reserve(mr, h->stream));
    CUDA_TRY(h, h->d_rb_key_off.reserve(mr, h->stream)); CUDA_TRY(h, h->d_rb_key_len.reserve(mr, h->stream));
    CUDA_TRY(h, h->d_rb_corr_off.reserve(mr, h->stream)); CUDA_TRY(h, h->d_rb_corr_len.reserve(mr, h->stream));
    CUDA_TRY(h, h->d_rb_rec_bad.reserve(mr, h->stream));
    CUDA_TRY(h, h->h_rb_boff.reserve(mr, h->stream)); CUDA_TRY(h, h->h_rb_rbase.reserve(mr, h->stream));
    if (!h->rb_ev) CUDA_TRY(h, cudaEventCreateWithFlags(&h->rb_ev, cudaEventDisableTiming));
    // the frame index is staged in page-locked memory the handle owns: its copies are asynchronous.  The staging is reused
    // once the copies of the previous call have been done (normally long ago: it waits for those copies only)
    CUDA_TRY(h, cudaEventSynchronize(h->rb_ev));
    long long* boff = h->h_rb_boff.p; u32* rbase = h->h_rb_rbase.p;
    uint64_t pos = 0; uint64_t total = 0; u32 nb = 0;
    bool decoded = false, has_lz4 = false, has_gz = false, has_zs = false, has_sn = false;   // decoded: a batch is decoded into a slot
    u32 nsn = 0;                                       // entries of the snappy chunk table
    bool flagged = false;                              // some batch is flagged bad or skipped by the host
    uint64_t dbytes = 0;                               // slot bytes so far (the LZ4 and zstd bounds, the gzip ISIZEs, the snappy lengths)
    uint64_t end;
    while ((end = ck_txn_frame_end(host_buf, nbytes, pos)) != 0) {   // stops at a truncated trailing frame: legal in a fetch response
        uint32_t cnt = host_be32(host_buf + pos + 57);
        if (total + cnt > h->max_records || nb >= h->max_records) return fail(h, "ck_submit_recordbatch: more records than max_records");
        u32 codec = host_buf[pos + 22] & 7u;
        int type = 0;
        u32 flag = (host_buf[pos + 22] & CK_TXN_CONTROL) ? (u32)ck_txn_control(host_buf + pos, end - pos, &type)
                 : hide && nb < h->rb_hide.size() && h->rb_hide[nb] ? (u32)CK_TXN_HIDE : (u32)CK_TXN_SHOW;
        if (flag && !flagged) {                        // the batches before the first flagged one are delivered
            CUDA_TRY(h, h->d_rb_flag.reserve(mr, h->stream)); CUDA_TRY(h, h->h_rb_flag.reserve(mr, h->stream));
            for (u32 b = 0; b < nb; b++) h->h_rb_flag.p[b] = 0;
            flagged = true;
        }
        if (flagged) h->h_rb_flag.p[nb] = flag;
        if (!flag && (codec == CK_RB_LZ4 || codec == CK_RB_GZIP || codec == CK_RB_ZSTD || codec == CK_RB_SNAPPY)) {
            if (!decoded) {                            // the batches before the first decoded one have empty slots
                CUDA_TRY(h, h->d_rb_dec_off.reserve(mr, h->stream)); CUDA_TRY(h, h->d_rb_dec_len.reserve(mr, h->stream));
                CUDA_TRY(h, h->h_rb_dec_off.reserve(mr, h->stream));
                for (u32 b = 0; b <= nb; b++) h->h_rb_dec_off.p[b] = 0;
                decoded = true;
            }
            // the slot: LZ4, what the block chain decodes to at most; gzip, the member's ISIZE; zstd, what the blocks
            // decode to at most (compressed ones Block_Maximum_Size, even when Frame_Content_Size says less: their literals
            // are decoded into the end of that room); snappy, exactly the sum of its blocks' declared lengths.  0 (the
            // device marks the batch bad) when the chain or the blocks cannot be walked or the member header parsed, or the
            // decoded batch would not fit the 32-bit lengths of the record split
            unsigned long long bound = 0;
            const u8* z = host_buf + pos + CK_RB_HEADER;
            if (codec == CK_RB_LZ4) {
                ck_lz_desc d; u32 k = 0;
                if (!ck_lz_parse_desc(z, end - pos - CK_RB_HEADER, d) || !ck_lz_walk(z, end - pos - CK_RB_HEADER, d, &k, &bound) ||
                    CK_RB_HEADER + bound > 0x7fffffffull) bound = 0;
                has_lz4 = true;
            } else if (codec == CK_RB_ZSTD) {
                ck_zs_frame f;
                if (!ck_zs_header(z, end - pos - CK_RB_HEADER, f) || !ck_zs_walk(z, end - pos - CK_RB_HEADER, f, &bound) ||
                    CK_RB_HEADER + bound > 0x7fffffffull) bound = 0;
                has_zs = true;
            } else if (codec == CK_RB_SNAPPY) {
                // one chunk table entry per block; a section the walk refuses has its entries dropped and gets one entry of
                // no input, which the device refuses (so it marks the batch bad)
                u32 first = nsn;
                ck_sn_walker w;
                ck_sn_begin(z, end - pos - CK_RB_HEADER, w);
                unsigned long long off, o = 0; u32 len, dl;
                int r;
                while ((r = ck_sn_next(z, end - pos - CK_RB_HEADER, w, &off, &len, &dl)) > 0) {
                    if (CK_RB_HEADER + o + dl > 0x7fffffffull) { r = -1; break; }
                    if (rb_sn_reserve(h, nsn + 1, nsn)) return 1;
                    h->h_rb_sn.p[nsn++] = ck_sn_chunk{(long long)(pos + CK_RB_HEADER + off), nb, len, (u32)o, dl};
                    o += dl;
                }
                if (r < 0) {
                    nsn = first;
                    if (rb_sn_reserve(h, nsn + 1, nsn)) return 1;
                    h->h_rb_sn.p[nsn++] = ck_sn_chunk{(long long)(pos + CK_RB_HEADER), nb, 0u, 0u, 0u};
                }
                bound = r < 0 ? 0 : o;
                has_sn = true;
            } else {
                u32 hdr = 0, isize = 0;
                if (ck_gz_member(z, end - pos - CK_RB_HEADER, &hdr, &isize) && CK_RB_HEADER + (unsigned long long)isize <= 0x7fffffffull) bound = isize;
                has_gz = true;
            }
            h->h_rb_dec_off.p[nb] = (long long)dbytes;
            dbytes += bound;
        } else if (decoded) h->h_rb_dec_off.p[nb] = (long long)dbytes;
        boff[nb] = (long long)pos; rbase[nb] = (u32)total; nb++;
        total += cnt; pos = end;
    }
    boff[nb] = (long long)pos; rbase[nb] = (u32)total;
    if (hide && h->rb_hide.size() != nb) return fail(h, "ck_submit_recordbatch: the mask of ck_set_fetch_hidden does not cover the fetch's batches");
    u32 n = (u32)total;
    if (n_records) *n_records = n;
    u8* buf = h->d_in.p;
    uint64_t base = 0, used = pos;
    if (decoded) {                                     // slots in value-offset space: behind the raw bytes, 16-byte aligned
        base = (pos + 15) & ~15ull; used = base + dbytes;
        for (u32 b = 0; b < nb; b++) h->h_rb_dec_off.p[b] += (long long)base;
        h->h_rb_dec_off.p[nb] = (long long)used;
        // the fetch buffer, grown as fr_grow grows the frame buffer
        if (used + CK_PAD > h->d_rb_fetch.cap) CUDA_TRY(h, h->d_rb_fetch.reserve(used + used / 8 + 4096 + CK_PAD, h->stream));
        buf = h->d_rb_fetch.p;
    }
    CUDA_TRY(h, cudaMemcpyAsync(buf, host_buf, pos, cudaMemcpyHostToDevice, h->stream));
    CUDA_TRY(h, cudaMemsetAsync(buf + pos, 0, decoded ? used - pos + 16 : 16, h->stream));
    CUDA_TRY(h, cudaMemcpyAsync(h->d_rb_batch_off.p, boff, sizeof(long long) * (nb + 1), cudaMemcpyHostToDevice, h->stream));
    CUDA_TRY(h, cudaMemcpyAsync(h->d_rb_rec_base.p, rbase, sizeof(u32) * (nb + 1), cudaMemcpyHostToDevice, h->stream));
    if (decoded) CUDA_TRY(h, cudaMemcpyAsync(h->d_rb_dec_off.p, h->h_rb_dec_off.p, sizeof(long long) * (nb + 1), cudaMemcpyHostToDevice, h->stream));
    if (nsn) {
        CUDA_TRY(h, h->d_rb_sn.reserve(h->h_rb_sn.cap, h->stream));   // the size of the staging
        CUDA_TRY(h, cudaMemcpyAsync(h->d_rb_sn.p, h->h_rb_sn.p, sizeof(ck_sn_chunk) * nsn, cudaMemcpyHostToDevice, h->stream));
    }
    if (flagged) CUDA_TRY(h, cudaMemcpyAsync(h->d_rb_flag.p, h->h_rb_flag.p, sizeof(u32) * nb, cudaMemcpyHostToDevice, h->stream));
    CUDA_TRY(h, cudaEventRecord(h->rb_ev, h->stream));
    h->rb_n = n; h->rb_dec_base = decoded ? base : 0; h->rb_dec_bytes = decoded ? dbytes : 0;
    if (nb) {
        KTimer t(h, CK_K_WALK);
        CKL(h) ck_rb_crc_kernel<<<(nb + 7) / 8, 256, 0, h->stream>>>(buf, h->d_rb_batch_off.p, flagged ? h->d_rb_flag.p : nullptr, nb, h->d_rb_batch_bad.p);
        if (has_lz4) CKL(h) ck_rb_lz4_kernel<<<(nb + 7) / 8, 256, 0, h->stream>>>(buf, h->d_rb_batch_off.p, h->d_rb_dec_off.p, nb, h->d_rb_batch_bad.p, h->d_rb_dec_len.p);
        if (has_gz) CKL(h) ck_rb_gzip_kernel<<<(nb + CK_GZ_WARPS - 1) / CK_GZ_WARPS, 32 * CK_GZ_WARPS, 0, h->stream>>>(buf, h->d_rb_batch_off.p, h->d_rb_dec_off.p, nb,
                                                                                                          h->d_rb_batch_bad.p, h->d_rb_dec_len.p);
        if (has_zs) CKL(h) ck_rb_zstd_kernel<<<(nb + CK_ZS_WARPS - 1) / CK_ZS_WARPS, 32 * CK_ZS_WARPS, 0, h->stream>>>(buf, h->d_rb_batch_off.p, h->d_rb_dec_off.p, nb,
                                                                                                          h->d_rb_batch_bad.p, h->d_rb_dec_len.p);
        if (has_sn) CKL(h) ck_rb_snappy_kernel<<<(nsn + CK_SN_WARPS - 1) / CK_SN_WARPS, 32 * CK_SN_WARPS, 0, h->stream>>>(buf, h->d_rb_sn.p, nsn, h->d_rb_dec_off.p,
                                                                                                              h->d_rb_batch_bad.p, h->d_rb_dec_len.p);
        CKL(h) ck_rb_split_kernel<<<(nb + 127) / 128, 128, 0, h->stream>>>(buf, h->d_rb_batch_off.p, decoded ? h->d_rb_dec_off.p : nullptr,
                                                                        decoded ? h->d_rb_dec_len.p : nullptr, h->d_rb_rec_base.p, nb,
                                                                        h->d_rb_batch_bad.p, h->d_rb_rec_pos.p, h->d_rb_rec_batch.p);
        if (n) CKL(h) ck_rb_fields_kernel<<<(n + 127) / 128, 128, 0, h->stream>>>(buf, (long long)used, h->d_rb_rec_pos.p, h->d_rb_rec_batch.p, h->d_rb_batch_bad.p, n,
            h->d_in_off.p, h->d_rb_val_len.p, h->d_rb_key_off.p, h->d_rb_key_len.p, h->d_rb_corr_off.p, h->d_rb_corr_len.p, h->d_rb_rec_bad.p);
        CUDA_TRY(h, cudaGetLastError());
    }
    h->cur_in = buf; h->cur_in_off = h->d_in_off.p; h->cur_len = h->d_rb_val_len.p; h->n = n; h->n_payloads = 0; h->n_pubs = 0;
    if (launch_decode(h)) return 1;
    if (n) { CKL(h) ck_rb_mark_bad_kernel<<<(n + 255) / 256, 256, 0, h->stream>>>(h->d_rb_rec_bad.p, n, h->d_cols.p, n); CUDA_TRY(h, cudaGetLastError()); }
    return 0;
}

// idempotent produce's sequence hand-off: the CRC32C of a span after 4 of its bytes changed (ck_txn_crc32c_patch)
extern "C" int ck_crc32c_patch(uint32_t* crc, uint64_t len, uint64_t pos, const uint8_t* old4, const uint8_t* new4) {
    if (len < 4 || pos > len - 4) { g_create_error = "ck_crc32c_patch: the 4 bytes lie outside the span"; return 1; }
    *crc = ck_txn_crc32c_patch(*crc, len, pos, old4, new4);
    return 0;
}

// a transaction marker as the broker appends it (ck_txn_control_batch): no handle, no device
extern "C" int ck_encode_control_batch(int64_t base_offset, int64_t timestamp_ms, int64_t producer_id, int16_t producer_epoch,
                                       int16_t type, uint8_t* out, uint64_t cap, uint64_t* len) {
    if (cap < CK_TXN_CONTROL_LEN) { g_create_error = "ck_encode_control_batch: buffer shorter than a control batch"; return 1; }
    ck_txn_control_batch(out, base_offset, timestamp_ms, producer_id, producer_epoch, type);
    if (len) *len = CK_TXN_CONTROL_LEN;
    return 0;
}

// the read_committed mask of a whole fetch (ck_txn_mask): no handle, no device
extern "C" int ck_fetch_txn_mask(const uint8_t* buf, uint64_t nbytes, const uint64_t* run_start, uint32_t nruns,
                                 const uint32_t* abort_run, const int64_t* abort_pid, const int64_t* abort_first, uint32_t naborts,
                                 uint8_t* mask, uint32_t cap, uint32_t* nbatches) {
    int64_t nb = ck_txn_mask(buf, nbytes, run_start, nruns, abort_run, abort_pid, abort_first, naborts, mask, cap);
    if (nb < 0) { g_create_error = "ck_fetch_txn_mask: partition starts out of order, or an aborted transaction of no partition"; return 1; }
    if (nbatches) *nbatches = (uint32_t)nb;
    if ((uint64_t)nb > cap) { g_create_error = "ck_fetch_txn_mask: mask shorter than the fetch's batches"; return 1; }
    return 0;
}

// the consumed positions of a fetch or a slice of one (ck_txn_positions): no handle, no device
extern "C" int ck_fetch_positions(const uint8_t* buf, uint64_t nbytes, const uint64_t* run_start, uint32_t nruns,
                                  int64_t* next, int64_t* batch_next, uint32_t cap, uint32_t* nbatches) {
    int64_t nb = ck_txn_positions(buf, nbytes, run_start, nruns, next, batch_next, cap);
    if (nb < 0) { g_create_error = "ck_fetch_positions: partition starts out of order"; return 1; }
    if (nbatches) *nbatches = (uint32_t)nb;
    if (batch_next && (uint64_t)nb > cap) { g_create_error = "ck_fetch_positions: batch_next shorter than the fetch's batches"; return 1; }
    return 0;
}

// per record of the last ck_submit_recordbatch: where value / key / correlation_id header lie in the submitted buffer
// (key_len / corr_len = -1: absent), and whether its frame failed the CRC / framing check
static int fetch_rb_index_impl(ck_handle* h, int64_t* val_off, uint32_t* val_len, int64_t* key_off, int32_t* key_len,
                               int64_t* corr_off, int32_t* corr_len, uint32_t* bad, bool wait);
extern "C" int ck_fetch_rb_index(ck_handle* h, int64_t* val_off, uint32_t* val_len, int64_t* key_off, int32_t* key_len,
                                 int64_t* corr_off, int32_t* corr_len, uint32_t* bad) {
    return fetch_rb_index_impl(h, val_off, val_len, key_off, key_len, corr_off, corr_len, bad, true);
}
// the same copies queued only (page-locked destinations): they ride along with the step's results, complete after ck_sync
extern "C" int ck_fetch_rb_index_async(ck_handle* h, int64_t* val_off, uint32_t* val_len, int64_t* key_off, int32_t* key_len,
                                       int64_t* corr_off, int32_t* corr_len, uint32_t* bad) {
    return fetch_rb_index_impl(h, val_off, val_len, key_off, key_len, corr_off, corr_len, bad, false);
}
static int fetch_rb_index_impl(ck_handle* h, int64_t* val_off, uint32_t* val_len, int64_t* key_off, int32_t* key_len,
                               int64_t* corr_off, int32_t* corr_len, uint32_t* bad, bool wait) {
    cudaSetDevice(h->device);
    u32 n = h->rb_n;
    if (!n) return 0;
    if (val_off) CUDA_TRY(h, cudaMemcpyAsync(val_off, h->d_in_off.p, sizeof(long long) * n, cudaMemcpyDeviceToHost, h->stream));
    if (val_len) CUDA_TRY(h, cudaMemcpyAsync(val_len, h->d_rb_val_len.p, sizeof(u32) * n, cudaMemcpyDeviceToHost, h->stream));
    if (key_off) CUDA_TRY(h, cudaMemcpyAsync(key_off, h->d_rb_key_off.p, sizeof(long long) * n, cudaMemcpyDeviceToHost, h->stream));
    if (key_len) CUDA_TRY(h, cudaMemcpyAsync(key_len, h->d_rb_key_len.p, sizeof(int) * n, cudaMemcpyDeviceToHost, h->stream));
    if (corr_off) CUDA_TRY(h, cudaMemcpyAsync(corr_off, h->d_rb_corr_off.p, sizeof(long long) * n, cudaMemcpyDeviceToHost, h->stream));
    if (corr_len) CUDA_TRY(h, cudaMemcpyAsync(corr_len, h->d_rb_corr_len.p, sizeof(int) * n, cudaMemcpyDeviceToHost, h->stream));
    if (bad) CUDA_TRY(h, cudaMemcpyAsync(bad, h->d_rb_rec_bad.p, sizeof(u32) * n, cudaMemcpyDeviceToHost, h->stream));
    if (wait) CUDA_TRY(h, cudaStreamSynchronize(h->stream));
    return 0;
}

// the decoded slots of the last ck_submit_recordbatch: value offsets from *base on index them.  Known on the host as soon
// as the call returns; dst NULL asks for the size only
extern "C" int ck_fetch_rb_decoded_async(ck_handle* h, uint8_t* dst, uint64_t cap, uint64_t* base, uint64_t* nbytes) {
    cudaSetDevice(h->device);
    if (base) *base = h->rb_dec_base;
    if (nbytes) *nbytes = h->rb_dec_bytes;
    if (!dst || !h->rb_dec_bytes) return 0;
    if (cap < h->rb_dec_bytes) return fail(h, "ck_fetch_rb_decoded_async: host buffer too small");
    CUDA_TRY(h, cudaMemcpyAsync(dst, h->d_rb_fetch.p + h->rb_dec_base, h->rb_dec_bytes, cudaMemcpyDeviceToHost, h->stream));
    return 0;
}

// ---- frame pass: the publishes of a step (or host-produced records) as RecordBatch v2 frames (csrc/ck_kafka.cuh) -------
static int fr_grow(ck_handle* h, uint64_t cap) {
    h->fr_cap = 0;
    CUDA_TRY(h, h->d_fr_frames.reserve(cap + CK_PAD, h->stream));
    CUDA_TRY(h, h->d_fr_partial.reserve(cap / CK_RB_CRC_CHUNK + (size_t)h->max_pubs + 2, h->stream));
    h->fr_cap = cap;
    return 0;
}
// the scratch of the LZ4 stage, sized for uncompressed frames of `cap` bytes: those frames, the block slots (a block's
// compressed bytes lie at its own offset, and are never longer), and a size per 64 KB block slot
static int lz_grow(ck_handle* h, uint64_t cap) {
    h->fr_raw_cap = 0;
    uint64_t bmax = cap / CK_LZ_BLOCK + (uint64_t)h->fr_max + 2;
    if (bmax > 0xffffffffull) return fail(h, "lz_grow: more than 2^32 LZ4 blocks");
    CUDA_TRY(h, h->d_fr_zoff.reserve((size_t)h->fr_max + 1, h->stream));
    CUDA_TRY(h, h->d_fr_raw.reserve(2 * (cap + CK_PAD), h->stream));
    CUDA_TRY(h, h->d_fr_bsize.reserve(bmax, h->stream));
    CUDA_TRY(h, h->d_fr_bscan.reserve(bmax + 1, h->stream));
    CUDA_TRY(h, h->d_fr_btile.reserve(bmax / CK_SCAN_TILE + 2, h->stream));
    h->fr_raw_cap = cap; h->fr_bmax = (u32)bmax;
    return 0;
}
static int fr_alloc(ck_handle* h) {
    size_t m = (size_t)h->max_pubs;
    h->fr_max = h->max_pubs;
    CUDA_TRY(h, h->d_fr_items.reserve(m, h->stream));
    CUDA_TRY(h, h->d_fr_gkey.reserve(m, h->stream));
    CUDA_TRY(h, h->d_fr_idx.reserve(m, h->stream));
    CUDA_TRY(h, h->d_fr_head.reserve(m, h->stream));
    CUDA_TRY(h, h->d_fr_fstart.reserve(m, h->stream));
    CUDA_TRY(h, h->d_fr_gfirst.reserve(m, h->stream));
    CUDA_TRY(h, h->d_fr_ffirst.reserve(m, h->stream));
    CUDA_TRY(h, h->d_fr_size.reserve(m, h->stream));
    CUDA_TRY(h, h->d_fr_nlive.reserve(1, h->stream));
    CUDA_TRY(h, h->d_fr_gscan.reserve(m + 1, h->stream));
    CUDA_TRY(h, h->d_fr_S.reserve(m + 1, h->stream));
    CUDA_TRY(h, h->d_fr_F.reserve(m + 1, h->stream));
    CUDA_TRY(h, h->d_fr_R.reserve(m + 1, h->stream));
    CUDA_TRY(h, h->d_fr_tile.reserve(m / CK_SCAN_TILE + 2, h->stream));
    CUDA_TRY(h, h->d_fr_grand.reserve(1, h->stream));
    CUDA_TRY(h, h->d_fr_table.reserve(m, h->stream));
    CUDA_TRY(h, h->d_fr_o1.reserve(m + 1, h->stream));
    CUDA_TRY(h, h->d_fr_o2.reserve(m + 1, h->stream));
    CUDA_TRY(h, h->h_fr_info.reserve(3, h->stream));
    // first size of the frame buffer: every payload framed twice (a payload slot carries at most two publishes) plus the
    // record and frame overhead of a publish with an id of up to 40 bytes.  A pass that needs more grows it (ck_frames_size)
    return h->fr_cap ? 0 : fr_grow(h, 2 * h->max_out + 160ull * m + 4096);
}

// group -> split -> size -> table + headers -> write -> CRC over items[0..n) that a source kernel built (gkey: group keys of
// 6 * passes bits, all ones = not framed; passes 0: one group in the given order).  Queued only.
static int frame_write(ck_handle* h);
static int lz_compress(ck_handle* h);
static int frame_pass(ck_handle* h, u32 n, u32 passes, u32 excl, unsigned long long window, long long base_offset, long long ts) {
    h->fr_n = n; h->fr_info = false; h->fr_sized = false; h->fr_pass_codec = h->fr_codec; h->fr_pass_level = h->fr_level; h->fr_prod = h->prod;
    if (!n) return 0;
    if (h->fr_pass_codec && !h->fr_raw_cap && lz_grow(h, h->fr_cap)) return 1;
    if (h->fr_pass_codec && ck_lz_hc_depth[h->fr_pass_level])
        CUDA_TRY(h, h->d_fr_chain.reserve((size_t)h->num_sms * CK_LZ_HC_CTAS_PER_SM * CK_LZ_WARPS * CK_LZ_BLOCK, h->stream));
    const u32* order = nullptr;
    if (passes) {
        if (group_alloc(h)) return 1;
        ck_key_arr kf; kf.k = h->d_fr_gkey.p;
        if (group_sort(h, kf, n, CK_K_FRAME, passes, nullptr, &order, h->d_fr_o1.p, h->d_fr_o2.p)) return 1;
    }
    h->fr_order = order; h->fr_base = base_offset; h->fr_ts = ts;
    u32 nb = (n + 255) / 256;
    unsigned long long* tile = h->d_fr_tile.p; unsigned long long* grand = h->d_fr_grand.p;
    {
        KTimer t(h, CK_K_FRAME);
        CUDA_TRY(h, cudaMemsetAsync(h->d_fr_nlive.p, 0, sizeof(u32), h->stream));
        CKL(h) ck_fr_heads_kernel<<<nb, 256, 0, h->stream>>>(order, h->d_fr_gkey.p, n, excl, h->d_fr_head.p, h->d_fr_nlive.p);
        CUDA_TRY(h, cudaGetLastError());
    }
    if (run_scan(h, h->d_fr_head.p, n, h->d_fr_gscan.p, 0, tile, grand, CK_K_FRAME)) return 1;
    {
        KTimer t(h, CK_K_FRAME);
        CKL(h) ck_fr_first_kernel<<<nb, 256, 0, h->stream>>>(h->d_fr_head.p, h->d_fr_gscan.p, n, h->d_fr_gfirst.p);
        CKL(h) ck_fr_size_kernel<<<nb, 256, 0, h->stream>>>(order, h->d_fr_items.p, h->d_fr_head.p, h->d_fr_gscan.p, h->d_fr_gfirst.p, n, h->d_fr_nlive.p, h->d_fr_size.p);
        CUDA_TRY(h, cudaGetLastError());
    }
    if (run_scan(h, h->d_fr_size.p, n, h->d_fr_S.p, 0, tile, grand, CK_K_FRAME)) return 1;
    {
        KTimer t(h, CK_K_FRAME);
        CKL(h) ck_fr_split_kernel<<<nb, 256, 0, h->stream>>>(h->d_fr_head.p, h->d_fr_gscan.p, h->d_fr_gfirst.p, h->d_fr_S.p, n, h->d_fr_nlive.p, window, h->d_fr_fstart.p);
        CUDA_TRY(h, cudaGetLastError());
    }
    if (run_scan(h, h->d_fr_fstart.p, n, h->d_fr_F.p, 0, tile, grand, CK_K_FRAME)) return 1;
    {
        KTimer t(h, CK_K_FRAME);
        CKL(h) ck_fr_first_kernel<<<nb, 256, 0, h->stream>>>(h->d_fr_fstart.p, h->d_fr_F.p, n, h->d_fr_ffirst.p);
        CKL(h) ck_fr_size_kernel<<<nb, 256, 0, h->stream>>>(order, h->d_fr_items.p, h->d_fr_fstart.p, h->d_fr_F.p, h->d_fr_ffirst.p, n, h->d_fr_nlive.p, h->d_fr_size.p);
        CUDA_TRY(h, cudaGetLastError());
    }
    if (run_scan(h, h->d_fr_size.p, n, h->d_fr_R.p, 0, tile, grand, CK_K_FRAME)) return 1;
    if (frame_write(h)) return 1;
    // frames and bytes, copied back with the step's results (ck_frames_size reads them)
    CUDA_TRY(h, cudaMemcpyAsync(h->h_fr_info.p, h->d_fr_F.p + n, sizeof(long long), cudaMemcpyDeviceToHost, h->stream));
    CUDA_TRY(h, cudaMemcpyAsync(h->h_fr_info.p + 1, h->d_fr_R.p + n, sizeof(long long), cudaMemcpyDeviceToHost, h->stream));
    h->fr_info = true;
    return 0;
}

// the half of the pass that writes into the frame buffer: table + headers, records, CRC.  Everything it reads stays on the
// device until the next pass, so it runs again into a larger buffer when the frames did not fit.  An LZ4 pass writes the
// uncompressed frames into the scratch buffer and compresses them into the frame buffer before the CRC
static int frame_write(ck_handle* h) {
    u32 n = h->fr_n, nb = (n + 255) / 256;
    const u32* order = h->fr_order;
    bool lz = h->fr_pass_codec != 0;
    u8* dst = lz ? h->d_fr_raw.p : h->d_fr_frames.p;
    uint64_t cap = lz ? h->fr_raw_cap : h->fr_cap;
    {
        KTimer t(h, CK_K_FRAME);   // chunk counts per frame go to d_fr_head (free again), their scan to d_fr_S
        CKL(h) ck_fr_table_kernel<<<nb, 256, 0, h->stream>>>(order, h->d_fr_items.p, h->d_fr_ffirst.p, h->d_fr_F.p, h->d_fr_R.p, n, h->d_fr_nlive.p,
                                                          h->fr_base, h->fr_ts, h->fr_prod, cap, h->d_fr_table.p, dst, h->d_fr_head.p);
        CUDA_TRY(h, cudaGetLastError());
    }
    if (!lz && run_scan(h, h->d_fr_head.p, n, h->d_fr_S.p, 0, h->d_fr_tile.p, h->d_fr_grand.p, CK_K_FRAME)) return 1;
    {
        KTimer t(h, CK_K_FRAME);
        CKL(h) ck_fr_write_kernel<<<(n + 7) / 8, 256, 0, h->stream>>>(order, h->d_fr_items.p, h->d_fr_fstart.p, h->d_fr_F.p, h->d_fr_ffirst.p, h->d_fr_R.p, n,
                                                                   h->d_fr_nlive.p, cap, dst);
        CUDA_TRY(h, cudaGetLastError());
    }
    if (lz && lz_compress(h)) return 1;
    {
        KTimer t(h, CK_K_FRAME);
        u32 cblocks = (n + 7) / 8; if (cblocks > h->num_sms * 8) cblocks = h->num_sms * 8;
        CKL(h) ck_fr_crc_chunks_kernel<<<cblocks, 256, 0, h->stream>>>(h->d_fr_table.p, h->d_fr_S.p, h->d_fr_F.p, n, h->d_fr_frames.p, h->d_fr_partial.p);
        CKL(h) ck_fr_crc_fold_kernel<<<nb, 256, 0, h->stream>>>(h->d_fr_table.p, h->d_fr_S.p, h->d_fr_F.p, n, h->d_fr_partial.p, h->d_fr_frames.p);
        CUDA_TRY(h, cudaGetLastError());
    }
    return 0;
}

// the LZ4 stage (csrc/ck_kafka.cuh): the uncompressed frames in d_fr_raw -> compressed frames in the frame buffer, their
// table entries and CRC chunk counts (scan in d_fr_S); h_fr_info[2] = bytes of the compressed frames.  Block scan in
// d_fr_gscan and frame lengths in d_fr_size: the first half of the pass is done with both
static int lz_compress(ck_handle* h) {
    u32 n = h->fr_n, nb = (n + 255) / 256;
    u8* slots = h->d_fr_raw.p + h->fr_raw_cap + CK_PAD;
    {
        KTimer t(h, CK_K_LZ4);
        CKL(h) ck_lz_blocks_kernel<<<nb, 256, 0, h->stream>>>(h->d_fr_table.p, h->d_fr_F.p, n, h->fr_raw_cap, h->d_fr_head.p);
        CUDA_TRY(h, cudaGetLastError());
    }
    if (run_scan(h, h->d_fr_head.p, n, h->d_fr_gscan.p, 0, h->d_fr_tile.p, h->d_fr_grand.p, CK_K_LZ4)) return 1;
    {
        KTimer t(h, CK_K_LZ4);
        u32 depth = ck_lz_hc_depth[h->fr_pass_level];
        if (!depth) CKL(h) ck_lz_compress_kernel<<<h->num_sms * 8, CK_LZ_WARPS * 32, 0, h->stream>>>(h->d_fr_table.p, h->d_fr_gscan.p, h->d_fr_F.p, n,
                                                                                                  h->d_fr_raw.p, slots, h->fr_bmax, h->d_fr_bsize.p);
        else CKL(h) ck_lz_compress_hc_kernel<<<h->num_sms * CK_LZ_HC_CTAS_PER_SM, CK_LZ_WARPS * 32, 0, h->stream>>>(h->d_fr_table.p, h->d_fr_gscan.p,
            h->d_fr_F.p, n, h->d_fr_raw.p, slots, h->fr_bmax, h->d_fr_bsize.p, h->d_fr_chain.p, depth);
        CUDA_TRY(h, cudaGetLastError());
    }
    if (run_scan(h, h->d_fr_bsize.p, h->fr_bmax, h->d_fr_bscan.p, 0, h->d_fr_btile.p, h->d_fr_grand.p, CK_K_LZ4)) return 1;
    {
        KTimer t(h, CK_K_LZ4);
        CKL(h) ck_lz_size_kernel<<<nb, 256, 0, h->stream>>>(h->d_fr_gscan.p, h->d_fr_bscan.p, n, h->d_fr_size.p);
        CUDA_TRY(h, cudaGetLastError());
    }
    if (run_scan(h, h->d_fr_size.p, n, h->d_fr_zoff.p, 0, h->d_fr_tile.p, h->d_fr_grand.p, CK_K_LZ4)) return 1;
    {
        KTimer t(h, CK_K_LZ4);
        CKL(h) ck_lz_gather_kernel<<<h->num_sms * 8, 256, 0, h->stream>>>(h->d_fr_table.p, h->d_fr_gscan.p, h->d_fr_F.p, n, h->d_fr_bscan.p, h->d_fr_bsize.p,
                                                                         h->d_fr_zoff.p, h->d_fr_size.p, h->d_fr_raw.p, slots, h->fr_cap, h->d_fr_frames.p);
        CKL(h) ck_lz_head_kernel<<<nb, 256, 0, h->stream>>>(h->d_fr_table.p, h->d_fr_F.p, n, h->d_fr_zoff.p, h->d_fr_size.p, h->d_fr_raw.p, h->fr_cap,
                                                           h->d_fr_frames.p, h->d_fr_head.p);
        CUDA_TRY(h, cudaGetLastError());
    }
    if (run_scan(h, h->d_fr_head.p, n, h->d_fr_S.p, 0, h->d_fr_tile.p, h->d_fr_grand.p, CK_K_FRAME)) return 1;
    CUDA_TRY(h, cudaMemcpyAsync(h->h_fr_info.p + 2, h->d_fr_zoff.p + n, sizeof(long long), cudaMemcpyDeviceToHost, h->stream));
    return 0;
}

// bits of the group key for `groups` groups (all ones is the key of unframed slots)
static u32 fr_passes(unsigned long long groups) { u32 p = 1; while (p < 6 && groups >= (1ull << (6 * p)) - 1) p++; return p; }

extern "C" int ck_set_frame_topics(ck_handle* h, const int32_t* topic_ids, uint32_t n) {
    cudaSetDevice(h->device);
    int32_t top = -1;
    for (u32 i = 0; i < n; i++) { if (topic_ids[i] < 0) return fail(h, "ck_set_frame_topics: ids must be >= 0"); if (topic_ids[i] > top) top = topic_ids[i]; }
    std::vector<int32_t> slot((size_t)top + 1, -1);
    for (u32 i = 0; i < n; i++) if (slot[topic_ids[i]] < 0) slot[topic_ids[i]] = (int32_t)i;
    CUDA_TRY(h, cudaStreamSynchronize(h->stream));    // the passes queued so far may read the old table
    ck_buf<int32_t> d_slot;
    if (n) {
        CUDA_TRY(h, d_slot.reserve(slot.size(), h->stream));
        CUDA_TRY(h, cudaMemcpy(d_slot.p, slot.data(), sizeof(int32_t) * slot.size(), cudaMemcpyHostToDevice));
    }
    h->d_fr_slot = std::move(d_slot); h->fr_nslots = (u32)slot.size(); h->fr_ntopics = n;
    return 0;
}

// the live publishes of the current plan to the frame topics, grouped by (topic, partition), as frames: queued only
extern "C" int ck_encode_frames(ck_handle* h, int64_t timestamp_ms) {
    cudaSetDevice(h->device);
    if (!h->fr_ntopics) return fail(h, "ck_encode_frames: call ck_set_frame_topics first");
    unsigned long long groups = (unsigned long long)h->fr_ntopics * ((unsigned long long)h->num_partitions + 1);
    u32 passes = fr_passes(groups);
    if (passes > 5) return fail(h, "ck_encode_frames: more than 2^30 (topic, partition) groups");
    if (fr_alloc(h)) return 1;
    u32 n = h->n_pubs, excl = (u32)((1ull << (6 * passes)) - 1);
    {
        KTimer t(h, CK_K_FRAME);
        if (n) CKL(h) ck_fr_src_pubs_kernel<<<(n + 255) / 256, 256, 0, h->stream>>>(view_of(h), h->d_pubs.p, nullptr, n, h->d_pay_len.p, h->d_out_off.p, h->d_out.p,
            h->d_cols.p, h->n, h->d_fr_slot.p, h->fr_nslots, h->num_partitions, excl, h->fr_sticky.empty() ? nullptr : h->d_fr_sticky.p,
            (u32)h->fr_sticky.size(), h->d_fr_items.p, h->d_fr_gkey.p);
        CUDA_TRY(h, cudaGetLastError());
    }
    return frame_pass(h, n, passes, excl, h->fr_window, 0, timestamp_ms);
}

// the producer fields of the following passes' frames: flags 0 none (producerId / producerEpoch -1), CK_PRODUCER_IDEMPOTENT
// pid and epoch, | CK_PRODUCER_TRANSACTIONAL and attributes bit 4
extern "C" int ck_set_producer(ck_handle* h, int64_t pid, int16_t epoch, uint32_t flags) {
    if (flags & ~(u32)(CK_PRODUCER_IDEMPOTENT | CK_PRODUCER_TRANSACTIONAL)) return fail(h, "ck_set_producer: unknown flags");
    if (flags && !(flags & CK_PRODUCER_IDEMPOTENT)) return fail(h, "ck_set_producer: a transactional producer is idempotent");
    if (flags && (pid < 0 || epoch < 0)) return fail(h, "ck_set_producer: producer id and epoch must be >= 0");
    h->prod = flags ? ck_producer{(long long)pid, (int)epoch, (flags & CK_PRODUCER_TRANSACTIONAL) ? 0x10u : 0u} : ck_producer{-1, -1, 0};
    return 0;
}

// parts[topic id] for ids < n: the partition of the topic's unkeyed publishes in the following passes (-1: they stay the
// partition -1 group); n = 0 clears the table.  The copy is queued on the stream, ahead of the passes that read it
extern "C" int ck_set_sticky_partitions(ck_handle* h, const int32_t* parts, uint32_t n) {
    cudaSetDevice(h->device);
    for (u32 i = 0; i < n; i++)
        if (parts[i] < -1 || (parts[i] >= 0 && (u32)parts[i] >= h->num_partitions))
            return fail(h, "ck_set_sticky_partitions: a partition outside [0, num_partitions)");
    std::vector<int32_t> host(parts, parts + n);
    ck_buf<int32_t> grown;                             // a larger table replaces the old one once its copy is queued
    if (n > h->d_fr_sticky.cap) {
        CUDA_TRY(h, cudaStreamSynchronize(h->stream));    // the passes queued so far may read the old table
        CUDA_TRY(h, grown.reserve(n, h->stream));
    }
    if (n) CUDA_TRY(h, cudaMemcpyAsync(grown.p ? grown.p : h->d_fr_sticky.p, host.data(), sizeof(int32_t) * n, cudaMemcpyHostToDevice, h->stream));
    if (grown.p) h->d_fr_sticky = std::move(grown);
    h->fr_sticky = std::move(host);
    return 0;
}

// records a host path produced for one topic (host tools, the LLM boundary, declined records re-run on the host)
extern "C" int ck_encode_frames_records(ck_handle* h, int32_t topic_id, const uint8_t* host_blob, uint64_t nbytes, const int64_t* host_desc,
                                        uint32_t n, int64_t timestamp_ms) {
    cudaSetDevice(h->device);
    if (n > h->max_pubs) return fail(h, "ck_encode_frames_records: more records than the publish table holds");
    if (nbytes > h->max_in) return fail(h, "ck_encode_frames_records: records larger than max_in_bytes");
    for (u32 i = 0; i < n; i++) {
        const int64_t* d = host_desc + 6 * (size_t)i;
        for (int f = 0; f < 3; f++) {
            if (d[2 * f + 1] < (f ? -1 : 0) || (d[2 * f + 1] >= 0 && (d[2 * f] < 0 || (uint64_t)(d[2 * f] + d[2 * f + 1]) > nbytes)))
                return fail(h, "ck_encode_frames_records: span outside the records");
        }
    }
    u32 passes = fr_passes((unsigned long long)h->num_partitions + 1);
    if (passes > 5) return fail(h, "ck_encode_frames_records: too many partitions");
    if (fr_alloc(h)) return 1;
    CUDA_TRY(h, h->d_fr_blob.reserve(h->max_in + CK_PAD, h->stream));
    CUDA_TRY(h, h->d_fr_desc.reserve(6 * (size_t)h->max_pubs, h->stream));
    if (nbytes) CUDA_TRY(h, cudaMemcpyAsync(h->d_fr_blob.p, host_blob, nbytes, cudaMemcpyHostToDevice, h->stream));
    CUDA_TRY(h, cudaMemsetAsync(h->d_fr_blob.p + nbytes, 0, 16, h->stream));
    if (n) CUDA_TRY(h, cudaMemcpyAsync(h->d_fr_desc.p, host_desc, sizeof(long long) * 6 * (size_t)n, cudaMemcpyHostToDevice, h->stream));
    {
        KTimer t(h, CK_K_FRAME);
        int32_t sticky = topic_id >= 0 && (size_t)topic_id < h->fr_sticky.size() ? h->fr_sticky[topic_id] : -1;
        if (n) CKL(h) ck_fr_src_recs_kernel<<<(n + 255) / 256, 256, 0, h->stream>>>(h->d_fr_blob.p, h->d_fr_desc.p, n, topic_id, h->num_partitions,
                                                                                   sticky, h->d_fr_items.p, h->d_fr_gkey.p);
        CUDA_TRY(h, cudaGetLastError());
    }
    return frame_pass(h, n, passes, (u32)((1ull << (6 * passes)) - 1), h->fr_window, 0, timestamp_ms);
}

// bytes of the last pass's frames: uncompressed (as the table kernel lays them out) and as they go out
static uint64_t fr_raw_bytes(ck_handle* h) { return h->fr_info ? (uint64_t)(h->h_fr_info.p[1] + (long long)CK_RB_HEADER * h->h_fr_info.p[0]) : 0; }
static uint64_t fr_bytes(ck_handle* h) { return !h->fr_info ? 0 : h->fr_pass_codec ? (uint64_t)h->h_fr_info.p[2] : fr_raw_bytes(h); }

// frames and bytes of the last pass (waits for it).  Frames that did not fit the frame buffer (or, compressed, the scratch
// buffer of the uncompressed frames) are written again into buffers grown to their size (one more wait each): a step is
// sized for whatever its ids and payloads need
extern "C" int ck_frames_size(ck_handle* h, uint32_t* n_frames, uint64_t* nbytes) {
    cudaSetDevice(h->device);
    CUDA_TRY(h, cudaStreamSynchronize(h->stream));
    for (;;) {
        uint64_t raw = fr_raw_bytes(h), nb = fr_bytes(h);
        bool grow_raw = h->fr_pass_codec && raw > h->fr_raw_cap, grow = nb > h->fr_cap;
        if (!grow_raw && !grow) break;
        if (grow_raw && lz_grow(h, raw + raw / 8 + 4096)) return 1;
        if (grow && fr_grow(h, nb + nb / 8 + 4096)) return 1;
        if (frame_write(h)) return 1;
        CUDA_TRY(h, cudaStreamSynchronize(h->stream));
    }
    h->fr_sized = true;
    if (n_frames) *n_frames = h->fr_info ? (u32)h->h_fr_info.p[0] : 0u;
    if (nbytes) *nbytes = fr_bytes(h);
    return 0;
}

// copies of the frame table and the frames of the last pass, queued only: page-locked destinations, complete after the
// next ck_sync.  ck_frames_size must have been called since the pass (it gives the sizes and makes sure the frames fit)
extern "C" int ck_fetch_frames_async(ck_handle* h, ck_frame* host_table, uint32_t table_cap, uint8_t* host_frames, uint64_t cap) {
    cudaSetDevice(h->device);
    if (h->fr_info && !h->fr_sized) return fail(h, "ck_fetch_frames_async: call ck_frames_size after the frame pass first");
    uint64_t nf = h->fr_info ? (uint64_t)h->h_fr_info.p[0] : 0, nb = fr_bytes(h);
    if (nb > h->fr_cap) return fail(h, "ck_fetch_frames_async: frames larger than the frame buffer");
    if (nf > table_cap || nb > cap) return fail(h, "ck_fetch_frames_async: host buffers too small");
    if (nf) CUDA_TRY(h, cudaMemcpyAsync(host_table, h->d_fr_table.p, sizeof(ck_frame) * (size_t)nf, cudaMemcpyDeviceToHost, h->stream));
    if (nb) CUDA_TRY(h, cudaMemcpyAsync(host_frames, h->d_fr_frames.p, (size_t)nb, cudaMemcpyDeviceToHost, h->stream));
    return 0;
}

// produce side, one topic-partition: the publishes host_idx[0..n) of the current plan (in send order) become ONE frame —
// the frame pass with one group, offsetDelta = position in the list — copied to host_frame (waits)
extern "C" int ck_encode_recordbatch(ck_handle* h, const uint32_t* host_idx, uint32_t n, int64_t base_offset, int64_t timestamp_ms,
                                     uint8_t* host_frame, uint64_t cap, uint64_t* frame_len) {
    cudaSetDevice(h->device);
    if (!n || n > h->n_pubs) return fail(h, "ck_encode_recordbatch: index list empty or longer than the publish table");
    if (fr_alloc(h)) return 1;
    CUDA_TRY(h, cudaMemcpyAsync(h->d_fr_idx.p, host_idx, sizeof(u32) * n, cudaMemcpyHostToDevice, h->stream));
    {
        KTimer t(h, CK_K_FRAME);
        CKL(h) ck_fr_src_pubs_kernel<<<(n + 255) / 256, 256, 0, h->stream>>>(view_of(h), h->d_pubs.p, h->d_fr_idx.p, n, h->d_pay_len.p, h->d_out_off.p, h->d_out.p,
            h->d_cols.p, h->n, nullptr, 0, 0, CK_RB_NONE, nullptr, 0, h->d_fr_items.p, h->d_fr_gkey.p);
        CUDA_TRY(h, cudaGetLastError());
    }
    if (frame_pass(h, n, 0, CK_RB_NONE, ~0ull, base_offset, timestamp_ms)) return 1;
    uint32_t nf = 0; uint64_t total = 0;
    if (ck_frames_size(h, &nf, &total)) return 1;
    if (nf != 1) return fail(h, "ck_encode_recordbatch: the index list holds no live publish");
    if (total > cap) return fail(h, "ck_encode_recordbatch: host buffer too small");
    CUDA_TRY(h, cudaMemcpyAsync(host_frame, h->d_fr_frames.p, total, cudaMemcpyDeviceToHost, h->stream));
    CUDA_TRY(h, cudaStreamSynchronize(h->stream));
    if (frame_len) *frame_len = total;
    return 0;
}

// ---- aggregation gate (csrc/ck_gate.cuh) ------------------------------------------------------------------------------
extern "C" int ck_gate_create(ck_handle* h, uint32_t max_entries, uint32_t max_slots, uint64_t arena_bytes) {
    cudaSetDevice(h->device);
    if (h->gate_set) return fail(h, "ck_gate_create: already created");
    if (arena_bytes >= (1ull << 32)) return fail(h, "ck_gate_create: arena must be smaller than 4 GiB (32-bit segment offsets)");
    if (max_entries == 0 || max_entries > (1u << 28)) return fail(h, "ck_gate_create: max_entries must be in [1, 2^28]");
    u32 cap = 64; while (cap < 4 * (uint64_t)max_entries) cap <<= 1;
    ck_gate_bufs b;
    CUDA_TRY(h, b.keys.reserve(cap, h->stream));
    CUDA_TRY(h, b.ctr.reserve(8, h->stream));
    // two sets of entries, slots and arena for ck_gate_compact: the gate holds twice what it is sized for
    for (int k = 0; k < 2; k++) {
        CUDA_TRY(h, b.entries[k].reserve((size_t)max_entries, h->stream));
        CUDA_TRY(h, b.slots[k].reserve((size_t)max_slots, h->stream));
        CUDA_TRY(h, b.arena[k].reserve(arena_bytes + CK_PAD, h->stream));
    }
    CUDA_TRY(h, b.src.reserve((size_t)max_entries, h->stream));
    CUDA_TRY(h, b.rec_entry.reserve((size_t)h->max_records, h->stream));
    CUDA_TRY(h, cudaMemsetAsync(b.keys.p, 0, sizeof(unsigned long long) * cap, h->stream));
    CUDA_TRY(h, cudaMemsetAsync(b.ctr.p, 0, sizeof(unsigned long long) * 8, h->stream));
    CUDA_TRY(h, cudaStreamSynchronize(h->stream));
    ck_gate g{};
    g.keys = b.keys.p; g.cap = cap; g.max_entries = max_entries; g.max_slots = max_slots; g.arena_cap = arena_bytes; g.ctr = b.ctr.p;
    ck_gate s = g;
    g.entries = b.entries[0].p; g.slots = b.slots[0].p; g.arena = b.arena[0].p;
    s.entries = b.entries[1].p; s.slots = b.slots[1].p; s.arena = b.arena[1].p;
    h->gate_bufs = std::move(b); h->gate = g; h->gate_spare = s; h->gate_set = true;
    return 0;
}

extern "C" int ck_gate_reset(ck_handle* h) {
    cudaSetDevice(h->device);
    if (!h->gate_set) return fail(h, "ck_gate_reset: call ck_gate_create first");
    CUDA_TRY(h, cudaMemsetAsync(h->gate.keys, 0, sizeof(unsigned long long) * h->gate.cap, h->stream));
    CUDA_TRY(h, cudaMemsetAsync(h->gate.ctr, 0, sizeof(unsigned long long) * 8, h->stream));
    return 0;
}

// give back what finished fan-outs used: the live entries (with their slots, blobs and collected values) move to the
// spare buffers, which become the gate's, and the key table is rebuilt from them.  Asynchronous; the pending state
// and every later result are exactly what they would have been without it.
extern "C" int ck_gate_compact(ck_handle* h) {
    cudaSetDevice(h->device);
    if (!h->gate_set) return fail(h, "ck_gate_compact: call ck_gate_create first");
    ck_gate g = h->gate, d = h->gate_spare;
    CUDA_TRY(h, cudaMemsetAsync(g.keys, 0, sizeof(unsigned long long) * g.cap, h->stream));
    CKL(h) ck_gate_compact_plan_kernel<<<1, 1024, 0, h->stream>>>(g, d, h->gate_bufs.src.p);
    CKL(h) ck_gate_compact_move_kernel<<<(g.max_entries + 7) / 8, 256, 0, h->stream>>>(g, d, h->gate_bufs.src.p);
    CUDA_TRY(h, cudaGetLastError());
    h->gate = d; h->gate_spare = g;
    return 0;
}

extern "C" int ck_gate_stats(ck_handle* h, uint64_t* out5) {
    cudaSetDevice(h->device);
    if (!h->gate_set) return fail(h, "ck_gate_stats: call ck_gate_create first");
    CUDA_TRY(h, cudaMemcpyAsync(out5, h->gate.ctr, sizeof(unsigned long long) * 5, cudaMemcpyDeviceToHost, h->stream));
    CUDA_TRY(h, cudaStreamSynchronize(h->stream));
    return 0;
}

// after ck_fanout_plan on a batch of post-LLM envelopes: every record that went out as list[Call] becomes a pending entry
extern "C" int ck_gate_register(ck_handle* h, uint32_t min_pending) {
    cudaSetDevice(h->device);
    if (!h->gate_set) return fail(h, "ck_gate_register: call ck_gate_create first");
    u32 n = h->n;
    CUDA_TRY(h, cudaMemsetAsync(h->gate.ctr + 4, 0, sizeof(unsigned long long), h->stream));   // failures of this call
    if (!n) return 0;
    KTimer t(h, CK_K_FANOUT);
    CKL(h) ck_gate_register_kernel<<<(n + 127) / 128, 128, 0, h->stream>>>(view_of(h), n, h->d_cols.p, n, h->gate, min_pending,
                                                                              h->gate_reg_seq, h->gate_bufs.rec_entry.p);
    h->gate_reg_seq += n;
    CKL(h) ck_gate_copy_base_kernel<<<(n + 7) / 8, 256, 0, h->stream>>>(view_of(h), n, h->gate, h->gate_bufs.rec_entry.p);
    CUDA_TRY(h, cudaGetLastError());
    return 0;
}

// a batch of records arriving at the agent's topic: probe -> resolve -> merge -> encode.  Per record (column ACTION):
// CK_ACT_SILENT (collected, set still incomplete: only the handler-return publish), CK_ACT_GATE_COMPLETE (payload i = the
// envelope carrying base_state + collected results), CK_ACT_GATE_PASS (no pending fan-out: continue with the inbound state).
extern "C" int ck_gate_arrive(ck_handle* h, uint64_t stamp_base) {
    cudaSetDevice(h->device);
    if (!h->gate_set) return fail(h, "ck_gate_arrive: call ck_gate_create first");
    if (!h->tool_set) return fail(h, "ck_gate_arrive: call ck_set_tool_node (publish topic) first");
    u32 n = h->n;
    CUDA_TRY(h, cudaMemsetAsync(h->gate.ctr + 4, 0, sizeof(unsigned long long), h->stream));   // failures of this call
    {
        KTimer t(h, CK_K_PLAN);
        if (n) {
            CKL(h) ck_gate_probe_kernel<<<(n + 127) / 128, 128, 0, h->stream>>>(view_of(h), n, h->d_cols.p, n, h->gate, stamp_base, h->gate_bufs.rec_entry.p);
            CKL(h) ck_gate_resolve_kernel<<<(n + 127) / 128, 128, 0, h->stream>>>(view_of(h), n, h->d_cols.p, n, h->gate, stamp_base, h->gate_bufs.rec_entry.p,
                h->h_tool_cfg.publish_topic_id, h->d_glue.p, h->d_descs.p, h->d_pay_len.p, h->d_pubs.p);
            CKL(h) ck_gate_merge_kernel<<<(n + 3) / 4, 128, 0, h->stream>>>(view_of(h), n, h->d_cols.p, n, h->gate, h->gate_bufs.rec_entry.p, h->d_glue.p, h->d_descs.p, h->d_pay_len.p);
        }
        CUDA_TRY(h, cudaGetLastError());
    }
    if (scan_emit(h, n, h->gate.arena)) return 1;
    h->n_pubs = 2 * n;
    return 0;
}

// ---- cross-partition forward over peer memory (csrc/ck_xsend.cuh) --------------------------------------------------------
static int x_alloc(ck_handle* h) {
    u32 nb_max = (h->max_pubs + CK_X_BLOCK - 1) / CK_X_BLOCK;
    size_t nh = (size_t)CK_X_MAXWORLD * nb_max;
    CUDA_TRY(h, h->d_x_hist.reserve(nh, h->stream));
    CUDA_TRY(h, h->d_x_base.reserve(nh + 1, h->stream));
    CUDA_TRY(h, h->d_x_nbytes.reserve(CK_X_MAXWORLD, h->stream));
    CUDA_TRY(h, h->d_x_src_off.reserve((size_t)h->max_pubs + 1, h->stream));
    CUDA_TRY(h, h->d_x_len.reserve((size_t)h->max_pubs + 1, h->stream));
    CUDA_TRY(h, h->d_x_dst_off.reserve((size_t)h->max_pubs + 1, h->stream));
    CUDA_TRY(h, h->d_x_len32.reserve((size_t)h->max_pubs + 1, h->stream));
    CUDA_TRY(h, h->d_x_pub.reserve((size_t)h->max_pubs + 1, h->stream));
    size_t nt = (nh > h->max_pubs ? nh : h->max_pubs) / CK_SCAN_TILE + 2;
    CUDA_TRY(h, h->d_x_tile.reserve(nt, h->stream));
    CUDA_TRY(h, h->d_x_grand.reserve(1, h->stream));
    CUDA_TRY(h, h->d_x_grand2.reserve(1, h->stream));
    CUDA_TRY(h, h->h_x.reserve(2 * CK_X_MAXWORLD + 2, h->stream));
    return 0;
}

// receive buffer of this rank: `world` regions (one per source rank), each max_fwd meta entries + data_cap payload bytes.
// ipc_handle_out (64 bytes): give it to every peer (any side channel: the Python binding all-gathers it).
extern "C" int ck_comm_create(ck_handle* h, uint32_t rank, uint32_t world, uint32_t max_fwd, uint64_t data_cap, uint8_t* ipc_handle_out) {
    cudaSetDevice(h->device);
    if (world < 1 || world > CK_X_MAXWORLD || rank >= world) return fail(h, "ck_comm_create: world must be 1..16 and rank < world");
    if (h->d_recv.p) return fail(h, "ck_comm_create: already created");
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "ipc handle size");
    unsigned long long data = (data_cap + 15) & ~15ull;
    unsigned long long stride = (CK_X_HDR + (unsigned long long)max_fwd * sizeof(ck_xmeta) + data + 255) & ~255ull;
    ck_buf<u8> recv; ck_buf<u32> overflow;
    CUDA_TRY(h, recv.reserve(stride * world + CK_X_FLAGS_BYTES + CK_PAD, h->stream));
    CUDA_TRY(h, cudaMemset(recv.p, 0, stride * world + CK_X_FLAGS_BYTES));
    CUDA_TRY(h, overflow.reserve(CK_X_MAXWORLD + 1, h->stream));
    CUDA_TRY(h, cudaMemset(overflow.p, 0, sizeof(u32) * (CK_X_MAXWORLD + 1)));     // [world]: barrier timeout flag
    cudaIpcMemHandle_t ih;
    CUDA_TRY(h, cudaIpcGetMemHandle(&ih, recv.p));
    // the exchange is a dozen small dependent kernels: on a highest-priority stream their blocks are scheduled as soon as
    // any SM slot frees up instead of queueing behind the other lane's million-record kernels
    int lo = 0, hi = 0;
    CUDA_TRY(h, cudaDeviceGetStreamPriorityRange(&lo, &hi));
    cudaStream_t xs = nullptr; cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    cudaError_t stream_err = cudaStreamCreateWithPriority(&xs, cudaStreamNonBlocking, hi);
    if (stream_err == cudaSuccess) stream_err = cudaEventCreateWithFlags(&ev0, cudaEventDisableTiming);
    if (stream_err == cudaSuccess) stream_err = cudaEventCreateWithFlags(&ev1, cudaEventDisableTiming);
    if (stream_err != cudaSuccess) {
        if (ev0) cudaEventDestroy(ev0);
        if (xs) cudaStreamDestroy(xs);
        CUDA_TRY(h, stream_err);
    }
    memcpy(ipc_handle_out, &ih, 64);
    h->comm_rank = rank; h->comm_world = world; h->max_fwd = max_fwd; h->region_data_cap = data; h->region_stride = stride;
    h->d_recv = std::move(recv); h->d_x_overflow = std::move(overflow); h->xstream = xs; h->x_ev0 = ev0; h->x_ev1 = ev1;
    return 0;
}

// handles[world][64]: every rank's ck_comm_create output, in rank order (this rank's own entry is ignored)
extern "C" int ck_comm_connect(ck_handle* h, const uint8_t* handles) {
    cudaSetDevice(h->device);
    if (!h->d_recv.p) return fail(h, "ck_comm_connect: call ck_comm_create first");
    for (u32 d = 0; d < h->comm_world; d++) {
        if (d == h->comm_rank) { h->peers.recv[d] = h->d_recv.p; continue; }
        cudaIpcMemHandle_t ih; memcpy(&ih, handles + 64 * (size_t)d, 64);
        void* p = nullptr;
        CUDA_TRY(h, cudaIpcOpenMemHandle(&p, ih, cudaIpcMemLazyEnablePeerAccess));
        h->peer_opened[d] = p; h->peers.recv[d] = (u8*)p;
    }
    h->comm_ready = true;
    return 0;
}

// plan + pack + transfer of the keyed publishes of the current plan whose partition another rank owns: queued on the
// handle's stream, no host synchronisation.  The caller brackets it with two barriers (peers consumed the previous
// contents / every peer's stores have landed).
static int exchange_send_on_stream(ck_handle* h, uint64_t step);
extern "C" int ck_exchange_send(ck_handle* h, uint64_t step) {
    cudaSetDevice(h->device);
    if (!h->comm_ready) return fail(h, "ck_exchange_send: call ck_comm_create / ck_comm_connect first");
    if (x_alloc(h)) return 1;
    // fork: everything below runs on the high-priority side stream, after what is queued on the handle's stream so far
    CUDA_TRY(h, cudaEventRecord(h->x_ev0, h->stream));
    CUDA_TRY(h, cudaStreamWaitEvent(h->xstream, h->x_ev0, 0));
    cudaStream_t main_stream = h->stream;
    h->stream = h->xstream;
    int rc = exchange_send_on_stream(h, step);
    h->stream = main_stream;
    if (rc) return rc;
    CUDA_TRY(h, cudaEventRecord(h->x_ev1, h->xstream));                  // join
    CUDA_TRY(h, cudaStreamWaitEvent(h->stream, h->x_ev1, 0));
    return 0;
}

static int exchange_send_on_stream(ck_handle* h, uint64_t step) {
    u32 rank = h->comm_rank, world = h->comm_world, npubs = h->n_pubs;
    u32 nb = (npubs + CK_X_BLOCK - 1) / CK_X_BLOCK;
    if (!nb) nb = 1;
    h->x_nb = nb;
    u32 nh = world * nb;
    {
        KTimer t(h, CK_K_ROUTE);
        CUDA_TRY(h, cudaMemsetAsync(h->d_x_nbytes.p, 0, sizeof(unsigned long long) * CK_X_MAXWORLD, h->stream));
        CKL(h) ck_xplan_count_kernel<<<nb, CK_X_BLOCK, 0, h->stream>>>(h->d_pubs.p, npubs, h->d_pay_len.p, rank, world, h->d_x_hist.p, h->d_x_nbytes.p);
        CUDA_TRY(h, cudaGetLastError());
    }
    if (run_scan(h, h->d_x_hist.p, nh, h->d_x_base.p, 0, h->d_x_tile.p, h->d_x_grand.p)) return 1;       // d_x_grand = payloads selected
    {
        KTimer t(h, CK_K_ROUTE);
        CUDA_TRY(h, cudaMemsetAsync(h->d_x_len32.p, 0, sizeof(u32) * ((size_t)npubs + 1), h->stream));
        CKL(h) ck_xplan_scatter_kernel<<<nb, CK_X_BLOCK, 0, h->stream>>>(h->d_pubs.p, npubs, h->d_pay_len.p, h->d_out_off.p, rank, world, h->d_x_base.p,
                                                                  h->d_x_src_off.p, h->d_x_len.p, h->d_x_len32.p, h->d_x_pub.p);
        CUDA_TRY(h, cudaGetLastError());
    }
    // byte offsets of the (16-byte padded) payloads in destination order; scanned over all publish slots so that the
    // launch does not need the selected count on the host (unselected tail entries are zero)
    if (run_scan(h, h->d_x_len32.p, npubs ? npubs : 1, h->d_x_dst_off.p, 15, h->d_x_tile.p, h->d_x_grand2.p)) return 1;
    unsigned long long flags_off = h->region_stride * world;
    {
        KTimer t(h, CK_K_EMIT);
        // barrier 1: every peer has consumed what it received last time (its own stream order puts that before this point)
        CKL(h) ck_xbarrier_kernel<<<1, 32, 0, h->stream>>>(h->peers, rank, world, flags_off, 0, step, h->d_x_overflow.p + CK_X_MAXWORLD);
        if (npubs) CKL(h) ck_xsend_kernel<<<h->num_sms * 4, 256, 0, h->stream>>>(h->d_pubs.p, h->d_x_pub.p, h->d_x_src_off.p, h->d_x_len32.p, h->d_x_dst_off.p, h->d_x_base.p, nb,
            h->d_x_grand.p, h->d_out.p, h->peers, rank, world, h->region_stride, h->max_fwd, h->region_data_cap, h->d_x_overflow.p);
        CKL(h) ck_xhdr_kernel<<<1, 32, 0, h->stream>>>(h->d_x_dst_off.p, h->d_x_base.p, nb, h->d_x_grand.p, h->peers, rank, world, h->region_stride, step, h->d_x_overflow.p);
        // barrier 2: everybody's stores (to everybody) have landed
        CKL(h) ck_xbarrier_kernel<<<1, 32, 0, h->stream>>>(h->peers, rank, world, flags_off, 1, step, h->d_x_overflow.p + CK_X_MAXWORLD);
        CUDA_TRY(h, cudaGetLastError());
    }
    return 0;
}

// what this rank received (after the caller's closing barrier): per source rank the header {step, count, overflow, bytes};
// ck_recv_buffer gives the device address and layout for in-place use, ck_fetch_received copies region `src` to the host
extern "C" int ck_recv_info(ck_handle* h, void** dev_recv, uint64_t* region_stride, uint32_t* max_fwd, uint64_t* data_cap) {
    if (!h->d_recv.p) return fail(h, "ck_recv_info: call ck_comm_create first");
    if (dev_recv) *dev_recv = h->d_recv.p;
    if (region_stride) *region_stride = h->region_stride;
    if (max_fwd) *max_fwd = h->max_fwd;
    if (data_cap) *data_cap = h->region_data_cap;
    return 0;
}
extern "C" int ck_fetch_received(ck_handle* h, uint32_t src, uint64_t* hdr4 /* step, count, overflow, nbytes */, uint8_t* host_meta, uint8_t* host_data, uint64_t data_cap) {
    cudaSetDevice(h->device);
    if (!h->d_recv.p || src >= h->comm_world) return fail(h, "ck_fetch_received: no such region");
    const u8* region = h->d_recv.p + (size_t)src * h->region_stride;
    ck_xregion_hdr hd{};
    CUDA_TRY(h, cudaMemcpyAsync(&hd, region, sizeof hd, cudaMemcpyDeviceToHost, h->stream));
    CUDA_TRY(h, cudaStreamSynchronize(h->stream));
    hdr4[0] = hd.step; hdr4[1] = hd.count; hdr4[2] = hd.overflow; hdr4[3] = hd.nbytes;
    { u32 to = 0; CUDA_TRY(h, cudaMemcpy(&to, h->d_x_overflow.p + CK_X_MAXWORLD, sizeof to, cudaMemcpyDeviceToHost)); if (to) return fail(h, "exchange barrier timed out: a peer did not arrive"); }
    if (hd.nbytes > data_cap) return fail(h, "ck_fetch_received: host buffer too small");
    if (host_meta && hd.count) CUDA_TRY(h, cudaMemcpyAsync(host_meta, region + CK_X_HDR, sizeof(ck_xmeta) * (size_t)hd.count, cudaMemcpyDeviceToHost, h->stream));
    if (host_data && hd.nbytes) CUDA_TRY(h, cudaMemcpyAsync(host_data, region + CK_X_HDR + (size_t)h->max_fwd * sizeof(ck_xmeta), hd.nbytes, cudaMemcpyDeviceToHost, h->stream));
    CUDA_TRY(h, cudaStreamSynchronize(h->stream));
    return 0;
}

// the pipelined form: ck_peek_received reads every region header with one small copy (one synchronisation of the engine's
// stream, which the caller has normally just done anyway), ck_fetch_received_async queues the copies of one region into
// page-locked memory and returns; they are complete after the next ck_sync
extern "C" int ck_peek_received(ck_handle* h, uint64_t* hdr4 /* [world][4]: step, count, overflow, nbytes */) {
    cudaSetDevice(h->device);
    if (!h->d_recv.p) return fail(h, "ck_peek_received: call ck_comm_create first");
    ck_xregion_hdr hd[CK_X_MAXWORLD];
    CUDA_TRY(h, cudaMemcpy2DAsync(hd, sizeof(ck_xregion_hdr), h->d_recv.p, h->region_stride, sizeof(ck_xregion_hdr), h->comm_world,
                                  cudaMemcpyDeviceToHost, h->stream));
    u32 to = 0;
    CUDA_TRY(h, cudaMemcpyAsync(&to, h->d_x_overflow.p + CK_X_MAXWORLD, sizeof to, cudaMemcpyDeviceToHost, h->stream));
    CUDA_TRY(h, cudaStreamSynchronize(h->stream));
    if (to) return fail(h, "exchange barrier timed out: a peer did not arrive");
    for (u32 r = 0; r < h->comm_world; r++) {
        hdr4[4 * r] = hd[r].step; hdr4[4 * r + 1] = hd[r].count; hdr4[4 * r + 2] = hd[r].overflow; hdr4[4 * r + 3] = hd[r].nbytes;
    }
    return 0;
}
extern "C" int ck_fetch_received_async(ck_handle* h, uint32_t src, uint64_t count, uint64_t nbytes, uint8_t* host_meta, uint8_t* host_data) {
    cudaSetDevice(h->device);
    if (!h->d_recv.p || src >= h->comm_world) return fail(h, "ck_fetch_received_async: no such region");
    if (count > h->max_fwd || nbytes > h->region_data_cap) return fail(h, "ck_fetch_received_async: count / nbytes beyond the region");
    const u8* region = h->d_recv.p + (size_t)src * h->region_stride;
    if (host_meta && count) CUDA_TRY(h, cudaMemcpyAsync(host_meta, region + CK_X_HDR, sizeof(ck_xmeta) * (size_t)count, cudaMemcpyDeviceToHost, h->stream));
    if (host_data && nbytes) CUDA_TRY(h, cudaMemcpyAsync(host_data, region + CK_X_HDR + (size_t)h->max_fwd * sizeof(ck_xmeta), nbytes, cudaMemcpyDeviceToHost, h->stream));
    return 0;
}

// multi-GPU exchange planning: see ck_xplan_*_kernel.  One host synchronisation (the all-to-all needs the split
// sizes on the host); the scatter and the offset scan are queued behind it.
extern "C" int ck_exchange_plan(ck_handle* h, uint32_t rank, uint32_t world, const int64_t** dev_src_off, const int64_t** dev_len,
                                const int64_t** dev_dst_off, const uint32_t** dev_pub, int64_t* host_counts, int64_t* host_nbytes,
                                uint32_t* n_sel) {
    cudaSetDevice(h->device);
    if (world < 1 || world > CK_X_MAXWORLD || rank >= world) return fail(h, "ck_exchange_plan: world must be 1..16 and rank < world");
    if (x_alloc(h)) return 1;
    u32 npubs = h->n_pubs;
    u32 nb = (npubs + CK_X_BLOCK - 1) / CK_X_BLOCK;
    for (u32 d = 0; d < world; d++) { host_counts[d] = 0; host_nbytes[d] = 0; }
    *n_sel = 0;
    if (dev_src_off) *dev_src_off = (const int64_t*)h->d_x_src_off.p;
    if (dev_len) *dev_len = (const int64_t*)h->d_x_len.p;
    if (dev_dst_off) *dev_dst_off = (const int64_t*)h->d_x_dst_off.p;
    if (dev_pub) *dev_pub = h->d_x_pub.p;
    if (!nb) return 0;
    u32 nh = world * nb;
    {
        KTimer t(h, CK_K_ROUTE);
        CUDA_TRY(h, cudaMemsetAsync(h->d_x_nbytes.p, 0, sizeof(unsigned long long) * CK_X_MAXWORLD, h->stream));
        CKL(h) ck_xplan_count_kernel<<<nb, CK_X_BLOCK, 0, h->stream>>>(h->d_pubs.p, npubs, h->d_pay_len.p, rank, world, h->d_x_hist.p, h->d_x_nbytes.p);
        CUDA_TRY(h, cudaGetLastError());
    }
    if (run_scan(h, h->d_x_hist.p, nh, h->d_x_base.p, 0, h->d_x_tile.p, h->d_x_grand.p)) return 1;
    // first slot of every destination (= base[d * nb]), the total, and the bytes per destination
    CUDA_TRY(h, cudaMemcpy2DAsync(h->h_x.p, sizeof(long long), h->d_x_base.p, sizeof(long long) * nb, sizeof(long long), world,
                                  cudaMemcpyDeviceToHost, h->stream));
    CUDA_TRY(h, cudaMemcpyAsync(h->h_x.p + CK_X_MAXWORLD, h->d_x_nbytes.p, sizeof(long long) * world, cudaMemcpyDeviceToHost, h->stream));
    CUDA_TRY(h, cudaMemcpyAsync(h->h_x.p + 2 * CK_X_MAXWORLD, h->d_x_grand.p, sizeof(long long), cudaMemcpyDeviceToHost, h->stream));
    CUDA_TRY(h, cudaStreamSynchronize(h->stream));
    long long total = h->h_x.p[2 * CK_X_MAXWORLD];
    for (u32 d = 0; d < world; d++) {
        long long next = d + 1 < world ? h->h_x.p[d + 1] : total;
        host_counts[d] = next - h->h_x.p[d];
        host_nbytes[d] = h->h_x.p[CK_X_MAXWORLD + d];
    }
    *n_sel = (u32)total;
    {
        KTimer t(h, CK_K_ROUTE);
        CKL(h) ck_xplan_scatter_kernel<<<nb, CK_X_BLOCK, 0, h->stream>>>(h->d_pubs.p, npubs, h->d_pay_len.p, h->d_out_off.p, rank, world, h->d_x_base.p,
                                                                  h->d_x_src_off.p, h->d_x_len.p, h->d_x_len32.p, h->d_x_pub.p);
        CUDA_TRY(h, cudaGetLastError());
    }
    if (total && run_scan(h, h->d_x_len32.p, (u32)total, h->d_x_dst_off.p, 0, h->d_x_tile.p, h->d_x_grand.p)) return 1;
    return 0;
}

extern "C" uint64_t ck_launch_count(ck_handle* h) { return h->n_launch; }

extern "C" int ck_sync(ck_handle* h) {
    cudaSetDevice(h->device);
    CUDA_TRY(h, cudaStreamSynchronize(h->stream));
    return 0;
}

extern "C" int ck_out_size(ck_handle* h, uint64_t* out_bytes, uint32_t* n_payloads, uint32_t* n_publishes) {
    cudaSetDevice(h->device);
    *h->h_grand.p = 0;
    if (h->n_payloads) {
        CUDA_TRY(h, cudaMemcpyAsync(h->h_grand.p, h->d_grand.p, sizeof(unsigned long long), cudaMemcpyDeviceToHost, h->stream));
    }
    CUDA_TRY(h, cudaStreamSynchronize(h->stream));
    if (out_bytes) *out_bytes = *h->h_grand.p;
    if (n_payloads) *n_payloads = h->n_payloads;
    if (n_publishes) *n_publishes = h->n_pubs;
    return 0;
}

extern "C" int ck_fetch_columns(ck_handle* h, uint32_t* host_cols) {
    cudaSetDevice(h->device);
    CUDA_TRY(h, cudaMemcpyAsync(host_cols, h->d_cols.p, sizeof(u32) * (size_t)CK_NUM_COLS * h->n, cudaMemcpyDeviceToHost, h->stream));
    CUDA_TRY(h, cudaStreamSynchronize(h->stream));
    return 0;
}

// selected column rows only (a worker needs status / action / the key span, not all 55 columns of a million records)
static int fetch_cols_impl(ck_handle* h, const uint32_t* which, uint32_t k, uint32_t* host_rows, bool wait);
extern "C" int ck_fetch_cols(ck_handle* h, const uint32_t* which, uint32_t k, uint32_t* host_rows) { return fetch_cols_impl(h, which, k, host_rows, true); }
extern "C" int ck_fetch_cols_async(ck_handle* h, const uint32_t* which, uint32_t k, uint32_t* host_rows) { return fetch_cols_impl(h, which, k, host_rows, false); }
static int fetch_cols_impl(ck_handle* h, const uint32_t* which, uint32_t k, uint32_t* host_rows, bool wait) {
    cudaSetDevice(h->device);
    for (uint32_t j = 0; j < k; j++) {
        if (which[j] >= CK_NUM_COLS) return fail(h, "ck_fetch_cols: no such column");
        if (h->n) CUDA_TRY(h, cudaMemcpyAsync(host_rows + (size_t)j * h->n, h->d_cols.p + (size_t)which[j] * h->n, sizeof(u32) * (size_t)h->n,
                                             cudaMemcpyDeviceToHost, h->stream));
    }
    if (wait) CUDA_TRY(h, cudaStreamSynchronize(h->stream));
    return 0;
}

// how many records of the current batch went through the canonicaliser pass, and the overlay bytes it produced (waits)
extern "C" int ck_canon_stats(ck_handle* h, uint32_t* n_listed, uint64_t* overlay_bytes) {
    cudaSetDevice(h->device);
    ck_canon_ctl c{};
    if (h->n) CUDA_TRY(h, cudaMemcpyAsync(&c, h->d_canon_ctl.p, sizeof c, cudaMemcpyDeviceToHost, h->stream));
    CUDA_TRY(h, cudaStreamSynchronize(h->stream));
    if (n_listed) *n_listed = c.count;
    if (overlay_bytes) *overlay_bytes = c.cursor;
    return 0;
}

// page-locked host memory for the batch arenas (calfkit/engine/lane.py): what cudaMemcpyAsync needs to overlap the
// two PCIe directions with the kernels
extern "C" int ck_host_alloc(uint64_t bytes, void** out) {
    *out = nullptr;
    cudaError_t e = cudaHostAlloc(out, bytes ? bytes : 1, cudaHostAllocPortable);
    if (e != cudaSuccess) { g_create_error = std::string("ck_host_alloc: ") + cudaGetErrorString(e); return 1; }
    return 0;
}
extern "C" void ck_host_free(void* p) { if (p) cudaFreeHost(p); }

static int fetch_output_impl(ck_handle* h, uint8_t* host_out, uint64_t cap, int64_t* host_out_off, uint32_t* host_out_len,
                             ck_publish* host_pubs, bool wait) {
    cudaSetDevice(h->device);
    uint64_t total = 0;
    if (ck_out_size(h, &total, nullptr, nullptr)) return 1;
    if (total > cap) return fail(h, "ck_fetch_output: host buffer too small");
    if (total > h->max_out) return fail(h, "ck_fetch_output: device output buffer overflowed (raise max_out_bytes)");
    if (host_out && total) CUDA_TRY(h, cudaMemcpyAsync(host_out, h->d_out.p, total, cudaMemcpyDeviceToHost, h->stream));
    if (host_out_off && h->n_payloads) CUDA_TRY(h, cudaMemcpyAsync(host_out_off, h->d_out_off.p, sizeof(long long) * ((size_t)h->n_payloads + 1), cudaMemcpyDeviceToHost, h->stream));
    if (host_out_len && h->n_payloads) CUDA_TRY(h, cudaMemcpyAsync(host_out_len, h->d_pay_len.p, sizeof(u32) * (size_t)h->n_payloads, cudaMemcpyDeviceToHost, h->stream));
    if (host_pubs && h->n_pubs) CUDA_TRY(h, cudaMemcpyAsync(host_pubs, h->d_pubs.p, sizeof(ck_pub) * (size_t)h->n_pubs, cudaMemcpyDeviceToHost, h->stream));
    if (wait) CUDA_TRY(h, cudaStreamSynchronize(h->stream));
    return 0;
}
extern "C" int ck_fetch_output(ck_handle* h, uint8_t* host_out, uint64_t cap, int64_t* host_out_off, uint32_t* host_out_len,
                               ck_publish* host_pubs) {
    return fetch_output_impl(h, host_out, cap, host_out_off, host_out_len, host_pubs, true);
}
// same copies, queued only (the destination must be page-locked for them to be asynchronous): the caller overlaps its
// own work and calls ck_sync before reading
extern "C" int ck_fetch_output_async(ck_handle* h, uint8_t* host_out, uint64_t cap, int64_t* host_out_off, uint32_t* host_out_len,
                                     ck_publish* host_pubs) {
    return fetch_output_impl(h, host_out, cap, host_out_off, host_out_len, host_pubs, false);
}

extern "C" int ck_fetch_overlay(ck_handle* h, uint8_t* host_ovl, uint64_t cap, int64_t* host_off, uint32_t* host_len, uint64_t* used) {
    cudaSetDevice(h->device);
    if (!h->n) { if (used) *used = 0; return 0; }
    long long total = 0;
    CUDA_TRY(h, cudaMemcpyAsync(&total, &h->d_canon_ctl.p->cursor, sizeof(long long), cudaMemcpyDeviceToHost, h->stream));
    CUDA_TRY(h, cudaMemcpyAsync(host_off, h->d_ovl_off.p, sizeof(long long) * (size_t)h->n, cudaMemcpyDeviceToHost, h->stream));
    CUDA_TRY(h, cudaMemcpyAsync(host_len, h->d_ovl_len.p, sizeof(u32) * (size_t)h->n, cudaMemcpyDeviceToHost, h->stream));
    CUDA_TRY(h, cudaStreamSynchronize(h->stream));
    if ((uint64_t)total > h->max_ovl) total = (long long)h->max_ovl;
    if ((uint64_t)total > cap) return fail(h, "ck_fetch_overlay: host buffer too small");
    if (total) CUDA_TRY(h, cudaMemcpyAsync(host_ovl, h->d_ovl.p, (size_t)total, cudaMemcpyDeviceToHost, h->stream));
    CUDA_TRY(h, cudaStreamSynchronize(h->stream));
    if (used) *used = (uint64_t)total;
    return 0;
}

extern "C" int ck_fetch_topic_hist(ck_handle* h, uint32_t* host_hist, uint32_t n) {
    cudaSetDevice(h->device);
    if (n > h->hist_cap) n = h->hist_cap;
    CUDA_TRY(h, cudaMemcpyAsync(host_hist, h->d_topic_hist.p, sizeof(u32) * n, cudaMemcpyDeviceToHost, h->stream));
    CUDA_TRY(h, cudaStreamSynchronize(h->stream));
    return 0;
}

extern "C" void* ck_stream(ck_handle* h) { return (void*)h->stream; }

extern "C" int ck_device_buffers2(ck_handle* h, void** pubs, void** pay_len, void** descs) {
    if (pubs) *pubs = h->d_pubs.p;
    if (pay_len) *pay_len = h->d_pay_len.p;
    if (descs) *descs = h->d_descs.p;
    return 0;
}

extern "C" int ck_device_buffers(ck_handle* h, void** in, void** in_off, void** out, void** out_off, void** cols) {
    if (in) *in = h->d_in.p;
    if (in_off) *in_off = h->d_in_off.p;
    if (out) *out = h->d_out.p;
    if (out_off) *out_off = h->d_out_off.p;
    if (cols) *cols = h->d_cols.p;
    return 0;
}

extern "C" int ck_profile(ck_handle* h, int enable) { cudaSetDevice(h->device); profile_collect(h); h->profile = enable != 0; return 0; }

extern "C" int ck_profile_read(ck_handle* h, float* ms, uint32_t* launches, int reset) {
    cudaSetDevice(h->device);
    profile_collect(h);
    for (int k = 0; k < CK_NUM_KERNELS; k++) { ms[k] = h->k_ms[k]; launches[k] = h->k_n[k]; if (reset) { h->k_ms[k] = 0; h->k_n[k] = 0; } }
    return 0;
}
