// Grouping the publish table by destination topic on the device.
//
// Reference analogue: every broker.publish(topic=...) of a handler goes to its own topic (calfkit/nodes/base.py:82-87,
// worker/worker.py:52-53); a producer then accumulates records per topic-partition.  A lane produces up to two publishes
// per record, a million records per step: splitting that table per topic with host-side scans of a 64 MB structure cost
// more than the PCIe copies of the step.  Here the table is partitioned on the device by a stable two-pass LSD radix sort
// over 12-bit keys (6 bits per pass, 64 buckets: per-block histograms -> scan -> stable scatter, the same scheme as the
// exchange planner):
//     key 0           live publish whose topic has no registered id (named by a span of the source record)
//     key 1 + id      live publish to registered topic `id` (ids above 4093 share the last live key)
//     key 4095        unused slot
// Result: order[] = publish indices grouped by key, send order preserved inside a group, and the number of publishes per
// key — the host slices, it never scans.
#ifndef CK_GROUP_CUH
#define CK_GROUP_CUH

#define CK_G_BLOCK 256
#define CK_G_KEYS 4096u

__device__ __forceinline__ u32 ck_group_key(const ck_pub& p) {
    if (p.payload == 0xffffffffu) return CK_G_KEYS - 1;
    if (p.topic_id < 0) return 0;
    u32 k = (u32)p.topic_id + 1;
    return k < CK_G_KEYS - 2 ? k : CK_G_KEYS - 2;
}

// key functors: the publish table by destination topic; the records of a batch by length (32-byte classes) — the second
// one buckets a heterogeneous batch before the thread-per-record walk: lanes of a warp then walk records of one size class
// (a warp takes as long as its longest record) and, since a topic's records of one size mostly share a shape, of one shape
// (lanes on different schema branches execute one after the other)
struct ck_key_pub {
    const ck_pub* pubs; u32 rank, world;        // world > 1: keyed publishes whose partition another rank owns were forwarded (ck_exchange_send): not produced here
    __device__ __forceinline__ u32 operator()(u32 i) const {
        ck_pub p = pubs[i];
        if (world > 1 && p.payload != 0xffffffffu && p.has_key == 1 && p.partition >= 0 && (u32)p.partition % world != rank) return CK_G_KEYS - 1;
        return ck_group_key(p);
    }
};
struct ck_key_len {
    ck_view v;
    // longest first: the walk's blocks start in this order, so the records that take longest start first and the short ones
    // fill in behind them (a 16 KB record alone keeps a thread busy far longer than a short one; started last it would be
    // the kernel's tail)
    __device__ __forceinline__ u32 operator()(u32 i) const { u32 len; ck_rec_in(v, i, len); u32 k = len >> 5; return CK_G_KEYS - 1 - (k < CK_G_KEYS - 1 ? k : CK_G_KEYS - 1); }
};

// pass over `in` (NULL = identity order): digit histogram per block -> hist[digit][block]; pass 0 also counts whole keys
template <int SHIFT, class KeyFn>
__global__ void __launch_bounds__(CK_G_BLOCK)
ck_group_count_kernel(KeyFn keyf, const u32* __restrict__ in, u32 n, u32* __restrict__ hist, u32* __restrict__ key_hist) {
    __shared__ u32 s_cnt[64];
    if (threadIdx.x < 64) s_cnt[threadIdx.x] = 0;
    __syncthreads();
    u32 j = blockIdx.x * blockDim.x + threadIdx.x;
    bool live = j < n;
    u32 key = 0;
    if (live) { key = keyf(in ? in[j] : j); atomicAdd(&s_cnt[(key >> SHIFT) & 63u], 1u); }
    if (SHIFT == 0) {
        u32 act = __ballot_sync(0xffffffffu, live);
        if (live) {
            u32 peers = __match_any_sync(act, key);
            if ((threadIdx.x & 31) == (u32)(__ffs(peers) - 1)) atomicAdd(key_hist + key, __popc(peers));
        }
    }
    __syncthreads();
    if (threadIdx.x < 64) hist[(size_t)threadIdx.x * gridDim.x + blockIdx.x] = s_cnt[threadIdx.x];
}

template <int SHIFT, class KeyFn>
__global__ void __launch_bounds__(CK_G_BLOCK)
ck_group_scatter_kernel(KeyFn keyf, const u32* __restrict__ in, u32 n, const long long* __restrict__ base, u32* __restrict__ out) {
    __shared__ u32 s_w[CK_G_BLOCK / 32][64];
    u32 lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (u32 k = threadIdx.x; k < (CK_G_BLOCK / 32) * 64; k += CK_G_BLOCK) (&s_w[0][0])[k] = 0;
    __syncthreads();
    u32 j = blockIdx.x * blockDim.x + threadIdx.x;
    bool live = j < n;
    u32 idx = 0, digit = 0, rank_in_warp = 0;
    if (live) { idx = in ? in[j] : j; digit = (keyf(idx) >> SHIFT) & 63u; }
    u32 act = __ballot_sync(0xffffffffu, live);
    if (live) {
        u32 same = __match_any_sync(act, digit);
        rank_in_warp = __popc(same & ((1u << lane) - 1u));
        if (rank_in_warp == 0) s_w[warp][digit] = __popc(same);
    }
    __syncthreads();
    if (live) {
        u32 before = 0;
        for (u32 w = 0; w < warp; w++) before += s_w[w][digit];
        out[base[(size_t)digit * gridDim.x + blockIdx.x] + before + rank_in_warp] = idx;
    }
}

#endif  // CK_GROUP_CUH
