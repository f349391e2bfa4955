// TEST INFRASTRUCTURE ONLY.  Launchers that run the shipped device code (csrc/ck_kernels.cuh) on inputs a test makes
// itself, so that the emitter, the offset scan and the Kafka key hash can be compared with plain references kernel by
// kernel, at edges the producers never reach.  Every pointer is a device pointer (a torch tensor's data_ptr()).  Nothing
// in the product links or loads this file.
#include <cstring>
#include "ck_kernels.cuh"

static ck_view dev_view(const u8* in, const long long* off, const long long* ovl_off) {
    ck_view v;
    memset(&v, 0, sizeof v);
    v.in = in; v.off = off; v.ovl_off = ovl_off;     // no overlay; len, perm, hist_skip stay NULL
    return v;
}

// ovl_off of `nrec` records without an overlay (all -1), for the life of one launch
static long long* no_overlay(u32 nrec) {
    long long* p = nullptr;
    if (cudaMalloc((void**)&p, sizeof(long long) * ((size_t)nrec + 1)) != cudaSuccess) return nullptr;
    cudaMemset(p, 0xff, sizeof(long long) * ((size_t)nrec + 1));
    return p;
}

static int finish(long long* ovl) {
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    cudaFree(ovl);
    return (int)e;
}

// ck_emit_kernel on caller-made descriptors, launched as scan_emit (ck_api.cu) launches it
extern "C" int ck_dev_emit(const u8* in, const long long* rec_off, u32 nrec, const u8* lit, const u8* aux, const u8* glue,
                           const ck_out_desc* descs, const long long* out_off, u32 n, u8* out, long long out_cap) {
    long long* ovl = no_overlay(nrec);
    if (!ovl) return (int)cudaErrorMemoryAllocation;
    if (n) ck_emit_kernel<<<(n + 7) / 8, 256>>>(dev_view(in, rec_off, ovl), lit, aux, glue, descs, out_off, n, out, out_cap);
    return finish(ovl);
}

// the three scan kernels, launched as run_scan (ck_api.cu) launches them; tile_sum holds n / CK_SCAN_TILE + 2 entries
extern "C" int ck_dev_scan(const u32* len, u32 n, long long* out_off, u32 pad, unsigned long long* tile_sum,
                           unsigned long long* grand) {
    u32 ntiles = (n + CK_SCAN_TILE - 1) / CK_SCAN_TILE;
    if (n) {
        ck_scan_tiles_kernel<<<ntiles, CK_SCAN_BLOCK>>>(len, n, tile_sum, pad);
        ck_scan_sums_kernel<<<1, CK_SCAN_BLOCK>>>(tile_sum, ntiles, grand);
        ck_scan_apply_kernel<<<ntiles, CK_SCAN_BLOCK>>>(len, n, tile_sum, out_off, pad);
    }
    return finish(nullptr);
}

// a reader that counts its byte reads: ck_murmur2_key reads bytes only to decode a key that holds an escape
template <class R> struct ck_dev_counted : R {
    u32 nat;
    __device__ __forceinline__ u8 at(u32 pos) { nat++; return R::at(pos); }
};
template <class R> __device__ __forceinline__ void ck_dev_reset(R&) {}
template <class R> __device__ __forceinline__ void ck_dev_reset(ck_dev_counted<R>& r) { r.nat = 0; }
template <class R> __device__ __forceinline__ u32 ck_dev_reads(const R&) { return 0; }
template <class R> __device__ __forceinline__ u32 ck_dev_reads(const ck_dev_counted<R>& r) { return r.nat; }

// ck_murmur2_key of the raw JSON string content key[j] = (record, offset, length, prime) of the batch: the full 32-bit
// hash.  prime != ~0u: the reader reads that byte of the record first, as the plan reads the callback topic before the
// correlation id, which places the key anywhere in a PRd window.  Each thread hashes several keys one after the other, and
// its window slot starts filled with backslashes, so bytes the window holds past a record's end are stale, never zero.
template <class R>
__global__ void __launch_bounds__(CK_P2_THREADS)
ck_dev_key_kernel(ck_view v, const uint4* __restrict__ keys, u32 n, u32* __restrict__ hash, u32* __restrict__ reads) {
    if (R::kWindow) {
        u8* slot = (u8*)ck_win_smem + threadIdx.x * CK_P2_WSTRIDE;
        for (u32 k = 0; k < CK_P2_WSTRIDE; k++) slot[k] = '\\';
    }
    for (u32 j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += gridDim.x * blockDim.x) {
        uint4 q = keys[j];
        u32 rlen; const u8* rec = ck_rec(v, q.x, rlen);
        R r; r.init(rec, rlen);
        if (q.w != 0xffffffffu) (void)r.at(q.w);
        ck_dev_reset(r);
        hash[j] = ck_murmur2_key(r, q.y, q.z);
        if (reads) reads[j] = ck_dev_reads(r);
    }
}

// reader: 0 = PRd (the plan's shared-memory window), 1 = GRd (ck_route_kernel's global loads), 2 = GRd counting its
// byte reads into `reads`
extern "C" int ck_dev_murmur2_key(int reader, const u8* in, const long long* rec_off, u32 nrec, const uint4* keys, u32 n,
                                  u32* hash, u32* reads) {
    long long* ovl = no_overlay(nrec);
    if (!ovl) return (int)cudaErrorMemoryAllocation;
    ck_view v = dev_view(in, rec_off, ovl);
    u32 grid = (n + CK_P2_THREADS * 4 - 1) / (CK_P2_THREADS * 4);    // about four keys per thread
    grid = grid ? grid : 1;
    if (reader == 0) ck_dev_key_kernel<PRd><<<grid, CK_P2_THREADS, CK_P2_SMEM>>>(v, keys, n, hash, nullptr);
    else if (reader == 1) ck_dev_key_kernel<GRd><<<grid, CK_P2_THREADS>>>(v, keys, n, hash, nullptr);
    else ck_dev_key_kernel<ck_dev_counted<GRd>><<<grid, CK_P2_THREADS>>>(v, keys, n, hash, reads);
    return finish(ovl);
}
