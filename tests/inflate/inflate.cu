// TEST INFRASTRUCTURE ONLY.  The shipped inflate core (ck_inflate, csrc/ck_inflate.cuh) alone, one warp per stream with
// its workspace in shared memory as ck_rb_gzip_kernel runs it: the raw deflate stream i = src[soff[i], soff[i+1])
// inflates into dst[doff[i], doff[i+1]); out_len[i] = inflated bytes (-1 = refused), used[i] = the bytes the stream took.
// Every pointer is a device pointer.
#include <cuda_runtime.h>
#include "ck_inflate.cuh"

#define WARPS 4
__global__ void __launch_bounds__(32 * WARPS)
inflate_kernel(const u8* __restrict__ src, const long long* __restrict__ soff, u32 n, u8* dst, const long long* __restrict__ doff,
               long long* __restrict__ out_len, long long* __restrict__ used) {
    __shared__ ck_gz_ws ws[WARPS];
    u32 wi = threadIdx.x >> 5, b = blockIdx.x * WARPS + wi, lane = threadIdx.x & 31;
    if (b >= n) return;
    unsigned long long u = 0;
    long long r = ck_inflate(src + soff[b], (unsigned long long)(soff[b + 1] - soff[b]), dst + doff[b],
                             (unsigned long long)(doff[b + 1] - doff[b]), ws[wi], lane, &u);
    if (lane == 0) { out_len[b] = r; used[b] = (long long)u; }
}

// the same with ck_gz_decode on whole gzip members (header, stream, trailer position and ISIZE; not the CRC32), each
// into a slot of doff[i+1] - doff[i] bytes: out_len[i] = inflated bytes or -1
__global__ void __launch_bounds__(32 * WARPS)
inflate_member_kernel(const u8* __restrict__ src, const long long* __restrict__ soff, u32 n, u8* dst, const long long* __restrict__ doff,
                      long long* __restrict__ out_len) {
    __shared__ ck_gz_ws ws[WARPS];
    u32 wi = threadIdx.x >> 5, b = blockIdx.x * WARPS + wi, lane = threadIdx.x & 31;
    if (b >= n) return;
    long long r = ck_gz_decode(src + soff[b], (unsigned long long)(soff[b + 1] - soff[b]), dst + doff[b],
                               (unsigned long long)(doff[b + 1] - doff[b]), ws[wi], lane);
    if (lane == 0) out_len[b] = r;
}

extern "C" int inflate_members(const u8* src, const long long* soff, u32 n, u8* dst, const long long* doff, long long* out_len) {
    if (n) inflate_member_kernel<<<(n + WARPS - 1) / WARPS, 32 * WARPS>>>(src, soff, n, dst, doff, out_len);
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    return (int)e;
}

extern "C" int inflate_streams(const u8* src, const long long* soff, u32 n, u8* dst, const long long* doff, long long* out_len, long long* used) {
    if (n) inflate_kernel<<<(n + WARPS - 1) / WARPS, 32 * WARPS>>>(src, soff, n, dst, doff, out_len, used);
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    return (int)e;
}
