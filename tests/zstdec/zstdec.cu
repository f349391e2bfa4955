// TEST INFRASTRUCTURE ONLY.  The shipped zstd decoder (ck_zs_decode, csrc/ck_zstd.cuh) alone, one warp per frame with its
// workspace in shared memory as ck_rb_zstd_kernel runs it: frame i = src[soff[i], soff[i+1]) decodes into
// dst[doff[i], doff[i+1]); out_len[i] = decoded bytes (-1 = refused).  Every pointer is a device pointer.
#include <cuda_runtime.h>
#include "ck_zstd.cuh"

#define WARPS 3
__global__ void __launch_bounds__(32 * WARPS)
zstd_kernel(const u8* __restrict__ src, const long long* __restrict__ soff, u32 n, u8* dst, const long long* __restrict__ doff,
            long long* __restrict__ out_len) {
    __shared__ ck_zs_ws ws[WARPS];
    u32 wi = threadIdx.x >> 5, b = blockIdx.x * WARPS + wi, lane = threadIdx.x & 31;
    if (b >= n) return;
    long long r = ck_zs_decode(src + soff[b], (unsigned long long)(soff[b + 1] - soff[b]), dst + doff[b],
                               (unsigned long long)(doff[b + 1] - doff[b]), ws[wi], lane);
    if (lane == 0) out_len[b] = r;
}

extern "C" int zstd_frames(const u8* src, const long long* soff, u32 n, u8* dst, const long long* doff, long long* out_len) {
    if (n) zstd_kernel<<<(n + WARPS - 1) / WARPS, 32 * WARPS>>>(src, soff, n, dst, doff, out_len);
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    return (int)e;
}
