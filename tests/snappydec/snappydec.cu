// TEST INFRASTRUCTURE ONLY.  The shipped snappy block decoder (ck_sn_decode_block, csrc/ck_snappy.cuh) alone, one warp per
// raw block as ck_rb_snappy_kernel runs it: block i = src[soff[i], soff[i+1]) decodes into dst[doff[i], doff[i+1]) (its
// declared length); out_len[i] = decoded bytes (-1 = refused).  Every pointer is a device pointer.
#include <cuda_runtime.h>
#include "ck_snappy.cuh"

__global__ void __launch_bounds__(256)
snappy_kernel(const u8* __restrict__ src, const long long* __restrict__ soff, u32 n, u8* dst, const long long* __restrict__ doff,
              long long* __restrict__ out_len) {
    u32 b = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (b >= n) return;
    long long r = ck_sn_decode_block(src + soff[b], (u32)(soff[b + 1] - soff[b]), dst + doff[b], (u32)(doff[b + 1] - doff[b]), lane);
    if (lane == 0) out_len[b] = r;
}

extern "C" int snappy_blocks(const u8* src, const long long* soff, u32 n, u8* dst, const long long* doff, long long* out_len) {
    if (n) snappy_kernel<<<(n + 7) / 8, 256>>>(src, soff, n, dst, doff, out_len);
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    return (int)e;
}
