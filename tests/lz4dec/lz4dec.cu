// TEST INFRASTRUCTURE ONLY.  The shipped LZ4 block decoder (ck_lz4_decode_block, csrc/ck_lz4.cuh) alone, one warp per
// block as ck_rb_lz4_kernel runs it: block i = src[soff[i], soff[i+1]) decodes into the region dst[doff[i], doff[i+1]),
// behind hist[i] bytes of history already there (matches may reach into them, as in a linked frame), with block maximum
// block_max; out_len[i] = decoded bytes, -1 = malformed.  Every pointer is a device pointer.
#include <cuda_runtime.h>
#include "ck_lz4.cuh"

__global__ void __launch_bounds__(128)
lz4dec_kernel(const u8* __restrict__ src, const long long* __restrict__ soff, u32 n, u8* __restrict__ dst, const long long* __restrict__ doff,
              const u32* __restrict__ hist, u32 block_max, long long* __restrict__ out_len) {
    u32 b = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (b >= n) return;
    unsigned long long cap = (unsigned long long)(doff[b + 1] - doff[b]);
    long long r = ck_lz4_decode_block(src + soff[b], (u32)(soff[b + 1] - soff[b]), dst + doff[b], hist[b], 0, cap, block_max, lane);
    if (lane == 0) out_len[b] = r;
}

extern "C" int lz4dec_blocks(const u8* src, const long long* soff, u32 n, u8* dst, const long long* doff, const u32* hist,
                             u32 block_max, long long* out_len) {
    if (n) lz4dec_kernel<<<(n + 3) / 4, 128>>>(src, soff, n, dst, doff, hist, block_max, out_len);
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    return (int)e;
}
