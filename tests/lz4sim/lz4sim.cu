// TEST INFRASTRUCTURE ONLY.  The shipped LZ4 block compressor (csrc/ck_lz4.cuh) alone, one warp per block with its hash
// table in shared memory as ck_lz_compress_kernel runs it: block i = src[off[i], off[i+1]) (at most 64 KB), compressed into
// dst at the same offset; out_len[i] = compressed bytes, 0 = not smaller (stored raw).  Every pointer is a device pointer.
#include <cuda_runtime.h>
#include "ck_lz4.cuh"

__global__ void __launch_bounds__(CK_LZ_WARPS * 32)
lz4sim_kernel(const u8* __restrict__ src, const long long* __restrict__ off, u32 n, u8* __restrict__ dst, u32* __restrict__ out_len) {
    __shared__ uint16_t tabs[CK_LZ_WARPS][1u << CK_LZ_HBITS];
    u32 lane = threadIdx.x & 31, wid = threadIdx.x >> 5, b = blockIdx.x * CK_LZ_WARPS + wid;
    if (b >= n) return;
    u32 z = ck_lz4_block(src + off[b], (u32)(off[b + 1] - off[b]), dst + off[b], tabs[wid], lane);
    if (lane == 0) out_len[b] = z;
}

extern "C" int lz4sim_blocks(const u8* src, const long long* off, u32 n, u8* dst, u32* out_len) {
    if (n) lz4sim_kernel<<<(n + CK_LZ_WARPS - 1) / CK_LZ_WARPS, CK_LZ_WARPS * 32>>>(src, off, n, dst, out_len);
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    return (int)e;
}
