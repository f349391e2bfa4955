// TEST INFRASTRUCTURE ONLY.  The shipped hash-chain LZ4 block compressor (ck_lz4_block_hc, csrc/ck_lz4.cuh) alone, one warp
// per block with its head table in shared memory as ck_lz_compress_hc_kernel runs it: block i = src[off[i], off[i+1]) (at
// most 64 KB), compressed at search depth `depth` into dst at the same offset with its chain at chains + i * 64 K;
// out_len[i] = compressed bytes, 0 = not smaller (stored raw).  Every pointer is a device pointer.
#include <cuda_runtime.h>
#include "ck_lz4.cuh"

__global__ void __launch_bounds__(CK_LZ_WARPS * 32)
lz4hc_kernel(const u8* __restrict__ src, const long long* __restrict__ off, u32 n, u8* __restrict__ dst, u32* __restrict__ out_len,
             uint16_t* __restrict__ chains, u32 depth) {
    __shared__ uint16_t tabs[CK_LZ_WARPS][1u << CK_LZ_HBITS];
    u32 lane = threadIdx.x & 31, wid = threadIdx.x >> 5, b = blockIdx.x * CK_LZ_WARPS + wid;
    if (b >= n) return;
    u32 z = ck_lz4_block_hc(src + off[b], (u32)(off[b + 1] - off[b]), dst + off[b], tabs[wid], chains + (size_t)b * CK_LZ_BLOCK, depth, lane);
    if (lane == 0) out_len[b] = z;
}

extern "C" int lz4hc_blocks(const u8* src, const long long* off, u32 n, u8* dst, u32* out_len, uint16_t* chains, u32 depth) {
    if (n) lz4hc_kernel<<<(n + CK_LZ_WARPS - 1) / CK_LZ_WARPS, CK_LZ_WARPS * 32>>>(src, off, n, dst, out_len, chains, depth);
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    return (int)e;
}
