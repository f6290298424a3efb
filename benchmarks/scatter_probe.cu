// What bounds the multisplit key scatter?  Standalone kernels for benchmarks/scatter_probe.py (not part of the
// library).  All variants run the statements of the key scatter as it was before it staged its slices in shared
// memory (one 8-byte store per pair) on the library's real inputs, and differ only in where a key goes:
//   MODE 0  keys[pos]          that scatter
//   MODE 1  dummy[pos & mask]  same instructions and atomics, but the write set is a small buffer that stays in L2
//   MODE 2  no store           the returned shared-memory atomic is kept (its result feeds a never-taken branch)
// plus stream_kernel, a coalesced write of the same number of keys: the byte floor of the output.
#include <cuda_runtime.h>
#include <stdint.h>

#define GSR_MS_ITEMS 4

template <int MODE>
__global__ void __launch_bounds__(1024)
probe_scatter_kernel(int P, int per, int gx, int ntiles, uint32_t max_pairs, const uint4* __restrict__ rectdepth,
                     uint32_t* __restrict__ tile_cursor, const uint32_t* __restrict__ block_hist,
                     unsigned long long* __restrict__ keys, unsigned long long* __restrict__ dummy, uint32_t mask) {
    extern __shared__ uint32_t hist[];
    const int i0 = blockIdx.x * per;
    const int i1 = min(P, i0 + per);
    const uint32_t* my_hist = block_hist + (size_t)blockIdx.x * ntiles;
    uint4 rd[GSR_MS_ITEMS];
#pragma unroll
    for (int u = 0; u < GSR_MS_ITEMS; ++u) {
        const int i = i0 + u * 1024 + threadIdx.x;
        rd[u] = (i < i1) ? __ldg(rectdepth + i) : make_uint4(0u, 0u, 0u, 0u);
    }
    for (int t = threadIdx.x; t < ntiles; t += 1024) {
        const uint32_t c = my_hist[t];
        if (c) hist[t] = atomicAdd(tile_cursor + t, c);
    }
    __syncthreads();
#pragma unroll
    for (int u = 0; u < GSR_MS_ITEMS; ++u) {
        if (rd[u].w) {
            const int i = i0 + u * 1024 + threadIdx.x;
            const int minx = rd[u].x & 0xffff, miny = rd[u].x >> 16, maxx = rd[u].y & 0xffff, maxy = rd[u].y >> 16;
            const unsigned long long key = ((unsigned long long)rd[u].z << 32) | (uint32_t)i;
            for (int ty = miny; ty < maxy; ++ty)
                for (int tx = minx; tx < maxx; ++tx) {
                    const uint32_t pos = atomicAdd(&hist[ty * gx + tx], 1u);
                    if (MODE == 0) {
                        if (pos < max_pairs) keys[pos] = key;
                    } else if (MODE == 1) {
                        if (pos < max_pairs) dummy[pos & mask] = key;
                    } else {
                        if (pos == 0xffffffffu) keys[0] = key;
                    }
                }
        }
    }
}

__global__ void __launch_bounds__(256) stream_kernel(size_t n2, uint4* __restrict__ out) {
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n2; i += (size_t)gridDim.x * blockDim.x)
        out[i] = make_uint4((uint32_t)i, 0u, (uint32_t)i, 1u);
}

extern "C" int probe_launch(int mode, int P, int nblk, int per, int gx, int ntiles, uint32_t max_pairs,
                            const void* rectdepth, void* tile_cursor, const void* block_hist, void* keys, void* dummy,
                            uint32_t mask, unsigned long long num_keys, void* stream) {
    cudaStream_t s = (cudaStream_t)stream;
    const int smem = ntiles * (int)sizeof(uint32_t);
    const uint4* rd = (const uint4*)rectdepth;
    uint32_t* cur = (uint32_t*)tile_cursor;
    const uint32_t* bh = (const uint32_t*)block_hist;
    unsigned long long* k = (unsigned long long*)keys;
    unsigned long long* d = (unsigned long long*)dummy;
    switch (mode) {
    case 0:
        cudaFuncSetAttribute(probe_scatter_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        probe_scatter_kernel<0><<<nblk, 1024, smem, s>>>(P, per, gx, ntiles, max_pairs, rd, cur, bh, k, d, mask);
        break;
    case 1:
        cudaFuncSetAttribute(probe_scatter_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        probe_scatter_kernel<1><<<nblk, 1024, smem, s>>>(P, per, gx, ntiles, max_pairs, rd, cur, bh, k, d, mask);
        break;
    case 2:
        cudaFuncSetAttribute(probe_scatter_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        probe_scatter_kernel<2><<<nblk, 1024, smem, s>>>(P, per, gx, ntiles, max_pairs, rd, cur, bh, k, d, mask);
        break;
    case 3: {
        int dev = 0, sms = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
        stream_kernel<<<sms * 8, 256, 0, s>>>(num_keys / 2, (uint4*)keys);
        break;
    }
    default:
        return -1;
    }
    return (int)cudaGetLastError();
}
