// Reconstruction loss (DESIGN.md §0 f9): loss[v] = w * mean((fp16(image_v) - target[idx[v]])^2) and its image
// gradient in one streaming pass over the image and the target, the reference's
// `l2_loss(image.to(torch.float16), gt) * 100` with torch's dtype rules.
//
// The gradient is torch's autograd chain on CUDA, every intermediate rounded where torch stores it, written with
// explicit round-to-nearest intrinsics so that nvcc cannot contract it (the forms were pinned on the H100 against
// torch's own ops, DESIGN.md §5 f9).  Every torch op involved computes in fp32 ("opmath") and rounds its result to the
// tensor's dtype:
//   MulBackward (loss * w)    g1 = dt(go * w)
//   MeanBackward (/ N)        g2 = dt(g1 * fp32(1 / N))          div by a CPU scalar is a reciprocal multiply
//   PowBackward (** 2)        d  = dt(g2 * dt(2 * diff))
//   SubBackward + the cast    grad = fp32(fp16(d))                 the fp16 input's gradient is fp16
// where dt rounds to the loss dtype (fp16 for a float16 target, else fp32) and diff = dt(fp16(x) - t).
#include "common.cuh"
#include <cuda_fp16.h>

namespace {

__device__ __forceinline__ float h(float x) { return __half2float(__float2half_rn(x)); }

// dt(x) of the loss dtype
template <bool HALF>
__device__ __forceinline__ float dt(float x) { return HALF ? h(x) : x; }

// One element: returns the squared difference as the loss sums it (the fp16 square for a float16 target) and sets
// *d to the image gradient for the view's g2.
template <bool HALF>
__device__ __forceinline__ float l2_elem(float x, float t, float g2, float& d) {
    const float diff = dt<HALF>(__fsub_rn(h(x), t));
    d = h(dt<HALF>(__fmul_rn(g2, dt<HALF>(__fmul_rn(2.0f, diff)))));
    return dt<HALF>(__fmul_rn(diff, diff));
}

// 4 target elements as floats (fp16 values are exact in fp32)
template <bool HALF>
__device__ __forceinline__ float4 load_target4(const void* base, long long j) {
    if constexpr (HALF) {
        const uint2 u = __ldg(reinterpret_cast<const uint2*>(base) + j);
        const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&u.x));
        const float2 b = __half22float2(*reinterpret_cast<const __half2*>(&u.y));
        return make_float4(a.x, a.y, b.x, b.y);
    } else {
        return __ldg(reinterpret_cast<const float4*>(base) + j);
    }
}

template <bool HALF>
__device__ __forceinline__ float load_target(const void* base, long long i) {
    if constexpr (HALF) return __half2float(reinterpret_cast<const __half*>(base)[i]);
    else return __ldg(reinterpret_cast<const float*>(base) + i);
}

template <bool HALF>
__device__ __forceinline__ float load_loss_dtype(const void* base, int i) {
    if constexpr (HALF) return __half2float(reinterpret_cast<const __half*>(base)[i]);
    else return reinterpret_cast<const float*>(base)[i];
}

// Fixed-order sum of one double per thread; the result is valid in thread 0.
__device__ __forceinline__ double block_sum(double x) {
    __shared__ double warp_sum[GSR_L2_THREADS / 32];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) x += __shfl_down_sync(0xffffffffu, x, o);
    if ((threadIdx.x & 31) == 0) warp_sum[threadIdx.x >> 5] = x;
    __syncthreads();
    double s = 0.0;
    if (threadIdx.x == 0)
        for (int w = 0; w < GSR_L2_THREADS / 32; ++w) s += warp_sum[w];
    return s;
}

// grid (gsr_l2_blocks(N), B): CTA b of view v owns elements [b CHUNK, min((b + 1) CHUNK, N)).  The vector path needs
// the view's image, gradient and target rows 16-, 16- and 16/8-byte aligned (every chunk starts at a multiple of 4096
// elements, so the view's base decides); the < 4-element tail and unaligned views take the scalar loop.
template <bool HALF>
__global__ void __launch_bounds__(GSR_L2_THREADS) recon_l2_kernel(const GsrL2Args a) {
    const int v = blockIdx.y;
    const long long N = a.N;
    const long long start = (long long)blockIdx.x * GSR_L2_CHUNK;
    const long long end = start + GSR_L2_CHUNK < N ? start + GSR_L2_CHUNK : N;
    const int t = a.target_index ? __ldg(a.target_index + v) : v;
    const bool bad = t < 0 || t >= a.n_targets;
    const float* img = a.image + (long long)v * N;
    float* dimg = a.d_image ? a.d_image + (long long)v * N : nullptr;
    const void* tgt = static_cast<const char*>(a.target) + (bad ? 0 : t) * N * (HALF ? 2 : 4);
    const float nan = __int_as_float(0x7fffffff);
    float g2 = 0.0f;
    if (dimg) {
        const float g1 = dt<HALF>(__fmul_rn(load_loss_dtype<HALF>(a.grad_out, v), a.weight));
        g2 = bad ? nan : dt<HALF>(__fmul_rn(g1, a.inv_n));
    }
    float acc = bad ? nan : 0.0f;
    long long i0 = start;
    const uintptr_t al = reinterpret_cast<uintptr_t>(img) | reinterpret_cast<uintptr_t>(dimg);
    if ((al & 15) == 0 && (reinterpret_cast<uintptr_t>(tgt) & (HALF ? 7 : 15)) == 0) {
        const long long q0 = start >> 2;
        const int nv = (int)((end - start) >> 2);
        float4 X[4], T[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const int j = k * GSR_L2_THREADS + threadIdx.x;
            if (j < nv) { X[k] = __ldg(reinterpret_cast<const float4*>(img) + q0 + j); T[k] = load_target4<HALF>(tgt, q0 + j); }
        }
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const int j = k * GSR_L2_THREADS + threadIdx.x;
            if (j < nv) {
                float4 D;
                acc += l2_elem<HALF>(X[k].x, T[k].x, g2, D.x);
                acc += l2_elem<HALF>(X[k].y, T[k].y, g2, D.y);
                acc += l2_elem<HALF>(X[k].z, T[k].z, g2, D.z);
                acc += l2_elem<HALF>(X[k].w, T[k].w, g2, D.w);
                if (dimg) reinterpret_cast<float4*>(dimg)[q0 + j] = D;
            }
        }
        i0 = start + 4LL * nv;
    }
    for (long long i = i0 + threadIdx.x; i < end; i += GSR_L2_THREADS) {
        float d;
        acc += l2_elem<HALF>(__ldg(img + i), load_target<HALF>(tgt, i), g2, d);
        if (dimg) dimg[i] = d;
    }
    if (a.loss_out) {
        const double s = block_sum((double)acc);
        if (threadIdx.x == 0) a.partials[(long long)v * gridDim.x + blockIdx.x] = s;
    }
}

// grid B: view v's partials summed in a fixed order, then mean and weight in the loss dtype as torch rounds them.
template <bool HALF>
__global__ void __launch_bounds__(GSR_L2_THREADS) recon_l2_finish_kernel(const GsrL2Args a, int nblk) {
    const int v = blockIdx.x;
    double s = 0.0;
    for (int i = threadIdx.x; i < nblk; i += GSR_L2_THREADS) s += a.partials[(long long)v * nblk + i];
    s = block_sum(s);
    if (threadIdx.x == 0) {
        const double mean = s / (double)a.N;
        if constexpr (HALF) {
            const float m = __half2float(__double2half(mean));
            reinterpret_cast<__half*>(a.loss_out)[v] = __float2half_rn(__fmul_rn(m, a.weight));
        } else {
            reinterpret_cast<float*>(a.loss_out)[v] = __fmul_rn(__double2float_rn(mean), a.weight);
        }
    }
}

template <bool HALF>
cudaError_t launch(const GsrL2Args& a, cudaStream_t s) {
    const int nblk = (int)gsr_l2_blocks(a.N);
    recon_l2_kernel<HALF><<<dim3(nblk, a.B), GSR_L2_THREADS, 0, s>>>(a);
    if (a.loss_out) recon_l2_finish_kernel<HALF><<<a.B, GSR_L2_THREADS, 0, s>>>(a, nblk);
    return cudaGetLastError();
}

}  // namespace

cudaError_t gsr_launch_recon_l2(const GsrL2Args& a, bool half_target, cudaStream_t s) {
    return half_target ? launch<true>(a, s) : launch<false>(a, s);
}
