// Adam step (DESIGN.md §0 f6): torch.optim.Adam's default update for every tensor of one step() in ONE launch.
// torch's foreach path (_multi_tensor_adam) runs lerp, mul, addcmul, sqrt, div, add and addcdiv as separate
// kernels per parameter group, about 76 bytes of traffic per element; this kernel reads p, g, m, v and writes
// p, m, v once: 28 bytes per element.
//
// The arithmetic is that of the foreach kernels, every intermediate rounded to fp32 where they store it, and
// written with explicit round-to-nearest intrinsics so that nvcc cannot contract or reassociate it:
//   lerp     ATen/native/Lerp.h, contracted to one FMA as torch's own build does: |w| < 0.5 -> m + w (g - m),
//            else g - (g - m)(1 - w)
//   addcmul  ATen/native/cuda/DeviceAddCmulCdiv.cuh: fma(value, g * g, v), or fma(g, g, v) when value == 1
//   div      IEEE division (torch's CUDA code is compiled without fast division)
//   addcdiv  fma(step_size, m / d, p)
// Non-finite values go through the same instructions and so come out as the same bit patterns.
#include "common.cuh"
#include <type_traits>

namespace {

__device__ __forceinline__ void adam_update(float& p, float g, float& m, float& v, const GsrAdamEntry& e) {
    const float d = __fsub_rn(g, m);
    m = fabsf(e.w) < 0.5f ? __fmaf_rn(e.w, d, m) : __fmaf_rn(-d, __fsub_rn(1.0f, e.w), g);
    v = __fmul_rn(v, e.beta2);
    v = e.omb2 == 1.0f ? __fmaf_rn(g, g, v) : __fmaf_rn(e.omb2, __fmul_rn(g, g), v);
    const float den = __fadd_rn(__fdiv_rn(__fsqrt_rn(v), e.bc2_sqrt), e.eps);
    p = __fmaf_rn(e.step_size, __fdiv_rn(m, den), p);
}

__device__ __forceinline__ void adam_update4(float4& p, const float4& g, float4& m, float4& v, const GsrAdamEntry& e) {
    adam_update(p.x, g.x, m.x, v.x, e);
    adam_update(p.y, g.y, m.y, v.y, e);
    adam_update(p.z, g.z, m.z, v.z, e);
    adam_update(p.w, g.w, m.w, v.w, e);
}

// DYN (b200gsr_adam_step_dyn): the table of b200gsr_adam_step plus, per entry, the row of the device scalar array
// [n, 6] that holds its six scalars, so that a CUDA graph replays with the step's learning rate and bias corrections.
struct GsrAdamDynTable {
    GsrAdamTable t;
    const float* scalars;
    int row[B200GSR_ADAM_MAX_TENSORS];   // entries skip empty tensors, rows do not
};

// One CTA = one GSR_ADAM_CHUNK-element chunk of one tensor.  The vector path issues all of a thread's loads
// (4 x 4 float4) before the first use, so each thread keeps 256 bytes in flight.
__device__ __forceinline__ void adam_chunk(const GsrAdamEntry& e) {
    const GsrAdamChunk c = gsr_adam_chunk(e, blockIdx.x);
    if (c.vend > c.start) {
        const int nv = (int)((c.vend - c.start) >> 2);
        float4* p4 = reinterpret_cast<float4*>(e.p + c.start);
        const float4* g4 = reinterpret_cast<const float4*>(e.g + c.start);
        float4* m4 = reinterpret_cast<float4*>(e.m + c.start);
        float4* v4 = reinterpret_cast<float4*>(e.v + c.start);
        float4 P[GSR_ADAM_VEC], G[GSR_ADAM_VEC], Mv[GSR_ADAM_VEC], V[GSR_ADAM_VEC];
#pragma unroll
        for (int k = 0; k < GSR_ADAM_VEC; ++k) {
            const int j = k * GSR_ADAM_THREADS + threadIdx.x;
            if (j < nv) { P[k] = p4[j]; G[k] = __ldg(g4 + j); Mv[k] = m4[j]; V[k] = v4[j]; }
        }
#pragma unroll
        for (int k = 0; k < GSR_ADAM_VEC; ++k) {
            const int j = k * GSR_ADAM_THREADS + threadIdx.x;
            if (j < nv) {
                adam_update4(P[k], G[k], Mv[k], V[k], e);
                p4[j] = P[k]; m4[j] = Mv[k]; v4[j] = V[k];
            }
        }
    }
    for (long long i = c.vend + threadIdx.x; i < c.end; i += GSR_ADAM_THREADS) {
        float p = e.p[i], m = e.m[i], v = e.v[i];
        adam_update(p, __ldg(e.g + i), m, v, e);
        e.p[i] = p; e.m[i] = m; e.v[i] = v;
    }
}

// DYN: each CTA loads its entry's six scalars from device memory once, in place of the table's.
template <bool DYN = false>
__global__ void __launch_bounds__(GSR_ADAM_THREADS)
adam_step_kernel(const __grid_constant__ std::conditional_t<DYN, GsrAdamDynTable, GsrAdamTable> tab) {
    if constexpr (DYN) {
        const int k = gsr_adam_find(tab.t, blockIdx.x);
        GsrAdamEntry e = tab.t.e[k];
        const float* s = tab.scalars + 6 * (size_t)tab.row[k];
        e.w = __ldg(s); e.beta2 = __ldg(s + 1); e.omb2 = __ldg(s + 2); e.eps = __ldg(s + 3);
        e.step_size = __ldg(s + 4); e.bc2_sqrt = __ldg(s + 5);
        adam_chunk(e);
    } else {
        adam_chunk(tab.e[gsr_adam_find(tab, blockIdx.x)]);
    }
}

}  // namespace

cudaError_t gsr_launch_adam(int n, const b200gsr_adam_tensor* t, cudaStream_t s) {
    GsrAdamTable tab;
    const long long blocks = gsr_adam_plan(n, t, &tab);
    if (blocks == 0) return cudaSuccess;
    if (blocks > 0x7fffffffLL) return cudaErrorInvalidConfiguration;
    adam_step_kernel<<<(unsigned)blocks, GSR_ADAM_THREADS, 0, s>>>(tab);
    return cudaGetLastError();
}

cudaError_t gsr_launch_adam_dyn(int n, const b200gsr_adam_tensor* t, const float* scalars, cudaStream_t s) {
    GsrAdamDynTable tab;
    const long long blocks = gsr_adam_plan(n, t, &tab.t);
    if (blocks == 0) return cudaSuccess;
    if (blocks > 0x7fffffffLL) return cudaErrorInvalidConfiguration;
    tab.scalars = scalars;
    for (int i = 0, k = 0; i < n; ++i)
        if (t[i].n > 0) tab.row[k++] = i;
    adam_step_kernel<true><<<(unsigned)blocks, GSR_ADAM_THREADS, 0, s>>>(tab);
    return cudaGetLastError();
}
