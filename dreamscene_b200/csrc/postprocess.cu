// Depth/alpha -> normalised disparity (SURVEY.md 8 f1, second half): the post-processing DreamScene runs
// after every render (/root/reference/scene_gaussian.py:871-881)
//     depth, alpha = chunk(depth_alpha, 2)
//     disp  = focal / (depth + alpha * 10 + 1e-5)
//     min_d = disp[alpha <= 0.1].min()        # falls back to disp.min() when no pixel is opaque
//     disp  = clamp((disp - min_d) / (disp.max() - min_d), 0, 1)
// as two small kernels forward and two backward, for a batch of views, with NO host synchronisation
// (the boolean-mask indexing above forces a device->host copy of the mask population per view).
// Gradients follow torch autograd exactly: through the quotient, through min_d and disp.max()
// (evenly distributed over ties, as torch.min()/max() do) and through the clamp (pass-through on
// the closed interval).
#include "common.cuh"
#include "../../include/b200gsr_frames.h"

namespace {

// per-view reduction record (device memory, zero/identity-initialised by the first kernel's view-0 block? no:
// by a dedicated tiny init in the launcher via cudaMemsetAsync-free pattern: the reduce kernel for
// block 0 cannot know it runs first, so the record is initialised by reduce_init_kernel)
struct DispStats {
    unsigned int min_masked;   // float bits (disparities are positive: bit order == value order)
    unsigned int min_all;
    unsigned int max_all;
    unsigned int n_masked;
    // backward
    float sum_min, sum_max;    // sum_j dt_j (d_j - M)/(M-m)^2   and   sum_j -dt_j (d_j - m)/(M-m)^2
    unsigned int ties_min, ties_max;
};
static_assert(sizeof(DispStats) == 32, "stats record is 8 words");
static_assert(sizeof(DispStats) == B200GSR_FRAMES_STATS_BYTES, "b200gsr_frames' scratch is one record per view");

__global__ void disp_init_kernel(DispStats* st, int B) {
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v < B) {
        st[v].min_masked = 0x7f800000u; st[v].min_all = 0x7f800000u; st[v].max_all = 0u; st[v].n_masked = 0u;
        st[v].sum_min = 0.f; st[v].sum_max = 0.f; st[v].ties_min = 0u; st[v].ties_max = 0u;
    }
}

__device__ __forceinline__ float disp_raw(float depth, float alpha, float focal) {
    return __fdiv_rn(focal, __fadd_rn(__fadd_rn(depth, __fmul_rn(alpha, 10.0f)), 1e-5f));
}

// One block's share of view v's statistics over its N contiguous depth and alpha values (blockDim 256, grid x strided)
__device__ __forceinline__ void disp_reduce_view(const float* __restrict__ depth, const float* __restrict__ alpha,
                                                 const float f, int N, DispStats* st, int v) {
    unsigned int mm = 0x7f800000u, ma = 0x7f800000u, mx = 0u, nm = 0u;
    for (int i = blockIdx.x * 256 + threadIdx.x; i < N; i += gridDim.x * 256) {
        const float a = alpha[i];
        const unsigned int d = __float_as_uint(disp_raw(depth[i], a, f));
        ma = min(ma, d); mx = max(mx, d);
        if (a <= 0.1f) { mm = min(mm, d); ++nm; }
    }
    mm = __reduce_min_sync(0xffffffffu, mm); ma = __reduce_min_sync(0xffffffffu, ma);
    mx = __reduce_max_sync(0xffffffffu, mx); nm = __reduce_add_sync(0xffffffffu, nm);
    if ((threadIdx.x & 31) == 0) {
        atomicMin(&st[v].min_masked, mm); atomicMin(&st[v].min_all, ma); atomicMax(&st[v].max_all, mx);
        if (nm) atomicAdd(&st[v].n_masked, nm);
    }
}

// depth_alpha: [B][2][N]; grid (blocks, B)
__global__ void __launch_bounds__(256)
disp_reduce_kernel(const float* __restrict__ da, const float* __restrict__ focal, int N, DispStats* st) {
    const int v = blockIdx.y;
    const float* depth = da + (size_t)v * 2 * N;
    disp_reduce_view(depth, depth + N, focal[v], N, st, v);
}

__device__ __forceinline__ void disp_bounds(const DispStats& s, float& m, float& M) {
    m = __uint_as_float(s.n_masked > 0 ? s.min_masked : s.min_all);
    M = __uint_as_float(s.max_all);
}

__device__ __forceinline__ float disp_norm(float d, float m, float den) {
    const float t = __fdiv_rn(__fsub_rn(d, m), den);
    return fminf(fmaxf(t, 0.0f), 1.0f);       // NaN (den == 0) propagates like torch.clamp
}

__global__ void __launch_bounds__(256)
disp_normalise_kernel(const float* __restrict__ da, const float* __restrict__ focal, int N,
                      const DispStats* __restrict__ st, float* __restrict__ out) {
    const int v = blockIdx.y;
    const float* depth = da + (size_t)v * 2 * N;
    const float* alpha = depth + N;
    float m, M;
    disp_bounds(st[v], m, M);
    const float f = focal[v];
    const float den = __fsub_rn(M, m);
    for (int i = blockIdx.x * 256 + threadIdx.x; i < N; i += gridDim.x * 256) {
        const float d = disp_raw(depth[i], alpha[i], f);
        out[(size_t)v * N + i] = disp_norm(d, m, den);
    }
}

// ---- 8-bit video frames (b200gsr_frames).  The views come straight from a stacked forward's outputs, color
// [3][Hs][W] and depth_alpha [2][Hs][W]: view v's H*W pixels are contiguous from row v*Hp (Hp = Hs / B), so its
// pixel i of channel c is at c*Hs*W + v*Hp*W + i.  The reference quantises a frame as
//     rgb   = (clamp(color, 0, 1) * 255).round().astype(uint8)                         (float32, round half even)
//     depth = (clamp(disp / disp.max(), 0, 1) * 255).round().astype(uint8)    disp = disp_normalise_kernel's value
// where the cast of a NaN is undefined in numpy; here a NaN becomes 0 (fmaxf returns the non-NaN operand).

// the statistics of disp_reduce_kernel over the stacked layout; grid (blocks, B)
__global__ void __launch_bounds__(256)
frames_stats_kernel(const float* __restrict__ da, const float* __restrict__ focal, int HW, size_t view_stride,
                    size_t chan_stride, DispStats* st) {
    const int v = blockIdx.y;
    const float* depth = da + v * view_stride;
    disp_reduce_view(depth, depth + chan_stride, focal[v], HW, st, v);
}

__device__ __forceinline__ unsigned int quantise8(float x) {
    return (unsigned int)rintf(__fmul_rn(fminf(fmaxf(x, 0.0f), 1.0f), 255.0f));
}

// One thread per 4 consecutive pixels of the B views (flattened view-major, as rgb8 [B,H,W,3] / depth8 [B,H,W,1]):
// three 32-bit stores of packed RGB and one of depth.  The last B*H*W % 4 pixels are stored byte by byte.
__global__ void __launch_bounds__(256)
frames_kernel(int B, int HW, size_t view_stride, size_t chan_stride, const float* __restrict__ color,
              const float* __restrict__ da, const float* __restrict__ focal, const DispStats* __restrict__ st,
              uint8_t* __restrict__ rgb8, uint8_t* __restrict__ depth8) {
    __shared__ float s_m[B200GSR_MAX_VIEWS], s_den[B200GSR_MAX_VIEWS], s_max[B200GSR_MAX_VIEWS], s_f[B200GSR_MAX_VIEWS];
    if (threadIdx.x < B) {
        const int v = threadIdx.x;
        float m, M;
        disp_bounds(st[v], m, M);
        const float den = __fsub_rn(M, m);
        s_m[v] = m; s_den[v] = den; s_f[v] = focal[v];
        // max over the view of disp_norm(d): disp_norm is non-decreasing in d and M is attained, so it is
        // disp_norm(M) - 1 for M > m, 0 when den is 0 or NaN (every pixel is then 0, and 0 / 0 quantises to 0)
        s_max[v] = disp_norm(M, m, den);
    }
    __syncthreads();
    const int total = B * HW;
    for (int q = blockIdx.x * blockDim.x + threadIdx.x; 4 * q < total; q += gridDim.x * blockDim.x) {
        const int p0 = 4 * q;
        int v = p0 / HW, i = p0 - v * HW;
        unsigned int rgb[4], dep[4];
        const int n = min(4, total - p0);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            rgb[k] = dep[k] = 0u;
            if (k < n) {
                while (i >= HW) { i -= HW; ++v; }
                const size_t o = v * view_stride + i;
                rgb[k] = quantise8(color[o]) | quantise8(color[o + chan_stride]) << 8 |
                         quantise8(color[o + 2 * chan_stride]) << 16;
                const float t = disp_norm(disp_raw(da[o], da[o + chan_stride], s_f[v]), s_m[v], s_den[v]);
                dep[k] = quantise8(__fdiv_rn(t, s_max[v]));
                ++i;
            }
        }
        if (n == 4) {
            uint32_t* w = reinterpret_cast<uint32_t*>(rgb8 + 12 * (size_t)q);
            w[0] = rgb[0] | rgb[1] << 24;
            w[1] = rgb[1] >> 8 | rgb[2] << 16;
            w[2] = rgb[2] >> 16 | rgb[3] << 8;
            reinterpret_cast<uint32_t*>(depth8)[q] = dep[0] | dep[1] << 8 | dep[2] << 16 | dep[3] << 24;
        } else {
            for (int k = 0; k < n; ++k) {
                uint8_t* px = rgb8 + 3 * (size_t)(p0 + k);
                px[0] = (uint8_t)rgb[k]; px[1] = (uint8_t)(rgb[k] >> 8); px[2] = (uint8_t)(rgb[k] >> 16);
                depth8[p0 + k] = (uint8_t)dep[k];
            }
        }
    }
}

// backward pass 1: the two global sums feeding the min / max paths, and the tie counts.
// DET (deterministic mode): instead of float atomics, each block writes its two sums - its warps' sums added in
// warp order - to part[2 * (v * gridDim.x + blockIdx.x)], and disp_bwd_sum_kernel adds them up in block order.
template <bool DET>
__global__ void __launch_bounds__(256)
disp_bwd_reduce_kernel(const float* __restrict__ da, const float* __restrict__ focal, int N,
                       const float* __restrict__ g_out, DispStats* st, float* __restrict__ part) {
    const int v = blockIdx.y;
    const float* depth = da + (size_t)v * 2 * N;
    const float* alpha = depth + N;
    float m, M;
    disp_bounds(st[v], m, M);
    const bool masked_min = st[v].n_masked > 0;
    const float f = focal[v];
    const float den = M - m, inv2 = 1.0f / (den * den);
    float sm = 0.f, sM = 0.f;
    unsigned int tm = 0u, tM = 0u;
    for (int i = blockIdx.x * 256 + threadIdx.x; i < N; i += gridDim.x * 256) {
        const float a = alpha[i];
        const float d = disp_raw(depth[i], a, f);
        const float t = (d - m) / den;
        const float dt = (t >= 0.0f && t <= 1.0f) ? g_out[(size_t)v * N + i] : 0.0f;
        sm += dt * (d - M) * inv2;
        sM -= dt * (d - m) * inv2;
        if (d == m && (!masked_min || a <= 0.1f)) ++tm;
        if (d == M) ++tM;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        sm += __shfl_xor_sync(0xffffffffu, sm, o);
        sM += __shfl_xor_sync(0xffffffffu, sM, o);
    }
    tm = __reduce_add_sync(0xffffffffu, tm); tM = __reduce_add_sync(0xffffffffu, tM);
    if ((threadIdx.x & 31) == 0) {
        if (!DET) { atomicAdd(&st[v].sum_min, sm); atomicAdd(&st[v].sum_max, sM); }
        if (tm) atomicAdd(&st[v].ties_min, tm);       // integer counts: exact in any order
        if (tM) atomicAdd(&st[v].ties_max, tM);
    }
    if (DET) {
        __shared__ float ws[2][8];
        if ((threadIdx.x & 31) == 0) { ws[0][threadIdx.x >> 5] = sm; ws[1][threadIdx.x >> 5] = sM; }
        __syncthreads();
        if (threadIdx.x == 0) {
            float bm = 0.f, bM = 0.f;
            for (int w = 0; w < 8; ++w) { bm += ws[0][w]; bM += ws[1][w]; }
            float* o = part + 2 * ((size_t)v * gridDim.x + blockIdx.x);
            o[0] = bm; o[1] = bM;
        }
    }
}

// deterministic backward, between the two passes: one warp per view adds the block sums in a fixed order
__global__ void __launch_bounds__(32)
disp_bwd_sum_kernel(int nblk, const float* __restrict__ part, DispStats* st) {
    const int v = blockIdx.x, lane = threadIdx.x;
    const float* p = part + 2 * (size_t)v * nblk;
    float sm = 0.f, sM = 0.f;
    for (int b = lane; b < nblk; b += 32) { sm += p[2 * b]; sM += p[2 * b + 1]; }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        sm += __shfl_xor_sync(0xffffffffu, sm, o);
        sM += __shfl_xor_sync(0xffffffffu, sM, o);
    }
    if (lane == 0) { st[v].sum_min += sm; st[v].sum_max += sM; }
}

// backward pass 2: d depth_alpha = chain through d = focal / x, x = depth + 10 alpha + 1e-5 (+ the caller's own
// gradient on the alpha channel, which is returned alongside the disparity)
__global__ void __launch_bounds__(256)
disp_bwd_apply_kernel(const float* __restrict__ da, const float* __restrict__ focal, int N,
                      const float* __restrict__ g_out, const float* __restrict__ g_alpha,
                      const DispStats* __restrict__ st, float* __restrict__ d_da) {
    const int v = blockIdx.y;
    const float* depth = da + (size_t)v * 2 * N;
    const float* alpha = depth + N;
    float m, M;
    disp_bounds(st[v], m, M);
    const bool masked_min = st[v].n_masked > 0;
    const float f = focal[v];
    const float den = M - m, inv = 1.0f / den;
    const float gmin = st[v].ties_min ? st[v].sum_min / (float)st[v].ties_min : 0.0f;
    const float gmax = st[v].ties_max ? st[v].sum_max / (float)st[v].ties_max : 0.0f;
    for (int i = blockIdx.x * 256 + threadIdx.x; i < N; i += gridDim.x * 256) {
        const float a = alpha[i];
        const float d = disp_raw(depth[i], a, f);
        const float t = (d - m) * inv;
        float gd = (t >= 0.0f && t <= 1.0f) ? g_out[(size_t)v * N + i] * inv : 0.0f;
        if (d == m && (!masked_min || a <= 0.1f)) gd += gmin;
        if (d == M) gd += gmax;
        const float gx = -gd * d * d / f;                     // d(focal/x)/dx = -d^2/focal
        d_da[(size_t)v * 2 * N + i] = gx;
        d_da[(size_t)v * 2 * N + N + i] = 10.0f * gx + (g_alpha ? g_alpha[(size_t)v * N + i] : 0.0f);
    }
}

}  // namespace

cudaError_t gsr_launch_disparity_fwd(int B, int N, const float* da, const float* focal, float* out, void* stats,
                                     int num_sms, cudaStream_t s) {
    if (B <= 0 || N <= 0) return cudaSuccess;
    DispStats* st = static_cast<DispStats*>(stats);
    disp_init_kernel<<<(B + 63) / 64, 64, 0, s>>>(st, B);
    const int bx = max(1, min((N + 255) / 256, (num_sms * 8 + B - 1) / B));
    disp_reduce_kernel<<<dim3(bx, B), 256, 0, s>>>(da, focal, N, st);
    disp_normalise_kernel<<<dim3(bx, B), 256, 0, s>>>(da, focal, N, st, out);
    return cudaGetLastError();
}

cudaError_t gsr_launch_frames(int B, int H, int W, int Hs, const float* color, const float* da, const float* focal,
                              uint8_t* rgb8, uint8_t* depth8, void* stats, int num_sms, cudaStream_t s) {
    const int HW = H * W;
    const size_t view_stride = (size_t)(Hs / B) * W, chan_stride = (size_t)Hs * W;
    DispStats* st = static_cast<DispStats*>(stats);
    disp_init_kernel<<<(B + 63) / 64, 64, 0, s>>>(st, B);
    const int bx = max(1, min((HW + 255) / 256, (num_sms * 8 + B - 1) / B));
    frames_stats_kernel<<<dim3(bx, B), 256, 0, s>>>(da, focal, HW, view_stride, chan_stride, st);
    const int quads = (B * HW + 3) / 4;
    frames_kernel<<<max(1, min((quads + 255) / 256, num_sms * 8)), 256, 0, s>>>(B, HW, view_stride, chan_stride, color,
                                                                                 da, focal, st, rgb8, depth8);
    return cudaGetLastError();
}

cudaError_t gsr_launch_disparity_bwd(int B, int N, const float* da, const float* focal, const float* g_out,
                                     const float* g_alpha, void* stats, float* d_da, bool deterministic, int num_sms,
                                     cudaStream_t s) {
    if (B <= 0 || N <= 0) return cudaSuccess;
    DispStats* st = static_cast<DispStats*>(stats);
    const int bx = max(1, min((N + 255) / 256, (num_sms * 8 + B - 1) / B));
    if (deterministic) {
        // the block sums (2 * bx <= 2N floats per view) live in d_da until disp_bwd_apply_kernel overwrites it
        disp_bwd_reduce_kernel<true><<<dim3(bx, B), 256, 0, s>>>(da, focal, N, g_out, st, d_da);
        disp_bwd_sum_kernel<<<B, 32, 0, s>>>(bx, d_da, st);
    } else {
        disp_bwd_reduce_kernel<false><<<dim3(bx, B), 256, 0, s>>>(da, focal, N, g_out, st, nullptr);
    }
    disp_bwd_apply_kernel<<<dim3(bx, B), 256, 0, s>>>(da, focal, N, g_out, g_alpha, st, d_da);
    return cudaGetLastError();
}
