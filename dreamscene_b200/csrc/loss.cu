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

// ---- the guidance stages' regularisers (DESIGN.md §0 f10) ----------------------------------------------------------
// Total variation, tv(x) = 2 (h_tv / (C (H-1) W) + w_tv / (C H (W-1))) / B, and its gradient as torch's CUDA autograd
// computes it for an incoming g:
//   DivBackward (/ B), MulBackward (2 *)      g2 = 2 fp32(g * fp32(1 / B))       div by a CPU scalar: reciprocal multiply
//   DivBackward (/ count), PowBackward        ch = fp32(fp32(g2 * fp32(1 / count_h)) * fp32(2 dh)), cw likewise
//   SubBackward, SliceBackward                +c at the minuend, -c at the subtrahend, zero padded (+0)
//   the input's gradient buffer               ((w+ + w-) + h-) + h+, autograd's arrival order
// with w+ = +cw at [..., 1:], w- = -cw at [..., :-1], h+ / h- likewise along H.
// Scale loss, mean(mean(scales, -1)): MeanBackward0 then MeanBackward1 give every element fp32(fp32(g * fp32(1 / rows))
// * fp32(1 / 3)).
namespace {

// Fixed-order sums of two doubles per thread; the results are valid in thread 0.
__device__ __forceinline__ void block_sum2(double& a, double& b) {
    __shared__ double2 warp_sum[GSR_L2_THREADS / 32];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        a += __shfl_down_sync(0xffffffffu, a, o);
        b += __shfl_down_sync(0xffffffffu, b, o);
    }
    if ((threadIdx.x & 31) == 0) warp_sum[threadIdx.x >> 5] = make_double2(a, b);
    __syncthreads();
    if (threadIdx.x == 0) {
        a = 0.0; b = 0.0;
        for (int w = 0; w < GSR_L2_THREADS / 32; ++w) { a += warp_sum[w].x; b += warp_sum[w].y; }
    }
}

// V consecutive elements of row i starting at column j (zeros for an inactive lane)
template <int V>
__device__ __forceinline__ void load_row(const float* p, float (&v)[V], bool act) {
    if constexpr (V == 4) {
        const float4 q = act ? __ldg(reinterpret_cast<const float4*>(p)) : make_float4(0.f, 0.f, 0.f, 0.f);
        v[0] = q.x; v[1] = q.y; v[2] = q.z; v[3] = q.w;
    } else {
        v[0] = act ? __ldg(p) : 0.0f;
    }
}

// c = fp32(gs * fp32(2 (hi - lo))), one term of the gradient
__device__ __forceinline__ float tv_term(float gs, float hi, float lo) {
    return __fmul_rn(gs, __fmul_rn(2.0f, __fsub_rn(hi, lo)));
}

// grid gsr_tv_blocks(planes, H, W, V): warp task t covers rows [band 8, band 8 + 8) and columns [(chunk 32 + lane) V,
// + V) of one plane, with the band's rows and a halo row above and below loaded into registers first; the left /
// right neighbours come from the adjacent lanes, or from memory at the warp's edges.  V = 4 needs W % 4 == 0 and x, d_x 16-byte aligned.
template <int V>
__global__ void __launch_bounds__(GSR_L2_THREADS) tv_kernel(const GsrTvArgs a) {
    const int lane = threadIdx.x & 31;
    const int H = a.H, W = a.W;
    const int nchunk = (W + 32 * V - 1) / (32 * V);
    const int nband = (H + GSR_TV_ROWS - 1) / GSR_TV_ROWS;
    const long long task = (long long)blockIdx.x * (GSR_L2_THREADS / 32) + (threadIdx.x >> 5);
    double sh = 0.0, sw = 0.0;
    if (task < (long long)a.planes * nband * nchunk) {          // warp-uniform
        const int chunk = (int)(task % nchunk);
        const int band = (int)((task / nchunk) % nband);
        const long long plane = task / ((long long)nchunk * nband);
        const int j0 = (chunk * 32 + lane) * V;
        const bool act = j0 < W;
        const float* xp = a.x + plane * H * W;
        float* dp = a.d_x ? a.d_x + plane * H * W : nullptr;
        float gh = 0.0f, gw = 0.0f;
        if (dp) {
            const float g2 = __fmul_rn(2.0f, __fmul_rn(__ldg(a.grad_out), a.inv_b));
            gh = __fmul_rn(g2, a.inv_h);
            gw = __fmul_rn(g2, a.inv_w);
        }
        const int r0 = band * GSR_TV_ROWS;
        float xs[GSR_TV_ROWS + 2][V];       // rows r0 - 1 .. r0 + GSR_TV_ROWS, all loads in flight at once
#pragma unroll
        for (int r = 0; r < GSR_TV_ROWS + 2; ++r) {
            const int i = r0 - 1 + r;
            load_row<V>(xp + (long long)min(max(i, 0), H - 1) * W + j0, xs[r], act && i >= 0 && i < H);
        }
#pragma unroll
        for (int r = 1; r <= GSR_TV_ROWS; ++r) {
            const int i = r0 - 1 + r;
            if (i >= H) break;                                  // warp-uniform
            const float(&up)[V] = xs[r - 1];
            const float(&cur)[V] = xs[r];
            const float(&dn)[V] = xs[r + 1];
            const float* row = xp + (long long)i * W;
            float xl = __shfl_up_sync(0xffffffffu, cur[V - 1], 1);
            float xr = __shfl_down_sync(0xffffffffu, cur[0], 1);
            if (lane == 0 && act && j0 > 0) xl = __ldg(row + j0 - 1);
            if (lane == 31 && j0 + V < W) xr = __ldg(row + j0 + V);
            if (act) {
                float d[V];
#pragma unroll
                for (int k = 0; k < V; ++k) {
                    const int j = j0 + k;
                    const float left = k > 0 ? cur[k - 1] : xl;
                    const float right = k < V - 1 ? cur[k + 1] : xr;
                    if (a.loss_out) {
                        if (i + 1 < H) { const float e = __fsub_rn(dn[k], cur[k]); sh += (double)__fmul_rn(e, e); }
                        if (j + 1 < W) { const float e = __fsub_rn(right, cur[k]); sw += (double)__fmul_rn(e, e); }
                    }
                    if (dp) {
                        const float wp = j > 0 ? tv_term(gw, cur[k], left) : 0.0f;
                        const float wm = j + 1 < W ? -tv_term(gw, right, cur[k]) : 0.0f;
                        const float hm = i + 1 < H ? -tv_term(gh, dn[k], cur[k]) : 0.0f;
                        const float hp = i > 0 ? tv_term(gh, cur[k], up[k]) : 0.0f;
                        d[k] = __fadd_rn(__fadd_rn(__fadd_rn(wp, wm), hm), hp);
                    }
                }
                if (dp) {
                    float* o = dp + (long long)i * W + j0;
                    if constexpr (V == 4) {
                        float4 q = make_float4(d[0], d[1], d[2], d[3]);
                        if (a.accumulate) {
                            const float4 p = *reinterpret_cast<const float4*>(o);
                            q = make_float4(__fadd_rn(p.x, q.x), __fadd_rn(p.y, q.y), __fadd_rn(p.z, q.z),
                                            __fadd_rn(p.w, q.w));
                        }
                        *reinterpret_cast<float4*>(o) = q;
                    } else {
                        o[0] = a.accumulate ? __fadd_rn(o[0], d[0]) : d[0];
                    }
                }
            }
        }
    }
    if (a.loss_out) {
        block_sum2(sh, sw);
        if (threadIdx.x == 0) { a.partials[2 * blockIdx.x] = sh; a.partials[2 * blockIdx.x + 1] = sw; }
    }
}

// one CTA: the (h, w) partials summed in a fixed order, then the value in double, rounded once
__global__ void __launch_bounds__(GSR_L2_THREADS) tv_finish_kernel(const GsrTvArgs a, int nblk) {
    double h = 0.0, w = 0.0;
    for (int i = threadIdx.x; i < nblk; i += GSR_L2_THREADS) { h += a.partials[2 * i]; w += a.partials[2 * i + 1]; }
    block_sum2(h, w);
    if (threadIdx.x == 0) *a.loss_out = __double2float_rn(2.0 * (h / a.count_h + w / a.count_w) / (double)a.B);
}

// grid gsr_l2_blocks(3 rows): CTA b owns elements [b CHUNK, min((b + 1) CHUNK, n)); float4 path when scales and
// d_scales are 16-byte aligned, the < 4-element tail and unaligned buffers take the scalar loop.  The gradient is one
// constant and reads nothing but d_scales when accumulating.
__global__ void __launch_bounds__(GSR_L2_THREADS) scale_loss_kernel(const GsrScaleArgs a) {
    const long long n = 3LL * a.rows;
    const long long start = (long long)blockIdx.x * GSR_L2_CHUNK;
    const long long end = start + GSR_L2_CHUNK < n ? start + GSR_L2_CHUNK : n;
    float* ds = a.d_scales;
    const float c = ds ? __fmul_rn(__fmul_rn(__ldg(a.grad_out), a.inv_rows), a.inv_3) : 0.0f;
    double acc = 0.0;
    long long i0 = start;
    if (((reinterpret_cast<uintptr_t>(a.scales) | reinterpret_cast<uintptr_t>(ds)) & 15) == 0) {
        const long long q0 = start >> 2;
        const int nv = (int)((end - start) >> 2);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const int j = k * GSR_L2_THREADS + threadIdx.x;
            if (j < nv) {
                if (a.loss_out) {
                    const float4 s = __ldg(reinterpret_cast<const float4*>(a.scales) + q0 + j);
                    acc += ((double)s.x + (double)s.y) + ((double)s.z + (double)s.w);
                }
                if (ds) {
                    float4* o = reinterpret_cast<float4*>(ds) + q0 + j;
                    float4 q = make_float4(c, c, c, c);
                    if (a.accumulate) {
                        const float4 p = *o;
                        q = make_float4(__fadd_rn(p.x, c), __fadd_rn(p.y, c), __fadd_rn(p.z, c), __fadd_rn(p.w, c));
                    }
                    *o = q;
                }
            }
        }
        i0 = start + 4LL * nv;
    }
    for (long long i = i0 + threadIdx.x; i < end; i += GSR_L2_THREADS) {
        if (a.loss_out) acc += (double)__ldg(a.scales + i);
        if (ds) ds[i] = a.accumulate ? __fadd_rn(ds[i], c) : c;
    }
    if (a.loss_out) {
        const double s = block_sum(acc);
        if (threadIdx.x == 0) a.partials[blockIdx.x] = s;
    }
}

__global__ void __launch_bounds__(GSR_L2_THREADS) scale_finish_kernel(const GsrScaleArgs a, int nblk) {
    double s = 0.0;
    for (int i = threadIdx.x; i < nblk; i += GSR_L2_THREADS) s += a.partials[i];
    s = block_sum(s);
    if (threadIdx.x == 0) *a.loss_out = __double2float_rn(s / (3.0 * (double)a.rows));
}

// b200gsr_scale_loss_live: the live rows' count of group g, clamped to its capacity
__device__ __forceinline__ int scale_live_rows(const GsrScaleLiveArgs& a, int g) {
    return min(max(__ldg(a.live + g), 0), a.start[g + 1] - a.start[g]);
}
// fp32(1 / (B sum(live))) as the host forms fp32(1 / rows) for the compact layout
__device__ __forceinline__ float scale_live_inv_rows(const GsrScaleLiveArgs& a, long long& rows) {
    long long n = 0;
    for (int g = 0; g < a.num_groups; ++g) n += scale_live_rows(a, g);
    rows = (long long)a.B * n;
    return __fdiv_rn(1.0f, (float)rows);
}

// The scalar path of scale_loss_kernel over the live elements only (rows over the groups' capacities); a dead
// element adds nothing to the sum and gets a zero gradient (left as it is when accumulating).
__global__ void __launch_bounds__(GSR_L2_THREADS) scale_loss_live_kernel(const GsrScaleLiveArgs a) {
    const long long n = 3LL * a.rows;
    const long long start = (long long)blockIdx.x * GSR_L2_CHUNK;
    const long long end = start + GSR_L2_CHUNK < n ? start + GSR_L2_CHUNK : n;
    float* ds = a.d_scales;
    long long rows;
    const float inv_rows = scale_live_inv_rows(a, rows);
    const float c = ds ? __fmul_rn(__fmul_rn(__ldg(a.grad_out), inv_rows), a.inv_3) : 0.0f;
    double acc = 0.0;
    for (long long i = start + threadIdx.x; i < end; i += GSR_L2_THREADS) {
        const int r = (int)((i / 3) % a.P);
        int g = 0;
        while (g + 1 < a.num_groups && r >= a.start[g + 1]) ++g;
        const bool alive = r - a.start[g] < scale_live_rows(a, g);
        if (a.loss_out && alive) acc += (double)__ldg(a.scales + i);
        if (ds && alive) ds[i] = a.accumulate ? __fadd_rn(ds[i], c) : c;
        else if (ds && !a.accumulate) ds[i] = 0.0f;
    }
    if (a.loss_out) {
        const double s = block_sum(acc);
        if (threadIdx.x == 0) a.partials[blockIdx.x] = s;
    }
}

__global__ void __launch_bounds__(GSR_L2_THREADS) scale_finish_live_kernel(const GsrScaleLiveArgs a, int nblk) {
    double s = 0.0;
    for (int i = threadIdx.x; i < nblk; i += GSR_L2_THREADS) s += a.partials[i];
    s = block_sum(s);
    long long rows;
    scale_live_inv_rows(a, rows);
    if (threadIdx.x == 0) *a.loss_out = __double2float_rn(s / (3.0 * (double)rows));
}

}  // namespace

cudaError_t gsr_launch_scale_loss_live(const GsrScaleLiveArgs& a, cudaStream_t s) {
    const int nblk = (int)gsr_l2_blocks(3 * a.rows);
    scale_loss_live_kernel<<<nblk, GSR_L2_THREADS, 0, s>>>(a);
    if (a.loss_out) scale_finish_live_kernel<<<1, GSR_L2_THREADS, 0, s>>>(a, nblk);
    return cudaGetLastError();
}

cudaError_t gsr_launch_tv_loss(const GsrTvArgs& a, cudaStream_t s) {
    const bool vec = a.W % 4 == 0 &&
                     ((reinterpret_cast<uintptr_t>(a.x) | reinterpret_cast<uintptr_t>(a.d_x)) & 15) == 0;
    const int nblk = (int)gsr_tv_blocks(a.planes, a.H, a.W, vec ? 4 : 1);
    if (vec) tv_kernel<4><<<nblk, GSR_L2_THREADS, 0, s>>>(a);
    else tv_kernel<1><<<nblk, GSR_L2_THREADS, 0, s>>>(a);
    if (a.loss_out) tv_finish_kernel<<<1, GSR_L2_THREADS, 0, s>>>(a, nblk);
    return cudaGetLastError();
}

cudaError_t gsr_launch_scale_loss(const GsrScaleArgs& a, cudaStream_t s) {
    const int nblk = (int)gsr_l2_blocks(3 * a.rows);
    scale_loss_kernel<<<nblk, GSR_L2_THREADS, 0, s>>>(a);
    if (a.loss_out) scale_finish_kernel<<<1, GSR_L2_THREADS, 0, s>>>(a, nblk);
    return cudaGetLastError();
}
