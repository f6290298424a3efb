// Densification / pruning (SURVEY.md 8 f4): the index surgery DreamScene runs every 100 steps
// (/root/reference/gs_renderer.py:854-1087) and the important-score percentile prune
// (gs_renderer.py:1076-1081, scene_gaussian.py:1046-1103), as a handful of kernels instead of
// ~60 boolean-index / cat / repeat ops (each `x[mask]` is a nonzero() with a device->host copy
// of the count) over 6 parameters, 12 Adam moments and 3 statistics arrays.
//
//   densify_stats     add_densification_stats + the max_radii2D update (object_trainer.py:385-390)
//   densify_classify  per-Gaussian decisions of densify_and_prune, in the reference's order
//                     (clone -> split -> prune, including that the stats arrays are reset in between,
//                     so the screen-size criterion never fires inside densify_and_prune)
//   gsr_scan_u32      exclusive prefix sum (two-level; fields.cu uses it too)
//   densify_map       decisions + scans -> source map of the NEW point set, in the reference's
//                     output order [kept originals | clones | split children (N blocks)]
//   gather_rows       out[p,:] = in[src[p],:]  (or zeros for appended rows: Adam moments, stats)
//   split_children    positions / log-scales of the split children from the caller's normal draws
//   kth_smallest      radix select on float bits (the percentile of prune_gaussians without a sort)
#include "common.cuh"

namespace {

enum { kKeep = 0, kClone = 1, kChild = 2, kSplitSel = 3 };   // the four flag planes [4][P]

__global__ void densify_stats_kernel(int P, const float* __restrict__ vs_grad, const int32_t* __restrict__ radii,
                                     float* __restrict__ accum, float* __restrict__ denom, float* __restrict__ max_radii) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    const int r = radii[i];
    if (r <= 0) return;                                   // visibility_filter = radii > 0
    const float gx = vs_grad[3 * (size_t)i], gy = vs_grad[3 * (size_t)i + 1];
    accum[i] += gsr_screen_grad_norm(gx, gy);             // torch.norm(grad[:, :2], dim=-1)
    denom[i] += 1.0f;
    if (max_radii != nullptr) max_radii[i] = fmaxf(max_radii[i], (float)r);
}

// A split child's log-scale, log(exp(s) / (0.8 N)) (gs_renderer.py:984-992).  torch divides a CUDA tensor by a CPU
// scalar as a multiply by the fp32 reciprocal, inv = fp32(1 / fp32(0.8 N)); a true division differs in the last bit
// of the quotient on a fifth of the elements.  split_children_kernel stores this value and densify_classify_kernel
// decides the children's prune on it.
__device__ __forceinline__ float child_log_scale(float e, float inv) { return logf(__fmul_rn(e, inv)); }

// Decisions of densify_and_prune(max_grad, min_opacity, extent, max_screen_size) restated per ORIGINAL point:
//   grads = accum / denom, NaN -> 0
//   clone : |grads| >= max_grad  and  max(exp(scaling)) <= percent_dense * extent      (appended unchanged)
//   split : grads >= max_grad    and  max(exp(scaling)) >  percent_dense * extent      (N children, parent removed)
//   final prune over [originals, clones, children]: sigmoid(opacity) < min_opacity, or (max_screen_size given)
//   max(exp(scaling)) > 0.1 * extent; the screen-size test uses max_radii2D, which densification_postfix has
//   just reset to zero, so it is always false here.
__global__ void densify_classify_kernel(int P, const float* __restrict__ accum, const float* __restrict__ denom,
                                        const float* __restrict__ scaling, const float* __restrict__ opacity,
                                        float max_grad, float dense_extent, float min_opacity, float big_ws, float child_div,
                                        uint32_t* __restrict__ flags) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    float g = __fdiv_rn(accum[i], denom[i]);
    if (isnan(g)) g = 0.0f;
    const float e0 = expf(scaling[3 * (size_t)i]), e1 = expf(scaling[3 * (size_t)i + 1]), e2 = expf(scaling[3 * (size_t)i + 2]);
    const float s = fmaxf(fmaxf(e0, e1), e2);
    const bool clone = (fabsf(g) >= max_grad) && (s <= dense_extent);
    const bool split = (g >= max_grad) && (s > dense_extent);
    const bool low = gsr_sigmoid_rn(opacity[i]) < min_opacity;
    const bool pruned = low || (big_ws > 0.0f && s > big_ws);
    // the final prune sees the children's stored log-scales: max over the components of exp(child_log_scale(e_k))
    const float inv = __fdiv_rn(1.0f, child_div);
    const float sc = fmaxf(fmaxf(expf(child_log_scale(e0, inv)), expf(child_log_scale(e1, inv))), expf(child_log_scale(e2, inv)));
    const bool child_pruned = low || (big_ws > 0.0f && sc > big_ws);
    flags[(size_t)kKeep * P + i] = (!split && !pruned) ? 1u : 0u;
    flags[(size_t)kClone * P + i] = (clone && !pruned) ? 1u : 0u;
    flags[(size_t)kChild * P + i] = (split && !child_pruned) ? 1u : 0u;
    flags[(size_t)kSplitSel * P + i] = split ? 1u : 0u;
}

// ---- exclusive scan, 2 levels: 1024 threads x 4 items per block ------------------------------
__global__ void __launch_bounds__(1024)
scan_blocks_kernel(int n, const uint32_t* __restrict__ in, uint32_t* __restrict__ out, uint32_t* __restrict__ block_sums) {
    __shared__ uint32_t warp_tot[32];
    const int base = blockIdx.x * 4096 + threadIdx.x * 4;
    uint32_t v[4], s = 0;
#pragma unroll
    for (int k = 0; k < 4; ++k) { v[k] = (base + k < n) ? in[base + k] : 0u; s += v[k]; }
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    uint32_t incl = s;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += t;
    }
    if (lane == 31) warp_tot[w] = incl;
    __syncthreads();
    if (w == 0) {
        uint32_t x = warp_tot[lane], xi = x;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t t = __shfl_up_sync(0xffffffffu, xi, o);
            if (lane >= o) xi += t;
        }
        warp_tot[lane] = xi - x;
        if (lane == 31) block_sums[blockIdx.x] = xi;
    }
    __syncthreads();
    uint32_t run = warp_tot[w] + incl - s;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        if (base + k < n) out[base + k] = run;
        run += v[k];
    }
}
__global__ void __launch_bounds__(1024)
scan_sums_kernel(int nblocks, uint32_t* __restrict__ block_sums, uint32_t* __restrict__ total) {
    __shared__ uint32_t carry, warp_tot[32];
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    for (int base = 0; base < nblocks; base += 1024) {
        const int i = base + threadIdx.x;
        const uint32_t v = i < nblocks ? block_sums[i] : 0u;
        uint32_t incl = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += t;
        }
        if (lane == 31) warp_tot[w] = incl;
        __syncthreads();
        if (w == 0) {
            uint32_t x = warp_tot[lane], xi = x;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const uint32_t t = __shfl_up_sync(0xffffffffu, xi, o);
                if (lane >= o) xi += t;
            }
            warp_tot[lane] = xi - x;
        }
        __syncthreads();
        const uint32_t excl = carry + warp_tot[w] + incl - v;
        if (i < nblocks) block_sums[i] = excl;
        __syncthreads();
        if (threadIdx.x == 1023) carry = excl + v;
        __syncthreads();
    }
    if (threadIdx.x == 0 && total != nullptr) *total = carry;
}
__global__ void scan_add_kernel(int n, uint32_t* __restrict__ out, const uint32_t* __restrict__ block_sums) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] += block_sums[i / 4096];
}

// totals[4] = number of set flags per plane (offsets are scans over the concatenated [4][P] flag array:
// offs[plane*P + i] = #set flags before (plane, i) counting all earlier planes entirely)
// src map entry: bits 0..29 source row, bits 30..31 kind (0 original, 1 clone, 2 child)
__global__ void densify_map_kernel(int P, int N, const uint32_t* __restrict__ flags, const uint32_t* __restrict__ offs,
                                   const uint32_t* __restrict__ totals4, int32_t* __restrict__ src_map,
                                   int32_t* __restrict__ child_draw) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    const uint32_t n_keep = totals4[0], n_clone = totals4[1], n_child = totals4[2], n_sel = totals4[3];
    if (flags[(size_t)kKeep * P + i]) src_map[offs[(size_t)kKeep * P + i]] = i;
    if (flags[(size_t)kClone * P + i]) src_map[offs[(size_t)kClone * P + i]] = i | (1 << 30);     // offs already past the keeps
    if (flags[(size_t)kChild * P + i]) {
        const uint32_t rank_surv = offs[(size_t)kChild * P + i] - (n_keep + n_clone);
        const uint32_t rank_sel = offs[(size_t)kSplitSel * P + i] - (n_keep + n_clone + n_child);
        for (int k = 0; k < N; ++k) {
            const uint32_t pos = n_keep + n_clone + (uint32_t)k * n_child + rank_surv;
            src_map[pos] = i | (2 << 30);
            // row of the reference's torch.normal draw: samples = normal(std=get_scaling[sel].repeat(N,1))
            child_draw[(uint32_t)k * n_child + rank_surv] = (int32_t)((uint32_t)k * n_sel + rank_sel);
        }
    }
}

// per-plane totals from the scan of the concatenated flags
__global__ void plane_totals_kernel(int P, const uint32_t* __restrict__ flags, const uint32_t* __restrict__ offs,
                                    uint32_t* __restrict__ totals4) {
    const int p = threadIdx.x;
    if (p >= 4 || P <= 0) { if (p < 4) totals4[p] = 0; return; }
    const size_t last = (size_t)p * P + (P - 1);
    const uint32_t end = offs[last] + flags[last];
    const uint32_t beg = offs[(size_t)p * P];
    totals4[p] = end - beg;
}

// out[p, :] = (src kind allowed) ? in[src, :] : 0   ; row = `row` floats
__global__ void gather_rows_kernel(int n_out, int row, const int32_t* __restrict__ src_map, const float* __restrict__ in,
                                   float* __restrict__ out, int zero_appended) {
    const size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= (size_t)n_out * row) return;
    const int p = (int)(e / row), c = (int)(e - (size_t)p * row);
    const int32_t m = src_map[p];
    const int kind = ((uint32_t)m) >> 30;
    const int s = m & 0x3fffffff;
    out[e] = (kind != 0 && zero_appended) ? 0.0f : in[(size_t)s * row + c];
}

// split children: xyz = R(normalize(q)) (z * exp(scaling)) + xyz ; scaling = child_log_scale(exp(scaling))
// (gs_renderer.py:984-992; build_rotation normalises the quaternion: gs_renderer.py:124-147)
__global__ void split_children_kernel(int n_out, int first_child, float child_div, const int32_t* __restrict__ src_map,
                                      const int32_t* __restrict__ child_draw, const float* __restrict__ xyz,
                                      const float* __restrict__ scaling, const float* __restrict__ rotation,
                                      const float* __restrict__ z, float* __restrict__ xyz_out, float* __restrict__ scaling_out) {
    const int p = first_child + blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n_out) return;
    const int s = src_map[p] & 0x3fffffff;
    const int zr = child_draw[p - first_child];
    const float e0 = expf(scaling[3 * (size_t)s]), e1 = expf(scaling[3 * (size_t)s + 1]), e2 = expf(scaling[3 * (size_t)s + 2]);
    const float s0 = __fmul_rn(z[3 * (size_t)zr], e0), s1 = __fmul_rn(z[3 * (size_t)zr + 1], e1), s2 = __fmul_rn(z[3 * (size_t)zr + 2], e2);
    const float4 q = *reinterpret_cast<const float4*>(rotation + 4 * (size_t)s);
    const float nrm = sqrtf(q.x * q.x + q.y * q.y + q.z * q.z + q.w * q.w);
    const float r = q.x / nrm, x = q.y / nrm, y = q.z / nrm, w = q.w / nrm;
    const float R00 = 1 - 2 * (y * y + w * w), R01 = 2 * (x * y - r * w), R02 = 2 * (x * w + r * y);
    const float R10 = 2 * (x * y + r * w), R11 = 1 - 2 * (x * x + w * w), R12 = 2 * (y * w - r * x);
    const float R20 = 2 * (x * w - r * y), R21 = 2 * (y * w + r * x), R22 = 1 - 2 * (x * x + y * y);
    xyz_out[3 * (size_t)p] = R00 * s0 + R01 * s1 + R02 * s2 + xyz[3 * (size_t)s];
    xyz_out[3 * (size_t)p + 1] = R10 * s0 + R11 * s1 + R12 * s2 + xyz[3 * (size_t)s + 1];
    xyz_out[3 * (size_t)p + 2] = R20 * s0 + R21 * s1 + R22 * s2 + xyz[3 * (size_t)s + 2];
    const float inv = __fdiv_rn(1.0f, child_div);
    scaling_out[3 * (size_t)p] = child_log_scale(e0, inv);
    scaling_out[3 * (size_t)p + 1] = child_log_scale(e1, inv);
    scaling_out[3 * (size_t)p + 2] = child_log_scale(e2, inv);
}

// ---- k-th smallest of n floats (ascending, k 0-based): 4-pass radix select on order-preserving keys ------
// Every NaN maps to the largest key, whatever its sign bit, so NaNs sort last as in torch.sort.
__device__ __forceinline__ uint32_t float_key(float f) {
    if (isnan(f)) return 0xffffffffu;
    const uint32_t b = __float_as_uint(f);
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float key_float(uint32_t k) {
    return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}
// state[0] = prefix, state[1] = remaining k, hist[256]
__global__ void select_hist_kernel(int n, const float* __restrict__ v, int pass, const uint32_t* __restrict__ state,
                                   uint32_t* __restrict__ hist) {
    __shared__ uint32_t h[256];
    h[threadIdx.x] = 0u;
    __syncthreads();
    const int shift = 24 - 8 * pass;
    const uint32_t prefix = state[0];
    const uint32_t mask = pass == 0 ? 0u : (0xffffffffu << (shift + 8));
    for (int i = blockIdx.x * 256 + threadIdx.x; i < n; i += gridDim.x * 256) {
        const uint32_t k = float_key(v[i]);
        if ((k & mask) == (prefix & mask)) atomicAdd(&h[(k >> shift) & 0xffu], 1u);
    }
    __syncthreads();
    if (h[threadIdx.x]) atomicAdd(&hist[threadIdx.x], h[threadIdx.x]);
}
__global__ void select_pick_kernel(int pass, uint32_t k0, uint32_t* __restrict__ state, uint32_t* __restrict__ hist,
                                   float* __restrict__ out) {
    if (threadIdx.x == 0) {
        const int shift = 24 - 8 * pass;
        uint32_t k = pass == 0 ? k0 : state[1], d = 0;
        for (; d < 256; ++d) {
            if (k < hist[d]) break;
            k -= hist[d];
        }
        if (d > 255) d = 255;
        state[0] |= d << shift;
        state[1] = k;
        if (pass == 3) *out = key_float(state[0]);
    }
    __syncthreads();
    hist[threadIdx.x] = 0u;
}

}  // namespace

cudaError_t gsr_densify_stats(int P, const float* vs_grad, const int32_t* radii, float* accum, float* denom,
                              float* max_radii, cudaStream_t s) {
    if (P > 0) densify_stats_kernel<<<(P + 255) / 256, 256, 0, s>>>(P, vs_grad, radii, accum, denom, max_radii);
    return cudaGetLastError();
}

void gsr_scan_u32(int n, const uint32_t* in, uint32_t* out, uint32_t* bsums, uint32_t* total, cudaStream_t s) {
    const int nb = (n + 4095) / 4096;
    scan_blocks_kernel<<<nb, 1024, 0, s>>>(n, in, out, bsums);
    scan_sums_kernel<<<1, 1024, 0, s>>>(nb, bsums, total);
    scan_add_kernel<<<(n + 255) / 256, 256, 0, s>>>(n, out, bsums);
}

size_t gsr_densify_scratch_bytes(int P) {
    const size_t n = 4 * (size_t)(P > 0 ? P : 1);
    return (2 * n + (n + 4095) / 4096 + 16) * sizeof(uint32_t);
}

// scratch: flags[4P] | offs[4P] | block sums | totals4 + grand total
cudaError_t gsr_densify_plan(int P, const float* accum, const float* denom, const float* scaling, const float* opacity,
                             float max_grad, float dense_extent, float min_opacity, float big_ws, float child_div, void* scratch,
                             uint32_t* totals5, cudaStream_t s) {
    if (P <= 0) return cudaMemsetAsync(totals5, 0, 5 * sizeof(uint32_t), s);
    uint32_t* flags = static_cast<uint32_t*>(scratch);
    uint32_t* offs = flags + 4 * (size_t)P;
    uint32_t* bsums = offs + 4 * (size_t)P;
    densify_classify_kernel<<<(P + 255) / 256, 256, 0, s>>>(P, accum, denom, scaling, opacity, max_grad, dense_extent,
                                                             min_opacity, big_ws, child_div, flags);
    gsr_scan_u32(4 * P, flags, offs, bsums, totals5 + 4, s);
    plane_totals_kernel<<<1, 32, 0, s>>>(P, flags, offs, totals5);
    return cudaGetLastError();
}

cudaError_t gsr_densify_map(int P, int N, const void* scratch, const uint32_t* totals5, int32_t* src_map,
                            int32_t* child_draw, cudaStream_t s) {
    if (P <= 0) return cudaSuccess;
    const uint32_t* flags = static_cast<const uint32_t*>(scratch);
    const uint32_t* offs = flags + 4 * (size_t)P;
    densify_map_kernel<<<(P + 255) / 256, 256, 0, s>>>(P, N, flags, offs, totals5, src_map, child_draw);
    return cudaGetLastError();
}

// mask (uint8, 1 = keep) -> src_map of the kept rows + count
cudaError_t gsr_compact_plan(int P, const uint8_t* keep, void* scratch, int32_t* src_map, uint32_t* count, cudaStream_t s);

namespace {
__global__ void mask_to_u32_kernel(int P, const uint8_t* __restrict__ keep, uint32_t* __restrict__ flags) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < P) flags[i] = keep[i] ? 1u : 0u;
}
__global__ void compact_map_kernel(int P, const uint32_t* __restrict__ flags, const uint32_t* __restrict__ offs,
                                   int32_t* __restrict__ src_map) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < P && flags[i]) src_map[offs[i]] = i;
}
}  // namespace

cudaError_t gsr_compact_plan(int P, const uint8_t* keep, void* scratch, int32_t* src_map, uint32_t* count, cudaStream_t s) {
    if (P <= 0) return cudaMemsetAsync(count, 0, sizeof(uint32_t), s);
    uint32_t* flags = static_cast<uint32_t*>(scratch);
    uint32_t* offs = flags + 4 * (size_t)P;
    uint32_t* bsums = offs + 4 * (size_t)P;
    mask_to_u32_kernel<<<(P + 255) / 256, 256, 0, s>>>(P, keep, flags);
    gsr_scan_u32(P, flags, offs, bsums, count, s);
    compact_map_kernel<<<(P + 255) / 256, 256, 0, s>>>(P, flags, offs, src_map);
    return cudaGetLastError();
}

cudaError_t gsr_gather_rows(int n_out, int row_floats, const int32_t* src_map, const float* in, float* out,
                            int zero_appended, cudaStream_t s) {
    const size_t total = (size_t)n_out * row_floats;
    if (total == 0) return cudaSuccess;
    gather_rows_kernel<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(n_out, row_floats, src_map, in, out, zero_appended);
    return cudaGetLastError();
}

cudaError_t gsr_split_children(int n_out, int first_child, float child_div, const int32_t* src_map, const int32_t* child_draw,
                               const float* xyz, const float* scaling, const float* rotation, const float* z,
                               float* xyz_out, float* scaling_out, cudaStream_t s) {
    const int n = n_out - first_child;
    if (n <= 0) return cudaSuccess;
    split_children_kernel<<<(n + 255) / 256, 256, 0, s>>>(n_out, first_child, child_div, src_map, child_draw, xyz, scaling,
                                                          rotation, z, xyz_out, scaling_out);
    return cudaGetLastError();
}

// scratch: state[2] + hist[256] uint32 (zeroed here)
cudaError_t gsr_kth_smallest(int n, const float* v, uint32_t k, void* scratch, float* out, int num_sms, cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    uint32_t* state = static_cast<uint32_t*>(scratch);
    uint32_t* hist = state + 2;
    cudaError_t e = cudaMemsetAsync(state, 0, (2 + 256) * sizeof(uint32_t), s);
    if (e != cudaSuccess) return e;
    const int nb = max(1, min((n + 255) / 256, num_sms * 8));
    for (int pass = 0; pass < 4; ++pass) {
        select_hist_kernel<<<nb, 256, 0, s>>>(n, v, pass, state, hist);
        select_pick_kernel<<<1, 256, 0, s>>>(pass, k, state, hist, out);
    }
    return cudaGetLastError();
}
