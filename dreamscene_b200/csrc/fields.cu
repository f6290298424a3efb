// The opacity field of a Gaussian group on a voxel grid (include/b200gsr_fields.h): DreamScene's
// GaussianModel.extract_fields as five kernels instead of a Python loop over the grid's blocks.
//
//   fields_init      coordinates into scratch, reduction state reset
//   fields_reduce    opacity filter, per-axis min / max of the kept centres (ordered-integer atomics), kept count
//   fields_prepare   normalisation; per kept row a 48-byte record (centre, opacity, scaled inverse covariance) and the
//                    bit masks of the chunks its centre falls into on each axis
//   fields_count     per (block, chunk of B200GSR_FIELDS_CHUNK_ROWS rows) member counts, block-major; then an
//                    exclusive scan (gsr_scan_u32) gives every block's list and every chunk's place in it
//   fields_scatter   one warp per row chunk walks its rows in order, so every block lists its members in row order
//   fields_eval      one CTA per block: members staged through shared memory, each thread sums its grid points in
//                    registers in list order, so the field is the same on every call
//   fields_eval_rgb  the same, also summing the members' opacity-weighted colours beside occ and dividing them by it
//                    (include/b200gsr_mesh_colour.h); each member's colour is made as it is staged
#include "common.cuh"
#include "../../include/b200gsr_fields.h"

namespace {

constexpr int kEvalThreads = 256;

struct FieldsState {
    uint32_t mn[3], mx[3];   // ordered keys of the kept centres' per-axis min / max
    uint32_t kept;
    uint32_t total;          // (block, row) pairs, written by the scan
    uint32_t overflow;
};

struct FieldsCoords {
    float v[B200GSR_FIELDS_MAX_R];
};

struct FieldsArgs {
    int P, R, split, C, nblk, nchunks;
    const float *xyz, *opacity, *scaling, *rotation;
    float lo[B200GSR_FIELDS_MAX_CHUNKS], hi[B200GSR_FIELDS_MAX_CHUNKS];
    FieldsState* state;
    const float* grid;       // [R] coordinates
    float4* rec;             // [P][3]
    uint4* mask;             // [P]: chunk bit masks x, y, z
    uint32_t* hist;          // [nblk][nchunks]: counts, then (scanned) list offsets
    uint32_t* members;       // [capacity]
    uint32_t capacity;
    float* occ;
    b200gsr_fields_info* info;
};

// float -> uint32 with the same order (NaN aside)
__device__ __forceinline__ uint32_t order_key(float f) {
    const uint32_t b = __float_as_uint(f);
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float order_unkey(uint32_t k) {
    return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

__device__ __forceinline__ int nth_bit(uint32_t m, int n) {   // position of the n-th (from 0) set bit
    for (int k = 0; k < n; ++k) m &= m - 1;
    return __ffs(m) - 1;
}

__global__ void fields_init_kernel(FieldsCoords coords, int R, float* grid, FieldsState* st) {
    for (int i = threadIdx.x; i < R; i += blockDim.x) grid[i] = coords.v[i];
    if (threadIdx.x < 3) { st->mn[threadIdx.x] = 0xffffffffu; st->mx[threadIdx.x] = 0u; }
    if (threadIdx.x == 0) { st->kept = 0u; st->total = 0u; st->overflow = 0u; }
}

__global__ void __launch_bounds__(256) fields_reduce_kernel(int P, const float* __restrict__ xyz,
                                                            const float* __restrict__ opacity, FieldsState* st) {
    uint32_t mn[3] = {0xffffffffu, 0xffffffffu, 0xffffffffu}, mx[3] = {0u, 0u, 0u}, kept = 0u;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < P; i += gridDim.x * blockDim.x) {
        if (!(gsr_sigmoid_rn(opacity[i]) > 0.005f)) continue;
        ++kept;
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            const uint32_t k = order_key(xyz[3 * (size_t)i + a]);
            mn[a] = min(mn[a], k);
            mx[a] = max(mx[a], k);
        }
    }
    kept = __reduce_add_sync(0xffffffffu, kept);
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        mn[a] = __reduce_min_sync(0xffffffffu, mn[a]);
        mx[a] = __reduce_max_sync(0xffffffffu, mx[a]);
    }
    if ((threadIdx.x & 31) == 0 && kept) {
        atomicAdd(&st->kept, kept);
#pragma unroll
        for (int a = 0; a < 3; ++a) { atomicMin(&st->mn[a], mn[a]); atomicMax(&st->mx[a], mx[a]); }
    }
}

// Normalisation and per-row records.  Every product and difference that decides a membership is rounded alone
// (__fsub_rn / __fmul_rn), as torch's elementwise kernels round them, so xyz' equals torch's bit for bit.
__global__ void __launch_bounds__(256) fields_prepare_kernel(FieldsArgs a) {
    const FieldsState& st = *a.state;
    const int kept = (int)st.kept;
    float mn[3], mx[3], center[3];
    float ext = 0.0f;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        mn[k] = order_unkey(st.mn[k]);
        mx[k] = order_unkey(st.mx[k]);
        center[k] = __fmul_rn(__fadd_rn(mn[k], mx[k]), 0.5f);
        ext = k == 0 ? __fsub_rn(mx[k], mn[k]) : fmaxf(ext, __fsub_rn(mx[k], mn[k]));
    }
    const bool ok = kept > 0 && ext > 0.0f;
    const double scale = 1.8 / (double)ext;          // Python's 1.8 / (mx - mn).amax().item()
    const float s32 = __double2float_rn(scale);       // the scalar torch multiplies a float32 tensor by
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        b200gsr_fields_info* info = a.info;
        info->kept = kept;
        info->extent = kept > 0 ? ext : 0.0f;
        info->scale = ok ? scale : 0.0;
        for (int k = 0; k < 3; ++k) info->center[k] = kept > 0 ? center[k] : 0.0f;
    }
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= a.P) return;
    uint4 m = make_uint4(0u, 0u, 0u, 0u);
    const float op = gsr_sigmoid_rn(a.opacity[i]);
    if (ok && op > 0.005f) {
        float g[3];
        uint32_t bits[3];
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            g[k] = __fmul_rn(__fsub_rn(a.xyz[3 * (size_t)i + k], center[k]), s32);
            uint32_t b = 0u;
            for (int c = 0; c < a.C; ++c)
                if (g[k] > a.lo[c] && g[k] < a.hi[c]) b |= 1u << c;
            bits[k] = b;
        }
        m = make_uint4(bits[0], bits[1], bits[2], 0u);
        // covariance of L = R(q / |q|) diag(exp(scaling) * scale), then the reference's cofactor inverse
        float s[3];
#pragma unroll
        for (int k = 0; k < 3; ++k) s[k] = __fmul_rn(expf(a.scaling[3 * (size_t)i + k]), s32);
        const float4 q0 = *reinterpret_cast<const float4*>(a.rotation + 4 * (size_t)i);
        const float nrm = sqrtf(q0.x * q0.x + q0.y * q0.y + q0.z * q0.z + q0.w * q0.w);
        const float r = q0.x / nrm, x = q0.y / nrm, y = q0.z / nrm, z = q0.w / nrm;
        const float R[3][3] = {{1.f - 2.f * (y * y + z * z), 2.f * (x * y - r * z), 2.f * (x * z + r * y)},
                               {2.f * (x * y + r * z), 1.f - 2.f * (x * x + z * z), 2.f * (y * z - r * x)},
                               {2.f * (x * z - r * y), 2.f * (y * z + r * x), 1.f - 2.f * (x * x + y * y)}};
        float M[3][3];
#pragma unroll
        for (int u = 0; u < 3; ++u)
#pragma unroll
            for (int v = 0; v < 3; ++v) M[u][v] = R[u][v] * s[v];
        auto dot = [&](int u, int v) { return M[u][0] * M[v][0] + M[u][1] * M[v][1] + M[u][2] * M[v][2]; };
        const float ca = dot(0, 0), cb = dot(0, 1), cc = dot(0, 2), cd = dot(1, 1), ce = dot(1, 2), cf = dot(2, 2);
        const float inv_det = 1.0f / (ca * cd * cf + 2.f * ce * cc * cb - ce * ce * ca - cc * cc * cd - cb * cb * cf + 1e-24f);
        const float ia = (cd * cf - ce * ce) * inv_det, ib = (ce * cc - cb * cf) * inv_det;
        const float ic = (ce * cb - cc * cd) * inv_det, id = (ca * cf - cc * cc) * inv_det;
        const float ie = (cb * cc - ce * ca) * inv_det, iff = (ca * cd - cb * cb) * inv_det;
        // log2 of the weight: A x^2 + D y^2 + F z^2 + B xy + C xz + E yz
        const float h = -0.5f * GSR_LOG2E;
        float4* rec = a.rec + 3 * (size_t)i;
        rec[0] = make_float4(g[0], g[1], g[2], op);
        rec[1] = make_float4(h * ia, -GSR_LOG2E * ib, -GSR_LOG2E * ic, h * id);
        rec[2] = make_float4(-GSR_LOG2E * ie, h * iff, 0.0f, 0.0f);
    }
    a.mask[i] = m;
}

// Member counts of row chunk blockIdx.x per block, written block-major: hist[b * nchunks + chunk].
__global__ void __launch_bounds__(32) fields_count_kernel(FieldsArgs a) {
    extern __shared__ uint32_t cnt[];
    const int c = blockIdx.x, lane = threadIdx.x, C = a.C;
    for (int b = lane; b < a.nblk; b += 32) cnt[b] = 0u;
    __syncwarp();
    const int r1 = min(a.P, (c + 1) * B200GSR_FIELDS_CHUNK_ROWS);
    for (int r = c * B200GSR_FIELDS_CHUNK_ROWS + lane; r < r1; r += 32) {
        const uint4 m = a.mask[r];
        for (uint32_t mx = m.x; mx; mx &= mx - 1)
            for (uint32_t my = m.y; my; my &= my - 1)
                for (uint32_t mz = m.z; mz; mz &= mz - 1)
                    atomicAdd(&cnt[((__ffs(mx) - 1) * C + (__ffs(my) - 1)) * C + (__ffs(mz) - 1)], 1u);
    }
    __syncwarp();
    for (int b = lane; b < a.nblk; b += 32) a.hist[(size_t)b * a.nchunks + c] = cnt[b];
}

// Member lists: the warp of row chunk blockIdx.x takes its rows one at a time, in order; a row's blocks are distinct,
// so its lanes advance the per-block cursors without conflict.
__global__ void __launch_bounds__(32) fields_scatter_kernel(FieldsArgs a) {
    extern __shared__ uint32_t cursor[];
    const int c = blockIdx.x, lane = threadIdx.x, C = a.C;
    if (a.state->total > a.capacity) {
        if (c == 0 && lane == 0) a.state->overflow = 1u;
        return;
    }
    for (int b = lane; b < a.nblk; b += 32) cursor[b] = a.hist[(size_t)b * a.nchunks + c];
    __syncwarp();
    const int r0 = c * B200GSR_FIELDS_CHUNK_ROWS, r1 = min(a.P, r0 + B200GSR_FIELDS_CHUNK_ROWS);
    for (int base = r0; base < r1; base += 32) {
        const uint4 mine = base + lane < r1 ? a.mask[base + lane] : make_uint4(0u, 0u, 0u, 0u);
        const int n = min(32, r1 - base);
        for (int j = 0; j < n; ++j) {
            const uint32_t mx = __shfl_sync(0xffffffffu, mine.x, j), my = __shfl_sync(0xffffffffu, mine.y, j),
                           mz = __shfl_sync(0xffffffffu, mine.z, j);
            const int cy = __popc(my), cz = __popc(mz), np = __popc(mx) * cy * cz;
            for (int p = lane; p < np; p += 32) {
                const int iz = p % cz, t = p / cz, iy = t % cy, ix = t / cy;
                const int b = (nth_bit(mx, ix) * C + nth_bit(my, iy)) * C + nth_bit(mz, iz);
                const uint32_t pos = cursor[b];
                a.members[pos] = (uint32_t)(base + j);
                cursor[b] = pos + 1u;
            }
            __syncwarp();
        }
    }
}

// op * clamp_min(SH2RGB(dc), 0) per channel: torch's float32 dc * SH_C0 + 0.5 (two roundings), then the clamp, which
// keeps NaN
__device__ __forceinline__ float4 weighted_colour(float op, const float* __restrict__ dc) {
    constexpr float kShC0 = 0.28209479177387814f;
    float c[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const float v = __fadd_rn(__fmul_rn(dc[k], kShC0), 0.5f);
        c[k] = __fmul_rn(op, v < 0.0f ? 0.0f : v);
    }
    return make_float4(c[0], c[1], c[2], 0.0f);
}

// One CTA per block; PT grid points per thread per pass, kEvalThreads * PT points per pass.  RGB adds three sums per
// point beside acc, whose fmaf sequence it leaves as it is, so occ is the same bits with and without them.
template <int PT, bool RGB>
__device__ __forceinline__ void fields_eval(const FieldsArgs& a, const float* dc, float* rgb) {
    __shared__ float4 s0[kEvalThreads], s1[kEvalThreads], s2[kEvalThreads];
    __shared__ float4 s3[kEvalThreads];      // RGB: op * colour of the staged members
    const int b = blockIdx.x, C = a.C, R = a.R, tid = threadIdx.x;
    const int bz = b % C, by = (b / C) % C, bx = b / (C * C);
    const int x0 = bx * a.split, y0 = by * a.split, z0 = bz * a.split;
    const int nx = min(a.split, R - x0), ny = min(a.split, R - y0), nz = min(a.split, R - z0);
    const int npts = nx * ny * nz;
    const uint32_t start = a.hist[(size_t)b * a.nchunks];
    uint32_t end = b + 1 < a.nblk ? a.hist[(size_t)(b + 1) * a.nchunks] : a.state->total;
    if (a.state->overflow) end = start;
    for (int pbase = 0; pbase < npts; pbase += kEvalThreads * PT) {
        float px[PT], py[PT], pz[PT], acc[PT], cr[RGB ? PT : 1], cg[RGB ? PT : 1], cb[RGB ? PT : 1];
        size_t out[PT];
#pragma unroll
        for (int k = 0; k < PT; ++k) {
            const int q = pbase + tid + kEvalThreads * k;
            const int i = q / (ny * nz), rem = q - i * ny * nz, j = rem / nz, l = rem - j * nz;
            const bool valid = q < npts;
            px[k] = valid ? a.grid[x0 + i] : 0.0f;
            py[k] = valid ? a.grid[y0 + j] : 0.0f;
            pz[k] = valid ? a.grid[z0 + l] : 0.0f;
            out[k] = valid ? ((size_t)(x0 + i) * R + (y0 + j)) * R + (z0 + l) : ~(size_t)0;
            acc[k] = 0.0f;
            if constexpr (RGB) cr[k] = cg[k] = cb[k] = 0.0f;
        }
        for (uint32_t m0 = start; m0 < end; m0 += kEvalThreads) {
            __syncthreads();
            if (m0 + tid < end) {
                const size_t r = a.members[m0 + tid];
                s0[tid] = a.rec[3 * r];
                s1[tid] = a.rec[3 * r + 1];
                s2[tid] = a.rec[3 * r + 2];
                if constexpr (RGB) s3[tid] = weighted_colour(a.rec[3 * r].w, dc + 3 * r);
            }
            __syncthreads();
            const int n = (int)min((uint32_t)kEvalThreads, end - m0);
            for (int j = 0; j < n; ++j) {
                const float4 g0 = s0[j], g1 = s1[j], g2 = s2[j];
#pragma unroll
                for (int k = 0; k < PT; ++k) {
                    const float x = px[k] - g0.x, y = py[k] - g0.y, z = pz[k] - g0.z;
                    const float e = x * fmaf(g1.x, x, fmaf(g1.y, y, g1.z * z)) + y * fmaf(g1.w, y, g2.x * z) + g2.y * z * z;
                    const float w = e > 0.0f ? 0.0f : exp2f(e);          // power > 0: the reference's weight 0
                    acc[k] = fmaf(g0.w, w, acc[k]);
                    if constexpr (RGB) {
                        const float4 c = s3[j];
                        cr[k] = fmaf(w, c.x, cr[k]);
                        cg[k] = fmaf(w, c.y, cg[k]);
                        cb[k] = fmaf(w, c.z, cb[k]);
                    }
                }
            }
        }
#pragma unroll
        for (int k = 0; k < PT; ++k)
            if (out[k] != ~(size_t)0) {
                a.occ[out[k]] = acc[k];
                if constexpr (RGB) {
                    const bool empty = acc[k] == 0.0f;
                    float* o = rgb + 3 * out[k];
                    o[0] = empty ? 0.0f : __fdiv_rn(cr[k], acc[k]);
                    o[1] = empty ? 0.0f : __fdiv_rn(cg[k], acc[k]);
                    o[2] = empty ? 0.0f : __fdiv_rn(cb[k], acc[k]);
                }
            }
    }
    if (b == 0 && tid == 0) {
        a.info->pairs = (int64_t)a.state->total;
        a.info->overflow = a.state->overflow;
    }
}

template <int PT>
__global__ void __launch_bounds__(kEvalThreads) fields_eval_kernel(FieldsArgs a) {
    fields_eval<PT, false>(a, nullptr, nullptr);
}

template <int PT>
__global__ void __launch_bounds__(kEvalThreads) fields_eval_rgb_kernel(FieldsArgs a, const float* __restrict__ dc,
                                                                       float* __restrict__ rgb) {
    fields_eval<PT, true>(a, dc, rgb);
}

template <int PT>
void launch_eval(const FieldsArgs& a, const float* dc, float* rgb, cudaStream_t s) {
    if (rgb) fields_eval_rgb_kernel<PT><<<a.nblk, kEvalThreads, 0, s>>>(a, dc, rgb);
    else fields_eval_kernel<PT><<<a.nblk, kEvalThreads, 0, s>>>(a);
}

size_t align256(size_t v) { return (v + 255) / 256 * 256; }

}  // namespace

void gsr_fields_plan(int P, int R, int num_blocks, double relax_ratio, const float* coords, GsrFieldsPlan* pl) {
    GsrFieldsPlan& p = *pl;
    p.P = P; p.R = R;
    p.split = R / num_blocks;
    p.C = (R + p.split - 1) / p.split;
    p.nblk = p.C * p.C * p.C;
    p.nchunks = (P + B200GSR_FIELDS_CHUNK_ROWS - 1) / B200GSR_FIELDS_CHUNK_ROWS;
    // torch: vmin = pts.amin(0) - r, vmax = pts.amax(0) + r on float32 tensors, r the Python double cast to float32
    p.r = (float)((2.0 / num_blocks) * relax_ratio);
    for (int c = 0; c < p.C; ++c) {
        float lo = coords[c * p.split], hi = lo;
        for (int i = c * p.split; i < R && i < (c + 1) * p.split; ++i) {
            lo = coords[i] < lo ? coords[i] : lo;
            hi = coords[i] > hi ? coords[i] : hi;
        }
        volatile float r = p.r;   // one float32 rounding each, as torch's sub / add
        p.lo[c] = lo - r;
        p.hi[c] = hi + r;
    }
    // The most open boxes (lo, hi) any point lies in: a point x in several boxes is in the one with the largest lo
    // below it, c, and every box holding x then has lo <= lo_c < hi.
    int m = 0;
    for (int c = 0; c < p.C; ++c) {
        int k = 0;
        for (int d = 0; d < p.C; ++d) k += p.lo[d] <= p.lo[c] && p.lo[c] < p.hi[d];
        m = k > m ? k : m;
    }
    p.max_per_axis = m;
    p.max_pairs = (long long)P * m * m * m;
    const size_t hist_n = (size_t)p.nblk * p.nchunks;
    p.off_state = 0;
    p.off_grid = align256(sizeof(uint32_t) * 16);
    p.off_rec = p.off_grid + align256(sizeof(float) * R);
    p.off_mask = p.off_rec + align256((size_t)P * 3 * sizeof(float4));
    p.off_hist = p.off_mask + align256((size_t)P * sizeof(uint4));
    p.off_bsums = p.off_hist + align256(hist_n * sizeof(uint32_t));
    p.off_members = p.off_bsums + align256(((hist_n + 4095) / 4096 + 1) * sizeof(uint32_t));
    p.total = p.off_members + align256((size_t)(p.max_pairs > 0 ? p.max_pairs : 1) * sizeof(uint32_t));
}

cudaError_t gsr_launch_fields(const GsrFieldsPlan& p, const float* coords, const float* xyz, const float* opacity,
                              const float* scaling, const float* rotation, const float* features_dc, float* occ,
                              float* rgb, b200gsr_fields_info* info, uint8_t* scratch, int num_sms, cudaStream_t s) {
    static_assert(sizeof(FieldsState) <= 16 * sizeof(uint32_t), "state must fit its slot");
    static std::atomic<unsigned long long> smem_count{0}, smem_scatter{0};
    FieldsArgs a;
    a.P = p.P; a.R = p.R; a.split = p.split; a.C = p.C; a.nblk = p.nblk; a.nchunks = p.nchunks;
    a.xyz = xyz; a.opacity = opacity; a.scaling = scaling; a.rotation = rotation;
    for (int c = 0; c < B200GSR_FIELDS_MAX_CHUNKS; ++c) {
        a.lo[c] = c < p.C ? p.lo[c] : 0.0f;
        a.hi[c] = c < p.C ? p.hi[c] : 0.0f;
    }
    a.state = reinterpret_cast<FieldsState*>(scratch + p.off_state);
    float* grid = reinterpret_cast<float*>(scratch + p.off_grid);
    a.grid = grid;
    a.rec = reinterpret_cast<float4*>(scratch + p.off_rec);
    a.mask = reinterpret_cast<uint4*>(scratch + p.off_mask);
    a.hist = reinterpret_cast<uint32_t*>(scratch + p.off_hist);
    a.members = reinterpret_cast<uint32_t*>(scratch + p.off_members);
    a.capacity = (uint32_t)p.max_pairs;
    a.occ = occ;
    a.info = info;

    FieldsCoords fc;
    for (int i = 0; i < B200GSR_FIELDS_MAX_R; ++i) fc.v[i] = i < p.R ? coords[i] : 0.0f;
    fields_init_kernel<<<1, 256, 0, s>>>(fc, p.R, grid, a.state);
    const int rb = (p.P + 255) / 256;
    fields_reduce_kernel<<<rb < 8 * num_sms ? rb : 8 * num_sms, 256, 0, s>>>(p.P, xyz, opacity, a.state);
    fields_prepare_kernel<<<rb, 256, 0, s>>>(a);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    // The opt-in limit is set once per device, so it is the largest any call uses (a block counter each for 32^3
    // blocks), not this call's size.
    constexpr int kMaxSmem = B200GSR_FIELDS_MAX_CHUNKS * B200GSR_FIELDS_MAX_CHUNKS * B200GSR_FIELDS_MAX_CHUNKS *
                             (int)sizeof(uint32_t);
    e = gsr_smem_once(fields_count_kernel, kMaxSmem, smem_count);
    if (e == cudaSuccess) e = gsr_smem_once(fields_scatter_kernel, kMaxSmem, smem_scatter);
    if (e != cudaSuccess) return e;
    const int smem = p.nblk * (int)sizeof(uint32_t);
    // each stage reads what the one before wrote: nothing more is issued after a launch that failed
    fields_count_kernel<<<p.nchunks, 32, smem, s>>>(a);
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    const int hist_n = p.nblk * p.nchunks;
    gsr_scan_u32(hist_n, a.hist, a.hist, reinterpret_cast<uint32_t*>(scratch + p.off_bsums), &a.state->total, s);
    fields_scatter_kernel<<<p.nchunks, 32, smem, s>>>(a);
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    // points per block: the first block is the largest
    const int pts = p.split * p.split * p.split, cover = pts < 16 * kEvalThreads ? pts : 16 * kEvalThreads;
    if (cover <= kEvalThreads) launch_eval<1>(a, features_dc, rgb, s);
    else if (cover <= 2 * kEvalThreads) launch_eval<2>(a, features_dc, rgb, s);
    else if (cover <= 4 * kEvalThreads) launch_eval<4>(a, features_dc, rgb, s);
    else if (cover <= 8 * kEvalThreads) launch_eval<8>(a, features_dc, rgb, s);
    else launch_eval<16>(a, features_dc, rgb, s);
    return cudaGetLastError();
}
