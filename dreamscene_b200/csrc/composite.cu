// composite_fwd / composite_bwd: per-tile front-to-back alpha blending and its backward.
//
// Replaces upstream's renderCUDA forward/backward (SURVEY.md 2.4 K6/K7, App. A.6/A.7; restated
// in oracle/splat_ref.py::composite).  Design:
//   * persistent CTAs pull work from a queue ordered longest-list-first.  FORWARD: a CTA
//     (8 warps x (8x4)-pixel blocks) takes a whole 16x16 tile and shares every gathered chunk;
//     BACKWARD: every warp is an independent worker on one 8x4 block (lists are truncated at the
//     block's own last contributor, so there is no long scan to share and no CTA barrier at all);
//   * a tile's list is its contiguous range of the depth-sorted key array; per chunk of 256
//     entries every thread reads ONE key (coalesced 8-B loads, prefetched two chunks ahead in a
//     register) and copies that Gaussian's 48-byte record from the per-Gaussian array (48 MB at 1M Gaussians: mostly L2-resident in H100's 50 MB L2)
//     straight into a double-buffered shared-memory ring with three 16-byte cp.async (LDGSTS):
//     no register staging, the copies for chunk c+1 fly while chunk c is being blended, and
//     - because saturated tiles stop early - records past the stopping point are never fetched;
//   * each warp tests 32 records at a time (one per lane) against its own 8x4 pixel block
//     (conservative extent test, never changes which pixels blend) and only evaluates the
//     survivors, in list order, reading them back with broadcast LDS.128;
//   * forward: warp/CTA early-out when every pixel is saturated (T < 1e-4 would follow);
//   * backward: per-(warp, Gaussian) partial gradients are reduced with a halving shuffle
//     butterfly (12 SHFL for 10 values) and committed with ONE coalesced RED instruction.
#include "common.cuh"
#include <cuda_fp16.h>
#include <type_traits>

namespace {

// BACKWARD work item = one warp's 8x4 pixel block of one non-empty tile (8 items per tile, queue
// ordered longest list first).  Every warp is an independent worker with a private ring of kSlots
// sub-chunks (32 records = one per lane): the backward kernel contains no CTA-wide barrier.
constexpr int kWarps = 8;      // warps per CTA (in the backward kernel just a container)
constexpr int kSlots = 3;      // backward ring depth per warp (kSlots-1 being gathered + 1 being blended); 1.5 KB per slot and warp
constexpr int kMinCtas = 4;    // backward CTAs per SM: launch bounds and grid size
struct __align__(128) SmemRing {
    GsrRec rec[kWarps][kSlots][32];
};

// Component-wise float2 arithmetic, each component rounded to nearest like the scalar intrinsics.
// sm_90 has no packed fp32 instructions, so each call is two scalar FADD / FMUL / FFMA.
__device__ __forceinline__ float2 fadd2_rn(float2 a, float2 b) {
    return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y));
}
__device__ __forceinline__ float2 fmul2_rn(float2 a, float2 b) {
    return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y));
}
__device__ __forceinline__ float2 ffma2_rn(float2 a, float2 b, float2 c) {
    return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y));
}

__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gsrc) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" :: "r"(smem_u32(smem_dst)), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" :: "n"(N) : "memory"); }

// copy geom[idx(key)] into rec (3 x 16 B)
__device__ __forceinline__ void gather_record(GsrRec* rec, const GsrRec* __restrict__ geom,
                                              unsigned long long key) {
    const char* src = reinterpret_cast<const char*>(geom + (uint32_t)key);
    char* dst = reinterpret_cast<char*>(rec);
    cp_async16(dst, src);
    cp_async16(dst + 16, src + 16);
    cp_async16(dst + 32, src + 32);
}

// Forward epilogue: a block that blended at least one entry becomes a work item of the backward, filed under
// the size class of its consumed list length (see GSR_BWD_CLASSES).  `n` is warp-uniform; call from lane 0.
__device__ __forceinline__ void bwd_item_append(uint32_t* fill, uint32_t* items, int ntiles, uint32_t tile,
                                                int blk, uint32_t n) {
    if (items == nullptr || n == 0u) return;
    const int k = gsr_bwd_class(n);
    const uint32_t slot = atomicAdd(fill + k, 1u);
    items[(size_t)k * ntiles * 8 + slot] = tile * 8u + (uint32_t)blk;
}

// The blending test, shared verbatim by forward and backward so both take identical decisions.
struct PairEval {
    float dx, dy, G, alpha;
    bool valid;
};
__device__ __forceinline__ PairEval eval_pair(float px, float py, float A, float B, float C,
                                              float opacity, float X, float Y) {
    PairEval e;
    const float2 d2 = fadd2_rn(make_float2(px, py), make_float2(-X, -Y));
    e.dx = d2.x;
    e.dy = d2.y;
#ifdef GSR_EXACT_EXP
    // oracle order (splat_ref.py::composite): power = -0.5*(A*dx*dx + C*dy*dy) - B*dx*dy, raw conic
    const float qs = __fadd_rn(__fmul_rn(__fmul_rn(A, e.dx), e.dx), __fmul_rn(__fmul_rn(C, e.dy), e.dy));
    const float p2 = __fsub_rn(__fmul_rn(-0.5f, qs), __fmul_rn(__fmul_rn(B, e.dx), e.dy));
    e.G = expf(fminf(p2, 0.0f));
#else
    const float u = __fmaf_rn(A, e.dx, __fmul_rn(B, e.dy));
    const float p2 = __fmaf_rn(__fmul_rn(C, e.dy), e.dy, __fmul_rn(u, e.dx));
    e.G = ex2_approx(p2);
#endif
    e.alpha = fminf(GSR_ALPHA_MAX, __fmul_rn(opacity, e.G));
    e.valid = (p2 <= 0.0f) && (e.alpha >= GSR_ALPHA_MIN);
    return e;
}

__device__ __forceinline__ bool cull_pass(float px, float py, uint32_t ext, float X0, float Y0) {
    // block covers pixel centres [X0, X0+7] x [Y0, Y0+3]
    const __half2 eh = *reinterpret_cast<const __half2*>(&ext);
    const float2 e = __half22float2(eh);
    const float ddx = fmaxf(fmaxf(X0 - px, px - (X0 + 7.0f)), 0.0f);
    const float ddy = fmaxf(fmaxf(Y0 - py, py - (Y0 + 3.0f)), 0.0f);
    return (ddx <= e.x) && (ddy <= e.y);
}

// slots of the optional diagnostic counters (b200gsr_debug_counters)
enum { GSR_STAT_BWD_EVAL = 0, GSR_STAT_BWD_CONTRIB = 1, GSR_STAT_BWD_LANES = 2, GSR_STAT_BWD_HIST = 3,   // 3..8
       GSR_STAT_FWD_EVAL = 10, GSR_STAT_FWD_LANES = 11,
       // load balance of the persistent kernels (globaltimer ns): sum of worker busy time, last exit,
       // ~(first entry) [so that atomicMax on a zeroed word yields the minimum], workers, largest item
       GSR_STAT_FWD_BUSY = 16, GSR_STAT_FWD_END = 17, GSR_STAT_FWD_NBEGIN = 18, GSR_STAT_FWD_WORKERS = 19,
       GSR_STAT_FWD_MAX_ITEM = 20,
       GSR_STAT_BWD_BUSY = 21, GSR_STAT_BWD_END = 22, GSR_STAT_BWD_NBEGIN = 23, GSR_STAT_BWD_WORKERS = 24,
       GSR_STAT_BWD_MAX_ITEM = 25, GSR_STAT_BWD_MAX_ITEM_NS = 26, GSR_STAT_WORDS = 32 };
__device__ __forceinline__ unsigned long long gsr_now_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}

// =============================================================================================
// Forward
// =============================================================================================
// Forward keeps the tile as the unit of work: blocks that never saturate (silhouettes, thin
// regions) must scan the whole list, and sharing each gathered 256-entry chunk between the 8
// warps of the tile makes that scan cheap (measured faster than independent warps).
constexpr int kChunk = 256;   // list entries per pipeline stage (one per thread)
constexpr int kIlp = 2;       // passing list entries in flight per warp
struct __align__(128) SmemCta {
    GsrRec rec[2][kChunk];   // 2 x 12 KB
    uint32_t work;           // broadcast slot for the tile queue
};

// One CTA of 8 warps per tile; warp w blends pixel block w, PPL rows of 8 pixels per lane.  PPL is 1, but the per-pixel
// state stays in PPL-element arrays: written as scalars, the kernel compiles to different code from the measured one.
// DET (deterministic mode, with SCORE): `score` points to the int64 fixed-point accumulators (GsrDetLayout::score_fx)
// and each warp's weight sum is committed as an integer (gsr_det_score_quantise).
// SCORE_ONLY (with SCORE; the score pass, b200gsr_score_views): the same tile loop, cull, blending test, T recurrence
// and early-outs, but no image, n_contrib or backward work list is written.  Every view of the stacked pass adds into
// ONE accumulator of P_view rows: entry idx of view v commits to row idx - v * P_view.  A pass that overflowed its pair
// capacity commits nothing, so re-issuing it with a larger capacity adds exactly what one complete pass adds.
template <bool SCORE, bool STATS, bool DET = false, bool SCORE_ONLY = false>
__global__ void __launch_bounds__(256)
composite_fwd_kernel(int H, int W, int gx, int gy_view, int Hs, int ntiles, const uint32_t* __restrict__ header,
                     const uint32_t* __restrict__ work_order,
                     const uint32_t* __restrict__ tile_start,
                     const unsigned long long* __restrict__ keys, const GsrRec* __restrict__ geom,
                     const float* __restrict__ bg, uint32_t* __restrict__ queue,
                     float* __restrict__ out_color, float* __restrict__ out_depth_alpha,
                     uint32_t* __restrict__ n_contrib, float* __restrict__ score,
                     unsigned long long* __restrict__ stats, uint32_t* bwd_fill, uint32_t* bwd_items, int P_view) {
    constexpr int PPL = 1;
    constexpr int kThreads = 256;
    unsigned int st_eval = 0, st_lanes = 0;
    unsigned long long st_t0 = 0, st_item_t0 = 0, st_max_item_ns = 0;
    if (STATS) st_t0 = gsr_now_ns();
    constexpr int kPer = kChunk / kThreads;   // list entries gathered per thread per chunk
    extern __shared__ __align__(128) unsigned char smem_raw[];
    SmemCta& sm = *reinterpret_cast<SmemCta*>(smem_raw);
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    if (SCORE_ONLY && header[GSR_H_OVERFLOW] != 0u) return;
    const uint32_t max_pairs = header[GSR_H_MAX_PAIRS];

    for (;;) {
        // one shared counter over ALL tiles (empty ones included, they come last): measured faster
        // here than the split queue + static empty tiles
        if (STATS) {
            const unsigned long long t = gsr_now_ns();
            if (st_item_t0 && t - st_item_t0 > st_max_item_ns) st_max_item_ns = t - st_item_t0;
            st_item_t0 = t;
        }
        if (tid == 0) sm.work = atomicAdd(queue, 1u);
        __syncthreads();
        const uint32_t w = sm.work;
        __syncthreads();   // everyone has read the slot before thread 0 may overwrite it
        if (w >= (uint32_t)ntiles) break;
        const uint32_t tile = work_order[w];
        const int blk = wid;      // 8x(4*PPL)-pixel block of the tile this warp renders
        uint32_t beg = tile_start[tile], end = tile_start[tile + 1];
        if (end > max_pairs) end = max_pairs;
        if (beg > end) beg = end;
        const int n = (int)(end - beg);
        const int nchunks = (n + kChunk - 1) / kChunk;
        const unsigned long long* tk = keys + beg;
        const int tys = tile / gx, txi = tile - tys * gx;
        // multi-view: tile row tys of the stacked image = row tyi of view `view`; everything is evaluated in
        // view-local pixel coordinates (bit-identical to a single-view render), only addressing is stacked
        const int view = tys / gy_view, tyi = tys - view * gy_view;
        const int row0 = view * gy_view * GSR_TILE;
        const float* bgv = bg + 3 * view;
        const float bg0 = SCORE_ONLY ? 0.f : __ldg(bgv), bg1 = SCORE_ONLY ? 0.f : __ldg(bgv + 1),
                    bg2 = SCORE_ONLY ? 0.f : __ldg(bgv + 2);
        const uint32_t idx0 = SCORE_ONLY ? (uint32_t)view * (uint32_t)P_view : 0u;   // first score row of this view
        const int X0i = txi * GSR_TILE + (blk & 1) * 8, Y0i = tyi * GSR_TILE + (blk >> 1) * (4 * PPL);
        const int Xi = X0i + (lane & 7), Yi = Y0i + (lane >> 3);
        const float X0 = (float)X0i, Y0 = (float)Y0i, X = (float)Xi;
        bool inside[PPL], done[PPL];
        float Y[PPL], T[PPL];
        float2 C01[PPL], C2D[PPL];         // (r, g) and (b, depth) accumulators: two fused multiply-adds each per blend
        uint32_t last[PPL];
        bool all_done = true;
#pragma unroll
        for (int q = 0; q < PPL; ++q) {
            inside[q] = Xi < W && (Yi + 4 * q) < H;
            done[q] = !inside[q];
            all_done = all_done && done[q];
            Y[q] = (float)(Yi + 4 * q);
            T[q] = 1.0f; C01[q] = make_float2(0.f, 0.f); C2D[q] = make_float2(0.f, 0.f); last[q] = 0;
        }

        // prologue: gather chunk 0, prefetch the keys of chunk 1
        unsigned long long knext[kPer];
#pragma unroll
        for (int u = 0; u < kPer; ++u) {
            const int e = u * kThreads + tid;
            if (e < n) gather_record(&sm.rec[0][e], geom, __ldg(tk + e));
            knext[u] = (kChunk + e < n) ? __ldg(tk + kChunk + e) : 0ull;
        }
        cp_async_commit();

        for (int c = 0; c < nchunks; ++c) {
            cp_async_wait<0>();   // my copies for chunk c have landed
            // barrier: everyone's copies for chunk c are visible, everyone is done with chunk c-1;
            // it doubles as the CTA-wide early-out vote.  all_done is done[0] (PPL is 1); SCORE_ONLY votes on done[0]
            // itself, which saves that instantiation the register a separate all_done costs.
            const int ndone = __syncthreads_count(SCORE_ONLY ? done[0] : all_done);
            if (ndone == kThreads) break;
            // issue the gathers for chunk c+1 (they fly while chunk c is blended), then fetch the
            // keys of chunk c+2
#pragma unroll
            for (int u = 0; u < kPer; ++u) {
                const int e = u * kThreads + tid;
                if ((c + 1) * kChunk + e < n) gather_record(&sm.rec[(c + 1) & 1][e], geom, knext[u]);
                knext[u] = ((c + 2) * kChunk + e < n) ? __ldg(tk + (c + 2) * kChunk + e) : 0ull;
            }
            cp_async_commit();

            const GsrRec* st = sm.rec[c & 1];
            const int cnt = min(kChunk, n - c * kChunk);
            if (__all_sync(0xffffffffu, SCORE_ONLY ? done[0] : all_done)) continue;   // this warp is saturated
            for (int sub = 0; sub * 32 < cnt; ++sub) {
                const int r = sub * 32 + lane;
                bool pass = false;
                if (r < cnt) {
                    const float4 q0 = *reinterpret_cast<const float4*>(&st[r]);
                    pass = cull_pass(q0.x, q0.y, __float_as_uint(q0.z), X0, Y0);
                }
                uint32_t mask = __ballot_sync(0xffffffffu, pass);
                const float4* sp = reinterpret_cast<const float4*>(&st[sub * 32]);
                const uint32_t pos0 = (uint32_t)(c * kChunk + sub * 32 + 1);
                // One list entry applied to this lane's pixel(s): the T / colour recurrences are the only
                // dependences between consecutive entries.
                auto blend = [&](const float4& q1, const float4& q2, const PairEval (&ev)[PPL], int b) {
                    float wsum = 0.f;
                    if (STATS) ++st_eval;
#pragma unroll
                    for (int q = 0; q < PPL; ++q) {
                        const PairEval& e = ev[q];
                        if (e.valid && !done[q]) {
                            const float Tn = T[q] * (1.0f - e.alpha);
                            if (Tn < GSR_T_STOP) {
                                done[q] = true;
                            } else {
                                const float wgt = e.alpha * T[q];
                                const float2 w2 = make_float2(wgt, wgt);
                                C01[q] = ffma2_rn(make_float2(q2.x, q2.y), w2, C01[q]);
                                C2D[q] = ffma2_rn(make_float2(q2.z, q1.w), w2, C2D[q]);
                                T[q] = Tn;
                                last[q] = pos0 + (uint32_t)b;
                                if (SCORE) wsum += wgt;
                                if (STATS) ++st_lanes;
                            }
                        }
                    }
                    if (SCORE) {
#pragma unroll
                        for (int o = 16; o > 0; o >>= 1) wsum += __shfl_xor_sync(0xffffffffu, wsum, o);
                        if (lane == 0 && wsum != 0.f) {
                            if (DET)
                                atomicAdd(reinterpret_cast<unsigned long long*>(score) + (__float_as_uint(q2.w) - idx0),
                                          (unsigned long long)gsr_det_score_quantise(wsum));
                            else
                                atomicAdd(score + (__float_as_uint(q2.w) - idx0), wsum);
                        }
                    }
                };
                while (mask) {
                    const int b = __ffs(mask) - 1;
                    mask &= mask - 1;
                    const float4* rp = sp + 3 * b;
                    const float4 q0 = rp[0], q1 = rp[1], q2 = rp[2];
                    // kIlp passing entries per trip: the record loads and exponents of the later ones are
                    // in flight while the first is evaluated (a warp issues in order, so this divides the
                    // dependent LDS -> FMA -> EX2 latency paid per entry on the longest tile, which bounds
                    // the kernel).  Same arithmetic and order per entry.
                    int bb[kIlp];
                    float4 r0[kIlp], r1[kIlp], r2[kIlp];
                    bb[0] = b; r0[0] = q0; r1[0] = q1; r2[0] = q2;
                    int have = 1;                                      // warp-uniform
#pragma unroll
                    for (int j = 1; j < kIlp; ++j) {
                        const bool more = mask != 0u;
                        bb[j] = more ? __ffs(mask) - 1 : b;
                        mask &= mask - 1;                              // 0 stays 0
                        have += more ? 1 : 0;
                        const float4* rj = sp + 3 * bb[j];
                        r0[j] = rj[0]; r1[j] = rj[1]; r2[j] = rj[2];
                    }
                    PairEval ev[kIlp][PPL];
#pragma unroll
                    for (int j = 0; j < kIlp; ++j)
#pragma unroll
                        for (int q = 0; q < PPL; ++q)
                            ev[j][q] = eval_pair(r0[j].x, r0[j].y, r0[j].w, r1[j].x, r1[j].y, r1[j].z, X, Y[q]);
#pragma unroll
                    for (int j = 0; j < kIlp; ++j)
                        if (j < have) blend(r1[j], r2[j], ev[j], bb[j]);
                }
                all_done = true;
#pragma unroll
                for (int q = 0; q < PPL; ++q) all_done = all_done && done[q];
                if (__all_sync(0xffffffffu, all_done)) break;
            }
        }
        cp_async_wait<0>();   // never leave copies in flight across tiles (early-out case)
        if constexpr (SCORE_ONLY) continue;   // no image, n_contrib or backward work list

        const size_t plane = (size_t)Hs * W;
#pragma unroll
        for (int q = 0; q < PPL; ++q) {
            if (inside[q]) {
                const size_t pix = (size_t)(row0 + Yi + 4 * q) * W + Xi;
                out_color[pix] = fmaf(T[q], bg0, C01[q].x);
                out_color[plane + pix] = fmaf(T[q], bg1, C01[q].y);
                out_color[2 * plane + pix] = fmaf(T[q], bg2, C2D[q].x);
                out_depth_alpha[pix] = C2D[q].y;
                out_depth_alpha[plane + pix] = T[q];
                n_contrib[pix] = last[q];
            }
            // this 8x4 block's entry in the backward's work lists (fwd block blk, pixel row set q)
            const uint32_t nb = __reduce_max_sync(0xffffffffu, last[q]);
            if (lane == 0) bwd_item_append(bwd_fill, bwd_items, ntiles, tile, ((blk >> 1) * PPL + q) * 2 + (blk & 1), nb);
        }
    }
    if (STATS && stats != nullptr) {
        const unsigned int tl = __reduce_add_sync(0xffffffffu, st_lanes);
        if (lane == 0) {
            atomicAdd(stats + GSR_STAT_FWD_EVAL, (unsigned long long)st_eval);
            atomicAdd(stats + GSR_STAT_FWD_LANES, (unsigned long long)tl);
        }
        if (threadIdx.x == 0) {
            const unsigned long long t1 = gsr_now_ns();
            atomicAdd(stats + GSR_STAT_FWD_BUSY, t1 - st_t0);
            atomicMax(stats + GSR_STAT_FWD_END, t1);
            atomicMax(stats + GSR_STAT_FWD_NBEGIN, ~st_t0);
            atomicAdd(stats + GSR_STAT_FWD_WORKERS, 1ull);
            atomicMax(stats + GSR_STAT_FWD_MAX_ITEM, st_max_item_ns);
        }
    }
}

// =============================================================================================
// Backward: the work items are the (tile, 8x4 block) lists the forward wrote, walked back to front.
//   * branch-free body: non-contributing lanes run the same arithmetic with alpha = G = 0 instead of a
//     divergent block + ten zero-initialisations;
//   * the four channel-parallel streams (r, g, b, depth) and the (x, y) geometry pairs are written
//     as float2 operations (fadd2_rn / fmul2_rn / ffma2_rn), two independent scalar ops each on sm_90;
//   * per (warp, Gaussian), the ten partials are reduced with a halving shuffle butterfly and
//     committed by ten lanes at once;
//   * the STATS instantiation counts evaluated / contributing (warp, Gaussian) pairs and the popcount
//     histogram for the secondary (pair-evaluation) roofline in bench.py; never timed.
// =============================================================================================
__device__ __forceinline__ int bwd_value_index(int lane) {
    // which of the 10 values this lane ends up owning (-1: a padding slot)
    int base = 0, n = 10;
    if (lane & 16) { base += 5; n = 5; } else { n = 5; }
    if (lane & 8) { base += 3; n = n - 3; } else { n = min(n, 3); }
    if (lane & 4) { base += 2; n = max(n - 2, 0); } else { n = min(n, 2); }
    if (lane & 2) { base += 1; n = max(n - 1, 0); } else { n = min(n, 1); }
    return n >= 1 ? base : -1;
}

// How composite_bwd_kernel commits a (warp item, Gaussian) partial of component c.
enum { GSR_ACC_FLOAT = 0,      // fp32 atomicAdd into dgeom (default)
       GSR_ACC_DET_MAX = 1,    // deterministic pass A: atomicMax of |partial|'s bits into dmax
       GSR_ACC_DET_SUM = 2 };  // deterministic pass B: int64 atomicAdd of the fixed-point partial into dfx
// mb (pass B): dmax of the component, loaded by the caller ahead of the arithmetic that produces v.
template <int ACC>
__device__ __forceinline__ void commit_partial(uint32_t* dmax, unsigned long long* dfx, uint32_t g, int c, float v,
                                               uint32_t mb) {
    if (ACC == GSR_ACC_DET_MAX) {
        atomicMax(dmax + GSR_DET_COMPONENTS * (size_t)g + c, __float_as_uint(fabsf(v)));
    } else if (ACC == GSR_ACC_DET_SUM) {
        // a non-finite component skips the sums: the result is NaN whatever they hold (gsr_det_dequantise)
        if (gsr_det_finite(mb))
            atomicAdd(dfx + GSR_DET_COMPONENTS * (size_t)g + c, (unsigned long long)gsr_det_quantise(v, gsr_det_shift(mb)));
    }
}

// One step of the halving butterfly: after the steps XOR = 16, 8, 4, 2 and a final XOR-1 shuffle, v[0] of
// lane L holds the warp-wide sum of value bwd_value_index(L); 5+3+2+1+1 = 12 shuffles for 10 values.
template <int N, int XOR>
__device__ __forceinline__ void halve2(float (&v)[10], bool hi) {
    constexpr int Hh = (N + 1) / 2;
    float keep[Hh], recv[Hh];
#pragma unroll
    for (int k = 0; k < Hh; ++k) {
        const float lo = v[k];
        const float hv = (Hh + k < N) ? v[Hh + k] : 0.0f;
        const float send = hi ? lo : hv;
        keep[k] = hi ? hv : lo;
        recv[k] = __shfl_xor_sync(0xffffffffu, send, XOR);
    }
#pragma unroll
    for (int k = 0; k + 1 < Hh; k += 2) {
        const float2 r = fadd2_rn(make_float2(keep[k], keep[k + 1]), make_float2(recv[k], recv[k + 1]));
        v[k] = r.x; v[k + 1] = r.y;
    }
    if (Hh & 1) v[Hh - 1] = keep[Hh - 1] + recv[Hh - 1];
}

// Frozen rows (GsrFrozenRanges) as merged half-open intervals [lo, lo + len): the caller's ranges of
// b200gsr_backward_views_frozen, or the packed rows of the scene backwards' frozen groups.  Adjacent frozen groups
// merge, so 24 groups give at most 12 intervals.
constexpr int kMaxFrozenIntervals = (B200GSR_MAX_GROUPS + 1) / 2;
static_assert(kMaxFrozenIntervals == B200GSR_MAX_FROZEN_RANGES, "b200gsr_views_frozen.h states the interval limit");
struct NoFrozen {};
struct FrozenRows {
    uint32_t n;                              // intervals in use
    uint32_t P_view;                         // record index q2.w of view v's row r is v * P_view + r
    uint32_t lo[kMaxFrozenIntervals], len[kMaxFrozenIntervals];
};
template <bool FROZEN>
using FrozenArg = std::conditional_t<FROZEN, FrozenRows, NoFrozen>;
// A loop over the intervals in use, reading them from the constant bank (fz is a __grid_constant__ parameter, so the
// dynamic index needs no local copy).  Unrolled over all twelve slots, the test cost every entry about as much as
// the gradient body it saves on a frozen one (composite_bwd 0.77 -> 1.00 ms with one interval, H100).
__device__ __forceinline__ bool row_frozen(const FrozenRows& f, uint32_t row) {
#pragma unroll 1
    for (uint32_t k = 0; k < f.n; ++k)
        if (row - f.lo[k] < f.len[k]) return true;
    return false;
}

// ACC: how the butterfly's per-(warp item, Gaussian) totals are committed (GSR_ACC_*).  Every commit is a
// butterfly total, a function of its work item alone, which the deterministic passes rely on.
// FROZEN (STATS false): an entry whose row lies in one of fz's intervals only advances the transmittance and colour
// recurrences, which the entries behind it need; its gradient body, butterfly, commit and (pass B) dmax load are
// skipped, so its dgeom / dmax / dfx rows are never written.  The test is warp-uniform (every lane reads the same
// record) and needs no load beyond the record part 2 that the recurrence reads anyway.
template <bool STATS, int ACC = GSR_ACC_FLOAT, bool FROZEN = false>
__global__ void __launch_bounds__(kWarps * 32, kMinCtas)
composite_bwd_kernel(int H, int W, int gx, int gy_view, int Hs, int ntiles, const uint32_t* __restrict__ header,
                     const uint32_t* __restrict__ work_order,
                     const uint32_t* __restrict__ tile_start,
                     const unsigned long long* __restrict__ keys, const GsrRec* __restrict__ geom,
                     const float* __restrict__ bg, uint32_t* __restrict__ queue,
                     const float* __restrict__ out_depth_alpha,
                     const uint32_t* __restrict__ n_contrib, const float* __restrict__ dL_dcolor,
                     const float* __restrict__ dL_ddepth_alpha, float* __restrict__ dgeom,
                     unsigned long long* __restrict__ stats, const uint32_t* __restrict__ bwd_items,
                     uint32_t* __restrict__ dmax, unsigned long long* __restrict__ dfx,
                     const __grid_constant__ FrozenArg<FROZEN> fz) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    SmemRing& sm = *reinterpret_cast<SmemRing*>(smem_raw);
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    GsrRec (*ring)[32] = sm.rec[wid];
    const uint32_t max_pairs = header[GSR_H_MAX_PAIRS];
    // Work lists written by the forward: (tile, block) items by size class of the consumed list length.
    // Lane l holds the END of class (31 - l) in the concatenated longest-first order.
    uint32_t cls_end = header[GSR_H_BWD_FILL + (GSR_BWD_CLASSES - 1 - lane)];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t t = __shfl_up_sync(0xffffffffu, cls_end, o);
        if (lane >= o) cls_end += t;
    }
    const uint32_t num_items = __shfl_sync(0xffffffffu, cls_end, 31);
    const size_t cls_cap = (size_t)ntiles * 8;
    static_assert(kWarps % GSR_NQUEUE == 0, "static first items must end on a sub-queue boundary");
    const uint32_t nworkers = gridDim.x * kWarps;            // the first item of every warp is static: no atomic
    const uint32_t i_first = (nworkers + GSR_NQUEUE - 1) / GSR_NQUEUE;
    bool first_item = true;
    const int vidx = bwd_value_index(lane);
    const bool commit_lane = (vidx >= 0) && !(lane & 1);
    const size_t plane = (size_t)Hs * W;
    unsigned long long st_eval = 0, st_contrib = 0, st_lanes = 0;
    unsigned long long st_hist[6] = {0, 0, 0, 0, 0, 0};
    unsigned long long st_t0 = 0, st_item_eval0 = 0, st_item_t0 = 0, st_max_item = 0, st_max_item_ns = 0;
    if (STATS) st_t0 = gsr_now_ns();

    uint32_t qsel = (blockIdx.x * kWarps + wid) % GSR_NQUEUE, qtried = 0;
    for (;;) {
        if (STATS) {
            if (st_eval - st_item_eval0 > st_max_item) st_max_item = st_eval - st_item_eval0;
            const unsigned long long t = gsr_now_ns();
            if (st_item_t0 && t - st_item_t0 > st_max_item_ns) st_max_item_ns = t - st_item_t0;
            st_item_eval0 = st_eval; st_item_t0 = t;
        }
        // position w in the longest-first order: warp g starts with w = g, later ones come from the split queue
        uint32_t w;
        if (first_item) {
            first_item = false;
            w = blockIdx.x * kWarps + wid;
            if (w >= num_items) break;
        } else {
            uint32_t i = 0xffffffffu;
            if (lane == 0) {
                while (qtried < GSR_NQUEUE) {
                    const uint32_t cand = (atomicAdd(queue + qsel, 1u) + i_first) * GSR_NQUEUE + qsel;
                    if (cand < num_items) { i = cand; break; }
                    qsel = (qsel + 1) % GSR_NQUEUE;
                    ++qtried;
                }
            }
            w = __shfl_sync(0xffffffffu, i, 0);
            if (w == 0xffffffffu) break;
        }
        const int cdone = __popc(__ballot_sync(0xffffffffu, cls_end <= w));          // classes entirely before w
        const uint32_t cstart = __shfl_sync(0xffffffffu, cls_end, (cdone + 31) & 31);
        const uint32_t item = __ldg(bwd_items + (size_t)(GSR_BWD_CLASSES - 1 - cdone) * cls_cap + (w - (cdone ? cstart : 0u)));
        const uint32_t tile = item >> 3;
        const int blk = (int)(item & 7u);
        uint32_t beg = tile_start[tile], end = tile_start[tile + 1];
        if (end > max_pairs) end = max_pairs;
        if (beg > end) beg = end;
        const unsigned long long* tk = keys + beg;
        const int tys = tile / gx, txi = tile - tys * gx;
        const int view = tys / gy_view, tyi = tys - view * gy_view;      // view-local evaluation, stacked addressing
        const int row0 = view * gy_view * GSR_TILE;
        const float* bgv = bg + 3 * view;
        const float bg0 = __ldg(bgv), bg1 = __ldg(bgv + 1), bg2 = __ldg(bgv + 2);
        const int X0i = txi * GSR_TILE + (blk & 1) * 8, Y0i = tyi * GSR_TILE + (blk >> 1) * 4;
        const int Xi = X0i + (lane & 7), Yi = Y0i + (lane >> 3);
        const float X0 = (float)X0i, Y0 = (float)Y0i;
        const float2 XY = make_float2(-(float)Xi, -(float)Yi);
        uint32_t last = 0;
        float Tfinal = 1.f, dT = 0.f;
        float2 dC01 = make_float2(0.f, 0.f), dC2D = make_float2(0.f, 0.f);
        if (Xi < W && Yi < H) {
            const size_t pix = (size_t)(row0 + Yi) * W + Xi;
            last = n_contrib[pix];
            Tfinal = out_depth_alpha[plane + pix];
            dC01.x = dL_dcolor[pix]; dC01.y = dL_dcolor[plane + pix]; dC2D.x = dL_dcolor[2 * plane + pix];
            dC2D.y = dL_ddepth_alpha[pix]; dT = dL_ddepth_alpha[plane + pix];
        }
        if ((int)last > (int)(end - beg)) last = end - beg;   // overflow safety
        const int n = (int)__reduce_max_sync(0xffffffffu, last);   // only entries [0, n) reached this block
        const int nsub = (n + 31) >> 5;
        const float bgT = Tfinal * (bg0 * dC01.x + bg1 * dC01.y + bg2 * dC2D.x + dT);   // Tfinal * bgterm
        float T = Tfinal;
        float2 acc01 = make_float2(0.f, 0.f), acc2D = make_float2(0.f, 0.f);

        // sub-chunks are visited from the back: visit v <-> sub-chunk nsub-1-v
        unsigned long long kq0, kq1;
        {
            unsigned long long kk[kSlots + 1];
#pragma unroll
            for (int j = 0; j < kSlots + 1; ++j) {
                const int e = (nsub - 1 - j) * 32 + lane;
                kk[j] = (j < nsub && e < n) ? __ldg(tk + e) : 0ull;
            }
#pragma unroll
            for (int j = 0; j < kSlots - 1; ++j) {
                const int e = (nsub - 1 - j) * 32 + lane;
                if (j < nsub && e < n) gather_record(&ring[j][lane], geom, kk[j]);
                cp_async_commit();
            }
            kq0 = kk[kSlots - 1]; kq1 = kk[kSlots];
        }
        for (int v = 0; v < nsub; ++v) {
            {
                const int g = v + kSlots - 1;
                if (g < nsub) gather_record(&ring[g % kSlots][lane], geom, kq0);   // earlier sub-chunks are full
                cp_async_commit();
                kq0 = kq1;
                const int g2 = v + kSlots + 1;
                kq1 = (g2 < nsub) ? __ldg(tk + (nsub - 1 - g2) * 32 + lane) : 0ull;
            }
            cp_async_wait<kSlots - 1>();
            __syncwarp();
            const GsrRec* st = ring[v % kSlots];
            const int sidx = nsub - 1 - v;
            const int cnt = min(32, n - sidx * 32);
            bool pass = false;
            if (lane < cnt) {
                const float4 q0 = *reinterpret_cast<const float4*>(&st[lane]);
                pass = cull_pass(q0.x, q0.y, __float_as_uint(q0.z), X0, Y0);
            }
            uint32_t mask = __ballot_sync(0xffffffffu, pass);
            const float4* sp = reinterpret_cast<const float4*>(st);
            const uint32_t pos0 = (uint32_t)(sidx * 32 + 1);
            while (mask) {
                const int b = 31 - __clz(mask);
                mask &= ~(1u << b);
                const float4* rp = sp + 3 * b;
                const float4 q0 = rp[0], q1 = rp[1];
                const uint32_t pos = pos0 + (uint32_t)b;
                // ---- the blending test ----
                const PairEval e = eval_pair(q0.x, q0.y, q0.w, q1.x, q1.y, q1.z, -XY.x, -XY.y);
                const float2 d = make_float2(e.dx, e.dy);
                const float G = e.G, alpha = e.alpha;
                const bool valid = e.valid;
                const bool contrib = valid && pos <= last;
                const uint32_t cm = __ballot_sync(0xffffffffu, contrib);
                if (STATS) ++st_eval;
                if (cm == 0u) continue;
                const float4 q2 = rp[2];
                if constexpr (FROZEN) {
                    if (row_frozen(fz, __float_as_uint(q2.w) - (uint32_t)view * fz.P_view)) {
                        // the recurrence statements of the body below, in its order
                        const float am = contrib ? alpha : 0.0f;
                        const float rom = rcp_approx(1.0f - am);
                        T = contrib ? T * rom : T;
                        const float2 c01 = make_float2(q2.x, q2.y), c2D = make_float2(q2.z, q1.w);
                        const float2 nacc01 = make_float2(-acc01.x, -acc01.y), nacc2D = make_float2(-acc2D.x, -acc2D.y);
                        const float2 d01 = fadd2_rn(c01, nacc01), d2D = fadd2_rn(c2D, nacc2D);
                        const float2 am2 = make_float2(am, am);
                        acc01 = ffma2_rn(am2, d01, acc01);
                        acc2D = ffma2_rn(am2, d2D, acc2D);
                        continue;
                    }
                }
                uint32_t det_mb = 0u;   // pass B: issued here so that its latency hides behind the body and butterfly
                if (ACC == GSR_ACC_DET_SUM && commit_lane)
                    det_mb = __ldg(dmax + GSR_DET_COMPONENTS * (size_t)__float_as_uint(q2.w) + vidx);
                // ---- branch-free body: non-contributing lanes carry alpha = G = 0 ----
                const float am = contrib ? alpha : 0.0f;
                const float Gm = contrib ? G : 0.0f;
                const float rom = rcp_approx(1.0f - am);
                T = contrib ? T * rom : T;                       // transmittance in front of this entry
                const float wgt = am * T;
                const float2 c01 = make_float2(q2.x, q2.y), c2D = make_float2(q2.z, q1.w);
                const float2 nacc01 = make_float2(-acc01.x, -acc01.y), nacc2D = make_float2(-acc2D.x, -acc2D.y);
                const float2 d01 = fadd2_rn(c01, nacc01), d2D = fadd2_rn(c2D, nacc2D);
                const float2 dot2 = ffma2_rn(d2D, dC2D, fmul2_rn(d01, dC01));
                const float dLda = (dot2.x + dot2.y) * T - bgT * rom;
                const float2 am2 = make_float2(am, am);
                acc01 = ffma2_rn(am2, d01, acc01);
                acc2D = ffma2_rn(am2, d2D, acc2D);
                float vv[10];
                vv[5] = Gm * dLda;
                const float gG = q1.z * vv[5];                   // dL/dG * G (no zeroing under the 0.99 clamp)
#ifdef GSR_EXACT_EXP
                const float2 gs = make_float2(-(q0.w * d.x + q1.x * d.y), -(q1.y * d.y + q1.x * d.x));
#else
                const float2 gs = ffma2_rn(make_float2(q0.w + q0.w, q1.y + q1.y), d, fmul2_rn(make_float2(q1.x, q1.x), make_float2(d.y, d.x)));
#endif
                const float2 gG2 = make_float2(gG, gG);
                const float2 v01 = fmul2_rn(gG2, gs);
                const float2 tu = fmul2_rn(gG2, d);             // (gG dx, gG dy)
                const float2 v24 = fmul2_rn(tu, d);             // (gG dx^2, gG dy^2)
                vv[0] = v01.x; vv[1] = v01.y; vv[2] = v24.x; vv[3] = tu.x * d.y; vv[4] = v24.y;
                const float2 w2 = make_float2(wgt, wgt);
                const float2 v67 = fmul2_rn(w2, dC01), v89 = fmul2_rn(w2, dC2D);
                vv[6] = v67.x; vv[7] = v67.y; vv[8] = v89.x; vv[9] = v89.y;
                float* row = dgeom + 12 * (size_t)__float_as_uint(q2.w);
                if (STATS) {
                    const int k = __popc(cm);
                    ++st_contrib; st_lanes += k;
                    ++st_hist[k == 1 ? 0 : k == 2 ? 1 : k <= 4 ? 2 : k <= 8 ? 3 : k <= 16 ? 4 : 5];
                }
                halve2<10, 16>(vv, lane & 16);
                halve2<5, 8>(vv, lane & 8);
                halve2<3, 4>(vv, lane & 4);
                halve2<2, 2>(vv, lane & 2);
                const float tot = vv[0] + __shfl_xor_sync(0xffffffffu, vv[0], 1);
                if (ACC == GSR_ACC_FLOAT) {
                    if (commit_lane) atomicAdd(row + vidx, tot);
                } else if (commit_lane) {
                    commit_partial<ACC>(dmax, dfx, __float_as_uint(q2.w), vidx, tot, det_mb);
                }
            }
            __syncwarp();
        }
        cp_async_wait<0>();
        __syncwarp();
    }
    if (STATS && lane == 0 && stats != nullptr) {
        atomicAdd(stats + GSR_STAT_BWD_EVAL, st_eval);
        atomicAdd(stats + GSR_STAT_BWD_CONTRIB, st_contrib);
        atomicAdd(stats + GSR_STAT_BWD_LANES, st_lanes);
#pragma unroll
        for (int j = 0; j < 6; ++j) atomicAdd(stats + GSR_STAT_BWD_HIST + j, st_hist[j]);
        const unsigned long long t1 = gsr_now_ns();
        atomicAdd(stats + GSR_STAT_BWD_BUSY, t1 - st_t0);
        atomicMax(stats + GSR_STAT_BWD_END, t1);
        atomicMax(stats + GSR_STAT_BWD_NBEGIN, ~st_t0);
        atomicAdd(stats + GSR_STAT_BWD_WORKERS, 1ull);
        atomicMax(stats + GSR_STAT_BWD_MAX_ITEM, st_max_item);
        atomicMax(stats + GSR_STAT_BWD_MAX_ITEM_NS, st_max_item_ns);
    }
}

// Deterministic mode, after pass B: the fixed-point sums of every visible Gaussian become the float dgeom row
// project_bwd reads, and both integer arrays are cleared for the next backward over this `saved` (read-and-clear,
// like dgeom itself).  Rows of culled Gaussians were never touched by the composite.
__global__ void __launch_bounds__(256)
det_resolve_kernel(int n, const int32_t* __restrict__ radii, uint32_t* __restrict__ dmax,
                   unsigned long long* __restrict__ dfx, float* __restrict__ dgeom, uint32_t* __restrict__ queue_b) {
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i < GSR_NQUEUE) queue_b[i] = 0u;   // pass B (the previous kernel) has drained its work queue
    if (i >= n || __ldg(radii + i) <= 0) return;
    uint32_t* mx = dmax + GSR_DET_COMPONENTS * (size_t)i;
    unsigned long long* fx = dfx + GSR_DET_COMPONENTS * (size_t)i;
    float* row = dgeom + 12 * (size_t)i;
#pragma unroll
    for (int c = 0; c < GSR_DET_COMPONENTS; ++c) {
        row[c] = gsr_det_dequantise((long long)fx[c], mx[c]);
        mx[c] = 0u;
        fx[c] = 0ull;
    }
}

// Deterministic mode, after composite_fwd: fixed-point important score -> float score (every row)
__global__ void __launch_bounds__(256)
det_score_kernel(int n, const unsigned long long* __restrict__ score_fx, float* __restrict__ score) {
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i < n) score[i] = gsr_det_score_dequantise((long long)score_fx[i]);
}

}  // namespace

struct CompPtrs {
    GsrTileGrid grid;
    int H;                 // height of the (stacked) image the kernels render
    const uint32_t *header, *tile_start, *work_order;
    const unsigned long long* keys;
    const GsrRec* geom;
    uint32_t* n_contrib;
    uint32_t *bwd_fill, *bwd_items;   // backward work lists (items == nullptr: the forward was issued without backward)
};
static CompPtrs comp_ptrs(const uint8_t* saved, const b200gsr_saved_layout& vl, int H, int W, int num_views, int gy_view) {
    CompPtrs c;
    c.grid = gsr_grid(H, W);
    c.H = H;
    if (num_views > 1) {   // views stacked vertically, each padded to whole tile rows
        c.grid.gy = num_views * gy_view; c.grid.ntiles = c.grid.gx * c.grid.gy;
        c.H = c.grid.gy * GSR_TILE;
    }
    c.header = reinterpret_cast<const uint32_t*>(saved + vl.header);
    c.tile_start = reinterpret_cast<const uint32_t*>(saved + vl.tile_start);
    c.work_order = reinterpret_cast<const uint32_t*>(saved + vl.work_order);
    c.keys = reinterpret_cast<const unsigned long long*>(saved + vl.keys);
    c.geom = reinterpret_cast<const GsrRec*>(saved + vl.geom);
    c.n_contrib = reinterpret_cast<uint32_t*>(const_cast<uint8_t*>(saved) + vl.n_contrib);
    c.bwd_fill = reinterpret_cast<uint32_t*>(const_cast<uint8_t*>(saved) + vl.header) + GSR_H_BWD_FILL;
    c.bwd_items = vl.bwd_items < vl.total ? reinterpret_cast<uint32_t*>(const_cast<uint8_t*>(saved) + vl.bwd_items) : nullptr;
    return c;
}

template <bool SCORE, bool STATS, bool DET = false, bool SCORE_ONLY = false>
static cudaError_t launch_fwd(const GsrFwdArgs& a, int nblocks, const CompPtrs& c, uint32_t* queue, float* score) {
    const int smem = (int)sizeof(SmemCta);
    static std::atomic<unsigned long long> attr_done{0};
    cudaError_t e = gsr_smem_once(composite_fwd_kernel<SCORE, STATS, DET, SCORE_ONLY>, smem, attr_done);
    if (e != cudaSuccess) return e;
    composite_fwd_kernel<SCORE, STATS, DET, SCORE_ONLY><<<nblocks, 256, smem, a.stream>>>(
        a.prm.image_height, a.prm.image_width, c.grid.gx, a.gy_view, c.H, c.grid.ntiles, c.header, c.work_order, c.tile_start,
        c.keys, c.geom, a.prm.bg, queue, a.out_color, a.out_depth_alpha, c.n_contrib, score, a.stats, c.bwd_fill, c.bwd_items,
        a.P_view);
    return cudaGetLastError();
}

cudaError_t gsr_launch_composite_fwd(const GsrFwdArgs& a) {
    const CompPtrs c = comp_ptrs(a.saved, a.vl, a.prm.image_height, a.prm.image_width, a.num_views, a.gy_view);
    if (c.grid.ntiles == 0) return cudaSuccess;
    uint32_t* queue = reinterpret_cast<uint32_t*>(a.scratch + a.sl.counters) + GSR_C_FWD_QUEUE;
    const int nblocks = min(c.grid.ntiles, a.num_sms * 6);
    if (a.det && a.prm.score_flag) {
        // deterministic important score: fixed-point commits, then one conversion pass over every row.  The
        // forward kernel is otherwise the default one (its outputs do not depend on scheduling); the
        // instrumented instantiation does not apply.
        unsigned long long* sfx = reinterpret_cast<unsigned long long*>(a.saved + a.dl.score_fx);
        cudaError_t e = launch_fwd<true, false, true>(a, nblocks, c, queue, reinterpret_cast<float*>(sfx));
        if (e != cudaSuccess) return e;
        const int n = a.num_views * a.P_view;
        if (n > 0) det_score_kernel<<<(n + 255) / 256, 256, 0, a.stream>>>(n, sfx, a.score);
        return cudaGetLastError();
    }
    if (a.det) return launch_fwd<false, false>(a, nblocks, c, queue, a.score);
    if (a.stats != nullptr)
        return a.prm.score_flag ? launch_fwd<true, true>(a, nblocks, c, queue, a.score)
                                : launch_fwd<false, true>(a, nblocks, c, queue, a.score);
    return a.prm.score_flag ? launch_fwd<true, false>(a, nblocks, c, queue, a.score)
                            : launch_fwd<false, false>(a, nblocks, c, queue, a.score);
}

cudaError_t gsr_launch_composite_score(const GsrFwdArgs& a, void* score_acc) {
    const CompPtrs c = comp_ptrs(a.saved, a.vl, a.prm.image_height, a.prm.image_width, a.num_views, a.gy_view);
    if (c.grid.ntiles == 0 || a.P_view == 0) return cudaSuccess;
    uint32_t* queue = reinterpret_cast<uint32_t*>(a.scratch + a.sl.counters) + GSR_C_FWD_QUEUE;
    const int nblocks = min(c.grid.ntiles, a.num_sms * 6);
    float* acc = static_cast<float*>(score_acc);   // int64 [P_view] with a.det (DET reinterprets it)
    return a.det ? launch_fwd<true, false, true, true>(a, nblocks, c, queue, acc)
                 : launch_fwd<true, false, false, true>(a, nblocks, c, queue, acc);
}

cudaError_t gsr_launch_score_finish(int n, const unsigned long long* score_fx, float* score, cudaStream_t s) {
    if (n == 0) return cudaSuccess;
    det_score_kernel<<<(n + 255) / 256, 256, 0, s>>>(n, score_fx, score);
    return cudaGetLastError();
}

template <bool STATS, int ACC = GSR_ACC_FLOAT, bool FROZEN = false>
static cudaError_t launch_bwd(const GsrBwdArgs& a, const CompPtrs& c, uint32_t* queue, float* dgeom,
                              uint32_t* dmax = nullptr, unsigned long long* dfx = nullptr,
                              const FrozenArg<FROZEN>& fz = {}) {
    const int smem = (int)sizeof(SmemRing);
    const int nblocks = min(c.grid.ntiles, a.num_sms * kMinCtas);
    static std::atomic<unsigned long long> attr_done{0};
    cudaError_t e = gsr_smem_once(composite_bwd_kernel<STATS, ACC, FROZEN>, smem, attr_done);
    if (e != cudaSuccess) return e;
    composite_bwd_kernel<STATS, ACC, FROZEN><<<nblocks, kWarps * 32, smem, a.stream>>>(
        a.prm.image_height, a.prm.image_width, c.grid.gx, a.gy_view, c.H, c.grid.ntiles, c.header, c.work_order, c.tile_start,
        c.keys, c.geom, a.prm.bg, queue, a.out_depth_alpha, c.n_contrib, a.dL_dcolor, a.dL_ddepth_alpha, dgeom,
        a.stats, c.bwd_items, dmax, dfx, fz);
    return cudaGetLastError();
}

// The frozen row ranges (validated and merged by the entry point).
static FrozenRows frozen_rows(const GsrFrozenRanges& r, int P_view) {
    FrozenRows f{};
    f.P_view = (uint32_t)P_view;
    f.n = (uint32_t)r.n;
    for (int k = 0; k < r.n; ++k) { f.lo[k] = r.lo[k]; f.len[k] = r.len[k]; }
    return f;
}

cudaError_t gsr_launch_composite_bwd(const GsrBwdArgs& a) {
    const CompPtrs c = comp_ptrs(a.saved, a.vl, a.prm.image_height, a.prm.image_width, a.num_views, a.gy_view);
    if (c.grid.ntiles == 0) return cudaSuccess;
    uint32_t* queue = reinterpret_cast<uint32_t*>(a.saved + a.vl.header) + GSR_H_BWD_QUEUE;
    float* dgeom = reinterpret_cast<float*>(a.saved + a.vl.dgeom);
    // Frozen rows: the FROZEN instantiations; the instrumented kernel has no such mode and the counters are left
    // untouched, as in deterministic mode.
    const bool frozen = a.frozen_rows != nullptr;
    const FrozenRows fz = frozen ? frozen_rows(*a.frozen_rows, a.P_view) : FrozenRows{};
    if (a.det) {
        // Deterministic mode: the default kernel with integer commits, run twice (instrumentation does not apply).
        // Pass B pops its own work queue (header words, zero between calls like the first one): no memset.
        uint32_t* dmax = reinterpret_cast<uint32_t*>(a.saved + a.dl.dmax);
        unsigned long long* dfx = reinterpret_cast<unsigned long long*>(a.saved + a.dl.dfx);
        uint32_t* queue_b = reinterpret_cast<uint32_t*>(a.saved + a.vl.header) + GSR_H_BWD_QUEUE_DET;
        cudaError_t e;
        if (frozen) {
            e = launch_bwd<false, GSR_ACC_DET_MAX, true>(a, c, queue, dgeom, dmax, dfx, fz);
            if (e == cudaSuccess) e = launch_bwd<false, GSR_ACC_DET_SUM, true>(a, c, queue_b, dgeom, dmax, dfx, fz);
        } else {
            e = launch_bwd<false, GSR_ACC_DET_MAX>(a, c, queue, dgeom, dmax, dfx);
            if (e == cudaSuccess) e = launch_bwd<false, GSR_ACC_DET_SUM>(a, c, queue_b, dgeom, dmax, dfx);
        }
        if (e != cudaSuccess) return e;
        const int n = a.num_views * a.P_view;
        // frozen rows: their dmax / dfx rows are zero, so they resolve to dgeom rows of zeros
        det_resolve_kernel<<<(n + 255) / 256, 256, 0, a.stream>>>(n, a.radii, dmax, dfx, dgeom, queue_b);
        return cudaGetLastError();
    }
    if (frozen) return launch_bwd<false, GSR_ACC_FLOAT, true>(a, c, queue, dgeom, nullptr, nullptr, fz);
    return a.stats != nullptr ? launch_bwd<true>(a, c, queue, dgeom) : launch_bwd<false>(a, c, queue, dgeom);
}
