// Tile binning and per-tile depth sort.
//
// Replaces upstream's InclusiveSum + duplicateWithKeys + global 64-bit cub::DeviceRadixSort +
// identifyTileRanges (SURVEY.md 2.4 K2-K5, App. A.6) with a counting-sort by tile followed by
// an independent in-shared-memory sort of every tile's list:
//   multisplit<count> : per-tile pair counts: 4096-Gaussian CTAs histogram their tile hits in shared
//                       memory, one global RED per (CTA, touched tile)   [large tile grids: privatised
//                       global REDs inside project_sh instead]
//   scan_order_kernel : exclusive scan -> tile_start[], cursors, total pair count (also written to a
//                       mapped host word), and the work order (tiles by list length, longest first)
//   multisplit<scatter>: every Gaussian appends (depth_bits<<32 | idx) to each tile it touches; a CTA
//                       reserves one slice per touched tile, ranks inside it come from smem atomics
//                       [fallback: scatter_kernel with returned global atomics]
//                       (arrival order inside a tile is arbitrary ...)
//   sort kernels      : ... and is then fixed by sorting each tile's keys on (depth bits, idx):
//                       identical to a stable sort of (tile<<32 | depth bits) over pairs emitted
//                       in Gaussian-index order, i.e. bit-exact with the oracle's lists.
//                       In-smem LSD radix sort (8-bit digits, match.any ranking, constant digit
//                       bytes skipped) on the depth bits + a tie pass ordering equal depths by
//                       index; lists longer than one chunk are merged with bitonic merge steps.
//                       The composite kernels gather the 48-B per-Gaussian records on demand
//                       (cp.async) from the sorted index list, so no record array is materialised.
#include "common.cuh"

namespace {

// ---------------------------------------------------------------------------------------------
// scan + work order: one CTA of 1024 threads (num_tiles is small: 4096 at 1024^2)
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ int size_bucket(uint32_t n) {   // 0 = longest lists
    return n == 0 ? 32 : __clz(n);                          // clz in [0,31] for n>0
}

__global__ void __launch_bounds__(1024)
scan_order_kernel(int ntiles, int ncopies, uint32_t max_pairs, const uint32_t* __restrict__ tile_count,
                  uint32_t* __restrict__ tile_start, uint32_t* __restrict__ tile_cursor,
                  uint32_t* __restrict__ work_order, uint32_t* __restrict__ header,
                  volatile uint32_t* host_notify, uint32_t notify_seq) {
    __shared__ uint32_t warp_sums[32];
    __shared__ uint32_t carry_s;
    __shared__ uint32_t bucket_cnt[33];
    __shared__ uint32_t bucket_pos[33];
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    if (tid == 0) carry_s = 0;
    if (tid < 33) bucket_cnt[tid] = 0;
    __syncthreads();
    for (int base = 0; base < ntiles; base += 1024) {
        const int t = base + tid;
        uint32_t cnt[GSR_COPIES];
        uint32_t v = 0;
#pragma unroll
        for (int c = 0; c < GSR_COPIES; ++c) {
            cnt[c] = (t < ntiles && c < ncopies) ? tile_count[(size_t)c * ntiles + t] : 0u;
            v += cnt[c];
        }
        uint32_t incl = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t n = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += n;
        }
        if (lane == 31) warp_sums[wid] = incl;
        __syncthreads();
        if (wid == 0) {
            uint32_t w = warp_sums[lane], wi = w;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const uint32_t n = __shfl_up_sync(0xffffffffu, wi, o);
                if (lane >= o) wi += n;
            }
            warp_sums[lane] = wi - w;   // exclusive
        }
        __syncthreads();
        const uint32_t excl = carry_s + warp_sums[wid] + incl - v;
        if (t < ntiles) {
            tile_start[t] = excl;
            uint32_t run = excl;
#pragma unroll
            for (int c = 0; c < GSR_COPIES; ++c) {
                tile_cursor[(size_t)c * ntiles + t] = run;
                run += cnt[c];
            }
            atomicAdd(&bucket_cnt[size_bucket(v)], 1u);
        }
        __syncthreads();
        if (tid == 1023) carry_s = excl + v;
        __syncthreads();
    }
    if (tid == 0) {
        const uint32_t total = carry_s;
        tile_start[ntiles] = total;
        header[GSR_H_NUM_PAIRS] = total;
        header[GSR_H_MAX_PAIRS] = max_pairs;
        header[GSR_H_NUM_TILES] = (uint32_t)ntiles;
        header[GSR_H_OVERFLOW] = total > max_pairs ? 1u : 0u;
        uint32_t run = 0, nbig = 0;
        for (int b = 0; b < 33; ++b) {
            bucket_pos[b] = run;
            run += bucket_cnt[b];
            // lists longer than GSR_SORT_SMALL_MAX (=2^12): n >= 4097 -> clz <= 19
            if (b <= 19) nbig = run;
        }
        header[GSR_H_NUM_BIG] = nbig;   // upper bound: includes n == 4096 exactly (clz 19)
        header[GSR_H_NUM_NONEMPTY] = run - bucket_cnt[32];
        for (int k = 0; k < GSR_NQUEUE; ++k) header[GSR_H_BWD_QUEUE + k] = 0u;
        for (int k = 0; k < GSR_BWD_CLASSES; ++k) header[GSR_H_BWD_FILL + k] = 0u;
        if (host_notify != nullptr) {   // mapped pinned host memory: tell the host the pair count now
            host_notify[1] = total;
            host_notify[2] = total > max_pairs ? 1u : 0u;
            host_notify[3] = (uint32_t)ntiles;
            __threadfence_system();
            host_notify[0] = notify_seq;
        }
    }
    __syncthreads();
    for (int t = tid; t < ntiles; t += 1024) {
        uint32_t v = 0;
#pragma unroll
        for (int c = 0; c < GSR_COPIES; ++c)
            if (c < ncopies) v += tile_count[(size_t)c * ntiles + t];
        const uint32_t pos = atomicAdd(&bucket_pos[size_bucket(v)], 1u);
        work_order[pos] = (uint32_t)t;
    }
}

// Single-pass variant for the multisplit path (one counter copy, ntiles <= 1024*kScanItems): every
// thread owns kScanItems consecutive tiles in registers, so there are two barriers in total and
// the counts are never re-read.
constexpr int kScanItems = GSR_MS_MAX_TILES / 1024;   // 12

__global__ void __launch_bounds__(1024)
scan_order_fast_kernel(int ntiles, uint32_t max_pairs, const uint32_t* __restrict__ tile_count,
                       uint32_t* __restrict__ tile_start, uint32_t* __restrict__ tile_cursor,
                       uint32_t* __restrict__ work_order, uint32_t* __restrict__ header,
                       volatile uint32_t* host_notify, uint32_t notify_seq) {
    extern __shared__ uint32_t cnt_s[];                  // [ntiles] copy of the counts for the last pass
    __shared__ uint32_t warp_sums[32];
    __shared__ uint32_t bucket_cnt[33];
    __shared__ uint32_t bucket_pos[33];
    __shared__ uint32_t total_s;
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const int per = (ntiles + 1023) / 1024;             // tiles per thread (<= kScanItems)
    if (tid < 33) bucket_cnt[tid] = 0;
    uint32_t v[kScanItems], sum = 0;
#pragma unroll
    for (int k = 0; k < kScanItems; ++k) {
        const int t = tid * per + k;
        v[k] = (k < per && t < ntiles) ? __ldg(tile_count + t) : 0u;
        if (k < per && t < ntiles) cnt_s[t] = v[k];
        sum += v[k];
    }
    uint32_t incl = sum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t n = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += n;
    }
    if (lane == 31) warp_sums[wid] = incl;
    __syncthreads();
    if (wid == 0) {
        const uint32_t w = warp_sums[lane];
        uint32_t wi = w;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t n = __shfl_up_sync(0xffffffffu, wi, o);
            if (lane >= o) wi += n;
        }
        warp_sums[lane] = wi - w;   // exclusive
        if (lane == 31) total_s = wi;
    }
#pragma unroll
    for (int k = 0; k < kScanItems; ++k) {
        const int t = tid * per + k;
        if (k < per && t < ntiles) atomicAdd(&bucket_cnt[size_bucket(v[k])], 1u);
    }
    __syncthreads();
    uint32_t run = warp_sums[wid] + incl - sum;
#pragma unroll
    for (int k = 0; k < kScanItems; ++k) {
        const int t = tid * per + k;
        if (k < per && t < ntiles) { tile_start[t] = run; tile_cursor[t] = run; }
        run += v[k];
    }
    if (wid == 0) {   // exclusive prefix over the 33 length buckets (bucket 32 = empty tiles, handled by lane 0)
        const uint32_t c = bucket_cnt[lane];
        uint32_t ci = c;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t n = __shfl_up_sync(0xffffffffu, ci, o);
            if (lane >= o) ci += n;
        }
        bucket_pos[lane] = ci - c;
        const uint32_t nonempty = __shfl_sync(0xffffffffu, ci, 31);
        const uint32_t nbig = __shfl_sync(0xffffffffu, ci, 19);   // buckets 0..19: n >= 4096
        if (lane == 0) {
            bucket_pos[32] = nonempty;
            const uint32_t total = total_s;
            tile_start[ntiles] = total;
            header[GSR_H_NUM_PAIRS] = total;
            header[GSR_H_MAX_PAIRS] = max_pairs;
            header[GSR_H_NUM_TILES] = (uint32_t)ntiles;
            header[GSR_H_OVERFLOW] = total > max_pairs ? 1u : 0u;
            header[GSR_H_NUM_BIG] = nbig;
            header[GSR_H_NUM_NONEMPTY] = nonempty;
#pragma unroll
            for (int k = 0; k < GSR_NQUEUE; ++k) header[GSR_H_BWD_QUEUE + k] = 0u;
#pragma unroll
            for (int k = 0; k < GSR_BWD_CLASSES; ++k) header[GSR_H_BWD_FILL + k] = 0u;
            if (host_notify != nullptr) {   // mapped pinned host memory: tell the host the pair count now
                host_notify[1] = total;
                host_notify[2] = total > max_pairs ? 1u : 0u;
                host_notify[3] = (uint32_t)ntiles;
                __threadfence_system();
                host_notify[0] = notify_seq;
            }
        }
    }
    __syncthreads();
    // Insertion order inside a length bucket matters: tiles are taken thread-strided (t, t+1024, ...)
    // so that spatially adjacent tiles - which share Gaussians and would contend on the same
    // gradient accumulators in composite_bwd - are not handed out back to back by a single thread.
    for (int t = tid; t < ntiles; t += 1024)
        work_order[atomicAdd(&bucket_pos[size_bucket(cnt_s[t])], 1u)] = (uint32_t)t;
}

// ---------------------------------------------------------------------------------------------
// scatter: one Gaussian per thread appends its key to every touched tile
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
scatter_kernel(int P, int gx, int ntiles, uint32_t max_pairs, const uint4* __restrict__ rectdepth,
               uint32_t* __restrict__ tile_cursor, unsigned long long* __restrict__ keys) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    const uint4 rd = __ldg(rectdepth + i);
    if (rd.w == 0) return;
    const int minx = rd.x & 0xffff, miny = rd.x >> 16, maxx = rd.y & 0xffff;
    const unsigned long long key = ((unsigned long long)rd.z << 32) | (uint32_t)i;
    uint32_t* cur = tile_cursor + (size_t)((i >> 5) & (GSR_COPIES - 1)) * ntiles;
    // The returned atomics are issued in batches of 8 before any dependent store, so up to 8
    // L2 round trips overlap per thread instead of serialising.
    const int w = maxx - minx, total = (int)rd.w;
    for (int base = 0; base < total; base += 8) {
        uint32_t pos[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) {
            const int t = base + u;
            if (t < total) {
                const int ry = t / w, rx = t - ry * w;
                pos[u] = atomicAdd(cur + (miny + ry) * gx + (minx + rx), 1u);
            }
        }
#pragma unroll
        for (int u = 0; u < 8; ++u)
            if (base + u < total && pos[u] < max_pairs) keys[pos[u]] = key;
    }
}

// ---------------------------------------------------------------------------------------------
// Block multisplit (default path).  count: smem histogram of the CTA's tile hits, then ONE global
// RED per touched tile; the histogram is kept in global memory.  scatter: re-reads it, ONE returned
// global atomic per touched tile reserves the CTA's contiguous slice of that tile's segment, then
// every pair takes its slot inside the slice from a shared-memory atomic.
// ---------------------------------------------------------------------------------------------
template <bool SCATTER>
__global__ void __launch_bounds__(1024)
multisplit_kernel(int P, int per, int gx, int ntiles, uint32_t max_pairs, const uint4* __restrict__ rectdepth,
                  uint32_t* __restrict__ tile_count, uint32_t* __restrict__ tile_cursor,
                  uint32_t* __restrict__ block_hist, unsigned long long* __restrict__ keys) {
    extern __shared__ uint32_t ms_smem[];
    uint32_t* hist = ms_smem;            // [ntiles] counts (count) / global write cursors of this CTA's slices (scatter)
    const int i0 = blockIdx.x * per;                 // this CTA's Gaussians: [i0, min(P, i0 + per)), per <= 4096
    const int i1 = min(P, i0 + per);
    uint32_t* my_hist = block_hist + (size_t)blockIdx.x * ntiles;   // written by count, re-read by scatter
    uint4 rd[GSR_MS_ITEMS];
#pragma unroll
    for (int u = 0; u < GSR_MS_ITEMS; ++u) {
        const int i = i0 + u * 1024 + threadIdx.x;
        rd[u] = (i < i1) ? __ldg(rectdepth + i) : make_uint4(0u, 0u, 0u, 0u);
    }
    if constexpr (!SCATTER) {
        for (int t = threadIdx.x; t < ntiles; t += 1024) hist[t] = 0u;
        __syncthreads();
#pragma unroll
        for (int u = 0; u < GSR_MS_ITEMS; ++u) {
            if (rd[u].w) {
                const int minx = rd[u].x & 0xffff, miny = rd[u].x >> 16, maxx = rd[u].y & 0xffff, maxy = rd[u].y >> 16;
                for (int ty = miny; ty < maxy; ++ty)
                    for (int tx = minx; tx < maxx; ++tx) atomicAdd(&hist[ty * gx + tx], 1u);
            }
        }
        __syncthreads();
        for (int t = threadIdx.x; t < ntiles; t += 1024) {
            const uint32_t c = hist[t];
            my_hist[t] = c;
            if (c) atomicAdd(tile_count + t, c);
        }
    } else {
        // reserve this CTA's slice of every touched tile: the in-slice cursor starts at the slice's
        // global position, so a pair's slot is ONE shared-memory atomic (no second lookup)
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
                        if (pos < max_pairs) keys[pos] = key;
                    }
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------
// In-smem LSD radix sort of n <= NT*ITEMS 64-bit keys on their HIGH 32 bits (depth), followed by a
// pass that orders runs of equal depth by the low 32 bits (Gaussian index).
// Element order is warp-major: warp w owns rows j = 0..rows-1 of 32 consecutive elements
//   e(w, j, lane) = (w*rows + j)*32 + lane.
// Per pass: (1) per-warp digit histogram, (2) scan over (digit, warp), (3) stable re-rank with
// match.any peer masks and scatter into the smem buffer, (4) read back into registers.
// ---------------------------------------------------------------------------------------------
template <int NT, int ITEMS>
__device__ __forceinline__ void radix_sort_smem(unsigned long long* s, uint32_t* hist /*[NT/32][256]*/,
                                                uint32_t* digit_base /*[256]*/, uint32_t* red /*[2]*/,
                                                int n, bool full64) {
    constexpr int NW = NT / 32;
    const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
    const uint32_t lt_mask = (1u << lane) - 1u;
    const int rows = (n + NW * 32 - 1) / (NW * 32);   // rows per warp actually used (<= ITEMS)
    unsigned long long k[ITEMS];
    uint32_t vor = 0u, vand = 0xffffffffu, lor = 0u, land = 0xffffffffu;
#pragma unroll
    for (int j = 0; j < ITEMS; ++j) {
        const int e = (w * rows + j) * 32 + lane;
        const bool ok = j < rows && e < n;
        k[j] = ok ? s[e] : ~0ull;
        if (ok) {
            vor |= (uint32_t)(k[j] >> 32); vand &= (uint32_t)(k[j] >> 32);
            lor |= (uint32_t)k[j]; land &= (uint32_t)k[j];
        }
    }
    vor = __reduce_or_sync(0xffffffffu, vor);
    vand = __reduce_and_sync(0xffffffffu, vand);
    lor = __reduce_or_sync(0xffffffffu, lor);
    land = __reduce_and_sync(0xffffffffu, land);
    if (tid == 0) { red[0] = 0u; red[1] = 0xffffffffu; red[2] = 0u; red[3] = 0xffffffffu; }
    __syncthreads();
    if (lane == 0) { atomicOr(&red[0], vor); atomicAnd(&red[1], vand); atomicOr(&red[2], lor); atomicAnd(&red[3], land); }
    __syncthreads();
    // bits that differ somewhere in the list (depth in the high word, index in the low word)
    const unsigned long long varying = ((unsigned long long)(red[0] ^ red[1]) << 32) |
                                       (full64 ? (unsigned long long)(red[2] ^ red[3]) : 0ull);
    __syncthreads();

#pragma unroll 1
    for (int shift = full64 ? 0 : 32; shift < 64; shift += 8) {
        if (((varying >> shift) & 0xffull) == 0ull) continue;   // constant digit: pass is a no-op
        // (1) per-warp histogram (native 32-bit shared-memory atomics)
        for (int d = lane; d < 256; d += 32) hist[w * 256 + d] = 0u;
        __syncwarp();
#pragma unroll
        for (int j = 0; j < ITEMS; ++j)
            if (j < rows) atomicAdd(&hist[w * 256 + ((uint32_t)(k[j] >> shift) & 0xffu)], 1u);
        __syncthreads();
        // (2) scan: for every digit, exclusive prefix over warps; then exclusive prefix over digits
        if (tid < 256) {
            uint32_t run = 0;
#pragma unroll 4
            for (int ww = 0; ww < NW; ++ww) {
                const uint32_t c = hist[ww * 256 + tid];
                hist[ww * 256 + tid] = run;
                run += c;
            }
            // exclusive scan of `run` over the 256 digit threads (8 warps)
            uint32_t incl = run;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
                if (lane >= o) incl += t;
            }
            if (lane == 31) digit_base[256 + w] = incl;   // per-warp totals (8 entries)
            __syncwarp();
            // all 8 warps see each other's totals only after a barrier: use named barrier 1 (256 thr)
            asm volatile("bar.sync 1, 256;" ::: "memory");
            uint32_t wbase = 0;
            for (int ww = 0; ww < w; ++ww) wbase += digit_base[256 + ww];
            digit_base[tid] = wbase + incl - run;
        }
        __syncthreads();
        // (3) stable rank + scatter (keys are in registers, so the buffer can be overwritten)
#pragma unroll
        for (int j = 0; j < ITEMS; ++j) {
            if (j < rows) {
                const uint32_t dg = (uint32_t)(k[j] >> shift) & 0xffu;
                const uint32_t peers = __match_any_sync(0xffffffffu, dg);   // lanes holding the same digit
                const int leader = __ffs(peers) - 1;
                uint32_t base = 0;
                if (lane == leader) {
                    base = hist[w * 256 + dg];
                    hist[w * 256 + dg] = base + __popc(peers);
                }
                base = __shfl_sync(0xffffffffu, base, leader);
                const uint32_t dst = digit_base[dg] + base + __popc(peers & lt_mask);
                if (dst < (uint32_t)n) s[dst] = k[j];   // padding keys (all ones) rank last: dropped
                __syncwarp();
            }
        }
        __syncthreads();
        // (4) back to registers in warp-major order
#pragma unroll
        for (int j = 0; j < ITEMS; ++j) {
            const int e = (w * rows + j) * 32 + lane;
            k[j] = (j < rows && e < n) ? s[e] : ~0ull;
        }
        __syncthreads();
    }
    if (full64) return;   // the index bytes were sorted too: nothing left to fix
    // tie pass: runs of equal depth bits are ordered by index (arrival order was arbitrary).
    // Short runs: the run head insertion-sorts them.  A long run (> 32, e.g. a plane at constant
    // view depth) would make that quadratic, so the caller re-sorts with the index bytes included.
    if (tid == 0) red[0] = 0u;
    __syncthreads();
    for (int i = tid; i < n; i += NT) {
        const uint32_t d = (uint32_t)(s[i] >> 32);
        const bool head = (i == 0 || (uint32_t)(s[i - 1] >> 32) != d) && (i + 1 < n) &&
                          (uint32_t)(s[i + 1] >> 32) == d;
        if (head) {
            int e = i + 1;
            while (e < n && e - i <= 32 && (uint32_t)(s[e] >> 32) == d) ++e;
            if (e - i > 32) { red[0] = 1u; continue; }
            for (int a = i + 1; a < e; ++a) {          // insertion sort of s[i, e)
                const unsigned long long x = s[a];
                int b = a - 1;
                while (b >= i && s[b] > x) { s[b + 1] = s[b]; --b; }
                s[b + 1] = x;
            }
        }
    }
    __syncthreads();
}

// ---------------------------------------------------------------------------------------------
// Fast path: one-pass interpolation bucket sort.  The keys are read from global memory straight into
// registers (g[0..n), coalesced); depth bits are mapped monotonically onto NB buckets between the
// list's min and max; a shared-memory atomic hands every key its arrival slot inside the bucket and
// the keys are scattered bucket by bucket into s.  Every key then counts the smaller FULL 64-bit
// keys of its own (tiny) bucket - one thread per key, no dependent read-modify-write chains - which
// is its final position (keys are distinct: the low word is the Gaussian index), and is written
// there.  If any bucket is larger than kBucketLimit (skewed depth distribution) the list falls back
// to the radix sort above.  Returns with s[0..n) sorted; the caller copies it out.
// ---------------------------------------------------------------------------------------------
constexpr int kBucketLimit = 32;

template <int NT, int ITEMS, int NB>
__device__ __forceinline__ void tile_sort_items(const unsigned long long* g, unsigned long long* s, uint32_t* hist,
                                               uint32_t* digit_base, uint32_t* red, int n) {
    static_assert(NB + 1 <= (NT / 32) * 256 + 32, "bucket counters alias the radix histogram (+32 spare words)");
    static_assert(NB % NT == 0, "whole number of buckets per thread");
    static_assert(NT / 32 <= 32 && ITEMS % 2 == 0, "one lane per warp total; positions are packed in pairs");
    constexpr int BPT = NB / NT;
    const int tid = threadIdx.x, lane = tid & 31;
    uint32_t* cnt = hist;   // NB counters, later NB + 1 exclusive starts
    unsigned long long k[ITEMS];
    uint32_t dmin = 0xffffffffu, dmax = 0u;
#pragma unroll
    for (int j = 0; j < ITEMS; ++j) {
        const int e = j * NT + tid;
        k[j] = ~0ull;
        if (e < n) {
            k[j] = __ldcg(g + e);                 // L2: the multi-chunk caller rewrites g between calls
            dmin = min(dmin, (uint32_t)(k[j] >> 32)); dmax = max(dmax, (uint32_t)(k[j] >> 32));
        }
    }
    dmin = __reduce_min_sync(0xffffffffu, dmin);
    dmax = __reduce_max_sync(0xffffffffu, dmax);
    if (tid == 0) { red[0] = 0xffffffffu; red[1] = 0u; red[2] = 0u; }
#pragma unroll
    for (int q = 0; q < BPT; ++q) cnt[q * NT + tid] = 0u;
    __syncthreads();
    if (lane == 0) { atomicMin(&red[0], dmin); atomicMax(&red[1], dmax); }
    __syncthreads();
    dmin = red[0]; dmax = red[1];
    const float scale = (float)NB / ((float)(dmax - dmin) + 1.0f);
    auto bucket_of = [&](unsigned long long key) {
        return min((uint32_t)(NB - 1), (uint32_t)((float)((uint32_t)(key >> 32) - dmin) * scale));
    };
    uint32_t rank8[(ITEMS + 3) / 4];   // arrival rank inside the bucket, one byte per item (saturating)
#pragma unroll
    for (int j = 0; j < (ITEMS + 3) / 4; ++j) rank8[j] = 0u;
#pragma unroll
    for (int j = 0; j < ITEMS; ++j) {
        const int e = j * NT + tid;
        if (e < n) rank8[j >> 2] |= min(atomicAdd(&cnt[bucket_of(k[j])], 1u), 255u) << (8 * (j & 3));
    }
    __syncthreads();
    // exclusive scan of the NB counters (BPT consecutive counters per thread) + largest bucket
    uint32_t c[BPT], sum = 0, big = 0;
#pragma unroll
    for (int q = 0; q < BPT; ++q) { c[q] = cnt[tid * BPT + q]; sum += c[q]; big = max(big, c[q]); }
    uint32_t incl = sum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += t;
    }
    big = __reduce_max_sync(0xffffffffu, big);
    if (lane == 31) digit_base[tid >> 5] = incl;
    if (lane == 0 && big > (uint32_t)kBucketLimit) red[2] = 1u;
    __syncthreads();
    if (red[2] != 0u) {   // skewed list (uniform branch): robust path, which sorts s in place
#pragma unroll
        for (int j = 0; j < ITEMS; ++j) {
            const int e = j * NT + tid;
            if (e < n) s[e] = k[j];
        }
        __syncthreads();
        for (bool full64 = false;; full64 = true) {     // one inlined copy; second trip only for long equal-depth runs
            radix_sort_smem<NT, ITEMS>(s, hist, digit_base, red, n, full64);
            if (full64 || red[0] == 0u) break;
            __syncthreads();
        }
        return;
    }
    // warps before mine: one lane per warp total, summed with a warp reduction
    const uint32_t wt = (lane < NT / 32 && lane < (tid >> 5)) ? digit_base[lane] : 0u;
    uint32_t run = __reduce_add_sync(0xffffffffu, wt) + incl - sum;
#pragma unroll
    for (int q = 0; q < BPT; ++q) { cnt[tid * BPT + q] = run; run += c[q]; }
    if (tid == NT - 1) cnt[NB] = (uint32_t)n;
    __syncthreads();
#pragma unroll
    for (int j = 0; j < ITEMS; ++j) {
        const int e = j * NT + tid;
        if (e < n) s[cnt[bucket_of(k[j])] + ((rank8[j >> 2] >> (8 * (j & 3))) & 0xffu)] = k[j];
    }
    __syncthreads();
    // s is now ordered bucket by bucket.  Each thread takes the keys at ITS positions (the registers'
    // original keys are dead): the lanes of a warp then sit in the same few neighbouring buckets, so
    // their counting loops have near-equal length and read the same addresses (broadcasts).
    uint32_t pos2[ITEMS / 2];          // final positions (< 65536), two per register
#pragma unroll
    for (int j = 0; j < ITEMS; ++j) {
        const int e = j * NT + tid;
        uint32_t pos = 0u;
        if (e < n) {
            const unsigned long long x = s[e];
            k[j] = x;
            const uint32_t b = bucket_of(x);
            const uint32_t b0 = cnt[b], b1 = cnt[b + 1];
            pos = b0;
            uint32_t a = b0;
#pragma unroll 1
            for (; a + 2 <= b1; a += 2) {              // two independent loads per trip (buckets hold ~1-3 keys)
                const unsigned long long y0 = s[a], y1 = s[a + 1];
                pos += (y0 < x) ? 1u : 0u;
                pos += (y1 < x) ? 1u : 0u;
            }
            if (a < b1) pos += (s[a] < x) ? 1u : 0u;
        }
        if (j & 1) pos2[j >> 1] |= pos << 16; else pos2[j >> 1] = pos;
    }
    __syncthreads();
#pragma unroll
    for (int j = 0; j < ITEMS; ++j) {
        const int e = j * NT + tid;
        if (e < n) s[(pos2[j >> 1] >> (16 * (j & 1))) & 0xffffu] = k[j];
    }
    __syncthreads();
}

// n <= NT * 16 keys; the per-thread item count is a compile-time constant of each instantiation, so
// short lists do not walk (predicated-off) rows they do not have.  The branch is CTA-uniform.
template <int NT, int NB>
__device__ __forceinline__ void tile_sort_smem(const unsigned long long* g, unsigned long long* s, uint32_t* hist,
                                               uint32_t* digit_base, uint32_t* red, int n) {
    if (n <= NT * 4) tile_sort_items<NT, 4, NB>(g, s, hist, digit_base, red, n);
    else if (n <= NT * 8) tile_sort_items<NT, 8, NB>(g, s, hist, digit_base, red, n);
    else if (n <= NT * 12) tile_sort_items<NT, 12, NB>(g, s, hist, digit_base, red, n);
    else tile_sort_items<NT, 16, NB>(g, s, hist, digit_base, red, n);
}

__device__ __forceinline__ int next_pow2(int n) {
    return n <= 1 ? 1 : 1 << (32 - __clz(n - 1));
}

struct SortSmemSmall {
    unsigned long long keys[GSR_SORT_SMALL_MAX];
    uint32_t hist[8 * 256 + 32];
    uint32_t digit_base[256 + 8];
    uint32_t red[4];
};
struct SortSmemBig {
    unsigned long long keys[GSR_SORT_BIG_CHUNK];
    uint32_t hist[32 * 256 + 32];
    uint32_t digit_base[256 + 8];
    uint32_t red[4];
};

// small tiles: n <= 4096, 256 threads x 16 items
__global__ void __launch_bounds__(256, 4)
sort_small_kernel(const uint32_t* __restrict__ header, const uint32_t* __restrict__ work_order,
                  const uint32_t* __restrict__ tile_start, unsigned long long* __restrict__ keys) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    SortSmemSmall& sm = *reinterpret_cast<SortSmemSmall*>(smem_raw);
    const uint32_t max_pairs = header[GSR_H_MAX_PAIRS];
    const uint32_t nonempty = header[GSR_H_NUM_NONEMPTY];
    for (uint32_t w = blockIdx.x; w < nonempty; w += gridDim.x) {
        const uint32_t tile = work_order[w];
        uint32_t beg = tile_start[tile], end = tile_start[tile + 1];
        if (end - beg > GSR_SORT_SMALL_MAX) continue;          // big kernel's job
        if (end > max_pairs) end = max_pairs;                  // overflow: stay in bounds
        if (beg >= end) continue;
        const int n = (int)(end - beg);
        tile_sort_smem<256, 2048>(keys + beg, sm.keys, sm.hist, sm.digit_base, sm.red, n);
        for (int i = threadIdx.x; i < n; i += 256) keys[beg + i] = sm.keys[i];
        __syncthreads();
    }
}

// big tiles: 1024 threads x 8 items per 8192-key chunk; lists longer than one chunk are sorted
// chunk by chunk (radix) and merged in place in global memory with bitonic merge steps.
__global__ void __launch_bounds__(1024)
sort_big_kernel(const uint32_t* __restrict__ header, const uint32_t* __restrict__ work_order,
                const uint32_t* __restrict__ tile_start, unsigned long long* __restrict__ keys) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    SortSmemBig& sm = *reinterpret_cast<SortSmemBig*>(smem_raw);
    unsigned long long* sb = sm.keys;
    constexpr int CH = GSR_SORT_BIG_CHUNK;
    const uint32_t max_pairs = header[GSR_H_MAX_PAIRS];
    const uint32_t nbig = header[GSR_H_NUM_BIG];
    for (uint32_t w = blockIdx.x; w < nbig; w += gridDim.x) {
        const uint32_t tile = work_order[w];
        uint32_t beg = tile_start[tile], end = tile_start[tile + 1];
        if (end - beg <= GSR_SORT_SMALL_MAX) continue;
        if (end > max_pairs) end = max_pairs;
        if (beg >= end) continue;
        const int n = (int)(end - beg);
        unsigned long long* gk = keys + beg;
        if (n <= CH) {
            tile_sort_smem<1024, 8192>(gk, sb, sm.hist, sm.digit_base, sm.red, n);
            for (int i = threadIdx.x; i < n; i += 1024) gk[i] = sb[i];
            __syncthreads();
            continue;
        }
        // ---- longer than one chunk: radix-sort CH-sized chunks, then bitonic merges ---------
        const int N = next_pow2(n);
        for (int c0 = 0; c0 < n; c0 += CH) {
            const int m = min(CH, n - c0);
            tile_sort_items<1024, 16, 8192>(gk + c0, sb, sm.hist, sm.digit_base, sm.red, m);
            for (int i = threadIdx.x; i < m; i += 1024) __stcg(gk + c0 + i, sb[i]);
            __syncthreads();
        }
        // flip-variant bitonic merge network: every comparator leaves the minimum at the lower
        // index, so the virtual +inf padding above n needs no storage (such comparators are no-ops)
        for (int k = 2 * CH; k <= N; k <<= 1) {
            const int half = k >> 1, lhalf = 31 - __clz(half);
            for (int t = threadIdx.x; t < N / 2; t += 1024) {          // flip step (global)
                const int b = t >> lhalf, off = t - b * half;
                const int i = b * k + off, l = b * k + k - 1 - off;
                if (i < n && l < n) {
                    const unsigned long long a = __ldcg(gk + i), c = __ldcg(gk + l);
                    if (a > c) { __stcg(gk + i, c); __stcg(gk + l, a); }
                }
            }
            __syncthreads();
            for (int j = half >> 1; j >= CH; j >>= 1) {                 // half cleaners (global)
                const int lj = 31 - __clz(j);
                for (int t = threadIdx.x; t < N / 2; t += 1024) {
                    const int i = ((t >> lj) << (lj + 1)) + (t & (j - 1)), l = i + j;
                    if (i < n && l < n) {
                        const unsigned long long a = __ldcg(gk + i), c = __ldcg(gk + l);
                        if (a > c) { __stcg(gk + i, c); __stcg(gk + l, a); }
                    }
                }
                __syncthreads();
            }
            for (int c0 = 0; c0 < n; c0 += CH) {                        // distances < CH: in smem
                const int m = min(CH, n - c0);
                for (int i = threadIdx.x; i < m; i += 1024) sb[i] = __ldcg(gk + c0 + i);
                __syncthreads();
                for (int j = CH >> 1; j > 0; j >>= 1) {
                    const int lj = 31 - __clz(j);
                    for (int t = threadIdx.x; ; t += 1024) {
                        const int i = ((t >> lj) << (lj + 1)) + (t & (j - 1)), l = i + j;
                        if (i >= m) break;
                        if (l < m) {
                            const unsigned long long a = sb[i], c = sb[l];
                            if (a > c) { sb[i] = c; sb[l] = a; }
                        }
                    }
                    __syncthreads();
                }
                for (int i = threadIdx.x; i < m; i += 1024) __stcg(gk + c0 + i, sb[i]);
                __syncthreads();
            }
        }
    }
}

struct BinPtrs {
    GsrTileGrid grid;
    uint32_t *header, *tile_start, *work_order, *tile_count, *tile_cursor;
    unsigned long long* keys;
    const uint4* rectdepth;
};
BinPtrs bin_ptrs(const GsrFwdArgs& a) {
    BinPtrs b;
    b.grid = gsr_grid(a.prm.image_height, a.prm.image_width);
    if (a.num_views > 1) { b.grid.gy = a.num_views * a.gy_view; b.grid.ntiles = b.grid.gx * b.grid.gy; }
    b.header = reinterpret_cast<uint32_t*>(a.saved + a.vl.header);
    b.tile_start = reinterpret_cast<uint32_t*>(a.saved + a.vl.tile_start);
    b.work_order = reinterpret_cast<uint32_t*>(a.saved + a.vl.work_order);
    b.tile_count = reinterpret_cast<uint32_t*>(a.scratch + a.sl.tile_count);
    b.tile_cursor = reinterpret_cast<uint32_t*>(a.scratch + a.sl.tile_cursor);
    b.keys = reinterpret_cast<unsigned long long*>(a.saved + a.vl.keys);
    b.rectdepth = reinterpret_cast<const uint4*>(a.scratch + a.sl.rectdepth);
    return b;
}
}  // namespace

cudaError_t gsr_launch_scan(const GsrFwdArgs& a) {
    const BinPtrs b = bin_ptrs(a);
    if (gsr_use_multisplit(b.grid.ntiles)) {
        // static + dynamic shared memory can exceed the 48 KB default at the top of the range
        static std::atomic<unsigned long long> attr_done{0};
        cudaError_t e = gsr_smem_once(scan_order_fast_kernel, GSR_MS_MAX_TILES * (int)sizeof(uint32_t), attr_done);
        if (e != cudaSuccess) return e;
        scan_order_fast_kernel<<<1, 1024, b.grid.ntiles * sizeof(uint32_t), a.stream>>>(b.grid.ntiles, a.max_pairs, b.tile_count, b.tile_start,
                                                          b.tile_cursor, b.work_order, b.header, a.host_notify,
                                                          a.notify_seq);
        return cudaGetLastError();
    }
    scan_order_kernel<<<1, 1024, 0, a.stream>>>(b.grid.ntiles, gsr_use_multisplit(b.grid.ntiles) ? 1 : GSR_COPIES,
                                                 a.max_pairs, b.tile_count, b.tile_start,
                                                 b.tile_cursor, b.work_order, b.header, a.host_notify,
                                                 a.notify_seq);
    return cudaGetLastError();
}

static cudaError_t launch_multisplit(const GsrFwdArgs& a, const BinPtrs& b, bool scatter) {
    const int P = a.num_views * a.P_view;     // virtual Gaussians (view-major)
    if (P == 0) return cudaSuccess;
    const int nblk = gsr_ms_blocks(P);
    const int per = (P + nblk - 1) / nblk;
    const int smem = b.grid.ntiles * (int)sizeof(uint32_t);
    const int smem_max = GSR_MS_MAX_TILES * (int)sizeof(uint32_t);
    static std::atomic<unsigned long long> done_scatter{0}, done_count{0};
    cudaError_t e = scatter ? gsr_smem_once(multisplit_kernel<true>, smem_max, done_scatter)
                            : gsr_smem_once(multisplit_kernel<false>, smem_max, done_count);
    if (e != cudaSuccess) return e;
    if (scatter)
        multisplit_kernel<true><<<nblk, 1024, smem, a.stream>>>(
            P, per, b.grid.gx, b.grid.ntiles, a.max_pairs, b.rectdepth, b.tile_count, b.tile_cursor,
            reinterpret_cast<uint32_t*>(a.scratch + a.sl.ms_hist), b.keys);
    else
        multisplit_kernel<false><<<nblk, 1024, smem, a.stream>>>(
            P, per, b.grid.gx, b.grid.ntiles, a.max_pairs, b.rectdepth, b.tile_count, b.tile_cursor,
            reinterpret_cast<uint32_t*>(a.scratch + a.sl.ms_hist), b.keys);
    return cudaGetLastError();
}

// multisplit path only: the fallback path counts inside project_sh
cudaError_t gsr_launch_count(const GsrFwdArgs& a) {
    const BinPtrs b = bin_ptrs(a);
    if (!gsr_use_multisplit(b.grid.ntiles)) return cudaSuccess;
    return launch_multisplit(a, b, false);
}

cudaError_t gsr_launch_scatter(const GsrFwdArgs& a) {
    const BinPtrs b = bin_ptrs(a);
    if (gsr_use_multisplit(b.grid.ntiles)) return launch_multisplit(a, b, true);
    const int PV = a.num_views * a.P_view;
    if (PV > 0)
        scatter_kernel<<<(PV + 255) / 256, 256, 0, a.stream>>>(PV, b.grid.gx, b.grid.ntiles,
                                                                     a.max_pairs, b.rectdepth, b.tile_cursor,
                                                                     b.keys);
    return cudaGetLastError();
}

// The two size classes touch disjoint tiles, so when the caller provides a forked stream the
// small-tile kernel runs there concurrently with the big-tile kernel (joined before returning).
cudaError_t gsr_launch_sort(const GsrFwdArgs& a, cudaStream_t side, cudaEvent_t fork, cudaEvent_t join) {
    const BinPtrs b = bin_ptrs(a);
    const int big_smem = (int)sizeof(SortSmemBig), small_smem = (int)sizeof(SortSmemSmall);
    static std::atomic<unsigned long long> done_big{0}, done_small{0};
    cudaError_t e = gsr_smem_once(sort_big_kernel, big_smem, done_big);
    if (e != cudaSuccess) return e;
    e = gsr_smem_once(sort_small_kernel, small_smem, done_small);
    if (e != cudaSuccess) return e;
    const int nsm = a.num_sms;
    const int small_grid = min(b.grid.ntiles, nsm * 4);
    const int big_grid = min(b.grid.ntiles, nsm);
    cudaStream_t s_small = a.stream;
    if (side != nullptr) {
        if ((e = cudaEventRecord(fork, a.stream)) != cudaSuccess) return e;
        if ((e = cudaStreamWaitEvent(side, fork, 0)) != cudaSuccess) return e;
        s_small = side;
    }
    sort_big_kernel<<<big_grid, 1024, big_smem, a.stream>>>(b.header, b.work_order, b.tile_start, b.keys);
    sort_small_kernel<<<small_grid, 256, small_smem, s_small>>>(b.header, b.work_order, b.tile_start, b.keys);
    if (side != nullptr) {
        if ((e = cudaEventRecord(join, side)) != cudaSuccess) return e;
        if ((e = cudaStreamWaitEvent(a.stream, join, 0)) != cudaSuccess) return e;
    }
    return cudaGetLastError();
}

// b200gsr_pair_report: a forward captured into a CUDA graph has no host notify slot, so this one-thread kernel,
// enqueued after it, folds the pair count and overflow flag the scan wrote into its header into a device report:
// report[0] = the largest pair count seen, report[1] = the number of forwards that overflowed their key buffer.
namespace {
__global__ void pair_report_kernel(const uint32_t* __restrict__ header, uint32_t* __restrict__ report) {
    report[0] = max(report[0], header[GSR_H_NUM_PAIRS]);
    report[1] += header[GSR_H_OVERFLOW] != 0u ? 1u : 0u;
}
}  // namespace

cudaError_t gsr_launch_pair_report(const uint32_t* header, uint32_t* report, cudaStream_t s) {
    pair_report_kernel<<<1, 1, 0, s>>>(header, report);
    return cudaGetLastError();
}
