// Quadric edge-collapse decimation in rounds of independent edges (include/b200gsr_mesh_decimate.h).  Every float64
// operation that decides anything is an explicit __d*_rn intrinsic, so nothing is contracted into an FMA, and the only
// atomics are integer counts, so every call gives the same bits.
//
//   dec_init          per vertex and per face: float64 positions, the working copy of the faces (a face with an index
//                     outside [0, V) is counted in bad and dropped); the state
//   dec_keys          per face slot: the sort key (the vertex, V for a dead face) and the face index
//   cub radix sort    stable, so each vertex's face list comes out in face-index order (no atomic append anywhere)
//   dec_starts        per sorted entry: the list starts of the vertices between the previous key and its own
//   dec_entries       per sorted entry: the fan entry (p, q) of its vertex, p = -1 for a face listing an index twice
//   dec_quadrics      per vertex (begin only): the sum of its faces' plane quadrics in list order
//   dec_regular       per vertex: the valence of a regular vertex (one closed, oriented fan), 0 for any other
//   dec_best          per regular vertex: m(v), the smallest candidate at v, and its placement
//   dec_min2          per regular vertex: M(v), the smallest m over v and its neighbours
//   dec_select        per vertex: its edge is selected (it is the smaller endpoint); S counted per warp
//   dec_plan          one CTA: how many selected edges this round applies (a radix select of the first j keys when
//                     they would overshoot the target), the new face count, the round count, whether to stop
//   dec_apply         per applied edge: the collapse, on faces no other applied edge touches
//   dec_ref_* / scan  the referenced vertices and the live faces, scanned (gsr_scan_u32) into V', F' and the offsets
//   dec_emit_*        gather the output like b200gsr_mesh_clean_emit
#include <cstddef>

#include <cub/device/device_radix_sort.cuh>

#include "common.cuh"
#include "../../include/b200gsr_mesh_decimate.h"

namespace {

constexpr int kThreads = 256;
constexpr int kPlanThreads = 1024;
constexpr int kMaxValence = B200GSR_DECIMATE_MAX_VALENCE;
constexpr unsigned long long kNone = ~0ull;

struct DecState {                 // the first B200GSR_DECIMATE_STATUS_WORDS words are the status
    int32_t F_live, rounds, done, bad, V_out, F_out;
    int32_t target, optimal;
    uint32_t S, pad;
    unsigned long long limit;     // this round applies the selected edges whose key is below limit
};
static_assert(offsetof(DecState, target) == 4 * B200GSR_DECIMATE_STATUS_WORDS, "status words lead the state");

struct DecArgs {
    int V, F, N;                  // N = 3 F sort entries
    int32_t* faces;               // [F,3] working faces, -1 -1 -1 once dead
    const uint32_t* skey;         // [N] sorted keys (vertices) of this round
    const uint32_t* sval;         // [N] sorted values (faces) of this round
    uint32_t* start;              // [V+1] list starts
    int32_t* ep;                  // [N] fan entries (p, q) in sorted order
    int32_t* eq;
    double* pos;                  // [V,3]
    double* Q;                    // [V,10]
    double* xb;                   // [V,3] placement of m(v)
    unsigned long long* m_hi;     // [V] (float32 bits of key cost) << 32 | a of m(v), kNone: none
    uint32_t* m_lo;               // [V] b of m(v)
    unsigned long long* M_hi;     // [V] M(v)
    uint32_t* M_lo;
    unsigned long long* sel;      // [V] key of the selected edge whose smaller endpoint is v, kNone: none
    uint8_t* kreg;                // [V] valence of a regular vertex, 0 otherwise
    uint8_t* moved;               // [V]
    uint8_t* ref;                 // [V]
    uint32_t* vstart;             // [V] flags, then offsets
    uint32_t* fstart;             // [F]
    DecState* st;
};

__device__ __forceinline__ double dadd(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double dsub(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ double dmul(double a, double b) { return __dmul_rn(a, b); }

struct D3 { double x, y, z; };
__device__ __forceinline__ D3 ld3(const double* p) { return D3{p[0], p[1], p[2]}; }
__device__ __forceinline__ D3 sub3(D3 u, D3 w) { return D3{dsub(u.x, w.x), dsub(u.y, w.y), dsub(u.z, w.z)}; }
__device__ __forceinline__ D3 cross3(D3 u, D3 w) {
    return D3{dsub(dmul(u.y, w.z), dmul(u.z, w.y)), dsub(dmul(u.z, w.x), dmul(u.x, w.z)),
              dsub(dmul(u.x, w.y), dmul(u.y, w.x))};
}
__device__ __forceinline__ double dot3(D3 u, D3 w) { return dadd(dadd(dmul(u.x, w.x), dmul(u.y, w.y)), dmul(u.z, w.z)); }

__device__ __forceinline__ bool face_ok(const int32_t* t, int V) {
    return (uint32_t)t[0] < (uint32_t)V && (uint32_t)t[1] < (uint32_t)V && (uint32_t)t[2] < (uint32_t)V;
}

// E(x) of rule 3
__device__ double qform(const double* q, D3 x) {
    const double r0 = dadd(dadd(dmul(q[0], x.x), dmul(q[1], x.y)), dadd(dmul(q[2], x.z), q[3]));
    const double r1 = dadd(dadd(dmul(q[1], x.x), dmul(q[4], x.y)), dadd(dmul(q[5], x.z), q[6]));
    const double r2 = dadd(dadd(dmul(q[2], x.x), dmul(q[5], x.y)), dadd(dmul(q[7], x.z), q[8]));
    const double r3 = dadd(dadd(dmul(q[3], x.x), dmul(q[6], x.y)), dadd(dmul(q[8], x.z), q[9]));
    return dadd(dadd(dmul(r0, x.x), dmul(r1, x.y)), dadd(dmul(r2, x.z), r3));
}

__device__ __forceinline__ double det3(double m00, double m01, double m02, double m10, double m11, double m12,
                                       double m20, double m21, double m22) {
    const double t0 = dsub(dmul(m11, m22), dmul(m12, m21));
    const double t1 = dsub(dmul(m10, m22), dmul(m12, m20));
    const double t2 = dsub(dmul(m10, m21), dmul(m11, m20));
    return dadd(dsub(dmul(m00, t0), dmul(m01, t1)), dmul(m02, t2));
}

__global__ void __launch_bounds__(kThreads) dec_init_kernel(DecArgs a, const float* __restrict__ vert, const int32_t* __restrict__ faces,
                                                            int target, int optimal) {
    const int i = blockIdx.x * kThreads + threadIdx.x;
    if (i == 0) {
        a.st->F_live = a.F;
        a.st->target = target;
        a.st->optimal = optimal;
    }
    if (i < a.V) {
        for (int k = 0; k < 3; ++k) a.pos[3 * (size_t)i + k] = (double)vert[3 * (size_t)i + k];
        a.moved[i] = 0;
    }
    if (i < a.F) {
        const int32_t* t = faces + 3 * (size_t)i;
        const bool ok = face_ok(t, a.V);
        if (!ok) atomicAdd(&a.st->bad, 1);
        int32_t* d = a.faces + 3 * (size_t)i;
        for (int k = 0; k < 3; ++k) d[k] = ok ? t[k] : -1;
    }
}

__global__ void dec_begin_done_kernel(DecState* st) {
    st->done = st->bad != 0 || st->F_live <= st->target;
}

__global__ void __launch_bounds__(kThreads) dec_keys_kernel(DecArgs a, uint32_t* __restrict__ key, uint32_t* __restrict__ val) {
    if (a.st->done) return;
    const int e = blockIdx.x * kThreads + threadIdx.x;
    if (e >= a.N) return;
    const int f = e / 3;
    const int32_t v = a.faces[e];
    key[e] = v < 0 ? (uint32_t)a.V : (uint32_t)v;
    val[e] = (uint32_t)f;
}

__global__ void __launch_bounds__(kThreads) dec_starts_kernel(DecArgs a) {
    if (a.st->done) return;
    const int i = blockIdx.x * kThreads + threadIdx.x;
    if (i > a.N) return;
    const long long prev = i == 0 ? -1 : (long long)a.skey[i - 1];
    const long long cur = i == a.N ? a.V : (long long)a.skey[i];
    for (long long v = prev + 1; v <= cur; ++v) a.start[v] = (uint32_t)i;
}

__global__ void __launch_bounds__(kThreads) dec_entries_kernel(DecArgs a) {
    if (a.st->done) return;
    const int i = blockIdx.x * kThreads + threadIdx.x;
    if (i >= (int)a.start[a.V]) return;
    const int v = (int)a.skey[i];
    const int32_t* t = a.faces + 3 * (size_t)a.sval[i];
    const int s = t[0] == v ? 0 : t[1] == v ? 1 : 2;
    const bool rep = t[0] == t[1] || t[1] == t[2] || t[0] == t[2];
    a.ep[i] = rep ? -1 : t[(s + 1) % 3];
    a.eq[i] = t[(s + 2) % 3];
}

// rule 1: the plane quadric of each face in v's list, added in list (face-index) order
__global__ void __launch_bounds__(kThreads) dec_quadrics_kernel(DecArgs a) {
    const int v = blockIdx.x * kThreads + threadIdx.x;
    if (v >= a.V) return;
    double acc[10];
#pragma unroll
    for (int k = 0; k < 10; ++k) acc[k] = 0.0;
    for (uint32_t i = a.start[v]; i < a.start[v + 1]; ++i) {
        const int32_t* t = a.faces + 3 * (size_t)a.sval[i];
        const D3 p0 = ld3(a.pos + 3 * (size_t)t[0]), p1 = ld3(a.pos + 3 * (size_t)t[1]), p2 = ld3(a.pos + 3 * (size_t)t[2]);
        const D3 n = cross3(sub3(p1, p0), sub3(p2, p0));
        const double l2 = dot3(n, n);
        if (l2 == 0.0) continue;                         // adds +0 to every value: acc is unchanged
        const double l = __dsqrt_rn(l2);
        const D3 u{__ddiv_rn(n.x, l), __ddiv_rn(n.y, l), __ddiv_rn(n.z, l)};
        const double s[4] = {u.x, u.y, u.z, -dot3(u, p0)};
        const double w = dmul(l, 0.5);
        int k = 0;
#pragma unroll
        for (int r = 0; r < 4; ++r)
#pragma unroll
            for (int c = r; c < 4; ++c, ++k) acc[k] = dadd(acc[k], dmul(w, dmul(s[r], s[c])));
    }
#pragma unroll
    for (int k = 0; k < 10; ++k) a.Q[10 * (size_t)v + k] = acc[k];
}

// rule 2's fan walk: regular vertices get their valence
__global__ void __launch_bounds__(kThreads) dec_regular_kernel(DecArgs a) {
    if (a.st->done) return;
    const int v = blockIdx.x * kThreads + threadIdx.x;
    if (v >= a.V) return;
    const uint32_t s = a.start[v];
    const int k = (int)(a.start[v + 1] - s);
    bool ok = k >= 3 && k <= kMaxValence;
    for (int i = 0; ok && i < k; ++i) ok = a.ep[s + i] >= 0;
    if (ok) {
        const int32_t p0 = a.ep[s];
        int32_t c = a.eq[s];
        int steps = 1;
        while (c != p0) {
            if (steps >= k) { ok = false; break; }
            int j = 0;
            while (j < k && a.ep[s + j] != c) ++j;
            if (j == k) { ok = false; break; }
            c = a.eq[s + j];
            ++steps;
        }
        ok = ok && steps == k;
    }
    a.kreg[v] = ok ? (uint8_t)k : 0;
}

// Rules 2 and 3 for the edge (ea, eb), ea < eb, both regular: whether it is a candidate, its placement and key cost.
__device__ bool evaluate(const DecArgs& a, int ea, int eb, bool optimal, D3& x, uint32_t& cost_bits) {
    const int ka = a.kreg[ea], kb = a.kreg[eb];
    if (ka + kb - 4 < 3) return false;
    const uint32_t sa = a.start[ea], sb = a.start[eb];
    int common = 0;
    for (int i = 0; i < ka; ++i) {
        const int32_t c = a.ep[sa + i];
        for (int j = 0; j < kb; ++j)
            if (a.ep[sb + j] == c) { ++common; break; }
    }
    if (common != 2) return false;
    double q[10];
#pragma unroll
    for (int k = 0; k < 10; ++k) q[k] = dadd(a.Q[10 * (size_t)ea + k], a.Q[10 * (size_t)eb + k]);
    const D3 pa = ld3(a.pos + 3 * (size_t)ea), pb = ld3(a.pos + 3 * (size_t)eb);
    bool solved = false;
    double e = 0.0;
    if (optimal) {
        const double r0 = -q[3], r1 = -q[6], r2 = -q[8];
        const double det = det3(q[0], q[1], q[2], q[1], q[4], q[5], q[2], q[5], q[7]);
        const double tr = dadd(dadd(q[0], q[4]), q[7]);
        if (fabs(det) > dmul(dmul(dmul(tr, tr), tr), B200GSR_DECIMATE_DET_TOL)) {
            x.x = __ddiv_rn(det3(r0, q[1], q[2], r1, q[4], q[5], r2, q[5], q[7]), det);
            x.y = __ddiv_rn(det3(q[0], r0, q[2], q[1], r1, q[5], q[2], r2, q[7]), det);
            x.z = __ddiv_rn(det3(q[0], q[1], r0, q[1], q[4], r1, q[2], q[5], r2), det);
            e = qform(q, x);
            solved = true;
        }
    }
    if (!solved) {
        x = pa;
        e = qform(q, pa);
        const double eb2 = qform(q, pb);
        if (eb2 < e) { x = pb; e = eb2; }
        const D3 mid{dmul(dadd(pa.x, pb.x), 0.5), dmul(dadd(pa.y, pb.y), 0.5), dmul(dadd(pa.z, pb.z), 0.5)};
        const double em = qform(q, mid);
        if (em < e) { x = mid; e = em; }
    }
    if (e <= 0.0) e = 0.0;
    if (isnan(e)) return false;
    for (int side = 0; side < 2; ++side) {
        const int mv = side ? eb : ea, other = side ? ea : eb;
        const uint32_t s = side ? sb : sa;
        const int k = side ? kb : ka;
        const D3 pv = ld3(a.pos + 3 * (size_t)mv);
        for (int i = 0; i < k; ++i) {
            const int32_t p = a.ep[s + i], r = a.eq[s + i];
            if (p == other || r == other) continue;
            const D3 pp = ld3(a.pos + 3 * (size_t)p), pr = ld3(a.pos + 3 * (size_t)r);
            const D3 nb = cross3(sub3(pp, pv), sub3(pr, pv));
            if (nb.x == 0.0 && nb.y == 0.0 && nb.z == 0.0) continue;
            const D3 na = cross3(sub3(pp, x), sub3(pr, x));
            if (!(dot3(nb, na) > 0.0)) return false;
        }
    }
    cost_bits = __float_as_uint(__double2float_ru(e));
    return true;
}

__device__ __forceinline__ bool less_key(unsigned long long h1, uint32_t l1, unsigned long long h2, uint32_t l2) {
    return h1 < h2 || (h1 == h2 && l1 < l2);
}

__global__ void __launch_bounds__(kThreads) dec_best_kernel(DecArgs a) {
    if (a.st->done) return;
    const int v = blockIdx.x * kThreads + threadIdx.x;
    if (v >= a.V) return;
    unsigned long long best_hi = kNone;
    uint32_t best_lo = ~0u;
    D3 best_x{0.0, 0.0, 0.0};
    const int k = a.kreg[v];
    const bool optimal = a.st->optimal != 0;
    for (int i = 0; i < k; ++i) {
        const int n = a.ep[a.start[v] + i];
        if (!a.kreg[n]) continue;
        const int ea = v < n ? v : n, eb = v < n ? n : v;
        D3 x;
        uint32_t cb;
        if (!evaluate(a, ea, eb, optimal, x, cb)) continue;
        const unsigned long long hi = (unsigned long long)cb << 32 | (uint32_t)ea;
        if (less_key(hi, (uint32_t)eb, best_hi, best_lo)) { best_hi = hi; best_lo = (uint32_t)eb; best_x = x; }
    }
    a.m_hi[v] = best_hi;
    a.m_lo[v] = best_lo;
    double* xb = a.xb + 3 * (size_t)v;
    xb[0] = best_x.x; xb[1] = best_x.y; xb[2] = best_x.z;
}

__global__ void __launch_bounds__(kThreads) dec_min2_kernel(DecArgs a) {
    if (a.st->done) return;
    const int v = blockIdx.x * kThreads + threadIdx.x;
    if (v >= a.V) return;
    unsigned long long hi = a.m_hi[v];
    uint32_t lo = a.m_lo[v];
    const int k = a.kreg[v];
    for (int i = 0; i < k; ++i) {
        const int n = a.ep[a.start[v] + i];
        const unsigned long long h = a.m_hi[n];
        const uint32_t l = a.m_lo[n];
        if (less_key(h, l, hi, lo)) { hi = h; lo = l; }
    }
    a.M_hi[v] = hi;
    a.M_lo[v] = lo;
}

__global__ void __launch_bounds__(kThreads) dec_select_kernel(DecArgs a) {
    if (a.st->done) return;
    const int v = blockIdx.x * kThreads + threadIdx.x;
    bool chosen = false;
    if (v < a.V) {
        const unsigned long long hi = a.m_hi[v];
        const uint32_t lo = a.m_lo[v];
        chosen = hi != kNone && (uint32_t)hi == (uint32_t)v && a.M_hi[v] == hi && a.M_lo[v] == lo &&
                 a.M_hi[lo] == hi && a.M_lo[lo] == lo;
        a.sel[v] = chosen ? hi : kNone;
    }
    const unsigned ballot = __ballot_sync(0xffffffffu, chosen);
    if ((threadIdx.x & 31) == 0 && ballot) atomicAdd(&a.st->S, (uint32_t)__popc(ballot));
}

// One CTA.  The j-th smallest selected key by an MSB-first radix select, 8 bits per pass, when the round would
// overshoot the target; otherwise every selected edge applies.
__global__ void __launch_bounds__(kPlanThreads) dec_plan_kernel(DecArgs a) {
    __shared__ uint32_t hist[256];
    __shared__ unsigned long long prefix;
    __shared__ long long rem;
    DecState* st = a.st;
    const int done = st->done;
    const long long S = st->S, F = st->F_live, T = st->target;
    __syncthreads();
    if (done || S == 0) {
        if (threadIdx.x == 0) { st->limit = 0ull; st->done = 1; st->S = 0; }
        return;
    }
    const long long j = (F - T + 1) / 2;
    unsigned long long limit = kNone;
    long long applied = S;
    if (S > j) {
        if (threadIdx.x == 0) { prefix = 0ull; rem = j; }
        for (int shift = 56; shift >= 0; shift -= 8) {
            if (threadIdx.x < 256) hist[threadIdx.x] = 0u;
            __syncthreads();
            const unsigned long long hmask = shift == 56 ? 0ull : ~0ull << (shift + 8);
            const unsigned long long pre = prefix;
            for (int v = threadIdx.x; v < a.V; v += kPlanThreads) {
                const unsigned long long key = a.sel[v];
                if ((key & hmask) == pre) atomicAdd(&hist[(key >> shift) & 255u], 1u);
            }
            __syncthreads();
            if (threadIdx.x == 0) {
                long long cum = 0;
                for (int d = 0; d < 256; ++d) {
                    if (cum + hist[d] >= rem) { prefix |= (unsigned long long)d << shift; rem -= cum; break; }
                    cum += hist[d];
                }
            }
            __syncthreads();
        }
        limit = prefix + 1;
        applied = j;
    }
    if (threadIdx.x == 0) {
        st->limit = limit;
        st->F_live = (int32_t)(F - 2 * applied);
        st->rounds += 1;
        st->S = 0;
        st->done = F - 2 * applied <= T;
    }
}

__global__ void __launch_bounds__(kThreads) dec_apply_kernel(DecArgs a) {
    const int v = blockIdx.x * kThreads + threadIdx.x;
    if (v >= a.V || a.sel[v] >= a.st->limit) return;
    const int b = (int)a.m_lo[v];
    double* qa = a.Q + 10 * (size_t)v;
    const double* qb = a.Q + 10 * (size_t)b;
#pragma unroll
    for (int k = 0; k < 10; ++k) qa[k] = dadd(qa[k], qb[k]);
    for (int k = 0; k < 3; ++k) a.pos[3 * (size_t)v + k] = a.xb[3 * (size_t)v + k];
    a.moved[v] = 1;
    const uint32_t s = a.start[b];
    const int kb = a.kreg[b];
    for (int i = 0; i < kb; ++i) {
        int32_t* t = a.faces + 3 * (size_t)a.sval[s + i];
        if (t[0] == v || t[1] == v || t[2] == v) {
            t[0] = t[1] = t[2] = -1;
        } else {
            for (int c = 0; c < 3; ++c)
                if (t[c] == b) t[c] = v;
        }
    }
}

__global__ void __launch_bounds__(kThreads) dec_ref_clear_kernel(DecArgs a) {
    const int v = blockIdx.x * kThreads + threadIdx.x;
    if (v < a.V) a.ref[v] = 0;
}

__global__ void __launch_bounds__(kThreads) dec_ref_mark_kernel(DecArgs a) {
    const int f = blockIdx.x * kThreads + threadIdx.x;
    if (f >= a.F) return;
    const int32_t* t = a.faces + 3 * (size_t)f;
    const bool live = t[0] >= 0;
    if (live) { a.ref[t[0]] = 1; a.ref[t[1]] = 1; a.ref[t[2]] = 1; }
    a.fstart[f] = live;
}

__global__ void __launch_bounds__(kThreads) dec_ref_flags_kernel(DecArgs a) {
    const int v = blockIdx.x * kThreads + threadIdx.x;
    if (v < a.V) a.vstart[v] = a.ref[v];
}

__global__ void __launch_bounds__(kThreads) dec_emit_vertices_kernel(DecArgs a, const float* __restrict__ vert,
                                                                     float* __restrict__ out, int32_t* __restrict__ kept,
                                                                     uint32_t V_out) {
    const int v = blockIdx.x * kThreads + threadIdx.x;
    if (v >= a.V || !a.ref[v]) return;
    const uint32_t o = a.vstart[v];
    if (o >= V_out) return;
    uint32_t* dst = reinterpret_cast<uint32_t*>(out) + 3 * (size_t)o;
    if (a.moved[v]) {
        for (int k = 0; k < 3; ++k) dst[k] = __float_as_uint(__double2float_rn(a.pos[3 * (size_t)v + k]));
    } else {
        const uint32_t* src = reinterpret_cast<const uint32_t*>(vert) + 3 * (size_t)v;   // the bits, NaN payloads too
        dst[0] = src[0]; dst[1] = src[1]; dst[2] = src[2];
    }
    kept[o] = v;
}

__global__ void __launch_bounds__(kThreads) dec_emit_faces_kernel(DecArgs a, int32_t* __restrict__ out, uint32_t F_out) {
    const int f = blockIdx.x * kThreads + threadIdx.x;
    if (f >= a.F) return;
    const int32_t* t = a.faces + 3 * (size_t)f;
    if (t[0] < 0) return;
    const uint32_t o = a.fstart[f];
    if (o >= F_out) return;
    int32_t* d = out + 3 * (size_t)o;
    d[0] = (int32_t)a.vstart[t[0]]; d[1] = (int32_t)a.vstart[t[1]]; d[2] = (int32_t)a.vstart[t[2]];
}

size_t align256(size_t v) { return (v + 255) / 256 * 256; }
int blocks(long long n) { return (int)((n + kThreads - 1) / kThreads); }

DecArgs dec_args(const GsrMeshDecimatePlan& p, uint8_t* s) {
    DecArgs a{};
    a.V = p.V; a.F = p.F; a.N = 3 * p.F;
    a.faces = reinterpret_cast<int32_t*>(s + p.off_faces);
    a.start = reinterpret_cast<uint32_t*>(s + p.off_start);
    a.ep = reinterpret_cast<int32_t*>(s + p.off_ep);
    a.eq = reinterpret_cast<int32_t*>(s + p.off_eq);
    a.pos = reinterpret_cast<double*>(s + p.off_pos);
    a.Q = reinterpret_cast<double*>(s + p.off_Q);
    a.xb = reinterpret_cast<double*>(s + p.off_xb);
    a.m_hi = reinterpret_cast<unsigned long long*>(s + p.off_m_hi);
    a.M_hi = reinterpret_cast<unsigned long long*>(s + p.off_M_hi);
    a.sel = reinterpret_cast<unsigned long long*>(s + p.off_sel);
    a.m_lo = reinterpret_cast<uint32_t*>(s + p.off_m_lo);
    a.M_lo = reinterpret_cast<uint32_t*>(s + p.off_M_lo);
    a.kreg = s + p.off_kreg;
    a.moved = s + p.off_moved;
    a.ref = s + p.off_ref;
    a.vstart = reinterpret_cast<uint32_t*>(s + p.off_vstart);
    a.fstart = reinterpret_cast<uint32_t*>(s + p.off_fstart);
    a.st = reinterpret_cast<DecState*>(s + p.off_state);
    return a;
}

int key_bits(int V) {                  // keys run over [0, V]
    int b = 1;
    while (b < 31 && ((long long)1 << b) <= V) ++b;
    return b;
}

// dec_keys, the stable sort and dec_starts / dec_entries: each vertex's fan, in face-index order
cudaError_t build_lists(const GsrMeshDecimatePlan& p, DecArgs& a, uint8_t* s, cudaStream_t st, bool entries) {
    uint32_t* k0 = reinterpret_cast<uint32_t*>(s + p.off_keys);
    uint32_t* k1 = k0 + a.N;
    uint32_t* v0 = reinterpret_cast<uint32_t*>(s + p.off_vals);
    uint32_t* v1 = v0 + a.N;
    dec_keys_kernel<<<blocks(a.N), kThreads, 0, st>>>(a, k0, v0);
    cub::DoubleBuffer<uint32_t> keys(k0, k1), vals(v0, v1);
    size_t need = 0;
    cudaError_t e = cub::DeviceRadixSort::SortPairs(nullptr, need, keys, vals, a.N, 0, key_bits(a.V), st);
    if (e != cudaSuccess) return e;
    if (need > p.cub_bytes) return cudaErrorInvalidValue;        // the plan's bound on cub's temporary storage
    e = cub::DeviceRadixSort::SortPairs(s + p.off_cub, need, keys, vals, a.N, 0, key_bits(a.V), st);
    if (e != cudaSuccess) return e;
    a.skey = keys.Current();
    a.sval = vals.Current();
    dec_starts_kernel<<<blocks((long long)a.N + 1), kThreads, 0, st>>>(a);
    if (entries) dec_entries_kernel<<<blocks(a.N), kThreads, 0, st>>>(a);
    return cudaGetLastError();
}

// the referenced vertices and live faces, scanned into V', F'; then the status words
cudaError_t count(const GsrMeshDecimatePlan& p, DecArgs& a, uint8_t* s, int32_t* status, cudaStream_t st) {
    dec_ref_clear_kernel<<<blocks(a.V), kThreads, 0, st>>>(a);
    if (a.F) dec_ref_mark_kernel<<<blocks(a.F), kThreads, 0, st>>>(a);
    dec_ref_flags_kernel<<<blocks(a.V), kThreads, 0, st>>>(a);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    uint32_t* bsums = reinterpret_cast<uint32_t*>(s + p.off_bsums);
    gsr_scan_u32(a.V, a.vstart, a.vstart, bsums, reinterpret_cast<uint32_t*>(&a.st->V_out), st);
    if (a.F) gsr_scan_u32(a.F, a.fstart, a.fstart, bsums, reinterpret_cast<uint32_t*>(&a.st->F_out), st);
    else if ((e = cudaMemsetAsync(&a.st->F_out, 0, sizeof(int32_t), st)) != cudaSuccess) return e;
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    return cudaMemcpyAsync(status, a.st, sizeof(int32_t) * B200GSR_DECIMATE_STATUS_WORDS, cudaMemcpyDeviceToDevice, st);
}

}  // namespace

void gsr_mesh_decimate_plan(int V, int F, GsrMeshDecimatePlan* pl) {
    GsrMeshDecimatePlan& p = *pl;
    p.V = V; p.F = F;
    const size_t v = (size_t)V, f = (size_t)F, n = 3 * (size_t)F;
    // cub's onesweep radix sort over a DoubleBuffer needs its bins, one lookback record of 256 counters per tile and
    // a few counters: under 4 bytes per item plus 1 MiB for any tile size of 256 items or more
    p.cub_bytes = align256(4 * n + (1u << 20));
    size_t o = 0;
    auto take = [&o](size_t bytes) { const size_t at = o; o += align256(bytes); return at; };
    p.off_state = take(256);
    p.off_faces = take(12 * f);
    p.off_keys = take(8 * n);
    p.off_vals = take(8 * n);
    p.off_cub = take(p.cub_bytes);
    p.off_start = take(4 * (v + 1));
    p.off_ep = take(4 * n);
    p.off_eq = take(4 * n);
    p.off_pos = take(24 * v);
    p.off_Q = take(80 * v);
    p.off_xb = take(24 * v);
    p.off_m_hi = take(8 * v);
    p.off_M_hi = take(8 * v);
    p.off_sel = take(8 * v);
    p.off_m_lo = take(4 * v);
    p.off_M_lo = take(4 * v);
    p.off_kreg = take(v);
    p.off_moved = take(v);
    p.off_ref = take(v);
    p.off_vstart = take(4 * v);
    p.off_fstart = take(4 * f);
    const size_t m = v > f ? v : f;
    p.off_bsums = take(((m + 4095) / 4096 + 1) * sizeof(uint32_t));
    p.total = o;
}

cudaError_t gsr_launch_mesh_decimate_begin(const GsrMeshDecimatePlan& p, const float* vertices, const int32_t* faces,
                                           int target_faces, bool optimal_placement, int32_t* status, uint8_t* scratch,
                                           cudaStream_t s) {
    DecArgs a = dec_args(p, scratch);
    cudaError_t e = cudaMemsetAsync(a.st, 0, sizeof(DecState), s);
    if (e != cudaSuccess) return e;
    dec_init_kernel<<<blocks(a.V > a.F ? a.V : a.F), kThreads, 0, s>>>(a, vertices, faces, target_faces,
                                                                         optimal_placement ? 1 : 0);
    if (a.F) {
        // the quadrics need every valid face, so the lists are built before the state may say done
        if ((e = build_lists(p, a, scratch, s, false)) != cudaSuccess) return e;
        dec_quadrics_kernel<<<blocks(a.V), kThreads, 0, s>>>(a);
    } else {
        cudaMemsetAsync(a.Q, 0, 80 * (size_t)a.V, s);
    }
    dec_begin_done_kernel<<<1, 1, 0, s>>>(a.st);
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    return count(p, a, scratch, status, s);
}

cudaError_t gsr_launch_mesh_decimate_rounds(const GsrMeshDecimatePlan& p, int rounds, int32_t* status,
                                            uint8_t* scratch, cudaStream_t s) {
    DecArgs a = dec_args(p, scratch);
    cudaError_t e;
    for (int r = 0; r < rounds && a.F; ++r) {
        if ((e = build_lists(p, a, scratch, s, true)) != cudaSuccess) return e;
        dec_regular_kernel<<<blocks(a.V), kThreads, 0, s>>>(a);
        dec_best_kernel<<<blocks(a.V), kThreads, 0, s>>>(a);
        dec_min2_kernel<<<blocks(a.V), kThreads, 0, s>>>(a);
        dec_select_kernel<<<blocks(a.V), kThreads, 0, s>>>(a);
        dec_plan_kernel<<<1, kPlanThreads, 0, s>>>(a);
        dec_apply_kernel<<<blocks(a.V), kThreads, 0, s>>>(a);
        if ((e = cudaGetLastError()) != cudaSuccess) return e;
    }
    return count(p, a, scratch, status, s);
}

cudaError_t gsr_launch_mesh_decimate_emit(const GsrMeshDecimatePlan& p, const float* vertices, const uint8_t* scratch,
                                          float* out_vertices, int32_t* out_faces, int32_t* kept, int32_t V_out,
                                          int32_t F_out, cudaStream_t s) {
    DecArgs a = dec_args(p, const_cast<uint8_t*>(scratch));
    dec_emit_vertices_kernel<<<blocks(a.V), kThreads, 0, s>>>(a, vertices, out_vertices, kept, (uint32_t)V_out);
    if (a.F) dec_emit_faces_kernel<<<blocks(a.F), kThreads, 0, s>>>(a, out_faces, (uint32_t)F_out);
    return cudaGetLastError();
}
