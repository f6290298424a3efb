// Connected components of a triangle mesh and the removal of small ones (include/b200gsr_mesh_clean.h).  Integer
// atomics only, each of them order-independent, so every call gives the same bits.
//
//   clean_init        per vertex: parent[v] = v, zero counts and flags, empty boxes; the mesh box, the largest
//                     candidate and the bad-face count reset
//   clean_union       per face: link its vertices' trees (lock-free union by CAS, smaller index wins)
//   clean_label       per vertex: label[v] = the root of v's tree, the smallest index of its component
//   clean_faces       per face: faces per root (warp-aggregated atomicAdd), referenced-vertex bytes
//   clean_boxes       per vertex: per-root and whole-mesh boxes, atomicMin / atomicMax of ordered uint32 encodings
//   clean_decide      per root: the face-count and float64 diameter tests; the largest candidate by one 64-bit
//                     atomicMax of (faces << 32) | ~label
//   clean_flags       per vertex and per face: kept or not, then gsr_scan_u32 (densify.cu) of both: offsets and the
//                     totals V', F'
//   clean_emit_*      gather the kept vertices and their indices, renumber the kept faces through the vertex offsets
//
// Termination of the union-find: parent[v] <= v holds at every moment for every v.  It holds after clean_init, a
// link only ever points a root at a smaller index, and path halving only stores an ancestor's ancestor, which is
// smaller again.  So every find walk visits strictly decreasing indices and ends within v steps, whatever values it
// reads (a stale read is still some earlier parent, which obeys the same bound), and there is no cycle to hang on.
#include "common.cuh"
#include "../../include/b200gsr_mesh_clean.h"

namespace {

constexpr int kThreads = 256;
constexpr uint32_t kEmptyMin = 0xffffffffu;   // box encodings an empty axis keeps; no float encodes to either
constexpr uint32_t kEmptyMax = 0u;

struct CleanArgs {
    int V, F;
    const float* vert;          // [V,3] (count / emit only)
    const int32_t* faces;       // [F,3]
    int32_t* parent;            // [V]
    int32_t* label;             // [V]
    int32_t* bad;               // faces with an index outside [0, V)
    uint8_t* ref;               // [V]: referenced by a face
    uint8_t* pass;              // [V]: root passes the face-count and diameter tests
    uint32_t* fcount;           // [V]: faces per root
    uint32_t* box;              // [V][6]: per-root min x, y, z, max x, y, z (encoded)
    uint32_t* vstart;           // [V]: kept flags, then (scanned) offsets
    uint32_t* fstart;           // [F]: kept flags, then (scanned) offsets
    uint32_t* mesh_box;         // [6]: the box of every referenced vertex
    unsigned long long* best;   // (faces << 32) | ~label of the largest passing component, 0 = none
    int min_faces;
    double min_diameter;
    bool keep_largest;
};

// order-preserving uint32 image of a float: a < b (both not NaN) iff enc(a) < enc(b)
__device__ __forceinline__ uint32_t enc(float x) {
    const uint32_t b = __float_as_uint(x);
    return b & 0x80000000u ? ~b : b | 0x80000000u;
}
__device__ __forceinline__ float dec(uint32_t e) { return __uint_as_float(e & 0x80000000u ? e & 0x7fffffffu : ~e); }

// the root of x's tree, halving the path on the way: every store puts an ancestor's ancestor (a smaller index) into
// a non-root, so parent[v] <= v stays true and the walk strictly decreases
__device__ __forceinline__ int find_root(int32_t* parent, int x) {
    while (true) {
        const int p = __ldcg(parent + x);
        if (p == x) return x;
        const int gp = __ldcg(parent + p);
        if (gp == p) return p;
        __stcg(parent + x, gp);
        x = gp;
    }
}

// link the trees of x and y: the larger root is pointed at the smaller one by CAS, only if it is still a root.  A
// failed CAS returns the root's new parent, smaller than the root; x + y strictly decreases from one try to the next.
__device__ __forceinline__ void unite(int32_t* parent, int x, int y) {
    while (true) {
        x = find_root(parent, x);
        y = find_root(parent, y);
        if (x == y) return;
        const int hi = x > y ? x : y, lo = x > y ? y : x;
        const int old = atomicCAS(parent + hi, hi, lo);
        if (old == hi) return;
        x = old;
        y = lo;
    }
}

__device__ __forceinline__ bool face_ok(const int32_t* f, int V) {
    return (uint32_t)f[0] < (uint32_t)V && (uint32_t)f[1] < (uint32_t)V && (uint32_t)f[2] < (uint32_t)V;
}

__global__ void __launch_bounds__(kThreads) clean_init_kernel(CleanArgs a) {
    const int v = blockIdx.x * kThreads + threadIdx.x;
    if (v == 0) {
        *a.bad = 0;
        *a.best = 0ull;
        for (int k = 0; k < 3; ++k) { a.mesh_box[k] = kEmptyMin; a.mesh_box[3 + k] = kEmptyMax; }
    }
    if (v >= a.V) return;
    a.parent[v] = v;
    if (!a.ref) return;                   // the components alone need the parents only
    a.ref[v] = 0;
    a.pass[v] = 0;
    a.fcount[v] = 0u;
    uint32_t* b = a.box + 6 * (size_t)v;
    for (int k = 0; k < 3; ++k) { b[k] = kEmptyMin; b[3 + k] = kEmptyMax; }
}

__global__ void __launch_bounds__(kThreads) clean_union_kernel(CleanArgs a) {
    const int f = blockIdx.x * kThreads + threadIdx.x;
    if (f >= a.F) return;
    const int32_t* t = a.faces + 3 * (size_t)f;
    if (!face_ok(t, a.V)) { atomicAdd(a.bad, 1); return; }
    const int x = t[0], y = t[1], z = t[2];
    unite(a.parent, x, y);
    unite(a.parent, x, z);
}

__global__ void __launch_bounds__(kThreads) clean_label_kernel(CleanArgs a) {
    const int v = blockIdx.x * kThreads + threadIdx.x;
    if (v < a.V) a.label[v] = find_root(a.parent, v);
}

__global__ void __launch_bounds__(kThreads) clean_faces_kernel(CleanArgs a) {
    const int f = blockIdx.x * kThreads + threadIdx.x;
    int root = -1;
    if (f < a.F) {
        const int32_t* t = a.faces + 3 * (size_t)f;
        if (face_ok(t, a.V)) {
            root = a.label[t[0]];
            a.ref[t[0]] = 1; a.ref[t[1]] = 1; a.ref[t[2]] = 1;
        }
    }
    // one atomicAdd per root present in the warp: a large component's faces sit together
    const unsigned peers = __match_any_sync(0xffffffffu, root);
    if (root >= 0 && (threadIdx.x & 31) == __ffs(peers) - 1) atomicAdd(a.fcount + root, (uint32_t)__popc(peers));
}

__global__ void __launch_bounds__(kThreads) clean_boxes_kernel(CleanArgs a) {
    __shared__ uint32_t sbox[6];
    if (threadIdx.x < 6) sbox[threadIdx.x] = threadIdx.x < 3 ? kEmptyMin : kEmptyMax;
    __syncthreads();
    const int v = blockIdx.x * kThreads + threadIdx.x;
    const bool on = v < a.V && a.ref[v];
    const int root = on ? a.label[v] : -1;
    uint32_t lo[3], hi[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const float x = on ? a.vert[3 * (size_t)v + k] : 0.0f;
        const bool use = on && !isnan(x);
        lo[k] = use ? enc(x) : kEmptyMin;
        hi[k] = use ? enc(x) : kEmptyMax;
    }
    const unsigned peers = __match_any_sync(0xffffffffu, root);
    const bool leader = (threadIdx.x & 31) == __ffs(peers) - 1;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const uint32_t mn = __reduce_min_sync(peers, lo[k]), mx = __reduce_max_sync(peers, hi[k]);
        if (leader && root >= 0 && mn != kEmptyMin) {
            atomicMin(a.box + 6 * (size_t)root + k, mn);
            atomicMax(a.box + 6 * (size_t)root + 3 + k, mx);
        }
        const uint32_t wmn = __reduce_min_sync(0xffffffffu, lo[k]), wmx = __reduce_max_sync(0xffffffffu, hi[k]);
        if ((threadIdx.x & 31) == 0 && wmn != kEmptyMin) {
            atomicMin(sbox + k, wmn);
            atomicMax(sbox + 3 + k, wmx);
        }
    }
    __syncthreads();
    if (threadIdx.x < 3 && sbox[threadIdx.x] != kEmptyMin) {
        atomicMin(a.mesh_box + threadIdx.x, sbox[threadIdx.x]);
        atomicMax(a.mesh_box + 3 + threadIdx.x, sbox[3 + threadIdx.x]);
    }
}

// the box diagonal of include/b200gsr_mesh_clean.h: float64, each operation rounded on its own, no FMA
__device__ double diagonal(const uint32_t* b) {
    double d[3];
#pragma unroll
    for (int k = 0; k < 3; ++k)
        d[k] = b[k] == kEmptyMin ? 0.0 : __dsub_rn((double)dec(b[3 + k]), (double)dec(b[k]));
    return __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(d[0], d[0]), __dmul_rn(d[1], d[1])), __dmul_rn(d[2], d[2])));
}

__global__ void __launch_bounds__(kThreads) clean_decide_kernel(CleanArgs a) {
    const int v = blockIdx.x * kThreads + threadIdx.x;
    if (v >= a.V || !a.ref[v] || a.label[v] != v) return;      // roots of components with a face
    const uint32_t n = a.fcount[v];
    bool ok = n >= (uint32_t)a.min_faces;
    if (ok && a.min_diameter != 0.0)
        ok = diagonal(a.box + 6 * (size_t)v) >= __dmul_rn(a.min_diameter, diagonal(a.mesh_box));
    if (!ok) return;
    a.pass[v] = 1;
    if (a.keep_largest) atomicMax(a.best, (unsigned long long)n << 32 | (uint32_t)~(uint32_t)v);
}

__device__ __forceinline__ bool kept_root(const CleanArgs& a, int r) {
    return a.pass[r] && (!a.keep_largest || (uint32_t)r == ~(uint32_t)*a.best);
}

__global__ void __launch_bounds__(kThreads) clean_flags_kernel(CleanArgs a) {
    const int i = blockIdx.x * kThreads + threadIdx.x;
    if (i < a.V) a.vstart[i] = a.ref[i] && kept_root(a, a.label[i]);
    if (i < a.F) {
        const int32_t* t = a.faces + 3 * (size_t)i;
        a.fstart[i] = face_ok(t, a.V) && kept_root(a, a.label[t[0]]);
    }
}

__global__ void __launch_bounds__(kThreads) clean_emit_vertices_kernel(CleanArgs a, float* __restrict__ out,
                                                                       int32_t* __restrict__ kept, uint32_t V_out) {
    const int v = blockIdx.x * kThreads + threadIdx.x;
    if (v >= a.V || !a.ref[v] || !kept_root(a, a.label[v])) return;
    const uint32_t o = a.vstart[v];
    if (o >= V_out) return;
    const uint32_t* src = reinterpret_cast<const uint32_t*>(a.vert) + 3 * (size_t)v;   // the bits, NaN payloads too
    uint32_t* dst = reinterpret_cast<uint32_t*>(out) + 3 * (size_t)o;
    dst[0] = src[0]; dst[1] = src[1]; dst[2] = src[2];
    kept[o] = v;
}

__global__ void __launch_bounds__(kThreads) clean_emit_faces_kernel(CleanArgs a, int32_t* __restrict__ out,
                                                                    uint32_t F_out) {
    const int f = blockIdx.x * kThreads + threadIdx.x;
    if (f >= a.F) return;
    const int32_t* t = a.faces + 3 * (size_t)f;
    if (!face_ok(t, a.V) || !kept_root(a, a.label[t[0]])) return;
    const uint32_t o = a.fstart[f];
    if (o >= F_out) return;
    int32_t* d = out + 3 * (size_t)o;
    d[0] = (int32_t)a.vstart[t[0]]; d[1] = (int32_t)a.vstart[t[1]]; d[2] = (int32_t)a.vstart[t[2]];
}

size_t align256(size_t v) { return (v + 255) / 256 * 256; }

CleanArgs clean_args(const GsrMeshCleanPlan& p, const float* vert, const int32_t* faces, uint8_t* s) {
    CleanArgs a{};
    a.V = p.V; a.F = p.F;
    a.vert = vert;
    a.faces = faces;
    a.parent = reinterpret_cast<int32_t*>(s + p.off_parent);
    a.label = reinterpret_cast<int32_t*>(s + p.off_label);
    a.ref = s + p.off_ref;
    a.pass = s + p.off_pass;
    a.fcount = reinterpret_cast<uint32_t*>(s + p.off_fcount);
    a.box = reinterpret_cast<uint32_t*>(s + p.off_box);
    a.vstart = reinterpret_cast<uint32_t*>(s + p.off_vstart);
    a.fstart = reinterpret_cast<uint32_t*>(s + p.off_fstart);
    a.best = reinterpret_cast<unsigned long long*>(s + p.off_misc);
    a.mesh_box = reinterpret_cast<uint32_t*>(s + p.off_misc + 8);
    return a;
}

int blocks(int n) { return (n + kThreads - 1) / kThreads; }

// clean_init, clean_union and clean_label: the parents in the scratch, the labels and the bad count where `a` says
cudaError_t components(const CleanArgs& a, cudaStream_t s) {
    clean_init_kernel<<<blocks(a.V), kThreads, 0, s>>>(a);
    if (a.F) clean_union_kernel<<<blocks(a.F), kThreads, 0, s>>>(a);
    clean_label_kernel<<<blocks(a.V), kThreads, 0, s>>>(a);
    return cudaGetLastError();
}

}  // namespace

void gsr_mesh_clean_plan(int V, int F, GsrMeshCleanPlan* pl) {
    GsrMeshCleanPlan& p = *pl;
    p.V = V; p.F = F;
    const size_t v = (size_t)V, f = (size_t)F;
    p.off_parent = 0;
    p.off_label = p.off_parent + align256(4 * v);
    p.off_ref = p.off_label + align256(4 * v);
    p.off_pass = p.off_ref + align256(v);
    p.off_fcount = p.off_pass + align256(v);
    p.off_box = p.off_fcount + align256(4 * v);
    p.off_vstart = p.off_box + align256(24 * v);
    p.off_fstart = p.off_vstart + align256(4 * v);
    p.off_misc = p.off_fstart + align256(4 * f);
    p.off_bsums = p.off_misc + 256;
    const size_t n = v > f ? v : f;
    p.total = p.off_bsums + align256(((n + 4095) / 4096 + 1) * sizeof(uint32_t));
}

cudaError_t gsr_launch_mesh_components(const GsrMeshCleanPlan& p, const int32_t* faces, int32_t* labels, int32_t* bad,
                                       uint8_t* scratch, cudaStream_t s) {
    CleanArgs a = clean_args(p, nullptr, faces, scratch);
    a.label = labels;
    a.bad = bad;
    a.ref = nullptr;
    return components(a, s);
}

cudaError_t gsr_launch_mesh_clean_count(const GsrMeshCleanPlan& p, const float* vertices, const int32_t* faces,
                                        int min_faces, double min_diameter, bool keep_largest, int32_t* totals,
                                        uint8_t* scratch, cudaStream_t s) {
    CleanArgs a = clean_args(p, vertices, faces, scratch);
    a.bad = totals + 2;
    a.min_faces = min_faces;
    a.min_diameter = min_diameter;
    a.keep_largest = keep_largest;
    cudaError_t e = components(a, s);
    if (e != cudaSuccess) return e;
    if (a.F) clean_faces_kernel<<<blocks(a.F), kThreads, 0, s>>>(a);
    clean_boxes_kernel<<<blocks(a.V), kThreads, 0, s>>>(a);
    clean_decide_kernel<<<blocks(a.V), kThreads, 0, s>>>(a);
    clean_flags_kernel<<<blocks(a.V > a.F ? a.V : a.F), kThreads, 0, s>>>(a);
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    // the two scans run one after the other on the stream, so they share the block sums
    uint32_t* bsums = reinterpret_cast<uint32_t*>(scratch + p.off_bsums);
    gsr_scan_u32(a.V, a.vstart, a.vstart, bsums, reinterpret_cast<uint32_t*>(totals), s);
    if (a.F) gsr_scan_u32(a.F, a.fstart, a.fstart, bsums, reinterpret_cast<uint32_t*>(totals) + 1, s);
    else if ((e = cudaMemsetAsync(totals + 1, 0, sizeof(int32_t), s)) != cudaSuccess) return e;
    return cudaGetLastError();
}

cudaError_t gsr_launch_mesh_clean_emit(const GsrMeshCleanPlan& p, const float* vertices, const int32_t* faces,
                                       bool keep_largest, const uint8_t* scratch, float* out_vertices,
                                       int32_t* out_faces, int32_t* kept, int32_t V_out, int32_t F_out,
                                       cudaStream_t s) {
    // the emit kernels only read the scratch: the count's decisions, so the thresholds are not needed again
    CleanArgs a = clean_args(p, vertices, faces, const_cast<uint8_t*>(scratch));
    a.keep_largest = keep_largest;
    clean_emit_vertices_kernel<<<blocks(a.V), kThreads, 0, s>>>(a, out_vertices, kept, (uint32_t)V_out);
    if (a.F) clean_emit_faces_kernel<<<blocks(a.F), kThreads, 0, s>>>(a, out_faces, (uint32_t)F_out);
    return cudaGetLastError();
}
