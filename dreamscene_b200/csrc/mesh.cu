// Marching cubes on a float32 volume (include/b200gsr_mesh.h): the cube table generated from the face rule at compile
// time, and two passes with no float atomics, so the output order is fixed and every call gives the same bits.
//
//   mesh_classify   per grid point: the crossing mask of its +x / +y / +z edges and its vertex count; per cell (by
//                   its corner 0): the case byte and its triangle count
//   gsr_scan_u32    exclusive scans of both counts (densify.cu); the sums are the totals V and F
//   mesh_vertices   per grid point: its vertices, in axis order, at its vertex offset
//   mesh_faces      per cell: its triangles in table order at its face offset, each corner the vertex offset of the
//                   edge's grid point plus the rank of the edge's axis among that point's crossing edges
//   mesh_attributes per grid point: its vertices' attributes, interpolated with the vertices' t, at the same offsets
//                   (include/b200gsr_mesh_colour.h)
//
// Built without fast-math: the interpolation is __fsub_rn / __fdiv_rn / __fadd_rn, one float32 rounding each.
#include "common.cuh"
#include "../../include/b200gsr_mesh.h"

#include <cstring>

namespace {

constexpr int kThreads = 256;
constexpr int kWidth = B200GSR_MESH_TABLE_WIDTH;

struct MeshTable {
    uint8_t count[256];
    int8_t edge[256][kWidth];
};

// edge e = 4 a + r: axis a, and r the rank of its corner b among the four corners with bit a clear
constexpr int edge_axis(int e) { return e >> 2; }
constexpr int edge_corner(int e) {
    const int a = e >> 2, r = e & 3;
    return (r & ((1 << a) - 1)) | ((r >> a) << (a + 1));
}
constexpr int edge_between(int c0, int c1) {       // the edge joining two corners that differ in one bit
    const int d = c0 ^ c1, a = d == 1 ? 0 : d == 2 ? 1 : 2, b = c0 < c1 ? c0 : c1;
    return 4 * a + ((b & ((1 << a) - 1)) | ((b >> (a + 1)) << a));
}

struct FaceWalks {
    int corner[6][4];     // counter-clockwise seen from outside the cube
    int edges[6];         // bit mask of the face's four edges
};

// face (axis n, side s): in-plane axes u = n + 1, v = n + 2 (mod 3), so e_u x e_v = e_n; the side-0 face looks down
// -e_n and walks the other way round
constexpr FaceWalks make_faces() {
    FaceWalks w{};
    const int up[4][2] = {{0, 0}, {1, 0}, {1, 1}, {0, 1}}, down[4][2] = {{0, 0}, {0, 1}, {1, 1}, {1, 0}};
    for (int n = 0; n < 3; ++n)
        for (int s = 0; s < 2; ++s) {
            const int f = 2 * n + s, u = (n + 1) % 3, v = (n + 2) % 3;
            for (int i = 0; i < 4; ++i) {
                const int du = s ? up[i][0] : down[i][0], dv = s ? up[i][1] : down[i][1];
                w.corner[f][i] = s << n | du << u | dv << v;
            }
            w.edges[f] = 0;
            for (int i = 0; i < 4; ++i) w.edges[f] |= 1 << edge_between(w.corner[f][i], w.corner[f][(i + 1) % 4]);
        }
    return w;
}

constexpr MeshTable make_table() {
    MeshTable t{};
    const FaceWalks fw = make_faces();
    for (int cs = 0; cs < 256; ++cs) {
        // the face rule: next[e] = the edge the segment from entry e runs to
        int next[12] = {-1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1};
        for (int f = 0; f < 6; ++f) {
            int in[4] = {}, cross[4] = {}, nc = 0;
            for (int i = 0; i < 4; ++i) in[i] = (cs >> fw.corner[f][i]) & 1;
            for (int i = 0; i < 4; ++i)
                if (in[i] != in[(i + 1) % 4]) cross[nc++] = i;
            for (int k = 0; k < nc; ++k) {
                const int i = cross[k], j = cross[(k + 1) % nc];
                if (!in[i])
                    next[edge_between(fw.corner[f][i], fw.corner[f][(i + 1) % 4])] =
                        edge_between(fw.corner[f][j], fw.corner[f][(j + 1) % 4]);
            }
        }
        // the loops, by their lowest edges; each fanned from its apex
        int seen = 0, ntri = 0;
        for (int e = 0; e < 12; ++e) {
            if (next[e] < 0 || (seen >> e & 1)) continue;
            int loop[12] = {}, m = 0, members = 0;
            for (int x = e; m == 0 || x != e; x = next[x]) { loop[m++] = x; members |= 1 << x; }
            seen |= members;
            int twice = 0;        // edges of the faces this loop crosses twice (all four of their edges in the loop)
            for (int f = 0; f < 6; ++f)
                if ((members & fw.edges[f]) == fw.edges[f]) twice |= fw.edges[f];
            int k0 = -1;          // the apex's place in the loop
            for (int k = 0; k < m; ++k)
                if (!(twice >> loop[k] & 1) && (k0 < 0 || loop[k] < loop[k0])) k0 = k;
            for (int i = 1; i + 1 < m; ++i, ++ntri) {
                t.edge[cs][3 * ntri] = (int8_t)loop[k0];
                t.edge[cs][3 * ntri + 1] = (int8_t)loop[(k0 + i) % m];
                t.edge[cs][3 * ntri + 2] = (int8_t)loop[(k0 + i + 1) % m];
            }
        }
        t.count[cs] = (uint8_t)ntri;
        for (int k = 3 * ntri; k < kWidth; ++k) t.edge[cs][k] = -1;
    }
    return t;
}

constexpr MeshTable kTable = make_table();
static_assert(kTable.count[0] == 0 && kTable.count[255] == 0 && kTable.count[1] == 1, "table generator");
__device__ const MeshTable d_table = kTable;

struct MeshArgs {
    int X, Y, Z, N;           // N = X Y Z points
    bool cells;               // every dimension >= 2
    float iso;
    const float* vol;
    uint8_t* emask;           // [N]: crossing +x / +y / +z edges (bits 0..2)
    uint8_t* cube;            // [N]: case of the cell at corner 0 = this point, 0 for points that start no cell
    uint32_t* vstart;         // [N]: vertex counts, then (scanned) offsets
    uint32_t* fstart;         // [N]: triangle counts, then (scanned) offsets
};

__global__ void __launch_bounds__(kThreads) mesh_classify_kernel(MeshArgs a) {
    const int p = blockIdx.x * kThreads + threadIdx.x;
    if (p >= a.N) return;
    const int YZ = a.Y * a.Z, i = p / YZ, j = (p / a.Z) % a.Y, k = p % a.Z;
    const bool nx = a.cells && i + 1 < a.X, ny = a.cells && j + 1 < a.Y, nz = a.cells && k + 1 < a.Z;
    // inside bits of the cell's corners that exist
    uint32_t in = 0u;
#pragma unroll
    for (int c = 0; c < 8; ++c) {
        const bool ok = (!(c & 1) || nx) && (!(c & 2) || ny) && (!(c & 4) || nz);
        if (ok && a.vol[p + (c & 1) * YZ + ((c >> 1) & 1) * a.Z + ((c >> 2) & 1)] > a.iso) in |= 1u << c;
    }
    const uint32_t m = (nx && ((in ^ (in >> 1)) & 1u) ? 1u : 0u) | (ny && ((in ^ (in >> 2)) & 1u) ? 2u : 0u) |
                       (nz && ((in ^ (in >> 4)) & 1u) ? 4u : 0u);
    const uint32_t cs = nx && ny && nz ? in : 0u;
    a.emask[p] = (uint8_t)m;
    a.cube[p] = (uint8_t)cs;
    a.vstart[p] = __popc(m);
    a.fstart[p] = d_table.count[cs];
}

__global__ void __launch_bounds__(kThreads) mesh_vertices_kernel(MeshArgs a, float* __restrict__ out, uint32_t V) {
    const int p = blockIdx.x * kThreads + threadIdx.x;
    if (p >= a.N) return;
    const uint32_t m = a.emask[p];
    if (!m) return;
    const int YZ = a.Y * a.Z, i = p / YZ, j = (p / a.Z) % a.Y, k = p % a.Z;
    const int step[3] = {YZ, a.Z, 1};
    const float f0 = a.vol[p], d0 = __fsub_rn(a.iso, f0);
    uint32_t v = a.vstart[p];
#pragma unroll
    for (int ax = 0; ax < 3; ++ax) {
        if (!(m >> ax & 1u)) continue;
        const float t = __fdiv_rn(d0, __fsub_rn(a.vol[p + step[ax]], f0));
        float xyz[3] = {(float)i, (float)j, (float)k};
        xyz[ax] = __fadd_rn(xyz[ax], t);
        if (v < V) {
            float* o = out + 3 * (size_t)v;
            o[0] = xyz[0]; o[1] = xyz[1]; o[2] = xyz[2];
        }
        ++v;
    }
}

__global__ void __launch_bounds__(kThreads) mesh_faces_kernel(MeshArgs a, int32_t* __restrict__ out, uint32_t F) {
    const int p = blockIdx.x * kThreads + threadIdx.x;
    if (p >= a.N) return;
    const uint32_t cs = a.cube[p], n = d_table.count[cs];
    if (!n) return;
    const int YZ = a.Y * a.Z;
    const uint32_t f = a.fstart[p];
    for (uint32_t t = 0; t < n; ++t) {
        if (f + t >= F) break;
        int32_t* o = out + 3 * (size_t)(f + t);
#pragma unroll
        for (int s = 0; s < 3; ++s) {
            const int e = d_table.edge[cs][3 * t + s], b = edge_corner(e);
            const int q = p + (b & 1) * YZ + ((b >> 1) & 1) * a.Z + ((b >> 2) & 1);
            o[s] = (int32_t)(a.vstart[q] + __popc(a.emask[q] & ((1u << edge_axis(e)) - 1u)));
        }
    }
}

// a + t (b - a) per channel, three roundings; t is mesh_vertices_kernel's, so each attribute sits where its vertex does
__global__ void __launch_bounds__(kThreads) mesh_attributes_kernel(MeshArgs a, const float* __restrict__ attr,
                                                                   float* __restrict__ out, uint32_t V) {
    const int p = blockIdx.x * kThreads + threadIdx.x;
    if (p >= a.N) return;
    const uint32_t m = a.emask[p];
    if (!m) return;
    const int step[3] = {a.Y * a.Z, a.Z, 1};
    const float f0 = a.vol[p], d0 = __fsub_rn(a.iso, f0);
    const float* a0 = attr + 3 * (size_t)p;
    uint32_t v = a.vstart[p];
#pragma unroll
    for (int ax = 0; ax < 3; ++ax) {
        if (!(m >> ax & 1u)) continue;
        const float t = __fdiv_rn(d0, __fsub_rn(a.vol[p + step[ax]], f0));
        const float* a1 = a0 + 3 * (size_t)step[ax];
        if (v < V) {
            float* o = out + 3 * (size_t)v;
#pragma unroll
            for (int c = 0; c < 3; ++c) o[c] = __fadd_rn(a0[c], __fmul_rn(t, __fsub_rn(a1[c], a0[c])));
        }
        ++v;
    }
}

size_t align256(size_t v) { return (v + 255) / 256 * 256; }

MeshArgs mesh_args(const GsrMeshPlan& p, const float* vol, float iso, uint8_t* scratch) {
    MeshArgs a;
    a.X = p.X; a.Y = p.Y; a.Z = p.Z; a.N = (int)p.points;
    a.cells = p.cells > 0;
    a.iso = iso;
    a.vol = vol;
    a.emask = scratch + p.off_emask;
    a.cube = scratch + p.off_cube;
    a.vstart = reinterpret_cast<uint32_t*>(scratch + p.off_vstart);
    a.fstart = reinterpret_cast<uint32_t*>(scratch + p.off_fstart);
    return a;
}

}  // namespace

void gsr_mesh_table(uint8_t* counts, int8_t* edges) {
    std::memcpy(counts, kTable.count, sizeof(kTable.count));
    std::memcpy(edges, kTable.edge, sizeof(kTable.edge));
}

void gsr_mesh_plan(int X, int Y, int Z, GsrMeshPlan* pl) {
    GsrMeshPlan& p = *pl;
    p.X = X; p.Y = Y; p.Z = Z;
    p.points = (long long)X * Y * Z;
    p.cells = X < 2 || Y < 2 || Z < 2 ? 0 : (long long)(X - 1) * (Y - 1) * (Z - 1);
    const size_t n = (size_t)p.points;
    p.off_emask = 0;
    p.off_cube = p.off_emask + align256(n);
    p.off_vstart = p.off_cube + align256(n);
    p.off_fstart = p.off_vstart + align256(n * sizeof(uint32_t));
    p.off_bsums = p.off_fstart + align256(n * sizeof(uint32_t));
    p.total = p.off_bsums + align256(((n + 4095) / 4096 + 1) * sizeof(uint32_t));
}

cudaError_t gsr_launch_mesh_count(const GsrMeshPlan& p, const float* vol, float iso, int32_t* totals, uint8_t* scratch,
                                  cudaStream_t s) {
    MeshArgs a = mesh_args(p, vol, iso, scratch);
    mesh_classify_kernel<<<(a.N + kThreads - 1) / kThreads, kThreads, 0, s>>>(a);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    // the two scans run one after the other on the stream, so they share the block sums
    uint32_t* bsums = reinterpret_cast<uint32_t*>(scratch + p.off_bsums);
    gsr_scan_u32(a.N, a.vstart, a.vstart, bsums, reinterpret_cast<uint32_t*>(totals), s);
    gsr_scan_u32(a.N, a.fstart, a.fstart, bsums, reinterpret_cast<uint32_t*>(totals) + 1, s);
    return cudaGetLastError();
}

cudaError_t gsr_launch_mesh_emit(const GsrMeshPlan& p, const float* vol, float iso, const uint8_t* scratch,
                                 float* vertices, int32_t V, int32_t* faces, int32_t F, cudaStream_t s) {
    // the emit kernels only read the scratch
    MeshArgs a = mesh_args(p, vol, iso, const_cast<uint8_t*>(scratch));
    const int blocks = (a.N + kThreads - 1) / kThreads;
    mesh_vertices_kernel<<<blocks, kThreads, 0, s>>>(a, vertices, (uint32_t)V);
    mesh_faces_kernel<<<blocks, kThreads, 0, s>>>(a, faces, (uint32_t)F);
    return cudaGetLastError();
}

cudaError_t gsr_launch_mesh_attributes(const GsrMeshPlan& p, const float* vol, float iso, const uint8_t* scratch,
                                       const float* attributes, float* out, int32_t V, cudaStream_t s) {
    MeshArgs a = mesh_args(p, vol, iso, const_cast<uint8_t*>(scratch));
    mesh_attributes_kernel<<<(a.N + kThreads - 1) / kThreads, kThreads, 0, s>>>(a, attributes, out, (uint32_t)V);
    return cudaGetLastError();
}
