// Device math shared by the scene assembly (assemble.cu) and the raw-parameter modes of project_sh / project_bwd
// (project.cu): the group table, the activations of the raw leaves and the in-kernel augmentation noise.
//
// Both kernels evaluate these with the same statements, which is what makes a render from the raw leaves
// (b200gsr_forward_scene) bit for bit the render of the assembled arrays: every value the rasterizer sees -
// sigmoid(_opacity), the augmented exp(_scaling), normalize(_rotation) and the augmented SH coefficients - is
// produced by one of the helpers below from the same inputs.
#pragma once
#include "common.cuh"
#include <cstring>

namespace {

constexpr int kMaxGroups = B200GSR_MAX_GROUPS;

struct GroupTable {
    const float* xyz[kMaxGroups];
    const float* opacity[kMaxGroups];
    const float* scaling[kMaxGroups];
    const float* rotation[kMaxGroups];
    const float* f_dc[kMaxGroups];
    const float* f_rest[kMaxGroups];
    int start[kMaxGroups + 1];     // first packed row of group g; start[num] = P
    int num;
};
struct GroupGradTable {
    float* xyz[kMaxGroups];
    float* opacity[kMaxGroups];
    float* scaling[kMaxGroups];
    float* rotation[kMaxGroups];
    float* f_dc[kMaxGroups];
    float* f_rest[kMaxGroups];
};

// The tables of `num_groups` host records (grads may be null) -> P, the number of packed rows.
inline int gsr_group_tables(int num_groups, const b200gsr_group* groups, const b200gsr_group_grad* grads,
                            GroupTable& tab, GroupGradTable& gtab) {
    memset(&tab, 0, sizeof(tab));
    memset(&gtab, 0, sizeof(gtab));
    int P = 0;
    for (int g = 0; g < num_groups; ++g) {
        tab.xyz[g] = groups[g].xyz; tab.opacity[g] = groups[g].opacity; tab.scaling[g] = groups[g].scaling;
        tab.rotation[g] = groups[g].rotation; tab.f_dc[g] = groups[g].f_dc; tab.f_rest[g] = groups[g].f_rest;
        tab.start[g] = P;
        P += groups[g].n;
        if (grads) {
            gtab.xyz[g] = grads[g].xyz; gtab.opacity[g] = grads[g].opacity; gtab.scaling[g] = grads[g].scaling;
            gtab.rotation[g] = grads[g].rotation; gtab.f_dc[g] = grads[g].f_dc; gtab.f_rest[g] = grads[g].f_rest;
        }
    }
    tab.start[num_groups] = P;
    tab.num = num_groups;
    return P;
}

__device__ __forceinline__ int find_group(const GroupTable& t, int row) {
    int g = 0;
#pragma unroll 1
    while (g + 1 < t.num && row >= t.start[g + 1]) ++g;
    return g;
}

// ---- Philox4x32-10 (Salmon et al. 2011), counter = (lo, hi, stream, 0), key = seed ------------
__device__ __forceinline__ uint4 philox4x32_10(uint4 ctr, uint2 key) {
    constexpr uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        const uint32_t hi0 = __umulhi(M0, ctr.x), lo0 = M0 * ctr.x;
        const uint32_t hi1 = __umulhi(M1, ctr.z), lo1 = M1 * ctr.z;
        ctr = make_uint4(hi1 ^ ctr.y ^ key.x, lo1, hi0 ^ ctr.w ^ key.y, lo0);
        key.x += W0; key.y += W1;
    }
    return ctr;
}
// four standard normals for quad index q of stream s (Box-Muller on the four 32-bit outputs)
__device__ __forceinline__ float4 normal4(unsigned long long seed, uint32_t stream, unsigned long long q) {
    const uint4 r = philox4x32_10(make_uint4((uint32_t)q, (uint32_t)(q >> 32), stream, 0u),
                                  make_uint2((uint32_t)seed, (uint32_t)(seed >> 32)));
    const float u0 = ((float)r.x + 0.5f) * 2.3283064365386963e-10f;   // (0, 1)
    const float u1 = ((float)r.y + 0.5f) * 2.3283064365386963e-10f;
    const float u2 = ((float)r.z + 0.5f) * 2.3283064365386963e-10f;
    const float u3 = ((float)r.w + 0.5f) * 2.3283064365386963e-10f;
    const float ra = sqrtf(-2.0f * __logf(u0)), rb = sqrtf(-2.0f * __logf(u2));
    float s0, c0, s1, c1;
    __sincosf(6.283185307179586f * u1, &s0, &c0);
    __sincosf(6.283185307179586f * u3, &s1, &c1);
    return make_float4(ra * c0, ra * s0, rb * c1, rb * s1);
}
// Streams of view v: SH noise 2v+1, scale noise 2v+2.  Counters: the packed row (scales) and the flat element index
// inside the view's packed [P, M, 3] array (SH), four elements per counter (element e uses component e & 3 of
// quad e >> 2).
enum { kStreamShs = 1u, kStreamScales = 2u };    // + 2 * view

// noise factor helpers: value v, standard normal z, coefficient c (0.2**0.5), divisor d (1 or 4):
// reference order  v + z * ((c * v) / d)
__device__ __forceinline__ float aug(float v, float z, float c, float d) {
    return __fadd_rn(v, __fmul_rn(z, __fdiv_rn(__fmul_rn(c, v), d)));
}
// augmented scale: clamp(e + z * ((c * e) / 4), 0)
__device__ __forceinline__ float aug_scale(float e, float z, float c) { return fmaxf(aug(e, z, c, 4.0f), 0.0f); }
// its derivative applied to d: 1 + z*c/4 where the clamp is inactive
__device__ __forceinline__ float aug_scale_grad(float d, float e, float z, float c) {
    return (aug(e, z, c, 4.0f) > 0.0f) ? d * (1.0f + z * (c * 0.25f)) : 0.0f;
}

// ---- activations (gs_renderer.py:464-488): individually rounded, in the reference's order --------------------
__device__ __forceinline__ float act_scale(float s) { return expf(s); }
__device__ __forceinline__ float act_opacity(float o) { return __fdiv_rn(1.0f, __fadd_rn(1.0f, expf(-o))); }
__device__ __forceinline__ float quat_norm(float4 q) {
    return fmaxf(sqrtf(__fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(q.x, q.x), __fmul_rn(q.y, q.y)), __fmul_rn(q.z, q.z)), __fmul_rn(q.w, q.w))), 1e-12f);
}
__device__ __forceinline__ float4 quat_normalize(float4 q, float nrm) {
    return make_float4(__fdiv_rn(q.x, nrm), __fdiv_rn(q.y, nrm), __fdiv_rn(q.z, nrm), __fdiv_rn(q.w, nrm));
}
// d normalize: (g - u (u.g)) / |q|   (the eps clamp is inactive for any usable quaternion)
__device__ __forceinline__ float4 quat_normalize_grad(float4 q, float nrm, float4 gq) {
    const float inv = 1.0f / nrm;
    const float4 u = make_float4(q.x * inv, q.y * inv, q.z * inv, q.w * inv);
    const float dot = u.x * gq.x + u.y * gq.y + u.z * gq.z + u.w * gq.w;
    return make_float4((gq.x - u.x * dot) * inv, (gq.y - u.y * dot) * inv, (gq.z - u.z * dot) * inv, (gq.w - u.w * dot) * inv);
}

}  // namespace
