// Scene assembly (SURVEY.md 8 f2): the per-render glue DreamScene runs in PyTorch before every
// rasterizer call, as ONE forward and ONE backward kernel.
//
// Reference (/root/reference/scene_gaussian.py:753-857, gs_renderer.py:464-488): for every visible
// group (environment, floor, object instances) take the raw leaf parameters, apply the activations
//     opacity = sigmoid(_opacity)   scales = exp(_scaling)   rotations = normalize(_rotation)
//     shs = cat(_features_dc, _features_rest, dim=1)         means3D = _xyz
// torch.cat the groups, then augment (scene_gaussian.py:848-856)
//     shs    = shs + randn_like(shs) * (0.2**0.5 * shs)
//     scales = clamp(scales + randn_like(scales) * (0.2**0.5 * scales / 4), 0)
// That is ~6 activation kernels + 5 cats per group list + 6 augmentation kernels per view, each a
// full pass over 2.6M-row tensors, and the same again (plus autograd's cat/split bookkeeping) in the
// backward.  Here: one pass that reads every raw parameter once and writes the five packed,
// rasterizer-ready arrays; one pass back that turns their gradients into the per-group leaf gradients.
//
// Numerics: every expression is evaluated with the reference's operation order and individually
// rounded fp32 ops (expf, IEEE division), so with the noise tensors passed in the outputs are
// bit-identical to the PyTorch expressions except `normalize` (sum-of-squares order, <= 1 ulp).
// Noise: either the caller's standard-normal tensors (z_shs[P,M,3], z_scales[P,3]: generate them with
// torch.randn in the reference's order and the random stream matches the reference's), or - z == NULL
// and seed given - a counter-based Philox4x32-10 generator evaluated in the kernel (no noise tensor
// is ever written or read; the backward regenerates the same numbers from (seed, element index)).
#include "scene_math.cuh"

namespace {

constexpr int kAsmBlock = 128;

// =============================================================================================
// forward: block = 128 packed rows; phase A one thread per Gaussian (11 floats), phase B the
// block's SH rows as a flat span of floats (coalesced stores; float4 when 3M % 4 == 0)
// =============================================================================================
// B = number of views: `scales` is [B][P,3] and `shs` [B][P,M,3] (one independently augmented copy per view, the
// raw parameters are read ONCE), means3D / opac / rots are written once; in the backward the per-view gradients of
// scales / shs are summed over the views in registers and every leaf gradient is written once.  View v uses the
// noise rows z[v] (caller's draws) or the Philox streams 2v+1 / 2v+2.
template <bool BACKWARD>
__global__ void __launch_bounds__(kAsmBlock)
assemble_kernel(GroupTable tab, GroupGradTable gtab, int P, int M, int B, float c_shs, float c_scale,
                const float* __restrict__ z_shs, const float* __restrict__ z_scales, unsigned long long seed,
                // forward outputs / backward incoming gradients (packed)
                float* __restrict__ means3D, float* __restrict__ opac, float* __restrict__ scales,
                float* __restrict__ rots, float* __restrict__ shs) {
    const int r0 = blockIdx.x * kAsmBlock;
    const int i = r0 + threadIdx.x;
    // ---- phase A ---------------------------------------------------------------------------
    if (i < P) {
        const int g = find_group(tab, i);
        const int l = i - tab.start[g];
        const float sx = tab.scaling[g][3 * (size_t)l], sy = tab.scaling[g][3 * (size_t)l + 1], sz = tab.scaling[g][3 * (size_t)l + 2];
        const float4 q = *reinterpret_cast<const float4*>(tab.rotation[g] + 4 * (size_t)l);
        const float o = tab.opacity[g][l];
        const float e[3] = {act_scale(sx), act_scale(sy), act_scale(sz)};
        const float sig = act_opacity(o);
        const float nrm = quat_norm(q);
        float dsum[3] = {0.f, 0.f, 0.f};
        for (int v = 0; v < B; ++v) {
            float zs[3] = {0.f, 0.f, 0.f};
            if (c_scale != 0.0f) {
                if (z_scales != nullptr) {
                    const float* zr = z_scales + ((size_t)v * P + i) * 3;
                    zs[0] = zr[0]; zs[1] = zr[1]; zs[2] = zr[2];
                } else {
                    const float4 n = normal4(seed, kStreamScales + 2u * (uint32_t)v, (unsigned long long)i);
                    zs[0] = n.x; zs[1] = n.y; zs[2] = n.z;
                }
            }
            float* sv = scales + ((size_t)v * P + i) * 3;
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                if (!BACKWARD) {
                    sv[k] = (c_scale != 0.0f) ? aug_scale(e[k], zs[k], c_scale) : e[k];
                } else {
                    float d = sv[k];
                    if (c_scale != 0.0f) d = aug_scale_grad(d, e[k], zs[k], c_scale);
                    dsum[k] += d;
                }
            }
        }
        if (!BACKWARD) {
            means3D[3 * (size_t)i] = tab.xyz[g][3 * (size_t)l];
            means3D[3 * (size_t)i + 1] = tab.xyz[g][3 * (size_t)l + 1];
            means3D[3 * (size_t)i + 2] = tab.xyz[g][3 * (size_t)l + 2];
            opac[i] = sig;
            *reinterpret_cast<float4*>(rots + 4 * (size_t)i) = quat_normalize(q, nrm);
        } else {
            // incoming gradients live in the packed arrays; outputs are the per-group leaf gradients
            gtab.xyz[g][3 * (size_t)l] = means3D[3 * (size_t)i];
            gtab.xyz[g][3 * (size_t)l + 1] = means3D[3 * (size_t)i + 1];
            gtab.xyz[g][3 * (size_t)l + 2] = means3D[3 * (size_t)i + 2];
            gtab.opacity[g][l] = opac[i] * sig * (1.0f - sig);
#pragma unroll
            for (int k = 0; k < 3; ++k) gtab.scaling[g][3 * (size_t)l + k] = dsum[k] * e[k];
            const float4 gq = *reinterpret_cast<const float4*>(rots + 4 * (size_t)i);
            *reinterpret_cast<float4*>(gtab.rotation[g] + 4 * (size_t)l) = quat_normalize_grad(q, nrm, gq);
        }
    }
    // ---- phase B: SH rows of the block as a flat span ----------------------------------------
    const int rows = min(kAsmBlock, P - r0);
    if (rows <= 0) return;
    const int row_f = 3 * M;
    const size_t base = (size_t)r0 * row_f;          // first float of the block's span in one view's packed array
    const size_t view_f = (size_t)P * row_f;         // floats per view
    const int total = rows * row_f;
    const bool vec = (row_f & 3) == 0;
    const int step = vec ? 4 : 1;
    for (int f = threadIdx.x * step; f < total; f += kAsmBlock * step) {
        const int row = f / row_f, col = f - row * row_f;       // vec: all 4 elements share the row
        const int gi = r0 + row;
        const int g = find_group(tab, gi);
        const size_t l = (size_t)(gi - tab.start[g]);
        float raw[4] = {0.f, 0.f, 0.f, 0.f}, dsum[4] = {0.f, 0.f, 0.f, 0.f};
        if (!BACKWARD) {
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                if (k >= step) break;
                const int c = col + k;
                raw[k] = (c < 3) ? tab.f_dc[g][3 * l + c] : tab.f_rest[g][(size_t)(row_f - 3) * l + (c - 3)];
            }
        }
        for (int v = 0; v < B; ++v) {
            float z[4] = {0.f, 0.f, 0.f, 0.f};
            const size_t e0 = base + f;                          // element index inside the view
            if (c_shs != 0.0f) {
                if (z_shs != nullptr) {
#pragma unroll
                    for (int k = 0; k < 4; ++k) if (k < step) z[k] = z_shs[(size_t)v * view_f + e0 + k];
                } else {
                    const float4 n = normal4(seed, kStreamShs + 2u * (uint32_t)v, (unsigned long long)(e0 >> 2));
                    if (vec) { z[0] = n.x; z[1] = n.y; z[2] = n.z; z[3] = n.w; }
                    else z[0] = (e0 & 3) == 0 ? n.x : (e0 & 3) == 1 ? n.y : (e0 & 3) == 2 ? n.z : n.w;
                }
            }
            float* sv = shs + (size_t)v * view_f + e0;
            if (!BACKWARD) {
                float out[4];
#pragma unroll
                for (int k = 0; k < 4; ++k) out[k] = (c_shs != 0.0f) ? aug(raw[k], z[k], c_shs, 1.0f) : raw[k];
                if (vec) *reinterpret_cast<float4*>(sv) = make_float4(out[0], out[1], out[2], out[3]);
                else sv[0] = out[0];
            } else {
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    if (k >= step) break;
                    float d = sv[k];
                    if (c_shs != 0.0f) d *= (1.0f + z[k] * c_shs);           // d(v + z*(c*v))/dv
                    dsum[k] += d;
                }
            }
        }
        if (BACKWARD) {
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                if (k >= step) break;
                const int c = col + k;
                if (c < 3) gtab.f_dc[g][3 * l + c] = dsum[k];
                else gtab.f_rest[g][(size_t)(row_f - 3) * l + (c - 3)] = dsum[k];
            }
        }
    }
}

}  // namespace

cudaError_t gsr_launch_assemble(bool backward, int num_groups, const b200gsr_group* groups,
                                const b200gsr_group_grad* grads, int M, int B, float c_shs, float c_scale,
                                const float* z_shs, const float* z_scales, unsigned long long seed,
                                float* means3D, float* opac, float* scales, float* rots, float* shs, cudaStream_t s) {
    GroupTable tab;
    GroupGradTable gtab;
    const int P = gsr_group_tables(num_groups, groups, backward ? grads : nullptr, tab, gtab);
    if (P == 0) return cudaSuccess;
    const int nblocks = (P + kAsmBlock - 1) / kAsmBlock;
    if (backward)
        assemble_kernel<true><<<nblocks, kAsmBlock, 0, s>>>(tab, gtab, P, M, B, c_shs, c_scale, z_shs, z_scales, seed,
                                                            means3D, opac, scales, rots, shs);
    else
        assemble_kernel<false><<<nblocks, kAsmBlock, 0, s>>>(tab, gtab, P, M, B, c_shs, c_scale, z_shs, z_scales, seed,
                                                             means3D, opac, scales, rots, shs);
    return cudaGetLastError();
}
