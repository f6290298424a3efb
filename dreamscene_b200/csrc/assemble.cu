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
    constexpr bool FROZEN = false;
    constexpr uint32_t frozen = 0u;
#include "assemble_body.cuh"
}

// The backward with frozen groups (b200gsr_assemble_backward_frozen): assemble_kernel<true>'s statements for the
// trainable groups' rows; a frozen group's rows are skipped, and a block of frozen rows only returns.
__global__ void __launch_bounds__(kAsmBlock)
assemble_bwd_frozen_kernel(GroupTable tab, GroupGradTable gtab, int P, int M, int B, float c_shs, float c_scale,
                           const float* __restrict__ z_shs, const float* __restrict__ z_scales,
                           unsigned long long seed, float* __restrict__ means3D, float* __restrict__ opac,
                           float* __restrict__ scales, float* __restrict__ rots, float* __restrict__ shs,
                           uint32_t frozen) {
    constexpr bool BACKWARD = true, FROZEN = true;
#include "assemble_body.cuh"
}

}  // namespace

cudaError_t gsr_launch_assemble(bool backward, int num_groups, const b200gsr_group* groups,
                                const b200gsr_group_grad* grads, int M, int B, float c_shs, float c_scale,
                                const float* z_shs, const float* z_scales, unsigned long long seed,
                                float* means3D, float* opac, float* scales, float* rots, float* shs, cudaStream_t s,
                                uint32_t frozen) {
    GroupTable tab;
    GroupGradTable gtab;
    const int P = gsr_group_tables(num_groups, groups, backward ? grads : nullptr, tab, gtab);
    if (P == 0) return cudaSuccess;
    const int nblocks = (P + kAsmBlock - 1) / kAsmBlock;
    if (backward && frozen)
        assemble_bwd_frozen_kernel<<<nblocks, kAsmBlock, 0, s>>>(tab, gtab, P, M, B, c_shs, c_scale, z_shs, z_scales,
                                                                 seed, means3D, opac, scales, rots, shs, frozen);
    else if (backward)
        assemble_kernel<true><<<nblocks, kAsmBlock, 0, s>>>(tab, gtab, P, M, B, c_shs, c_scale, z_shs, z_scales, seed,
                                                            means3D, opac, scales, rots, shs);
    else
        assemble_kernel<false><<<nblocks, kAsmBlock, 0, s>>>(tab, gtab, P, M, B, c_shs, c_scale, z_shs, z_scales, seed,
                                                             means3D, opac, scales, rots, shs);
    return cudaGetLastError();
}
