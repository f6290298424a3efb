/*
 * b200gsr_scene.h - scene renders: the views of one training step rendered straight from the raw parameter groups
 * (additive to b200gsr.h, same conventions and the same library, libb200gsr.so; ABI version unchanged).
 *
 * DreamScene's scene_render / object_render (scene_gaussian.py:673-893) activate and augment the raw leaves of every
 * group, concatenate them and rasterize.  b200gsr_assemble_forward + b200gsr_forward_views do that in two steps
 * that meet through B augmented copies of shs [B,P,M,3] and scales [B,P,3] in device memory (and their gradients
 * on the way back).  These entry points do it in one: project_sh reads the raw leaves, applies the activations and
 * the view's augmentation itself, and project_bwd chains each view's gradients straight to the leaf gradients.
 *
 *   groups / grads : HOST arrays of num_groups (<= B200GSR_MAX_GROUPS) b200gsr_group / b200gsr_group_grad records
 *                    as for b200gsr_assemble_forward / _backward; the packed row of group g's row l is
 *                    sum_{h<g} n_h + l and P = sum n.  rotation rows must be 16-byte aligned.
 *   prm[B]         : as b200gsr_forward_views (bg one contiguous [B,3] device array; cameras, sh_degree and
 *                    scale_modifier may differ per view), with P = sum n and M = SH coefficients per channel of every
 *                    group.  score_flag must be 0 (B200GSR_ERR_UNSUPPORTED otherwise).
 *   shs_noise[B], scale_noise[B] : HOST arrays, the per-view augmentation coefficients (0 = that augmentation is
 *                    off in that view; DreamScene's value is 0.2**0.5).
 *   seed           : the in-kernel Philox4x32-10 noise of b200gsr_assemble_forward with z == NULL.  View v draws the
 *                    SH noise from stream 2v+1 and the scale noise from stream 2v+2, with the same counters, so the
 *                    values the rasterizer sees are bit for bit those of b200gsr_assemble_forward(num_views = B,
 *                    seed) followed by b200gsr_forward_views on view v's slices.
 *
 * Forward: outputs, scratch, saved, max_pairs, flags (B200GSR_FWD_NO_BACKWARD, B200GSR_FWD_DETERMINISTIC),
 * host_notify and the pair-capacity protocol are those of b200gsr_forward_views (layouts for (B*P, Hs, W)).
 * out_scales: NULL, or [B,P,3] receiving every row's augmented scales per view (culled rows included).  The
 * profiling store records the call like b200gsr_forward.
 *
 * Backward: radii / out_depth_alpha / saved of the forward and the incoming stacked image gradients as for
 * b200gsr_backward_views; the same groups, noise coefficients and seed as the forward.  d_scales: NULL, or the
 * incoming gradient [B,P,3] of out_scales.  Outputs: grads (every row of every group fully overwritten, zeros where
 * no view contributes) and d_means2D [B,P,3] (per view, as b200gsr_backward_views).  The views run in order (view 0
 * writes, later views add into the rows they touched), so with flags = B200GSR_BWD_DETERMINISTIC the leaf
 * gradients are bitwise reproducible.  The profiling store records it like b200gsr_backward.
 */
#ifndef B200GSR_SCENE_H
#define B200GSR_SCENE_H

#include "b200gsr.h"

#ifdef __cplusplus
extern "C" {
#endif

int b200gsr_forward_scene(int32_t B, const b200gsr_params* prm, int32_t num_groups, const b200gsr_group* groups,
                          const float* shs_noise, const float* scale_noise, uint64_t seed, float* out_scales,
                          float* out_color, float* out_depth_alpha, int32_t* radii, void* scratch, size_t scratch_bytes,
                          void* saved, size_t saved_bytes, uint64_t max_pairs, uint32_t flags, uint32_t* host_notify,
                          uint32_t notify_seq, void* stream);
int b200gsr_backward_scene(int32_t B, const b200gsr_params* prm, int32_t num_groups, const b200gsr_group* groups,
                           const b200gsr_group_grad* grads, const float* shs_noise, const float* scale_noise,
                           uint64_t seed, const float* d_scales, const int32_t* radii, const float* out_depth_alpha,
                           const float* dL_dcolor, const float* dL_ddepth_alpha, void* saved, size_t saved_bytes,
                           uint64_t max_pairs, float* d_means2D, uint32_t flags, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B200GSR_SCENE_H */
