/*
 * b200gsr_reserve.h - the replayed step's entry points over parameter groups with reserved rows (additive to
 * b200gsr_step.h, b200gsr_loss.h and b200gsr_stats.h; same conventions and the same library, libb200gsr.so; ABI
 * version unchanged).
 *
 * A reserved group's leaves, Adam moments and statistics are allocated once at a row capacity; densify, prune and
 * opacity reset rewrite a prefix of the same tensors, so the pointers and shapes a captured CUDA graph holds stay
 * valid.  Each group's record keeps its capacity in `n` (P is the sum of the capacities, as before); the number of
 * rows in use - its live count - is read from device memory by the kernels at every launch:
 *
 *   live : DEVICE int32 array [num_groups], live[g] in [0, groups[g].n] (a value outside is clamped to that range).
 *          Row l of group g is live iff l < live[g]; a plain group passes live[g] = n.
 *
 * A dead row (l >= live[g]) is treated as culled before any of its parameters are read, so it may hold anything,
 * NaN included: radius 0, no tile pairs, a zero out_scales row, zero leaf gradients and d_means2D row, no statistics.
 * The augmentation noise of a live row is keyed by the row the compact layout would give it, sum_{h<g} live[h] + l
 * (computed on the device), so that a render over reserved groups equals the render over their live prefixes packed
 * back to back, bit for bit.
 */
#ifndef B200GSR_RESERVE_H
#define B200GSR_RESERVE_H

#include "b200gsr_step.h"
#include "b200gsr_loss.h"
#include "b200gsr_stats.h"

#ifdef __cplusplus
extern "C" {
#endif

/* b200gsr_forward_scene_dyn plus `live`. */
int b200gsr_forward_scene_dyn_live(int32_t B, const b200gsr_params* prm, int32_t num_groups,
                                   const b200gsr_group* groups, const b200gsr_step_view* views, const uint64_t* seed,
                                   float* out_scales, float* out_color, float* out_depth_alpha, int32_t* radii,
                                   void* scratch, size_t scratch_bytes, void* saved, size_t saved_bytes,
                                   uint64_t max_pairs, uint32_t flags, uint32_t* host_notify, uint32_t notify_seq,
                                   const int32_t* live, void* stream);

/* b200gsr_backward_scene_dyn_stats plus `live` (frozen_groups = 0 and stats = NULL give the plain _dyn backward).
 * The backward of a forward_scene_dyn_live with the same `live` values. */
int b200gsr_backward_scene_dyn_live(int32_t B, const b200gsr_params* prm, int32_t num_groups,
                                    const b200gsr_group* groups, const b200gsr_group_grad* grads,
                                    const b200gsr_step_view* views, const uint64_t* seed, const float* d_scales,
                                    const int32_t* radii, const float* out_depth_alpha, const float* dL_dcolor,
                                    const float* dL_ddepth_alpha, void* saved, size_t saved_bytes,
                                    uint64_t max_pairs, float* d_means2D, uint32_t flags, uint32_t frozen_groups,
                                    const b200gsr_group_stats* stats, const int32_t* stats_view,
                                    const int32_t* live, void* stream);

/* b200gsr_scale_loss over the [B,P,3] augmented scales of a render over `groups` (P = sum of their n): the mean over
 * the live rows only, i.e. the divisor is B * sum(live) * 3, read on the device.  The live elements' gradient is the
 * compact layout's bit for bit; a dead element's is 0 (accumulate = 0) or left as it is (accumulate = 1).  scratch as
 * b200gsr_scale_loss_scratch_bytes(B * P). */
int b200gsr_scale_loss_live(int32_t B, int32_t num_groups, const b200gsr_group* groups, const int32_t* live,
                            const float* scales, const float* grad_out, float* loss_out, float* d_scales,
                            int32_t accumulate, void* scratch, size_t scratch_bytes, void* stream);

/* Per tensor of b200gsr_adam_step_dyn_live: its live element count is *rows * row_floats (rows: DEVICE int32, or NULL
 * = the whole tensor).  Elements past it are left untouched. */
typedef struct b200gsr_adam_live {
    const int32_t* rows;
    int32_t row_floats;
    int32_t reserved;
} b200gsr_adam_live;

/* b200gsr_adam_step_dyn plus a HOST array of n_tensors live records. */
int b200gsr_adam_step_dyn_live(int32_t n_tensors, const b200gsr_adam_tensor* tensors, const float* scalars,
                               const b200gsr_adam_live* live, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B200GSR_RESERVE_H */
