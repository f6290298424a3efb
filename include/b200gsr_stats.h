/*
 * b200gsr_stats.h - scene-render backwards that also gather the densification statistics (additive to
 * b200gsr_frozen.h, same conventions and the same library, libb200gsr.so; ABI version unchanged).
 *
 * While it densifies, DreamScene follows every backward with the statistics of the step's last rendered view, per row
 * of each trained group whose radius in that view is positive:
 *
 *   xyz_gradient_accum += |d_means2D[view][row][0:2]|      (torch.norm of the screen-space gradient's x, y)
 *   denom              += 1
 *   max_radii2D         = max(max_radii2D, radii[view][row])
 *
 * These backwards add them inside the backward itself, in the same launch that computes the view's screen-space
 * gradient: each row is read and written by one thread, with the arithmetic of b200gsr_densify_stats (the norm is
 * bit for bit the one b200gsr_densify_stats computes from the stored d_means2D row).  The [B,P,3] d_means2D
 * array is then optional.
 *
 *   stats        : HOST array of num_groups records, or NULL (no group gathers).  A record whose pointers are all
 *                  NULL gathers nothing for its group.  xyz_gradient_accum and denom are both set or both NULL;
 *                  max_radii2D may be NULL when they are set (then it is not updated).  Each is a DEVICE float32 array
 *                  of the group's n rows ([n] or [n,1]), updated in place.  A frozen group's record must be empty: a
 *                  frozen row's screen-space gradient is zero, so it would still count in denom.
 *   stats_view   : the view whose launch gathers, in [-1, B); -1 = none.  By value (b200gsr_backward_scene_stats), or
 *                  a DEVICE int32 read by the kernels at every launch (b200gsr_backward_scene_dyn_stats), so that a
 *                  captured graph switches the view, or gathering off (-1), without a re-capture.  The device value
 *                  is trusted: a value outside [0, B) gathers nothing.  NULL is allowed when no group gathers.
 *   d_means2D    : as b200gsr_backward_scene_frozen, or NULL: then no per-view screen-space gradient is stored.
 *
 * Refused with B200GSR_ERR_BAD_ARG before any device work: a by-value stats_view outside [-1, B); a record with only
 * one of xyz_gradient_accum / denom, or with max_radii2D alone; a record with statistics on a frozen group; a NULL
 * device stats_view with a group that gathers.
 *
 * In every other respect exactly b200gsr_backward_scene_frozen / b200gsr_backward_scene_dyn_frozen (same validation,
 * layouts, flags, gradients and d_means2D rows; the `saved` buffer is left as they leave it).  A second backward over
 * the same `saved` adds the statistics a second time.
 */
#ifndef B200GSR_STATS_H
#define B200GSR_STATS_H

#include "b200gsr_frozen.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct b200gsr_group_stats {   /* per group; all NULL = this group gathers nothing */
    float* xyz_gradient_accum;         /* [n] or [n,1] float32 */
    float* denom;                      /* [n] or [n,1] float32 */
    float* max_radii2D;                /* [n] float32, may be NULL */
} b200gsr_group_stats;

int b200gsr_backward_scene_stats(int32_t B, const b200gsr_params* prm, int32_t num_groups, const b200gsr_group* groups,
                                 const b200gsr_group_grad* grads, const float* shs_noise, const float* scale_noise,
                                 uint64_t seed, const float* d_scales, const int32_t* radii,
                                 const float* out_depth_alpha, const float* dL_dcolor, const float* dL_ddepth_alpha,
                                 void* saved, size_t saved_bytes, uint64_t max_pairs, float* d_means2D,
                                 uint32_t flags, uint32_t frozen_groups, const b200gsr_group_stats* stats,
                                 int32_t stats_view, void* stream);
int b200gsr_backward_scene_dyn_stats(int32_t B, const b200gsr_params* prm, int32_t num_groups,
                                     const b200gsr_group* groups, const b200gsr_group_grad* grads,
                                     const b200gsr_step_view* views, const uint64_t* seed, const float* d_scales,
                                     const int32_t* radii, const float* out_depth_alpha, const float* dL_dcolor,
                                     const float* dL_ddepth_alpha, void* saved, size_t saved_bytes,
                                     uint64_t max_pairs, float* d_means2D, uint32_t flags, uint32_t frozen_groups,
                                     const b200gsr_group_stats* stats, const int32_t* stats_view, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B200GSR_STATS_H */
