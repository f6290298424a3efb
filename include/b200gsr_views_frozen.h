/*
 * b200gsr_views_frozen.h - frozen rows on the two-step scene route, b200gsr_assemble_forward + b200gsr_forward_views
 * (additive to b200gsr.h and b200gsr_frozen.h, same conventions and the same library, libb200gsr.so; ABI version
 * unchanged).
 *
 * b200gsr_frozen.h freezes parameter groups of the one-call scene render.  These two entry points do the same for the
 * route that packs the groups first (b200gsr_assemble_forward, whose noise may be the caller's own draws) and then
 * rasterizes the packed arrays (b200gsr_forward_views): the frozen rows are still rendered, and their entries still
 * take part in the compositing recurrence behind which the trainable ones sit, but no gradient of theirs is
 * computed, accumulated or written.
 *
 * b200gsr_backward_views_frozen: b200gsr_backward_views_ex plus
 *   frozen     : HOST array of num_frozen row ranges [lo, lo + len) over the P rows of one view (the same rows in
 *                every view).  Sorted, non-overlapping, non-empty and inside [0, P); ranges that touch are merged,
 *                and at most B200GSR_MAX_FROZEN_RANGES may remain.  Anything else is refused (B200GSR_ERR_BAD_ARG)
 *                before any device work.  num_frozen = 0 is b200gsr_backward_views_ex (frozen may then be NULL).
 *   Every output row is still written: a frozen row's gradient rows and d_means2D row are zeros (added to the
 *   output where `accumulate` says so).  The trainable rows' gradients and d_means2D rows are those of the call
 *   without ranges: bit for bit with B200GSR_BWD_DETERMINISTIC, within float atomics' rounding otherwise.  The
 *   `saved` buffer is left as the plain backward leaves it, so a later backward over it is unaffected.  The debug
 *   counters (b200gsr_debug_counters) are not written by a call with ranges.
 *
 * b200gsr_assemble_backward_frozen: b200gsr_assemble_backward plus
 *   frozen_groups : bit g set = group g is frozen, as b200gsr_backward_scene_frozen.  A bit at or above num_groups is
 *                   refused (B200GSR_ERR_BAD_ARG) before any device work.  A frozen group's `grads` pointers may be
 *                   NULL: no packed gradient row of the group is read and nothing is written for it.
 *   frozen_groups = 0 is b200gsr_assemble_backward.
 */
#ifndef B200GSR_VIEWS_FROZEN_H
#define B200GSR_VIEWS_FROZEN_H

#include "b200gsr.h"

#ifdef __cplusplus
extern "C" {
#endif

#define B200GSR_MAX_FROZEN_RANGES 12       /* merged frozen row ranges per call: (B200GSR_MAX_GROUPS + 1) / 2 */

typedef struct b200gsr_row_range {
    int32_t lo;                            /* first row */
    int32_t len;                           /* rows in the range, > 0 */
} b200gsr_row_range;

int b200gsr_backward_views_frozen(int32_t B, const b200gsr_params* prm, const b200gsr_view_inputs* in,
                                  const int32_t* radii, const float* out_depth_alpha, const float* dL_dcolor,
                                  const float* dL_ddepth_alpha, void* saved, size_t saved_bytes, uint64_t max_pairs,
                                  const b200gsr_view_grads* out, uint32_t flags, const b200gsr_row_range* frozen,
                                  int32_t num_frozen, void* stream);
int b200gsr_assemble_backward_frozen(int32_t num_groups, const b200gsr_group* groups, const b200gsr_group_grad* grads,
                                     int32_t M, int32_t num_views, float shs_noise, float scale_noise,
                                     const float* z_shs, const float* z_scales, uint64_t seed, const float* d_means3D,
                                     const float* d_opacities, const float* d_scales, const float* d_rotations,
                                     const float* d_shs, uint32_t frozen_groups, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B200GSR_VIEWS_FROZEN_H */
