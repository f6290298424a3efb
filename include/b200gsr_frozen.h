/*
 * b200gsr_frozen.h - scene-render backwards with frozen parameter groups (additive to b200gsr_scene.h and
 * b200gsr_step.h, same conventions and the same library, libb200gsr.so; ABI version unchanged).
 *
 * DreamScene's scene stages render every visible group but train only some of them (the environment alone, then the
 * floor alone).  These backwards compute the gradients of the trainable groups only: the forward is unchanged, and
 * the frozen groups' entries still take part in the compositing recurrence behind which the trainable ones sit, but
 * no gradient of a frozen group is computed, accumulated or written.
 *
 *   frozen_groups : bit g set = group g is frozen.  A bit at or above num_groups is refused (B200GSR_ERR_BAD_ARG)
 *                   before any device work.
 *   grads         : as b200gsr_backward_scene for a trainable group (every pointer required).  A frozen group's
 *                   pointers may be NULL; nothing is written through them.
 *   d_means2D     : every row written; the rows of frozen groups are zeros.
 *
 * Otherwise exactly b200gsr_backward_scene / b200gsr_backward_scene_dyn (same validation, layouts and flags).  The
 * trainable groups' gradients and d_means2D rows are those of the call without a mask: bit for bit with
 * B200GSR_BWD_DETERMINISTIC, within float atomics' rounding otherwise.  frozen_groups = 0 is that call.  The `saved`
 * buffer is left as the plain backward leaves it, so a later backward over it, with or without a mask, is unaffected.
 * The debug counters (b200gsr_debug_counters) are not written by a call with a non-zero mask.
 */
#ifndef B200GSR_FROZEN_H
#define B200GSR_FROZEN_H

#include "b200gsr_step.h"

#ifdef __cplusplus
extern "C" {
#endif

int b200gsr_backward_scene_frozen(int32_t B, const b200gsr_params* prm, int32_t num_groups, const b200gsr_group* groups,
                                  const b200gsr_group_grad* grads, const float* shs_noise, const float* scale_noise,
                                  uint64_t seed, const float* d_scales, const int32_t* radii,
                                  const float* out_depth_alpha, const float* dL_dcolor, const float* dL_ddepth_alpha,
                                  void* saved, size_t saved_bytes, uint64_t max_pairs, float* d_means2D,
                                  uint32_t flags, uint32_t frozen_groups, void* stream);
int b200gsr_backward_scene_dyn_frozen(int32_t B, const b200gsr_params* prm, int32_t num_groups,
                                      const b200gsr_group* groups, const b200gsr_group_grad* grads,
                                      const b200gsr_step_view* views, const uint64_t* seed, const float* d_scales,
                                      const int32_t* radii, const float* out_depth_alpha, const float* dL_dcolor,
                                      const float* dL_ddepth_alpha, void* saved, size_t saved_bytes,
                                      uint64_t max_pairs, float* d_means2D, uint32_t flags, uint32_t frozen_groups,
                                      void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B200GSR_FROZEN_H */
