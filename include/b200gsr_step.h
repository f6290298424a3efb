/*
 * b200gsr_step.h - a training step replayed from CUDA graphs: the scene render and the Adam step with their per-step
 * values read from device memory (additive to b200gsr.h and b200gsr_scene.h, same conventions and the same library,
 * libb200gsr.so; ABI version unchanged).
 *
 * A kernel parameter passed by value is frozen into a captured graph, so a replay of b200gsr_forward_scene would reuse
 * the seed, noise coefficients, FoV and SH degree of the capture.  These entry points read those values through
 * device pointers instead; the caller rewrites the device records before each replay.
 *
 *   views [B]  : DEVICE array of b200gsr_step_view, one record per view.  The kernels trust the records: the caller
 *                validates them when it writes them (tanfov > 0, 0 <= sh_degree <= 3 with (sh_degree + 1)^2 <= M).
 *   seed       : DEVICE pointer to the uint64 Philox seed (b200gsr_forward_scene's `seed`).
 *   prm[B]     : as b200gsr_forward_scene for P, M, the image size, scale_modifier and the bg / viewmatrix /
 *                projmatrix / campos device pointers (whose contents may change between replays).  The host values of
 *                tanfovx, tanfovy and sh_degree are ignored.
 *
 * b200gsr_forward_scene_dyn / b200gsr_backward_scene_dyn: otherwise exactly b200gsr_forward_scene /
 * b200gsr_backward_scene (same validation, layouts, flags and outputs); for equal values the results are bit for bit
 * theirs.
 *
 * b200gsr_adam_step_dyn: b200gsr_adam_step with the six per-tensor scalars of record i (lerp_weight, beta2,
 * one_minus_beta2, eps, step_size, bc2_sqrt) read from scalars[6 i .. 6 i + 5] (DEVICE float [n_tensors, 6]); the
 * scalar fields of the host records are ignored.  Pointers and lengths stay host values.
 *
 * b200gsr_pair_report: enqueue after a forward that had no host_notify slot (a captured one).  It folds that forward's
 * pair count and overflow flag from the header of its `saved` buffer into report (DEVICE uint32[2]):
 * report[0] = max(report[0], pairs), report[1] += 1 if the pairs exceeded the forward's max_pairs.  The caller zeroes
 * the report and reads it when it wants to know whether a replay overflowed.
 */
#ifndef B200GSR_STEP_H
#define B200GSR_STEP_H

#include "b200gsr_scene.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct b200gsr_step_view {
    float tanfovx, tanfovy;
    float shs_noise, scale_noise;    /* 0 = that augmentation is off in this view */
    int32_t sh_degree;
    int32_t reserved[3];             /* pads the record to 32 bytes; not read */
} b200gsr_step_view;

int b200gsr_forward_scene_dyn(int32_t B, const b200gsr_params* prm, int32_t num_groups, const b200gsr_group* groups,
                              const b200gsr_step_view* views, const uint64_t* seed, float* out_scales,
                              float* out_color, float* out_depth_alpha, int32_t* radii, void* scratch,
                              size_t scratch_bytes, void* saved, size_t saved_bytes, uint64_t max_pairs, uint32_t flags,
                              uint32_t* host_notify, uint32_t notify_seq, void* stream);
int b200gsr_backward_scene_dyn(int32_t B, const b200gsr_params* prm, int32_t num_groups, const b200gsr_group* groups,
                               const b200gsr_group_grad* grads, const b200gsr_step_view* views, const uint64_t* seed,
                               const float* d_scales, const int32_t* radii, const float* out_depth_alpha,
                               const float* dL_dcolor, const float* dL_ddepth_alpha, void* saved, size_t saved_bytes,
                               uint64_t max_pairs, float* d_means2D, uint32_t flags, void* stream);
int b200gsr_adam_step_dyn(int32_t n_tensors, const b200gsr_adam_tensor* tensors, const float* scalars, void* stream);
int b200gsr_pair_report(const void* saved, uint32_t* report, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B200GSR_STEP_H */
