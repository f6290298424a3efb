/*
 * b200gsr_views_stats.h - the two-step scene route's backward that also gathers the densification statistics
 * (additive to b200gsr_views_frozen.h and b200gsr_stats.h, same conventions and the same library, libb200gsr.so; ABI
 * version unchanged).
 *
 * b200gsr_stats.h gathers DreamScene's densification statistics inside the one-call scene backward.  This entry point
 * does the same for the route that packs the groups first (b200gsr_assemble_forward) and rasterizes the packed arrays
 * (b200gsr_forward_views): in the launch of view stats_view, for each row of a record whose radius in that view is
 * positive,
 *
 *   xyz_gradient_accum[row - lo] += |d_means2D[stats_view][row][0:2]|
 *   denom[row - lo]              += 1
 *   max_radii2D[row - lo]         = max(max_radii2D[row - lo], radii[stats_view][row])
 *
 * with the arithmetic of b200gsr_densify_stats, bit for bit (the same device helper computes the norm), in the thread
 * that computes the row's screen-space gradient.  The [B,P,3] d_means2D arrays are then optional.
 *
 * b200gsr_backward_views_stats: b200gsr_backward_views_frozen plus
 *   stats      : HOST array of num_stats records, one per trained row range of the packed P rows (a group packed by
 *                b200gsr_assemble_forward), sorted, non-overlapping, non-empty and inside [0, P).  Each record's
 *                xyz_gradient_accum and denom are both set or both NULL (then the record gathers nothing); max_radii2D
 *                may be NULL when they are set (then it is not updated), but not set alone.  Each is a DEVICE float32
 *                array of the record's len rows ([len] or [len,1]), indexed by row - lo, updated in place.  A record
 *                may not overlap a frozen range: a frozen row's screen-space gradient is zero, so it would still count
 *                in denom.  NULL is allowed when num_stats = 0.
 *   num_stats  : records in stats, in [0, B200GSR_MAX_GROUPS].
 *   stats_view : the view whose launch gathers, in [-1, B); -1 = none.
 *   out[v].d_means2D may be NULL: then no screen-space gradient of view v is stored.
 *
 * Refused with B200GSR_ERR_BAD_ARG before any device work: a stats_view outside [-1, B); num_stats outside
 * [0, B200GSR_MAX_GROUPS], or NULL records with num_stats > 0; a record that is empty, outside [0, P), unsorted or
 * overlapping another; a record with only one of xyz_gradient_accum / denom, or with max_radii2D alone; a record that
 * overlaps a frozen range.  Every refusal of b200gsr_backward_views_frozen, except a NULL d_means2D.
 *
 * In every other respect exactly b200gsr_backward_views_frozen: the gradients, the `accumulate` bits, the frozen
 * ranges, B200GSR_BWD_DETERMINISTIC, and the `saved` buffer, left as the plain backward leaves it.  A second backward
 * over the same `saved` adds the statistics a second time.  num_stats = 0 with stats_view = -1 and every d_means2D set
 * is b200gsr_backward_views_frozen.  b200gsr_backward_views[_ex] and b200gsr_backward_views_frozen still require
 * every d_means2D.
 */
#ifndef B200GSR_VIEWS_STATS_H
#define B200GSR_VIEWS_STATS_H

#include "b200gsr_views_frozen.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct b200gsr_row_stats {     /* one trained row range of the packed P rows */
    int32_t lo, len;                   /* rows [lo, lo + len) */
    float* xyz_gradient_accum;         /* [len] or [len,1] float32, indexed by row - lo (the group's own tensors) */
    float* denom;                      /* [len] or [len,1] float32 */
    float* max_radii2D;                /* [len] float32, may be NULL */
} b200gsr_row_stats;

int b200gsr_backward_views_stats(int32_t B, const b200gsr_params* prm, const b200gsr_view_inputs* in,
                                 const int32_t* radii, const float* out_depth_alpha, const float* dL_dcolor,
                                 const float* dL_ddepth_alpha, void* saved, size_t saved_bytes, uint64_t max_pairs,
                                 const b200gsr_view_grads* out, uint32_t flags, const b200gsr_row_range* frozen,
                                 int32_t num_frozen, const b200gsr_row_stats* stats, int32_t num_stats,
                                 int32_t stats_view, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B200GSR_VIEWS_STATS_H */
