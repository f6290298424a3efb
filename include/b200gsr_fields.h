/*
 * b200gsr_fields.h - the opacity field of a Gaussian group on a voxel grid (additive to b200gsr.h; same conventions and
 * the same library, libb200gsr.so; ABI version unchanged).
 *
 * DreamScene's GaussianModel.extract_fields(resolution, num_blocks, relax_ratio) (gs_renderer.py), the field a user
 * turns into a mesh:
 *   1. keep the rows with sigmoid(opacity) > 0.005f;
 *   2. mn, mx = per-axis min / max of the kept centres; center = (mn + mx) / 2, scale = 1.8 / max(mx - mn) in double;
 *   3. xyz' = (xyz - center) * float(scale), std' = exp(scaling) * float(scale), cov = strip_symmetric(L L^T) with
 *      L = R(normalize(rotation)) diag(std');
 *   4. the grid coordinates coords[R] (torch.linspace(-1, 1, R) in float32) are cut into chunks of split = R / num_blocks
 *      points, the last chunk possibly shorter: C = ceil(R / split) chunks per axis, C^3 blocks;
 *   5. a row belongs to block (bx, by, bz) when on every axis lo[c] < xyz'[axis] < hi[c], strictly, with
 *      lo[c] = first coordinate of chunk c - r and hi[c] = last coordinate + r, float32, r = float((2 / num_blocks) *
 *      relax_ratio);
 *   6. weight = exp(power) with power = -1/2 d^T Sigma^-1 d from the cofactor inverse (1e-24 added to the determinant),
 *      and weight 0 where power > 0;
 *   7. occ[i,j,k] (ij meshgrid order, [R,R,R]) = sum over the members of the block holding grid point (i, j, k) of
 *      opacity * weight, summed in row order, in a fixed order on every call (no float atomics).
 * Steps 1-5 are bit for bit torch's float32 evaluation of the same expressions; the sum is held to a tolerance.
 *
 * b200gsr_fields_layout_query sizes the scratch for P rows and the grid; coords is a HOST array of R floats (the same
 * values b200gsr_fields takes).  The scratch holds, per row, one 48-byte record and one 16-byte block mask, a block x
 * row-chunk count table, and the member lists, sized for the most blocks a centre can fall into on each axis
 * (max_blocks_per_axis, found from the block boxes): max_pairs = P * max_blocks_per_axis^3.
 *
 * b200gsr_fields: xyz [P,3], opacity [P,1], scaling [P,3], rotation [P,4] device float32, contiguous; occ [R,R,R]
 * device float32 (every element written); info a device b200gsr_fields_info (written); coords the host array above,
 * read during the call only; scratch of at least the queried total bytes, 256-byte aligned.  The call enqueues its
 * kernels on `stream` and returns without waiting for them (no host sync).  It does not refuse degenerate input, which
 * it cannot see without waiting: info.kept == 0 (no row passes the filter) or info.extent == 0 (all kept centres
 * coincide) mark the inputs the reference cannot evaluate, and occ is then all zero.
 *
 * Limits, else B200GSR_ERR_BAD_ARG before any device work: 1 <= P, 1 <= R <= B200GSR_FIELDS_MAX_R (so R^3 < 2^31),
 * 1 <= num_blocks <= R, fmod(R, 2 / num_blocks) == 0 (the reference's assert), C <= B200GSR_FIELDS_MAX_CHUNKS,
 * relax_ratio finite, max_pairs < 2^31 and C^3 * ceil(P / B200GSR_FIELDS_CHUNK_ROWS) < 2^31.
 */
#ifndef B200GSR_FIELDS_H
#define B200GSR_FIELDS_H

#include "b200gsr.h"

#define B200GSR_FIELDS_MAX_R 1024
#define B200GSR_FIELDS_MAX_CHUNKS 32       /* chunks per axis: 32^3 blocks */
#define B200GSR_FIELDS_CHUNK_ROWS 1024     /* rows per binning chunk */

typedef struct {
    size_t total;                  /* scratch bytes */
    int32_t blocks_per_axis;       /* C */
    int32_t max_blocks_per_axis;
    int64_t max_pairs;             /* member-list capacity */
} b200gsr_fields_layout;

typedef struct {
    double scale;                  /* 1.8 / extent, the reference's self.scale */
    float center[3];               /* (mn + mx) / 2, the reference's self.center */
    float extent;                  /* max(mx - mn) over the axes */
    int32_t kept;                  /* rows that passed the opacity filter */
    uint32_t overflow;             /* 1: the member lists did not fit (not expected; occ is then all zero) */
    int64_t pairs;                 /* (block, row) memberships */
} b200gsr_fields_info;

#ifdef __cplusplus
extern "C" {
#endif

int b200gsr_fields_layout_query(int32_t P, int32_t R, int32_t num_blocks, double relax_ratio, const float* coords,
                                b200gsr_fields_layout* out);
int b200gsr_fields(int32_t P, const float* xyz, const float* opacity, const float* scaling, const float* rotation,
                   int32_t R, int32_t num_blocks, double relax_ratio, const float* coords, float* occ,
                   b200gsr_fields_info* info, void* scratch, size_t scratch_bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B200GSR_FIELDS_H */
