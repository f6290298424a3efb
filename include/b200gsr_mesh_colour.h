/*
 * b200gsr_mesh_colour.h - the colour of a Gaussian group's mesh (additive to b200gsr.h; same conventions and the same
 * library, libb200gsr.so; ABI version unchanged).  A colour field evaluated beside the opacity field of
 * b200gsr_fields.h, and per-vertex attributes carried onto the vertices of b200gsr_mesh.h.
 *
 * Symbols: P rows of a Gaussian group; occ the opacity field b200gsr_fields computes, [R,R,R]; a block's members the
 * rows steps 1-5 of b200gsr_fields.h assign to that block, and w_m, op_m the weight and sigmoid opacity of its step 7.
 *   1. Per-row colour: c_m = clamp_min(dc_m * SH_C0 + 0.5, 0) per channel, SH_C0 = float(0.28209479177387814): the
 *      reference's SH2RGB followed by a clamp at 0, as torch evaluates it in float32 (one rounded multiply, one rounded
 *      add, no FMA; NaN stays NaN).  It is the mean of the SH colour over all view directions, because the higher
 *      bands integrate to zero, so the colour is view-independent.
 *   2. Colour field: rgb[i,j,k,:] = (sum_m op_m w_m c_m) / occ[i,j,k], the sum over the same members in the same row
 *      order as occ's sum, with the same w_m; the division is IEEE; rgb is 0 where occ == 0.  Each term is
 *      fmaf(w_m, float(op_m * c_m), sum): op_m * c_m is rounded once per row.  The result is a weighted mean: every
 *      value lies between the smallest and largest member colour, up to rounding, where occ is well inside float32's
 *      normal range (below it both sums keep few bits, and the ratio is only >= 0).
 *   3. The occ b200gsr_fields_rgb writes is bit for bit the occ b200gsr_fields writes for the same arguments.
 *   4. Vertex attributes: the vertex on the edge from grid point p along axis a, with t as b200gsr_mesh.h defines it,
 *      gets attr[p] + t * (attr[p + e_a] - attr[p]) per channel, each operation rounded to float32 (no FMA); a NaN t
 *      gives a NaN attribute.  Attributes come in the vertices' order.
 *
 * b200gsr_fields_rgb_layout_query sizes the scratch of b200gsr_fields_rgb; it takes what b200gsr_fields_layout_query
 * takes and refuses what it refuses, and also the grids with 3 R^3 >= 2^31.
 *
 * b200gsr_fields_rgb: the arguments of b200gsr_fields, in its order, with features_dc [P,1,3] device float32
 * (contiguous) after rotation, and rgb [R,R,R,3] device float32 (every element written) after occ.  Same info,
 * conventions and refusals as b200gsr_fields; info.kept == 0 or info.extent == 0 leave occ and rgb all zero.
 *
 * b200gsr_mesh_attributes: after b200gsr_mesh_count of the same X, Y, Z, volume and iso, whose scratch it reads (the
 * scratch b200gsr_mesh_emit reads), writes out [V,3] float32 from attributes [X,Y,Z,3] float32 (device, contiguous,
 * point (i, j, k) at ((i*Y + j)*Z + k)*3); V the vertex total of that count.  It writes no attribute past V.
 *
 * None of the three waits for the device.  Limits, else B200GSR_ERR_BAD_ARG before any device work: those of
 * b200gsr_fields.h and b200gsr_mesh.h, 3 R^3 < 2^31 for the colour field, no null pointer, attributes and out 4-byte
 * aligned, V >= 0.
 */
#ifndef B200GSR_MESH_COLOUR_H
#define B200GSR_MESH_COLOUR_H

#include "b200gsr.h"
#include "b200gsr_fields.h"
#include "b200gsr_mesh.h"

#ifdef __cplusplus
extern "C" {
#endif

int b200gsr_fields_rgb_layout_query(int32_t P, int32_t R, int32_t num_blocks, double relax_ratio, const float* coords,
                                    b200gsr_fields_layout* out);
int b200gsr_fields_rgb(int32_t P, const float* xyz, const float* opacity, const float* scaling, const float* rotation,
                       const float* features_dc, int32_t R, int32_t num_blocks, double relax_ratio, const float* coords,
                       float* occ, float* rgb, b200gsr_fields_info* info, void* scratch, size_t scratch_bytes,
                       void* stream);
int b200gsr_mesh_attributes(int32_t X, int32_t Y, int32_t Z, const float* volume, float iso, const void* scratch,
                            size_t scratch_bytes, const float* attributes, float* out, int32_t V, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B200GSR_MESH_COLOUR_H */
