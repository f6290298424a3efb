/*
 * b200gsr_mesh_clean.h - connected components of a triangle mesh and the removal of small ones ("floaters"), on the
 * device (additive to b200gsr.h; same conventions and the same library, libb200gsr.so; ABI version unchanged).  The
 * step after marching cubes (b200gsr_mesh.h) that DreamGaussian's clean_mesh does with pymeshlab's "remove connected
 * components by face count / by diameter" filters.
 *
 * Input: vertices float32 [V,3], faces int32 [F,3] (device, contiguous), every index in [0, V).
 *
 * Components.  Two vertices are connected when some face contains both; a component is a connected set of vertices,
 * and a face belongs to the component of its vertices.  A degenerate face (a repeated index) is an ordinary face.  A
 * vertex's label is the smallest vertex index in its component; a vertex no face references is its own component,
 * with no faces.
 *
 * Per component c:
 *   - faces_c, its number of faces;
 *   - its box, the per-axis min and max over its vertices, NaN coordinates skipped (fmin / fmax); an axis whose
 *     coordinates are all NaN has extent 0;
 *   - d_c, the box diagonal in float64, each operation IEEE-rounded with no FMA, in this order:
 *       dx = (double)max_x - (double)min_x, likewise dy and dz;  d2 = (dx*dx + dy*dy) + dz*dz;  d_c = sqrt(d2).
 * d_all is the same diagonal over every referenced vertex.
 *
 * A component is kept when it has a face and
 *   - faces_c >= min_faces, and
 *   - min_diameter == 0, or d_c >= min_diameter * d_all, the product rounded in float64 (min_diameter is a fraction of
 *     the whole mesh's diagonal: 0.1 is 10 %, as pymeshlab's PercentageValue), and
 *   - with keep_largest set, it also has the most faces among the components passing the first two tests, ties to
 *     the smallest label (none passes: nothing is kept).
 *
 * Output.  The kept vertices are the referenced vertices of kept components in input order (an unreferenced vertex is
 * always dropped): kept int32 [V'] their input indices, vertices float32 [V',3] copies of their input bits.  The kept
 * faces are the faces of kept components in input order, their indices renumbered into the kept vertices: int32
 * [F',3].  With the defaults (min_faces = 1, min_diameter = 0, keep_largest = 0) every referenced vertex and every
 * face is kept: a mesh whose vertices are all referenced comes back unchanged, kept = 0 .. V-1.
 *
 * Calls.  b200gsr_mesh_clean_layout_query gives the scratch bytes for (V, F); the scratch serves all three calls.
 *   - b200gsr_mesh_components writes labels int32 [V] and bad, an int32 in device memory.
 *   - b200gsr_mesh_clean_count runs the components, the statistics and the decision, and writes totals = {V', F', bad}
 *     (three int32, device memory).
 *   - b200gsr_mesh_clean_emit, after a count with the same inputs and scratch, writes out_vertices [V_out,3],
 *     out_faces [F_out,3] and kept [V_out]; it writes no vertex past V_out and no face past F_out.
 * bad is the number of faces with an index outside [0, V).  No call can refuse those on the host: the kernels skip
 * such a face (it connects nothing, counts nowhere and is never kept) and never read or write through its indices.
 * None of the calls waits for the device; every result is deterministic, two calls give the same bits.
 *
 * Refusals, B200GSR_ERR_BAD_ARG before any device work: 1 <= V < 2^31, 0 <= F and 3 F < 2^31; a null pointer (faces
 * may be null when F = 0); vertices, faces, labels, bad, totals and the outputs not 4-byte aligned, scratch not
 * 256-byte aligned or smaller than the queried size; min_faces < 0; min_diameter negative or not finite; V_out or
 * F_out negative.
 */
#ifndef B200GSR_MESH_CLEAN_H
#define B200GSR_MESH_CLEAN_H

#include "b200gsr.h"

#ifdef __cplusplus
extern "C" {
#endif

int b200gsr_mesh_clean_layout_query(int32_t V, int32_t F, size_t* scratch_bytes);
int b200gsr_mesh_components(int32_t V, int32_t F, const int32_t* faces, int32_t* labels, int32_t* bad, void* scratch,
                            size_t scratch_bytes, void* stream);
int b200gsr_mesh_clean_count(int32_t V, int32_t F, const float* vertices, const int32_t* faces, int32_t min_faces,
                             double min_diameter, int32_t keep_largest, int32_t* totals, void* scratch,
                             size_t scratch_bytes, void* stream);
int b200gsr_mesh_clean_emit(int32_t V, int32_t F, const float* vertices, const int32_t* faces, int32_t min_faces,
                            double min_diameter, int32_t keep_largest, const void* scratch, size_t scratch_bytes,
                            float* out_vertices, int32_t* out_faces, int32_t* kept, int32_t V_out, int32_t F_out,
                            void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B200GSR_MESH_CLEAN_H */
