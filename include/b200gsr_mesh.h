/*
 * b200gsr_mesh.h - marching cubes on a float32 volume (additive to b200gsr.h; same conventions and the same library,
 * libb200gsr.so; ABI version unchanged).  The step that turns an opacity field (b200gsr_fields.h) into a mesh.
 *
 * The cube table.  Corner c = dx | dy << 1 | dz << 2 of a cell.  Edge (axis a, corner b), bit a of b clear, runs from
 * b to b | 1 << a; the twelve edges are numbered axis by axis and within an axis by b: x 0..3 (b = 0, 2, 4, 6),
 * y 4..7 (b = 0, 1, 4, 5), z 8..11 (b = 0, 1, 2, 3).  A point is inside when its value is > iso, strictly (NaN is
 * outside); a cell's case is the sum of 1 << c over its inside corners.  The table is generated from one rule when the
 * library is compiled, not typed in:
 *   - Face rule.  Each cube face's four corners are walked counter-clockwise as seen from outside the cube.  An edge
 *     crossed from an outside corner into an inside one is an entry, and each entry gets the directed segment from it
 *     to the next crossing edge of the walk.  A face with four crossings has its inside corners on a diagonal; each of
 *     them gets its own segment.  The rule reads the face's four signs only and the neighbouring cell walks the
 *     shared face the other way round, so both cells make the same segments there, in opposite directions: the
 *     surface has no cracks.
 *   - Loops.  The segments of the six faces chain into closed loops, ordered by their lowest edges.  Each loop is
 *     fanned from its apex l0, followed along its segments l0, l1, ...: triangles (l0, l_i, l_i+1).  The apex is the
 *     loop's lowest edge whose two faces the loop crosses once only; a fan from an edge of a face crossed twice would
 *     lay a triangle flat in that face, which the neighbouring cell can lay too.
 *   - Orientation.  Seen from outside (v <= iso) every triangle turns counter-clockwise (the OBJ / PLY convention):
 *     (b - a) x (c - a) points from inside to outside.
 * At most B200GSR_MESH_MAX_TRIANGLES triangles per cell.  b200gsr_mesh_table copies the table the kernels use; it
 * needs no device.
 *
 * The mesh of a volume v [X,Y,Z] (float32, contiguous, point (i, j, k) at i*Y*Z + j*Z + k):
 *   - vertices: one per crossing edge (p, a) of the grid, none duplicated between cells, ordered by p's linear index
 *     and then by a; the vertex is p with coordinate a replaced by p_a + t, t = (iso - v[p]) / (v[p + e_a] - v[p]),
 *     each operation rounded to float32 (IEEE division), in index space;
 *   - faces: int32 vertex indices, cell by cell in linear order of the cell's corner 0, each cell's triangles in table
 *     order.
 * A grid with a dimension below 2 has no cells and gives V = F = 0, as does an iso that no edge crosses.  The surface
 * is closed wherever no grid-boundary point is inside.
 *
 * Two calls.  b200gsr_mesh_count classifies the grid and scans the counts into the scratch, and writes totals =
 * {V, F} (two int32, device memory).  The caller reads the totals back and allocates vertices [V,3] float32 and faces
 * [F,3] int32 (device), then b200gsr_mesh_emit, with the same volume, iso and scratch, writes them; it writes no
 * vertex past V and no face past F.  Neither call waits for the device.
 *
 * Limits, else B200GSR_ERR_BAD_ARG before any device work: 1 <= X, Y, Z <= B200GSR_FIELDS_MAX_R; 3 X Y Z < 2^31 and
 * B200GSR_MESH_MAX_TRIANGLES (X-1)(Y-1)(Z-1) < 2^31, so no count, scan or index overflows (512^3 fits); iso finite;
 * no null pointer; scratch 256-byte aligned and at least the queried total; V, F >= 0.
 */
#ifndef B200GSR_MESH_H
#define B200GSR_MESH_H

#include "b200gsr.h"
#include "b200gsr_fields.h"

#define B200GSR_MESH_MAX_TRIANGLES 5      /* triangles per cell */
#define B200GSR_MESH_TABLE_WIDTH 15       /* edges per case in the table: 3 per triangle, -1 past the last */

typedef struct {
    size_t total;                  /* scratch bytes */
    int64_t points;                /* X Y Z */
    int64_t cells;                 /* (X-1)(Y-1)(Z-1), 0 when a dimension is below 2 */
} b200gsr_mesh_layout;

#ifdef __cplusplus
extern "C" {
#endif

/* counts[256]: triangles per case; edges[256 * B200GSR_MESH_TABLE_WIDTH]: their cube edges, three per triangle. */
int b200gsr_mesh_table(uint8_t* counts, int8_t* edges);
int b200gsr_mesh_layout_query(int32_t X, int32_t Y, int32_t Z, b200gsr_mesh_layout* out);
int b200gsr_mesh_count(int32_t X, int32_t Y, int32_t Z, const float* volume, float iso, int32_t* totals, void* scratch,
                       size_t scratch_bytes, void* stream);
int b200gsr_mesh_emit(int32_t X, int32_t Y, int32_t Z, const float* volume, float iso, const void* scratch,
                      size_t scratch_bytes, float* vertices, int32_t V, int32_t* faces, int32_t F, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B200GSR_MESH_H */
