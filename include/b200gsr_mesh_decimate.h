/*
 * b200gsr_mesh_decimate.h - quadric edge-collapse decimation of a triangle mesh to a target face count, on the device
 * (additive to b200gsr.h; same conventions and the same library, libb200gsr.so; ABI version unchanged).  The step after
 * cleaning (b200gsr_mesh_clean.h) that DreamGaussian's export does with pymeshlab's quadric edge collapse.  Edges are
 * collapsed in rounds of independent edges, so a round's collapses touch disjoint faces and are applied together.
 *
 * Input: vertices float32 [V,3], faces int32 [F,3] (device, contiguous), every index in [0, V); target_faces >= 0.
 * Notation: all arithmetic below is float64 with every operation IEEE-rounded on its own (no FMA), evaluated in the
 * order the parentheses give.  For 3-vectors, u - w and u * s are per component;
 *   cross(u, w) = (u.y*w.z - u.z*w.y, u.z*w.x - u.x*w.z, u.x*w.y - u.y*w.x),  dot(u, w) = (u.x*w.x + u.y*w.y) + u.z*w.z.
 *
 * 1. Quadrics.  pos[v] = (double) vertices[v].  Face (i0, i1, i2) has n = cross(p1 - p0, p2 - p0) (pk = pos[ik]) and
 *    l2 = dot(n, n).  If l2 == 0 its quadric is 0.  Otherwise l = sqrt(l2), u = (n.x / l, n.y / l, n.z / l),
 *    d = -dot(u, p0), w = l * 0.5 (its area) and, with s = (u.x, u.y, u.z, d), its quadric is the 10 values
 *      q = (w*(s0*s0), w*(s0*s1), w*(s0*s2), w*(s0*s3), w*(s1*s1), w*(s1*s2), w*(s1*s3), w*(s2*s2), w*(s2*s3), w*(s3*s3)).
 *    A vertex's quadric Q[v] starts at +0 and adds, per value, the quadric of each face that lists v, in face-index
 *    order (a face listing v twice is added twice).  The 10 values of Q are named xx, xy, xz, xd, yy, yz, yd, zz, zd,
 *    dd in that order.  Positions and quadrics are carried in float64 between rounds.
 *
 * 2. Rounds.  Each round reads the live faces (current indices) only.
 *    Fan.  Each live face listing v gives v a fan entry (p, q): the face's indices rotated to start at v, v p q (for a
 *    face listing v twice, the entry of each slot).  The entries are ordered by face index.  v is *regular* when it has
 *    k entries, 3 <= k <= B200GSR_DECIMATE_MAX_VALENCE, none of its faces lists an index twice, and the entries chain
 *    into one cycle: starting at entry 0 with c = q_0, repeatedly take the first entry (in order) with p == c and set
 *    c to its q; c comes back to p_0 after exactly k entries, every step finding an entry.  This is one closed,
 *    consistently oriented fan, so every edge at a regular v has exactly two faces: it excludes boundaries,
 *    non-manifold edges, inconsistently oriented faces and pinch vertices (two sheets of surface touching at v, whose
 *    entries form two or more cycles, which the link condition alone does not see).  N(v) = {p_i}, deg(v) = k.
 *    Candidate.  The edge (a, b), a < b, of two regular vertices that are neighbours is a candidate when
 *      - deg(a) + deg(b) - 4 >= 3 (valence; with the link condition this excludes a tetrahedron and any fold),
 *      - |N(a) & N(b)| == 2 (link condition),
 *      - its cost (3.) is not NaN, and
 *      - no flip: for v in {a, b} and each entry (p, q) of v with p and q both not the other endpoint,
 *        nb = cross(pos[p] - pos[v], pos[q] - pos[v]) and na = cross(pos[p] - x, pos[q] - x) (x from 3.): nb is
 *        (0, 0, 0) (a zero-area face, which has no orientation to keep; marching cubes makes them where a grid value
 *        equals iso) or dot(nb, na) > 0.
 *
 * 3. Placement and cost.  Q = Q[a] + Q[b] per value.  The quadric form of a point x is
 *      r0 = (xx*x.x + xy*x.y) + (xz*x.z + xd),  r1 = (xy*x.x + yy*x.y) + (yz*x.z + yd),
 *      r2 = (xz*x.x + yz*x.y) + (zz*x.z + zd),  r3 = (xd*x.x + yd*x.y) + (zd*x.z + dd),
 *      E(x) = (r0*x.x + r1*x.y) + (r2*x.z + r3).
 *    det3 of a row-major 3x3 m is (m00*t0 - m01*t1) + m02*t2 with t0 = m11*m22 - m12*m21, t1 = m10*m22 - m12*m20,
 *    t2 = m10*m21 - m11*m20.  With optimal_placement, A = [[xx, xy, xz], [xy, yy, yz], [xz, yz, zz]], r = (-xd, -yd,
 *    -zd), det = det3(A), tr = (xx + yy) + zz: if |det| > ((tr*tr)*tr) * B200GSR_DECIMATE_DET_TOL (a relative test,
 *    NaN fails it), x = (det3(A_0) / det, det3(A_1) / det, det3(A_2) / det), A_j being A with column j replaced by r
 *    (Cramer's rule), and e = E(x).  Otherwise, and always without optimal_placement, x is the first of pos[a],
 *    pos[b], mid = (pos[a] + pos[b]) * 0.5 whose E is smaller than every earlier one's (x = pos[a], e = E(pos[a]);
 *    then e2 < e replaces, then e3 < e replaces), and e its E.  The cost is +0 when e <= 0, e itself otherwise (NaN
 *    stays NaN).  Its key cost is the cost rounded to float32 toward +infinity.
 *
 * 4. Selection.  Candidates are ordered by (key cost, a, b) lexicographically, which is the order of the key
 *    (float32 bits of the key cost) << 32 | (the edge's index in (a, b) order): every candidate has its own place.
 *    m(v) is the smallest candidate at v, M(v) the smallest of m over v and N(v).  A candidate is selected when it is
 *    m(a), M(a) and M(b).  No two selected edges share or neighbour an endpoint (if c neighbours a, M(a) <= m(c) and
 *    M(c) <= m(a), so the edges are the same), so their collapses touch disjoint faces; the smallest candidate is always
 *    selected.  Let S selected edges and F live faces, F > target_faces, and j = ceil((F - target_faces) / 2): if
 *    S <= j all are applied, otherwise the first j in candidate order, so F ends at target_faces or target_faces - 1.
 *    Collapsing (a, b): pos[a] = x, Q[a] = Q[a] + Q[b]; the two faces listing both a and b die; b is replaced by a in
 *    its other faces.  a is then *moved*.
 *
 * 5. Stopping.  Rounds run while F > target_faces and a candidate exists; `rounds` counts the rounds that collapsed.
 *
 * Output.  The vertices some live face lists, in input order: kept int32 [V'] their input indices, vertices float32
 * [V',3] pos rounded to nearest float32 for a moved vertex and the input's bits for any other.  The live faces in input
 * order, renumbered into them: int32 [F',3].  When nothing collapses (F <= target_faces or no candidate) this is
 * b200gsr_mesh_clean's output with its defaults.  A face with an index outside [0, V) is counted in bad and takes no
 * part (nothing runs when bad != 0).
 *
 * Calls.  b200gsr_mesh_decimate_layout_query gives the scratch bytes for (V, F); the scratch holds all state between
 * calls.
 *   - b200gsr_mesh_decimate_begin reads vertices and faces, builds the quadrics and writes status.
 *   - b200gsr_mesh_decimate_rounds runs up to `rounds` more rounds, reading F and whether to stop from the scratch
 *     (rounds past the end do nothing), then writes status; rounds = 0 only writes status.
 *   - b200gsr_mesh_decimate_emit, after status reports done, writes out_vertices [V_out,3], out_faces [F_out,3] and
 *     kept [V_out]; it writes no vertex past V_out and no face past F_out.
 * status is B200GSR_DECIMATE_STATUS_WORDS int32 in device memory: {F live, rounds, done (no round would collapse
 * anything), bad, V', F'}.  None of the calls waits for the device; every result is deterministic, two runs give the
 * same bits.
 *
 * Refusals, B200GSR_ERR_BAD_ARG before any device work: 1 <= V < 2^31, 0 <= F and 3 F < 2^31; target_faces < 0;
 * rounds < 0; a null pointer (faces may be null when F = 0); vertices, faces, status and the outputs not 4-byte aligned,
 * scratch not 256-byte aligned or smaller than the queried size; V_out or F_out negative.
 */
#ifndef B200GSR_MESH_DECIMATE_H
#define B200GSR_MESH_DECIMATE_H

#include "b200gsr.h"

#define B200GSR_DECIMATE_MAX_VALENCE 32
#define B200GSR_DECIMATE_DET_TOL 1e-9
#define B200GSR_DECIMATE_STATUS_WORDS 6

#ifdef __cplusplus
extern "C" {
#endif

int b200gsr_mesh_decimate_layout_query(int32_t V, int32_t F, size_t* scratch_bytes);
int b200gsr_mesh_decimate_begin(int32_t V, int32_t F, const float* vertices, const int32_t* faces, int32_t target_faces,
                                int32_t optimal_placement, int32_t* status, void* scratch, size_t scratch_bytes,
                                void* stream);
int b200gsr_mesh_decimate_rounds(int32_t V, int32_t F, int32_t rounds, int32_t* status, void* scratch,
                                 size_t scratch_bytes, void* stream);
int b200gsr_mesh_decimate_emit(int32_t V, int32_t F, const float* vertices, const void* scratch, size_t scratch_bytes,
                               float* out_vertices, int32_t* out_faces, int32_t* kept, int32_t V_out, int32_t F_out,
                               void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B200GSR_MESH_DECIMATE_H */
