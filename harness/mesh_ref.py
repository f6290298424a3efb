"""Marching cubes restated in numpy from the rule of include/b200gsr_mesh.h: the cube table generated from the face rule,
and the surface of a volume with the same vertices, in the same order, with the same float32 rounding.  The checker of
dreamscene_b200.mesh.marching_cubes; not product code.  Also the components and the cleaning of include/b200gsr_mesh_clean.h
(components, clean_mesh), with scipy's connected_components, the checker of mesh_components and clean_mesh.

Corner c = dx | dy << 1 | dz << 2.  Edge (axis a, corner b), bit a of b clear, runs from b to b | 1 << a; the twelve
edges are numbered axis by axis, and within an axis by b: x 0..3 (b = 0, 2, 4, 6), y 4..7 (b = 0, 1, 4, 5), z 8..11
(b = 0, 1, 2, 3).  A corner is inside when its value is > iso (NaN is outside); the case is the sum of 1 << c over the
inside corners.

Face rule: walk each cube face's four corners counter-clockwise as seen from outside the cube.  An edge crossed from an
outside corner into an inside one is an entry; each entry gets the directed segment from it to the next crossing edge
of the walk (with four crossings that is the next edge, so each inside corner is cut off on its own).  The rule reads
the face's four signs only, and the neighbouring cell walks the shared face the other way round, so it makes the same
segments there in the opposite direction.  Every crossing edge is the entry of one of its two faces and the exit of
the other, so the segments chain into closed loops.  Loops come in the order of their lowest edges.  Each loop is
fanned from its apex l0, followed along its segments l0, l1, ...: triangles (l0, l_i, l_i+1).  The apex is the loop's
lowest edge whose two faces the loop crosses once only.  (A loop can cross a face twice, through all four of its edges;
a fan from one of those edges would lay a triangle flat in that face, and the neighbouring cell could lay the same one,
reversed, so the surface would not be a manifold.  Every loop of the 256 cases has such an edge.)  Seen from outside
(v <= iso) the triangles turn counter-clockwise: (b - a) x (c - a) points from inside to outside.
"""
from __future__ import annotations

import numpy as np
import scipy.sparse
from scipy.sparse.csgraph import connected_components

MAX_TRIANGLES = 5

EDGES = [(a, b) for a in range(3) for b in range(8) if not (b >> a) & 1]     # edge number -> (axis, corner)
EDGE_OF = {(b, b | 1 << a): e for e, (a, b) in enumerate(EDGES)}


def _face_walks():
    """The six faces' corners, counter-clockwise seen from outside the cube: face (axis n, side s) with in-plane axes
    u = n + 1, v = n + 2 (mod 3), so e_u x e_v = e_n."""
    walks = []
    for n in range(3):
        u, v = (n + 1) % 3, (n + 2) % 3
        for s in (0, 1):
            uv = [(0, 0), (1, 0), (1, 1), (0, 1)] if s else [(0, 0), (0, 1), (1, 1), (1, 0)]
            walks.append([s << n | du << u | dv << v for du, dv in uv])
    return walks


FACES = _face_walks()


def _edge(c0, c1):
    return EDGE_OF[(min(c0, c1), max(c0, c1))]


def face_segments(case):
    """The directed segments (from edge, to edge) of the face rule, face by face."""
    out = []
    for walk in FACES:
        inside = [(case >> c) & 1 for c in walk]
        crossing = [i for i in range(4) if inside[i] != inside[(i + 1) % 4]]
        for k, i in enumerate(crossing):
            if not inside[i]:                                # outside -> inside: an entry
                out.append((_edge(walk[i], walk[(i + 1) % 4]),
                            _edge(walk[crossing[(k + 1) % len(crossing)]], walk[(crossing[(k + 1) % len(crossing)] + 1) % 4])))
    return out


FACE_EDGES = [{_edge(w[i], w[(i + 1) % 4]) for i in range(4)} for w in FACES]


def case_loops(case):
    """The closed loops of a case, in the order of their lowest edges, each rotated to start at its apex."""
    nxt = dict(face_segments(case))
    loops, seen = [], set()
    for e in sorted(nxt):
        if e in seen:
            continue
        loop = [e]
        seen.add(e)
        while nxt[loop[-1]] != e:
            loop.append(nxt[loop[-1]])
            seen.add(loop[-1])
        twice = [f for f in FACE_EDGES if f <= set(loop)]
        apex = min(a for a in loop if not any(a in f for f in twice))
        k = loop.index(apex)
        loops.append(loop[k:] + loop[:k])
    return loops


def make_table():
    """-> (counts uint8 [256], edges int8 [256, 15]): triangles per case and their edges, -1 past the last."""
    counts = np.zeros(256, np.uint8)
    edges = np.full((256, 3 * MAX_TRIANGLES), -1, np.int8)
    for case in range(256):
        tris = [(lp[0], lp[i], lp[i + 1]) for lp in case_loops(case) for i in range(1, len(lp) - 1)]
        assert len(tris) <= MAX_TRIANGLES
        counts[case] = len(tris)
        edges[case, :3 * len(tris)] = np.array(tris, np.int8).reshape(-1)
    return counts, edges


COUNTS, TABLE = make_table()


def marching_cubes(volume, iso):
    """-> (vertices float32 [V,3] in index space, faces int32 [F,3]) of a float32 volume [X,Y,Z] at iso (a float32).

    Vertices: one per crossing edge (p, a) of the grid, ordered by p's linear index and then a; at p with coordinate a
    replaced by p_a + t, t = (iso - v[p]) / (v[p + e_a] - v[p]), each operation rounded to float32.  Faces: cell by
    cell in linear order, each cell's triangles in table order.  A grid with a dimension below 2 has no cells: no
    vertices and no faces."""
    vol = np.ascontiguousarray(volume, dtype=np.float32)
    iso = np.float32(iso)
    X, Y, Z = vol.shape
    if min(X, Y, Z) < 2:
        return np.zeros((0, 3), np.float32), np.zeros((0, 3), np.int32)
    inside = vol > iso
    idx = np.arange(X * Y * Z).reshape(X, Y, Z)
    # crossing mask of every point's +x / +y / +z edge
    mask = np.zeros((X, Y, Z), np.int64)
    mask[:-1] |= (inside[:-1] != inside[1:]) * 1
    mask[:, :-1] |= (inside[:, :-1] != inside[:, 1:]) * 2
    mask[:, :, :-1] |= (inside[:, :, :-1] != inside[:, :, 1:]) * 4
    pts, axes = np.nonzero(((mask.reshape(-1, 1) >> np.arange(3)) & 1).astype(bool))     # point-major, then axis
    nvert = np.bitwise_count(mask.reshape(-1).astype(np.uint8)).astype(np.int64)
    vstart = np.cumsum(nvert) - nvert
    step = np.array([Y * Z, Z, 1])
    f0 = vol.reshape(-1)[pts]
    f1 = vol.reshape(-1)[pts + step[axes]]
    t = (iso - f0) / (f1 - f0)
    verts = np.stack(np.unravel_index(pts, (X, Y, Z)), 1).astype(np.float32)
    verts[np.arange(len(pts)), axes] += t
    # cases of the cells, by their corner 0
    case = np.zeros((X - 1, Y - 1, Z - 1), np.int64)
    for c in range(8):
        dx, dy, dz = c & 1, (c >> 1) & 1, (c >> 2) & 1
        case |= inside[dx:X - 1 + dx, dy:Y - 1 + dy, dz:Z - 1 + dz].astype(np.int64) << c
    cells = idx[:-1, :-1, :-1].reshape(-1)
    case = case.reshape(-1)
    n = COUNTS[case].astype(np.int64)
    cell_of = np.repeat(np.arange(len(cells)), n)
    tri = np.arange(n.sum()) - np.repeat(np.cumsum(n) - n, n)          # triangle number within its cell
    e = TABLE[case[cell_of][:, None], 3 * tri[:, None] + np.arange(3)].astype(np.int64)     # [F, 3] cube edges
    ax = np.array([a for a, _ in EDGES])[e]
    corner = np.array([b for _, b in EDGES])[e]
    q = cells[cell_of][:, None] + (corner & 1) * step[0] + ((corner >> 1) & 1) * step[1] + ((corner >> 2) & 1) * step[2]
    rank = np.bitwise_count((mask.reshape(-1)[q] & ((1 << ax) - 1)).astype(np.uint8)).astype(np.int64)
    faces = (vstart[q] + rank).astype(np.int32)
    return verts, faces.reshape(-1, 3)


def vertex_attributes(volume, iso, attributes):
    """-> [V,3] float32: step 4 of include/b200gsr_mesh_colour.h, the attributes [X,Y,Z,3] of a float32 volume's grid
    points carried onto marching_cubes(volume, iso)'s vertices, in their order: a[p] + t * (a[p + e_a] - a[p]) per
    channel with the vertex's t, each operation rounded to float32."""
    vol = np.ascontiguousarray(volume, dtype=np.float32)
    attr = np.ascontiguousarray(attributes, dtype=np.float32).reshape(-1, 3)
    iso = np.float32(iso)
    X, Y, Z = vol.shape
    if min(X, Y, Z) < 2:
        return np.zeros((0, 3), np.float32)
    inside = vol > iso
    mask = np.zeros((X, Y, Z), np.int64)
    mask[:-1] |= (inside[:-1] != inside[1:]) * 1
    mask[:, :-1] |= (inside[:, :-1] != inside[:, 1:]) * 2
    mask[:, :, :-1] |= (inside[:, :, :-1] != inside[:, :, 1:]) * 4
    pts, axes = np.nonzero(((mask.reshape(-1, 1) >> np.arange(3)) & 1).astype(bool))
    q = pts + np.array([Y * Z, Z, 1])[axes]
    f0 = vol.reshape(-1)[pts]
    t = ((iso - f0) / (vol.reshape(-1)[q] - f0))[:, None]
    a0, a1 = attr[pts], attr[q]
    return a0 + t * (a1 - a0)


def _faces(faces, V):
    f = np.asarray(faces, dtype=np.int64).reshape(-1, 3)
    if f.size and (f.min() < 0 or f.max() >= V):
        raise ValueError("a face index is outside [0, V)")
    return f


def components(faces, V):
    """-> int64 [V]: each vertex's label, the smallest vertex index of its component.  Two vertices are connected when
    some face contains both; an unreferenced vertex is its own component."""
    f = _faces(faces, V)
    rows = np.concatenate([f[:, 0], f[:, 0]])
    cols = np.concatenate([f[:, 1], f[:, 2]])
    graph = scipy.sparse.coo_matrix((np.ones(len(rows), np.int8), (rows, cols)), shape=(V, V))
    _, lab = connected_components(graph, directed=False)
    first = np.full(lab.max() + 1, V, np.int64)
    np.minimum.at(first, lab, np.arange(V))
    return first[lab]


def _diagonal(lo, hi):
    """Box diagonals in float64 from per-axis float32 min / max [..., 3] (NaN: an empty axis, extent 0), each operation
    rounded on its own: sqrt((dx*dx + dy*dy) + dz*dz)."""
    d = np.where(np.isnan(lo), 0.0, hi.astype(np.float64) - lo.astype(np.float64))
    return np.sqrt((d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2])


def clean_mesh(vertices, faces, min_faces=1, min_diameter=0.0, keep_largest=False):
    """-> (vertices float32 [V',3], faces int32 [F',3], kept int32 [V']) of include/b200gsr_mesh_clean.h: the kept
    components' referenced vertices in input order (their bits), their input indices, and their faces in input order
    renumbered into them."""
    v = np.ascontiguousarray(vertices, dtype=np.float32).reshape(-1, 3)
    V = len(v)
    f = _faces(faces, V)
    label = components(f, V)
    ref = np.zeros(V, bool)
    ref[f.reshape(-1)] = True
    nfaces = np.bincount(label[f[:, 0]], minlength=V) if len(f) else np.zeros(V, np.int64)
    # per-root boxes over the referenced vertices, NaN skipped (fmin / fmax); an axis with no value stays NaN
    lo = np.full((V, 3), np.nan, np.float32)
    hi = np.full((V, 3), np.nan, np.float32)
    np.fmin.at(lo, label[ref], v[ref])
    np.fmax.at(hi, label[ref], v[ref])
    with np.errstate(all="ignore"):
        mesh_lo = np.fmin.reduce(v[ref], axis=0, initial=np.nan) if ref.any() else np.full(3, np.nan, np.float32)
        mesh_hi = np.fmax.reduce(v[ref], axis=0, initial=np.nan) if ref.any() else np.full(3, np.nan, np.float32)
        d_all = float(_diagonal(mesh_lo, mesh_hi))
        roots = np.flatnonzero(ref & (label == np.arange(V)))
        ok = nfaces[roots] >= min_faces
        if min_diameter != 0:
            ok &= _diagonal(lo[roots], hi[roots]) >= float(min_diameter) * d_all
    keep_root = np.zeros(V, bool)
    passing = roots[ok]
    if keep_largest:
        if len(passing):
            keep_root[passing[np.argmax(nfaces[passing])]] = True        # argmax: the first, the smallest label
    else:
        keep_root[passing] = True
    vkeep = ref & keep_root[label]
    fkeep = keep_root[label[f[:, 0]]] if len(f) else np.zeros(0, bool)
    kept = np.flatnonzero(vkeep)
    new_index = np.cumsum(vkeep) - 1
    return v[kept], new_index[f[fkeep]].astype(np.int32).reshape(-1, 3), kept.astype(np.int32)
