"""Marching cubes restated in numpy from the rule of include/b200gsr_mesh.h: the cube table generated from the face rule,
and the surface of a volume with the same vertices, in the same order, with the same float32 rounding.  The checker of
dreamscene_b200.mesh.marching_cubes; not product code.  Also the components and the cleaning of include/b200gsr_mesh_clean.h
(components, clean_mesh), with scipy's connected_components, the checker of mesh_components and clean_mesh.
And the decimation of include/b200gsr_mesh_decimate.h (decimate_mesh), round by round in elementwise float64 numpy,
the checker of dreamscene_b200.mesh.decimate_mesh.

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


# ---- decimation (include/b200gsr_mesh_decimate.h) ------------------------------------------------------------------

DEC_MAX_VALENCE = 32            # B200GSR_DECIMATE_MAX_VALENCE
DEC_DET_TOL = 1e-9              # B200GSR_DECIMATE_DET_TOL
_QPAIRS = [(0, 0), (0, 1), (0, 2), (0, 3), (1, 1), (1, 2), (1, 3), (2, 2), (2, 3), (3, 3)]


def _cross(u, w):
    return np.stack([u[..., 1] * w[..., 2] - u[..., 2] * w[..., 1], u[..., 2] * w[..., 0] - u[..., 0] * w[..., 2],
                     u[..., 0] * w[..., 1] - u[..., 1] * w[..., 0]], -1)


def _dot(u, w):
    return (u[..., 0] * w[..., 0] + u[..., 1] * w[..., 1]) + u[..., 2] * w[..., 2]


def _face_quadrics(p0, p1, p2):
    """[F,10]: rule 1, each face's plane quadric (unit normal, weighted by area), 0 for a zero-area face."""
    n = _cross(p1 - p0, p2 - p0)
    l2 = _dot(n, n)
    with np.errstate(all="ignore"):
        ln = np.sqrt(l2)
        u = n / ln[:, None]
        s = [u[:, 0], u[:, 1], u[:, 2], -_dot(u, p0)]
        w = ln * 0.5
        q = np.stack([w * (s[i] * s[j]) for i, j in _QPAIRS], -1)
    q[l2 == 0] = 0.0
    return q


def _det3(m):
    """m: 9 arrays, row-major; the header's expansion along the first row."""
    m00, m01, m02, m10, m11, m12, m20, m21, m22 = m
    t0 = m11 * m22 - m12 * m21
    t1 = m10 * m22 - m12 * m20
    t2 = m10 * m21 - m11 * m20
    return (m00 * t0 - m01 * t1) + m02 * t2


def _qform(q, x):
    """x^T Q x of the homogeneous point (x, 1), in the header's order."""
    X, Y, Z = x[:, 0], x[:, 1], x[:, 2]
    r0 = (q[:, 0] * X + q[:, 1] * Y) + (q[:, 2] * Z + q[:, 3])
    r1 = (q[:, 1] * X + q[:, 4] * Y) + (q[:, 5] * Z + q[:, 6])
    r2 = (q[:, 2] * X + q[:, 5] * Y) + (q[:, 7] * Z + q[:, 8])
    r3 = (q[:, 3] * X + q[:, 6] * Y) + (q[:, 8] * Z + q[:, 9])
    return (r0 * X + r1 * Y) + (r2 * Z + r3)


def _placement(q, pa, pb, optimal):
    """-> (x [E,3], cost [E]) of rule 3: Cramer's rule when |det| passes, else the best of a, b and the midpoint."""
    with np.errstate(all="ignore"):
        ca, cb = _qform(q, pa), _qform(q, pb)
        mid = (pa + pb) * 0.5
        cm = _qform(q, mid)
        x, c = pa.copy(), ca.copy()
        tb = cb < c
        x[tb], c[tb] = pb[tb], cb[tb]
        tm = cm < c
        x[tm], c[tm] = mid[tm], cm[tm]
        if optimal:
            A = [q[:, 0], q[:, 1], q[:, 2], q[:, 1], q[:, 4], q[:, 5], q[:, 2], q[:, 5], q[:, 7]]
            r = [-q[:, 3], -q[:, 6], -q[:, 8]]
            det = _det3(A)
            tr = (q[:, 0] + q[:, 4]) + q[:, 7]
            ok = np.abs(det) > ((tr * tr) * tr) * DEC_DET_TOL
            cols = []
            for j in range(3):
                m = list(A)
                m[j], m[3 + j], m[6 + j] = r
                cols.append(_det3(m) / det)
            xo = np.stack(cols, -1)
            x[ok] = xo[ok]
            c[ok] = _qform(q[ok], xo[ok])
        c = np.where(c <= 0, 0.0, c)                  # -0 and negatives to +0; NaN stays NaN
    return x, c


def _round_up_f32(c):
    with np.errstate(all="ignore"):
        c32 = c.astype(np.float32)
        up = c32.astype(np.float64) < c
        c32[up] = np.nextafter(c32[up], np.float32(np.inf))
    return c32


def _fans(f, live, V):
    """The per-vertex face lists of the live faces, sorted by (vertex, face, slot), and each entry's (p, q)."""
    lf = np.flatnonzero(live)
    ent_v = f[lf].reshape(-1)
    ent_f = np.repeat(lf, 3)
    ent_s = np.tile(np.arange(3), len(lf))
    order = np.argsort(ent_v, kind="stable")
    ev, ef, es = ent_v[order], ent_f[order], ent_s[order]
    start = np.searchsorted(ev, np.arange(V + 1))
    p = f[ef, (es + 1) % 3]
    q = f[ef, (es + 2) % 3]
    return start, ev, ef, p, q


def _regular(start, ev, ef, p, q, f, V):
    """k [V]: the valence of a regular vertex (rule 2: one closed, consistently oriented fan of 3 .. 32 faces with
    no repeated index), 0 for every other vertex."""
    k = np.diff(start)
    fdeg = (f[:, 0] == f[:, 1]) | (f[:, 1] == f[:, 2]) | (f[:, 0] == f[:, 2])
    bad = np.zeros(V, bool)
    bad[ev[fdeg[ef]]] = True
    out = np.zeros(V, np.int64)
    for kk in range(3, DEC_MAX_VALENCE + 1):
        vs = np.flatnonzero((k == kk) & ~bad)
        if not len(vs):
            continue
        idx = start[vs][:, None] + np.arange(kk)
        P, Qn = p[idx], q[idx]
        eq = Qn[:, :, None] == P[:, None, :]                 # [n, i, j]: target of i is the source of j
        found = eq.any(2).all(1)
        distinct = (np.diff(np.sort(P, 1), axis=1) != 0).all(1)
        succ = eq.argmax(2)
        cur = np.zeros(len(vs), np.int64)
        ok = found & distinct
        for t in range(1, kk):
            cur = succ[np.arange(len(vs)), cur]
            ok &= cur != 0
        ok &= succ[np.arange(len(vs)), cur] == 0
        out[vs[ok]] = kk
    return out


def _segments(starts, counts):
    """Flattened index arrays of the segments [starts, starts + counts) and each element's segment number."""
    seg = np.repeat(np.arange(len(starts)), counts)
    off = np.arange(counts.sum()) - np.repeat(np.cumsum(counts) - counts, counts)
    return seg, np.repeat(starts, counts) + off


def _candidates(a, b, k, start, p, q, pos, Q, optimal, V):
    """Rule 2 and 3 for edges a < b between regular vertices: -> (candidate mask, x, float32 cost)."""
    ok = k[a] + k[b] - 4 >= 3
    # link condition: |N(a) & N(b)| == 2
    reg = np.flatnonzero(k)
    rv, ridx = _segments(start[reg], k[reg])
    adj = np.sort(reg[rv] * (V + 1) + p[ridx])
    seg, idx = _segments(start[a], k[a])
    key = b[seg] * (V + 1) + p[idx]
    hit = adj[np.minimum(np.searchsorted(adj, key), len(adj) - 1)] == key
    ok &= np.bincount(seg, weights=hit, minlength=len(a)) == 2
    x, c = _placement(Q[a] + Q[b], pos[a], pos[b], optimal)
    ok &= ~np.isnan(c)
    # no flip: every face of a or b that survives keeps a positive dot product of its normals (zero-area: skipped)
    for moved, other in ((a, b), (b, a)):
        seg, idx = _segments(start[moved], k[moved])
        keep = (p[idx] != other[seg]) & (q[idx] != other[seg])
        seg, idx = seg[keep], idx[keep]
        pp, pq, pv = pos[p[idx]], pos[q[idx]], pos[moved[seg]]
        with np.errstate(all="ignore"):
            nb = _cross(pp - pv, pq - pv)
            na = _cross(pp - x[seg], pq - x[seg])
            good = (nb == 0).all(1) | (_dot(nb, na) > 0)
        ok &= np.bincount(seg, weights=~good, minlength=len(a)) == 0
    return ok, x, _round_up_f32(c)


def decimate_mesh(vertices, faces, target_faces, optimal_placement=True, return_rounds=False):
    """-> (vertices float32 [V',3], faces int32 [F',3], kept int32 [V']) of include/b200gsr_mesh_decimate.h, round by
    round; with return_rounds also the number of rounds that collapsed an edge."""
    v32 = np.ascontiguousarray(vertices, dtype=np.float32).reshape(-1, 3)
    V = len(v32)
    f = _faces(faces, V).copy()
    F, target = len(f), int(target_faces)
    pos = v32.astype(np.float64)
    moved = np.zeros(V, bool)
    live = np.ones(F, bool)
    # rule 1: vertex quadrics, each the sum of its faces' in face-index order
    start, ev, ef, p, q = _fans(f, live, V)
    fq = _face_quadrics(pos[f[:, 0]], pos[f[:, 1]], pos[f[:, 2]]) if F else np.zeros((0, 10))
    Q = np.zeros((V, 10))
    k = np.diff(start)
    for t in range(int(k.max()) if V else 0):
        vs = np.flatnonzero(k > t)
        Q[vs] = Q[vs] + fq[ef[start[vs] + t]]
    n_live, rounds = F, 0
    while n_live > target:
        start, ev, ef, p, q = _fans(f, live, V)
        k = _regular(start, ev, ef, p, q, f, V)
        seg, idx = _segments(start[:-1], k)                 # the fans of the regular vertices
        e = seg < p[idx]
        a, b = seg[e], p[idx][e]
        a, b = a[k[b] > 0], b[k[b] > 0]
        ok, x, c32 = _candidates(a, b, k, start, p, q, pos, Q, optimal_placement, V)
        a, b, x, c32 = a[ok], b[ok], x[ok], c32[ok]
        if not len(a):
            break
        order = np.lexsort((b, a, c32.view(np.uint32)))       # key order: (cost, a, b)
        rank = np.empty(len(a), np.int64)
        rank[order] = np.arange(len(a))
        m = np.full(V, len(a), np.int64)
        np.minimum.at(m, a, rank)
        np.minimum.at(m, b, rank)
        M = m.copy()
        np.minimum.at(M, seg, m[p[idx]])
        sel = np.flatnonzero((M[a] == rank) & (M[b] == rank))
        sel = sel[np.argsort(rank[sel])]
        need = (n_live - target + 1) // 2
        sel = sel[:need]
        sa, sb = a[sel], b[sel]
        remap = np.arange(V)
        remap[sb] = sa
        has_b = np.zeros(V, bool)
        has_b[sb] = True
        touched = live & has_b[f].any(1)
        nf = remap[f[touched]]
        dead = (nf[:, 0] == nf[:, 1]) | (nf[:, 1] == nf[:, 2]) | (nf[:, 0] == nf[:, 2])
        ti = np.flatnonzero(touched)
        f[ti] = nf
        live[ti[dead]] = False
        Q[sa] = Q[sa] + Q[sb]
        pos[sa] = x[sel]
        moved[sa] = True
        n_live -= 2 * len(sel)
        rounds += 1
    fl = f[live]
    ref = np.zeros(V, bool)
    ref[fl.reshape(-1)] = True
    kept = np.flatnonzero(ref)
    new_index = np.cumsum(ref) - 1
    out_v = np.where(moved[kept, None], pos[kept].astype(np.float32), v32[kept])
    out = (out_v, new_index[fl].astype(np.int32).reshape(-1, 3), kept.astype(np.int32))
    return out + (rounds,) if return_rounds else out
