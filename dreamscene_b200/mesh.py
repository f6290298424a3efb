"""Triangle meshes from volumes on the device: marching cubes (include/b200gsr_mesh.h), and the mesh of a Gaussian
group's opacity field.

``marching_cubes(volume, iso)`` puts a vertex on every grid edge the iso-surface crosses, at the same position as
``mcubes.marching_cubes(volume, iso)`` does, and triangulates each cell from a cube table generated from one face rule,
so the surface is crack-free and consistently oriented (counter-clockwise seen from outside, the OBJ / PLY convention).
The triangulation is not mcubes' table, so the faces differ from mcubes' faces.  ``extract_mesh(group)`` evaluates the
group's opacity field with ``fields.extract_fields`` and marches it, without the field leaving the device.
``marching_cubes(volume, iso, attributes)`` also interpolates a per-point attribute volume onto the vertices, and
``extract_coloured_mesh(group)`` uses it to colour the mesh with ``fields.extract_fields_rgb``'s colour field.
``mesh_components(faces, V)`` labels a mesh's connected components and ``clean_mesh(vertices, faces)`` removes the
small ones (include/b200gsr_mesh_clean.h), the floaters low-opacity Gaussians leave around an object.
``decimate_mesh(vertices, faces, target_faces)`` reduces a mesh to a target face count by quadric edge collapse
(include/b200gsr_mesh_decimate.h), as DreamGaussian's export does with pymeshlab before writing the mesh.
"""
from __future__ import annotations

import ctypes as C
import math
from numbers import Integral, Real
from typing import Optional, Tuple

import torch

from . import _lib
from .fields import extract_fields, extract_fields_rgb


def marching_cubes(volume: torch.Tensor, iso: float, attributes: Optional[torch.Tensor] = None):
    """The iso-surface of a float32 CUDA volume [X,Y,Z] at `iso`.

    -> (vertices float32 CUDA [V,3], faces int32 CUDA [F,3]).  Vertices are in index space: the vertex on the edge
    from grid point p along axis a is p with coordinate a replaced by p_a + (iso - v[p]) / (v[p + e_a] - v[p]), each
    operation rounded to float32.  There is one vertex per crossing edge, shared by the cells around it, ordered by
    the grid point's linear index and then the axis; faces come cell by cell in linear order.  A point is inside when
    its value is > iso (NaN is outside); iso is rounded to float32.  A dimension below 2, or an iso nothing crosses,
    gives V = F = 0.  Two calls give the same bits.

    Refused with ValueError: a CPU tensor, a volume that is not 3-D or not float32, a dimension above 1024 or a grid
    too large to index with int32 (3 X Y Z >= 2^31), and a non-finite iso.  The call reads the two totals back to
    allocate the outputs, so it waits for the device and cannot be captured into a CUDA graph (RuntimeError).

    attributes: None, or a float32 CUDA tensor [X,Y,Z,3] on the volume's device, a value per grid point (a colour,
    say).  Then the call returns (vertices, faces, vertex_attributes float32 CUDA [V,3]): the vertex on the edge from p
    along axis a gets attributes[p] + t * (attributes[p + e_a] - attributes[p]) per channel, with the vertex's t and
    each operation rounded to float32; a NaN t gives a NaN attribute.  It makes no further host sync.  A wrong shape,
    dtype or device of attributes is refused with ValueError before any device work."""
    if not isinstance(volume, torch.Tensor):
        raise ValueError(f"marching_cubes: volume must be a torch tensor, got {type(volume).__name__}")
    if volume.dim() != 3:
        raise ValueError(f"marching_cubes: volume must be 3-D [X,Y,Z], got shape {tuple(volume.shape)}")
    if volume.dtype != torch.float32:
        raise ValueError(f"marching_cubes: volume must be float32, got {volume.dtype}")
    if volume.device.type != "cuda":
        raise ValueError("marching_cubes (b200gsr): volume must be a CUDA tensor; there is no CPU fallback")
    if torch.cuda.is_current_stream_capturing():
        raise RuntimeError("marching_cubes reads its totals back to the host, so it cannot be captured into a CUDA graph")
    X, Y, Z = (int(d) for d in volume.shape)
    dev = volume.device
    if attributes is not None:
        if not isinstance(attributes, torch.Tensor):
            raise ValueError(f"marching_cubes: attributes must be a torch tensor, got {type(attributes).__name__}")
        if tuple(attributes.shape) != (X, Y, Z, 3):
            raise ValueError(f"marching_cubes: attributes have shape {tuple(attributes.shape)}, "
                             f"expected {(X, Y, Z, 3)}")
        if attributes.dtype != torch.float32:
            raise ValueError(f"marching_cubes: attributes must be float32, got {attributes.dtype}")
        if attributes.device != dev:
            raise ValueError(f"marching_cubes (b200gsr): attributes must be a CUDA tensor on the volume's device "
                             f"{dev}; there is no CPU fallback")
    lib = _lib.load()
    layout = _lib.MeshLayout()
    _lib.check(lib.b200gsr_mesh_layout_query(X, Y, Z, C.byref(layout)), "b200gsr_mesh_layout_query", ValueError)
    with torch.no_grad(), torch.cuda.device(dev):
        vol = volume.detach().contiguous()
        totals = torch.empty(2, dtype=torch.int32, device=dev)
        scratch = torch.empty(layout.total, dtype=torch.uint8, device=dev)
        ptr, st = _lib.ptr, _lib.stream(dev)
        _lib.check(lib.b200gsr_mesh_count(X, Y, Z, ptr(vol), iso, ptr(totals), ptr(scratch), scratch.numel(), st),
                   "b200gsr_mesh_count", ValueError)
        V, F = (int(n) for n in totals.tolist())          # the call's one host sync
        vertices = torch.empty((V, 3), dtype=torch.float32, device=dev)
        faces = torch.empty((F, 3), dtype=torch.int32, device=dev)
        if V:
            _lib.check(lib.b200gsr_mesh_emit(X, Y, Z, ptr(vol), iso, ptr(scratch), scratch.numel(), ptr(vertices), V,
                                             ptr(faces), F, st), "b200gsr_mesh_emit", ValueError)
        if attributes is None:
            return vertices, faces
        attr = attributes.detach().contiguous()
        out = torch.empty((V, 3), dtype=torch.float32, device=dev)
        if V:
            _lib.check(lib.b200gsr_mesh_attributes(X, Y, Z, ptr(vol), iso, ptr(scratch), scratch.numel(), ptr(attr),
                                                   ptr(out), V, st), "b200gsr_mesh_attributes", ValueError)
    return vertices, faces, out


def extract_mesh(group, resolution: int = 128, iso: float = 1.0, num_blocks: int = 16,
                 relax_ratio: float = 1.5) -> Tuple[torch.Tensor, torch.Tensor]:
    """The mesh of a Gaussian group's opacity field: extract_fields(group, resolution, num_blocks, relax_ratio), then
    marching_cubes(occ, iso), as DreamGaussian's extract_mesh does with mcubes on the host.

    group accepts what extract_fields accepts (a plain group or ReservedGroup.rows()) and is refused as it refuses.
    -> (vertices float32 CUDA [V,3] in world space, faces int32 CUDA [F,3]): the index-space vertices v mapped with
    torch float32 operations as (v / (R - 1) * 2 - 1) / scale + center, the normalisation extract_fields returns.
    Same faces and orientation as marching_cubes.  Waits for the device; no gradients."""
    occ, center, scale = extract_fields(group, resolution, num_blocks, relax_ratio)
    vertices, faces = marching_cubes(occ, iso)
    return (vertices / (int(resolution) - 1) * 2 - 1) / scale + center, faces


def extract_coloured_mesh(group, resolution: int = 128, iso: float = 1.0, num_blocks: int = 16,
                          relax_ratio: float = 1.5) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """The mesh of extract_mesh(group, resolution, iso, num_blocks, relax_ratio), coloured.

    extract_fields_rgb evaluates the opacity field and the colour field in one pass, and marching_cubes(occ, iso, rgb)
    interpolates the colour field onto the vertices.  group accepts what extract_fields_rgb accepts (it needs
    _features_dc [P,1,3]) and is refused as it refuses.
    -> (vertices float32 CUDA [V,3] in world space, faces int32 CUDA [F,3], colours float32 CUDA [V,3]): vertices and
    faces bit for bit extract_mesh's.  The colours are view-independent (each Gaussian's degree-0 SH colour, clamped
    at 0 as the renderer clamps it) and not clamped above 1.  Waits for the device; no gradients."""
    occ, rgb, center, scale = extract_fields_rgb(group, resolution, num_blocks, relax_ratio)
    vertices, faces, colours = marching_cubes(occ, iso, rgb)
    return (vertices / (int(resolution) - 1) * 2 - 1) / scale + center, faces, colours


def _faces_arg(faces, what: str) -> None:
    if not isinstance(faces, torch.Tensor):
        raise ValueError(f"{what}: faces must be a torch tensor, got {type(faces).__name__}")
    if faces.dim() != 2 or faces.shape[1] != 3:
        raise ValueError(f"{what}: faces must be [F,3], got shape {tuple(faces.shape)}")
    if faces.dtype != torch.int32:
        raise ValueError(f"{what}: faces must be int32, got {faces.dtype}")


def _on_cuda(t: torch.Tensor, name: str, what: str) -> None:
    if t.device.type != "cuda":
        raise ValueError(f"{what} (b200gsr): {name} must be a CUDA tensor; there is no CPU fallback")


def _no_capture(what: str) -> None:
    if torch.cuda.is_current_stream_capturing():
        raise RuntimeError(f"{what} reads its totals back to the host, so it cannot be captured into a CUDA graph")


def _bad_faces(what: str, bad: int, V: int) -> None:
    if bad:
        raise ValueError(f"{what}: {bad} face(s) have a vertex index outside [0, {V})")


def _scratch_bytes(lib, V: int, F: int, what: str) -> int:
    n = C.c_size_t(0)
    _lib.check(lib.b200gsr_mesh_clean_layout_query(V, F, C.byref(n)), what, ValueError)
    return int(n.value)


def mesh_components(faces: torch.Tensor, num_vertices: int) -> torch.Tensor:
    """The connected components of a triangle mesh with `num_vertices` vertices: int32 CUDA labels [V].

    Two vertices are connected when some face contains both; a vertex's label is the smallest vertex index in its
    component, so a vertex no face references is labelled with its own index.  faces: int32 CUDA [F,3] (marching_cubes'
    faces, say).  Two calls give the same labels.

    Refused with ValueError: faces that are not an int32 CUDA tensor [F,3], num_vertices not an integer in
    [0, 2^31), 3 F >= 2^31, and a face index outside [0, V) (checked on the device and read back: the call's one host
    sync, so it cannot be captured into a CUDA graph, RuntimeError)."""
    if isinstance(num_vertices, bool) or not isinstance(num_vertices, Integral) or not 0 <= num_vertices < 2**31:
        raise ValueError(f"mesh_components: num_vertices must be an integer in [0, 2^31), got {num_vertices!r}")
    _faces_arg(faces, "mesh_components")
    _on_cuda(faces, "faces", "mesh_components")
    _no_capture("mesh_components")
    V, F, dev = int(num_vertices), int(faces.shape[0]), faces.device
    if V == 0:
        _bad_faces("mesh_components", F, V)
        return torch.empty(0, dtype=torch.int32, device=dev)
    lib = _lib.load()
    nbytes = _scratch_bytes(lib, V, F, "b200gsr_mesh_clean_layout_query")
    with torch.no_grad(), torch.cuda.device(dev):
        f = faces.detach().contiguous()
        labels = torch.empty(V, dtype=torch.int32, device=dev)
        bad = torch.empty(1, dtype=torch.int32, device=dev)
        scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        ptr = _lib.ptr
        _lib.check(lib.b200gsr_mesh_components(V, F, ptr(f), ptr(labels), ptr(bad), ptr(scratch), nbytes,
                                               _lib.stream(dev)), "b200gsr_mesh_components", ValueError)
        _bad_faces("mesh_components", int(bad.item()), V)   # the call's one host sync
    return labels


def clean_mesh(vertices: torch.Tensor, faces: torch.Tensor, *, min_faces: int = 1, min_diameter: float = 0.0,
               keep_largest: bool = False) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """Remove a mesh's small connected components (the floaters), as DreamGaussian's clean_mesh does with pymeshlab's
    "remove connected components by face count / by diameter" filters.

    vertices float32 CUDA [V,3], faces int32 CUDA [F,3] on the same device.  Components are mesh_components'.  A
    component with a face is kept when it has at least `min_faces` faces, when min_diameter is 0 or its box diagonal is
    at least min_diameter times the diagonal of all referenced vertices (float64, see include/b200gsr_mesh_clean.h;
    NaN coordinates are skipped), and, with keep_largest, when it also has the most faces of those passing (ties to the
    smallest label).
    -> (vertices float32 CUDA [V',3], faces int32 CUDA [F',3], kept int32 CUDA [V']): the referenced vertices of the
    kept components in input order, their bits unchanged, kept their input indices, and the kept components' faces in
    input order renumbered into them.  Carry per-vertex data with data[kept].  Unreferenced vertices are always
    dropped, so the defaults return a mesh whose vertices are all referenced unchanged, kept = arange(V).  Two calls
    give the same bits; no gradients.

    Refused with ValueError: wrong types, shapes, dtypes or devices; min_faces not an integer in [0, 2^31);
    min_diameter negative or not finite; 3 F >= 2^31; a face index outside [0, V) (found on the device: the call reads
    its totals back once, before the outputs are allocated, so it cannot be captured into a CUDA graph, RuntimeError)."""
    if isinstance(min_faces, bool) or not isinstance(min_faces, Integral) or not 0 <= min_faces < 2**31:
        raise ValueError(f"clean_mesh: min_faces must be an integer in [0, 2^31), got {min_faces!r}")
    if isinstance(min_diameter, bool) or not isinstance(min_diameter, Real) or not math.isfinite(min_diameter) \
            or min_diameter < 0:
        raise ValueError(f"clean_mesh: min_diameter must be a finite number >= 0, got {min_diameter!r}")
    if not isinstance(keep_largest, bool):
        raise ValueError(f"clean_mesh: keep_largest must be a bool, got {keep_largest!r}")
    if not isinstance(vertices, torch.Tensor):
        raise ValueError(f"clean_mesh: vertices must be a torch tensor, got {type(vertices).__name__}")
    if vertices.dim() != 2 or vertices.shape[1] != 3:
        raise ValueError(f"clean_mesh: vertices must be [V,3], got shape {tuple(vertices.shape)}")
    if vertices.dtype != torch.float32:
        raise ValueError(f"clean_mesh: vertices must be float32, got {vertices.dtype}")
    _faces_arg(faces, "clean_mesh")
    _on_cuda(vertices, "vertices", "clean_mesh")
    _on_cuda(faces, "faces", "clean_mesh")
    if faces.device != vertices.device:
        raise ValueError(f"clean_mesh: faces are on {faces.device}, vertices on {vertices.device}")
    _no_capture("clean_mesh")
    V, F, dev = int(vertices.shape[0]), int(faces.shape[0]), vertices.device
    if V == 0:
        _bad_faces("clean_mesh", F, V)
        return (torch.empty((0, 3), dtype=torch.float32, device=dev), torch.empty((0, 3), dtype=torch.int32, device=dev),
                torch.empty(0, dtype=torch.int32, device=dev))
    lib = _lib.load()
    nbytes = _scratch_bytes(lib, V, F, "b200gsr_mesh_clean_layout_query")
    args = (int(min_faces), float(min_diameter), int(keep_largest))
    with torch.no_grad(), torch.cuda.device(dev):
        v = vertices.detach().contiguous()
        f = faces.detach().contiguous()
        totals = torch.empty(3, dtype=torch.int32, device=dev)
        scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        ptr, st = _lib.ptr, _lib.stream(dev)
        _lib.check(lib.b200gsr_mesh_clean_count(V, F, ptr(v), ptr(f), *args, ptr(totals), ptr(scratch), nbytes, st),
                   "b200gsr_mesh_clean_count", ValueError)
        V_out, F_out, bad = (int(n) for n in totals.tolist())      # the call's one host sync
        _bad_faces("clean_mesh", bad, V)
        out_v = torch.empty((V_out, 3), dtype=torch.float32, device=dev)
        out_f = torch.empty((F_out, 3), dtype=torch.int32, device=dev)
        kept = torch.empty(V_out, dtype=torch.int32, device=dev)
        if V_out:
            _lib.check(lib.b200gsr_mesh_clean_emit(V, F, ptr(v), ptr(f), *args, ptr(scratch), nbytes, ptr(out_v),
                                                   ptr(out_f), ptr(kept), V_out, F_out, st),
                       "b200gsr_mesh_clean_emit", ValueError)
    return out_v, out_f, kept


DECIMATE_BATCH = 8          # rounds per b200gsr_mesh_decimate_rounds call: one status read-back each


def decimate_mesh(vertices: torch.Tensor, faces: torch.Tensor, target_faces: int, *,
                  optimal_placement: bool = True) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """Reduce a mesh to `target_faces` faces by quadric edge collapse, as DreamGaussian's decimate_mesh does with
    pymeshlab's meshing_decimation_quadric_edge_collapse (include/b200gsr_mesh_decimate.h states every rule).

    vertices float32 CUDA [V,3], faces int32 CUDA [F,3] on the same device.  Each face's plane quadric, weighted by its
    area, is summed per vertex in float64; edges are collapsed in rounds of independent edges, each round's cheapest
    edges first.  An edge collapses only between two vertices whose faces form one closed, consistently oriented fan,
    when the two share exactly two neighbours, when the result keeps valence >= 3 and when no surviving face turns
    over, so boundaries, non-manifold parts and each component's topology stay as they are.  With optimal_placement the
    survivor moves to the quadric's minimum (Cramer's rule, falling back to the best of the two ends and the midpoint
    when the system is near singular), without it to that best of three.  Rounds run while F > target_faces and an
    edge can collapse; the last round applies only the cheapest of its edges, so F' is target_faces or
    target_faces - 1 unless the mesh runs out of collapsible edges first.
    -> (vertices float32 CUDA [V',3], faces int32 CUDA [F',3], kept int32 CUDA [V']): the surviving referenced
    vertices in input order, kept their input indices (carry per-vertex data with data[kept]; a vertex that absorbed
    others carries its own index), and the surviving faces in input order, renumbered.  With F <= target_faces, or no
    collapsible edge, this is clean_mesh(vertices, faces).  Two calls give the same bits; no gradients.

    The rounds run DECIMATE_BATCH (8) at a time on the device; after each batch the call reads back one status record,
    so it waits for the device 1 + ceil(rounds / 8) times (a tenfold reduction of the object meshes in
    BASELINE.md takes about 30 rounds), and it cannot be captured into a CUDA graph (RuntimeError).
    Refused with ValueError: what clean_mesh refuses; target_faces not an integer in [0, 2^31); optimal_placement not
    a bool; a face index outside [0, V) (found on the device)."""
    if isinstance(target_faces, bool) or not isinstance(target_faces, Integral) or not 0 <= target_faces < 2**31:
        raise ValueError(f"decimate_mesh: target_faces must be an integer in [0, 2^31), got {target_faces!r}")
    if not isinstance(optimal_placement, bool):
        raise ValueError(f"decimate_mesh: optimal_placement must be a bool, got {optimal_placement!r}")
    if not isinstance(vertices, torch.Tensor):
        raise ValueError(f"decimate_mesh: vertices must be a torch tensor, got {type(vertices).__name__}")
    if vertices.dim() != 2 or vertices.shape[1] != 3:
        raise ValueError(f"decimate_mesh: vertices must be [V,3], got shape {tuple(vertices.shape)}")
    if vertices.dtype != torch.float32:
        raise ValueError(f"decimate_mesh: vertices must be float32, got {vertices.dtype}")
    _faces_arg(faces, "decimate_mesh")
    _on_cuda(vertices, "vertices", "decimate_mesh")
    _on_cuda(faces, "faces", "decimate_mesh")
    if faces.device != vertices.device:
        raise ValueError(f"decimate_mesh: faces are on {faces.device}, vertices on {vertices.device}")
    _no_capture("decimate_mesh")
    V, F, dev = int(vertices.shape[0]), int(faces.shape[0]), vertices.device
    if V == 0:
        _bad_faces("decimate_mesh", F, V)
        return (torch.empty((0, 3), dtype=torch.float32, device=dev), torch.empty((0, 3), dtype=torch.int32, device=dev),
                torch.empty(0, dtype=torch.int32, device=dev))
    lib = _lib.load()
    n = C.c_size_t(0)
    _lib.check(lib.b200gsr_mesh_decimate_layout_query(V, F, C.byref(n)), "b200gsr_mesh_decimate_layout_query",
               ValueError)
    nbytes = int(n.value)
    with torch.no_grad(), torch.cuda.device(dev):
        v = vertices.detach().contiguous()
        f = faces.detach().contiguous()
        status = torch.empty(_lib.DECIMATE_STATUS_WORDS, dtype=torch.int32, device=dev)
        scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        ptr, st = _lib.ptr, _lib.stream(dev)
        _lib.check(lib.b200gsr_mesh_decimate_begin(V, F, ptr(v), ptr(f), int(target_faces), int(optimal_placement),
                                                   ptr(status), ptr(scratch), nbytes, st),
                   "b200gsr_mesh_decimate_begin", ValueError)
        _, _, done, bad, V_out, F_out = status.tolist()
        _bad_faces("decimate_mesh", bad, V)
        while not done:
            _lib.check(lib.b200gsr_mesh_decimate_rounds(V, F, DECIMATE_BATCH, ptr(status), ptr(scratch), nbytes, st),
                       "b200gsr_mesh_decimate_rounds", ValueError)
            _, _, done, _, V_out, F_out = status.tolist()
        out_v = torch.empty((V_out, 3), dtype=torch.float32, device=dev)
        out_f = torch.empty((F_out, 3), dtype=torch.int32, device=dev)
        kept = torch.empty(V_out, dtype=torch.int32, device=dev)
        if V_out:
            _lib.check(lib.b200gsr_mesh_decimate_emit(V, F, ptr(v), ptr(scratch), nbytes, ptr(out_v), ptr(out_f),
                                                      ptr(kept), V_out, F_out, st),
                       "b200gsr_mesh_decimate_emit", ValueError)
    return out_v, out_f, kept
