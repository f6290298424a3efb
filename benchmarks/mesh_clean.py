#!/usr/bin/env python
"""dreamscene_b200.mesh.mesh_components and clean_mesh on the marching-cubes meshes of the object layout of
benchmarks/fields.py (1.2 M Gaussians in a ball, 0.004 scales; num_blocks 16, relax_ratio 1.5), at R = 128 and R = 256.

  mesh_components : mesh_components(faces, V); `components` counts the components with a face
  defaults        : clean_mesh(v, f), which returns a marching-cubes mesh unchanged
  floaters        : clean_mesh(v, f, min_faces=64, min_diameter=0.1)
  largest         : clean_mesh(v, f, keep_largest=True)
  host            : harness/mesh_ref.py's restatement of `floaters` (scipy connected_components and numpy) on the
                    host, a host clock around one run with the mesh already on the host: the alternative of copying
                    the mesh to the host and cleaning it there.  Checked to give the same bits as the native call.

iso is half the maximum of the R = 128 field, the same iso at both resolutions (benchmarks/mesh.py's choice).  The
device timings use CUDA events around the call after one warm-up call, median and range over --reps calls; a call
includes its one read-back of the totals.  Peak memory is the peak allocated during one call above what was held
before it.  Prints one JSON line with the card's name, power limit and max SM clock.  Writes nothing to disk.

  python benchmarks/mesh_clean.py [--reps 20]
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
from dreamscene_b200.fields import extract_fields  # noqa: E402
from dreamscene_b200.mesh import clean_mesh, marching_cubes, mesh_components  # noqa: E402
from harness import mesh_ref  # noqa: E402
import fields as fields_bench  # noqa: E402  (benchmarks/fields.py: the object group and the card query)


def timed(fn, reps):
    out = fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        out = fn()
        b.record()
        torch.cuda.synchronize()
        ms.append(a.elapsed_time(b))
    del out
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    out = fn()
    peak = torch.cuda.max_memory_allocated() - base
    ms.sort()
    res = dict(median_ms=round(ms[len(ms) // 2], 3), min_ms=round(ms[0], 3), max_ms=round(ms[-1], 3),
               peak_mb=round(peak / 2**20, 1))
    if isinstance(out, tuple):
        res.update(V_out=len(out[0]), F_out=len(out[1]))
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "benchmarks/mesh_clean.py needs a GPU"
    dev = torch.device("cuda", 0)
    g = fields_bench.object_group(dev)
    occ128, _, _ = extract_fields(g, 128, 16, 1.5)
    iso = round(0.5 * float(occ128.max()), 4)
    out = dict(bench="mesh_clean", card=fields_bench.card(), rows=int(g["_xyz"].shape[0]), num_blocks=16,
               relax_ratio=1.5, iso=iso)
    floaters = dict(min_faces=64, min_diameter=0.1)
    for R in (128, 256):
        occ = occ128 if R == 128 else extract_fields(g, R, 16, 1.5)[0]
        v, f = marching_cubes(occ, iso)
        del occ
        V = len(v)
        lab = mesh_components(f, V)
        res = dict(V=V, F=len(f), components=int(torch.unique(lab[f[:, 0].long()]).numel()))
        res["mesh_components"] = timed(lambda: mesh_components(f, V), args.reps)
        res["defaults"] = timed(lambda: clean_mesh(v, f), args.reps)
        res["floaters"] = timed(lambda: clean_mesh(v, f, **floaters), args.reps)
        res["largest"] = timed(lambda: clean_mesh(v, f, keep_largest=True), args.reps)
        hv, hf = v.cpu().numpy(), f.cpu().numpy()
        t0 = time.perf_counter()
        rv, rf, rk = mesh_ref.clean_mesh(hv, hf, **floaters)
        s = time.perf_counter() - t0
        nv, nf, nk = clean_mesh(v, f, **floaters)
        same = bool(np.array_equal(nv.cpu().numpy().view(np.uint32), rv.view(np.uint32)) and
                    np.array_equal(nf.cpu().numpy(), rf) and np.array_equal(nk.cpu().numpy(), rk))
        res["host"] = dict(host_ms=round(1000 * s, 1), V_out=len(rv), F_out=len(rf))
        res["same_bits_as_restatement"] = same
        out[f"R{R}"] = res
    print(json.dumps(out))


if __name__ == "__main__":
    main()
