#!/usr/bin/env python
"""dreamscene_b200.mesh on the object layout of benchmarks/fields.py (1.2 M Gaussians in a ball, 0.004 scales), with
num_blocks 16 and relax_ratio 1.5.

  march   : marching_cubes(occ, iso) on the object's field at R = 128 and R = 256
  mesh    : extract_mesh(group, R, iso), the field evaluation and the march end to end, at R = 128 and R = 256
  numpy   : harness/mesh_ref.py's restatement of the march at R = 128, on the host: the alternative of copying the
            field to the host and marching it there.  Its output is checked against the native one.

iso is half the maximum of the R = 128 field (the object's field has no fixed scale; DreamGaussian's default of 1 lies
above it), the same iso at both resolutions.  The device timings use CUDA events around the call after one warm-up
call, median and range over --reps calls; a call includes its one read-back of the totals.  The host timing is a host
clock around one run.  Peak memory is the peak allocated during one call above what was held before it.

Prints one JSON line with the card's name, power limit and max SM clock.  Writes nothing to disk.

  python benchmarks/mesh.py [--reps 10]
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
from dreamscene_b200.mesh import extract_mesh, marching_cubes  # noqa: E402
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
    v, f = fn()
    peak = torch.cuda.max_memory_allocated() - base
    ms.sort()
    return dict(median_ms=round(ms[len(ms) // 2], 3), min_ms=round(ms[0], 3), max_ms=round(ms[-1], 3),
                peak_mb=round(peak / 2**20, 1), V=len(v), F=len(f))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "benchmarks/mesh.py needs a GPU"
    dev = torch.device("cuda", 0)
    g = fields_bench.object_group(dev)
    occ128, _, _ = extract_fields(g, 128, 16, 1.5)
    iso = round(0.5 * float(occ128.max()), 4)
    out = dict(bench="marching_cubes", card=fields_bench.card(), rows=int(g["_xyz"].shape[0]), num_blocks=16,
               relax_ratio=1.5, iso=iso)
    for R in (128, 256):
        occ = occ128 if R == 128 else extract_fields(g, R, 16, 1.5)[0]
        out[f"march_R{R}"] = timed(lambda: marching_cubes(occ, iso), args.reps)
        del occ
        out[f"mesh_R{R}"] = timed(lambda: extract_mesh(g, R, iso, 16, 1.5), max(2, args.reps // 3))
    host = occ128.cpu().numpy()
    t0 = time.perf_counter()
    rv, rf = mesh_ref.marching_cubes(host, np.float32(iso))
    s = time.perf_counter() - t0
    v, f = marching_cubes(occ128, iso)
    same = bool(np.array_equal(f.cpu().numpy(), rf) and np.array_equal(v.cpu().numpy().view(np.uint32),
                                                                       rv.view(np.uint32)))
    out["numpy_R128"] = dict(host_ms=round(1000 * s, 1), V=len(rv), F=len(rf), same_bits_as_native=same)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
