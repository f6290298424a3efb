#!/usr/bin/env python
"""The mesh colour (include/b200gsr_mesh_colour.h) on the object layout of benchmarks/fields.py (1.2 M Gaussians in a
ball, 0.004 scales, colours uniform in [0, 1)), with num_blocks 16 and relax_ratio 1.5, at R = 128 and R = 256.

  fields     : extract_fields against extract_fields_rgb, the same field with the colour field beside it; the two are
               timed in alternation, so both see the same state of the card
  attributes : the attribute pass alone, b200gsr_mesh_attributes over the scratch of one b200gsr_mesh_count, on the
               object's field and colour field (CUDA events around --reps launches, per launch)
  mesh       : extract_coloured_mesh(group, R, iso) end to end, against extract_mesh(group, R, iso)

iso is half the maximum of the R = 128 field, the same at both resolutions (as benchmarks/mesh.py).  Call timings use
CUDA events around the call after one warm-up call, median and range over --reps calls; a call that reads back its
normalisation or totals includes that sync.  Peak memory is the peak allocated during one call above what was held
before it.  The `_features_dc` leaf comes from the same scene_render.object_layout group fields.object_group cuts
its four leaves from.

Prints one JSON line with the card's name, power limit and max SM clock.  Writes nothing to disk.

  python benchmarks/mesh_colour.py [--reps 10]
"""
import argparse
import ctypes as C
import json
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
from dreamscene_b200 import _lib  # noqa: E402
from dreamscene_b200.fields import extract_fields, extract_fields_rgb  # noqa: E402
from dreamscene_b200.mesh import extract_coloured_mesh, extract_mesh, marching_cubes  # noqa: E402
import fields as fields_bench  # noqa: E402  (benchmarks/fields.py: the card query)
import scene_render  # noqa: E402


def object_group(dev):
    groups, _, _ = scene_render.object_layout(dev)
    return {k: groups[0][k].detach() for k in ("_xyz", "_opacity", "_scaling", "_rotation", "_features_dc")}


def stats(ms):
    ms = sorted(ms)
    return dict(median_ms=round(ms[len(ms) // 2], 3), min_ms=round(ms[0], 3), max_ms=round(ms[-1], 3))


def event_ms(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    out = fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b), out


def peak_mb(fn):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    out = fn()
    peak = torch.cuda.max_memory_allocated() - base
    del out
    return round(peak / 2**20, 1)


def alternate(fns, reps):
    """{name: stats} of each call, the calls taken in turn rep by rep after one warm-up each."""
    for fn in fns.values():
        fn()
    torch.cuda.synchronize()
    ms = {name: [] for name in fns}
    for _ in range(reps):
        for name, fn in fns.items():
            t, out = event_ms(fn)
            del out
            ms[name].append(t)
    return {name: dict(**stats(v), peak_mb=peak_mb(fns[name])) for name, v in ms.items()}


def attribute_pass(occ, rgb, iso, reps):
    """Per-launch time of b200gsr_mesh_attributes after one b200gsr_mesh_count, and V."""
    lib = _lib.load()
    X, Y, Z = occ.shape
    layout = _lib.MeshLayout()
    _lib.check(lib.b200gsr_mesh_layout_query(X, Y, Z, C.byref(layout)), "b200gsr_mesh_layout_query")
    totals = torch.empty(2, dtype=torch.int32, device=occ.device)
    scratch = torch.empty(layout.total, dtype=torch.uint8, device=occ.device)
    ptr, st = _lib.ptr, _lib.stream(occ.device)
    _lib.check(lib.b200gsr_mesh_count(X, Y, Z, ptr(occ), iso, ptr(totals), ptr(scratch), scratch.numel(), st),
               "b200gsr_mesh_count")
    V = int(totals[0])
    out = torch.empty((V, 3), dtype=torch.float32, device=occ.device)

    def launch():
        _lib.check(lib.b200gsr_mesh_attributes(X, Y, Z, ptr(occ), iso, ptr(scratch), scratch.numel(), ptr(rgb),
                                               ptr(out), V, st), "b200gsr_mesh_attributes")

    launch()
    torch.cuda.synchronize()
    runs = []
    for _ in range(reps):
        t, _ = event_ms(lambda: [launch() for _ in range(20)])
        runs.append(t / 20)
    same = bool(torch.equal(out, marching_cubes(occ, iso, rgb)[2]))
    return dict(**stats(runs), V=V, same_as_marching_cubes=same)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "benchmarks/mesh_colour.py needs a GPU"
    dev = torch.device("cuda", 0)
    g = object_group(dev)
    occ128, _, _ = extract_fields(g, 128, 16, 1.5)
    iso = round(0.5 * float(occ128.max()), 4)
    del occ128
    out = dict(bench="mesh_colour", card=fields_bench.card(), rows=int(g["_xyz"].shape[0]), num_blocks=16,
               relax_ratio=1.5, iso=iso)
    for R in (128, 256):
        f = alternate(dict(extract_fields=lambda: extract_fields(g, R, 16, 1.5),
                           extract_fields_rgb=lambda: extract_fields_rgb(g, R, 16, 1.5)), args.reps)
        f["rgb_over_plain"] = round(f["extract_fields_rgb"]["median_ms"] / f["extract_fields"]["median_ms"], 3)
        out[f"fields_R{R}"] = f
        occ, rgb, _, _ = extract_fields_rgb(g, R, 16, 1.5)
        out[f"attributes_R{R}"] = attribute_pass(occ, rgb, iso, args.reps)
        del occ, rgb
        reps = max(2, args.reps // 3)
        m = alternate(dict(extract_mesh=lambda: extract_mesh(g, R, iso, 16, 1.5),
                           extract_coloured_mesh=lambda: extract_coloured_mesh(g, R, iso, 16, 1.5)), reps)
        v, f_, c = extract_coloured_mesh(g, R, iso, 16, 1.5)
        m["V"], m["F"] = len(v), len(f_)
        m["colour_min"], m["colour_max"] = round(float(c.min()), 4), round(float(c.max()), 4)
        del v, f_, c
        out[f"mesh_R{R}"] = m
        torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
