#!/usr/bin/env python
"""dreamscene_b200.mesh.decimate_mesh on the marching-cubes meshes of the object layout of benchmarks/fields.py (1.2 M
Gaussians in a ball, 0.004 scales; num_blocks 16, relax_ratio 1.5), at R = 128 and R = 256, to 100,000 faces and to
10 % of F (pymeshlab's default target in DreamGaussian's export, and a fixed fraction).

  device : decimate_mesh(v, f, target) with optimal placement; CUDA events around the whole call after one warm-up
           call, median and range over --reps calls (a call includes its status read-backs); rounds and ms per round
  host   : harness/mesh_ref.py's restatement at R = 128 on the host, a host clock around one run with the mesh already
           on the host, and whether it gives the same bits as the native call

iso is half the maximum of the R = 128 field at both resolutions (benchmarks/mesh.py's choice).  Peak memory is the
peak allocated during one call above what was held before it.  Prints one JSON line with the card's name, power limit
and max SM clock.  Writes nothing to disk.

  python benchmarks/mesh_decimate.py [--reps 10]
"""
import argparse
import ctypes as C
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
from dreamscene_b200.mesh import decimate_mesh, marching_cubes  # noqa: E402
from harness import mesh_ref  # noqa: E402
import fields as fields_bench  # noqa: E402  (benchmarks/fields.py: the object group and the card query)
from mesh_clean import timed  # noqa: E402  (benchmarks/mesh_clean.py: events, range and peak memory)
from dreamscene_b200 import _lib  # noqa: E402


def native_rounds(v, f, target):
    """The round count of the status record: decimate_mesh's own calls, run to the end."""
    lib, V, F, dev = _lib.load(), len(v), len(f), v.device
    n = C.c_size_t(0)
    _lib.check(lib.b200gsr_mesh_decimate_layout_query(V, F, C.byref(n)), "layout")
    st = torch.empty(_lib.DECIMATE_STATUS_WORDS, dtype=torch.int32, device=dev)
    scr = torch.empty(int(n.value), dtype=torch.uint8, device=dev)
    s, p = _lib.stream(dev), _lib.ptr
    _lib.check(lib.b200gsr_mesh_decimate_begin(V, F, p(v), p(f), target, 1, p(st), p(scr), n.value, s), "begin")
    while not st.tolist()[2]:
        _lib.check(lib.b200gsr_mesh_decimate_rounds(V, F, 8, p(st), p(scr), n.value, s), "rounds")
    return st.tolist()[1]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "benchmarks/mesh_decimate.py needs a GPU"
    dev = torch.device("cuda", 0)
    g = fields_bench.object_group(dev)
    occ128, _, _ = extract_fields(g, 128, 16, 1.5)
    iso = round(0.5 * float(occ128.max()), 4)
    out = dict(bench="mesh_decimate", card=fields_bench.card(), rows=int(g["_xyz"].shape[0]), num_blocks=16,
               relax_ratio=1.5, iso=iso)
    for R in (128, 256):
        occ = occ128 if R == 128 else extract_fields(g, R, 16, 1.5)[0]
        v, f = marching_cubes(occ, iso)
        del occ
        res = dict(V=len(v), F=len(f))
        hv, hf = v.cpu().numpy(), f.cpu().numpy()
        for name, target in (("to_100k", 100_000), ("to_10pct", len(f) // 10)):
            r = timed(lambda: decimate_mesh(v, f, target), args.reps)
            if R == 128 and name == "to_10pct":
                t0 = time.perf_counter()
                rv, rf, rk = mesh_ref.decimate_mesh(hv, hf, target, True)
                r["host_ms"] = round(1000 * (time.perf_counter() - t0), 1)
                nv, nf, nk = decimate_mesh(v, f, target)
                r["same_bits_as_restatement"] = bool(
                    np.array_equal(nv.cpu().numpy().view(np.int32), rv.view(np.int32)) and
                    np.array_equal(nf.cpu().numpy(), rf) and np.array_equal(nk.cpu().numpy(), rk))
            rounds = native_rounds(v, f, target)
            r.update(target=target, rounds=rounds, ms_per_round=round(r["median_ms"] / max(rounds, 1), 3))
            res[name] = r
        out[f"R{R}"] = res
    print(json.dumps(out))


if __name__ == "__main__":
    main()
