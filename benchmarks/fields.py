#!/usr/bin/env python
"""dreamscene_b200.fields.extract_fields against the reference's extract_fields restated in torch
(harness/fields_ref.py), on the object layout of benchmarks/scene_render.py (1.2 M Gaussians in a ball, 0.004 scales,
the synthetic harness).

  native : extract_fields(group, R, 16, 1.5) at R = 128 and R = 256, timed with CUDA events after one warm-up call,
           median and range over --reps calls; the peak allocated memory of a call above what was held before it
  torch  : the restatement on the same device, at R = 128, on the first --torch-rows rows and on all 1.2 M, each in a
           subprocess of its own with a deadline of --torch-timeout seconds: a run that does not finish is reported as
           "not measured", never extrapolated.  Host clock around the call, which ends in a device synchronise.

Prints one JSON line with the card's name, power limit and max SM clock.  Writes nothing to disk.

  python benchmarks/fields.py [--reps 5] [--torch-rows 100000] [--torch-timeout 600]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
from dreamscene_b200.fields import extract_fields  # noqa: E402
from harness import fields_ref  # noqa: E402
import scene_render  # noqa: E402


def card():
    try:
        return subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()),
                               "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        return torch.cuda.get_device_name()


def object_group(dev, rows=None):
    groups, _, _ = scene_render.object_layout(dev)
    g = {k: groups[0][k].detach() for k in ("_xyz", "_opacity", "_scaling", "_rotation")}
    return g if rows is None else {k: v[:rows].contiguous() for k, v in g.items()}


def time_native(g, R, reps):
    extract_fields(g, R, 16, 1.5)
    torch.cuda.synchronize()
    ms = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        occ, _, _ = extract_fields(g, R, 16, 1.5)
        b.record()
        torch.cuda.synchronize()
        ms.append(a.elapsed_time(b))
    del occ
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    occ, _, _ = extract_fields(g, R, 16, 1.5)
    peak = torch.cuda.max_memory_allocated() - base
    ms.sort()
    return dict(median_ms=round(ms[len(ms) // 2], 3), min_ms=round(ms[0], 3), max_ms=round(ms[-1], 3),
                peak_mb=round(peak / 2**20, 1), occ_mb=round(occ.numel() * 4 / 2**20, 1)), occ


def time_torch_subprocess(rows, R, timeout):
    cmd = [sys.executable, os.path.abspath(__file__), "--torch-run", str(rows), str(R)]
    try:
        out = subprocess.run(cmd, capture_output=True, text=True, timeout=timeout)
    except subprocess.TimeoutExpired:
        return dict(rows=rows, R=R, result=f"not measured (did not finish in {timeout} s)")
    lines = [ln for ln in out.stdout.splitlines() if ln.startswith("{")]
    if out.returncode != 0 or not lines:
        return dict(rows=rows, R=R, result="not measured (failed)", stderr=out.stderr[-400:])
    return json.loads(lines[-1])


def torch_run(rows, R):
    dev = torch.device("cuda", 0)
    g = object_group(dev, rows)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    ref, _, _ = fields_ref.extract_fields(g, R, 16, 1.5)
    torch.cuda.synchronize()
    s = time.perf_counter() - t0
    occ, _, _ = extract_fields(g, R, 16, 1.5)
    diff = float((occ - ref).abs().max())
    print(json.dumps(dict(rows=rows, R=R, torch_s=round(s, 2), max_abs_diff_vs_native=diff,
                          max_occ=float(ref.max()))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--torch-rows", type=int, default=100_000)
    ap.add_argument("--torch-timeout", type=int, default=600)
    ap.add_argument("--torch-run", nargs=2, type=int, help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.torch_run:
        torch_run(*args.torch_run)
        return
    assert torch.cuda.is_available(), "benchmarks/fields.py needs a GPU"
    dev = torch.device("cuda", 0)
    g = object_group(dev)
    out = dict(bench="extract_fields", card=card(), rows=int(g["_xyz"].shape[0]), num_blocks=16, relax_ratio=1.5)
    for R in (128, 256):
        res, occ = time_native(g, R, args.reps)
        out[f"native_R{R}"] = res
        del occ
    torch.cuda.empty_cache()
    out["torch_R128"] = [time_torch_subprocess(rows, 128, args.torch_timeout)
                         for rows in (args.torch_rows, out["rows"])]
    print(json.dumps(out))


if __name__ == "__main__":
    main()
