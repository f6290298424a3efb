#!/usr/bin/env python
"""Adam step cost: torch.optim.Adam's default (foreach) path, torch.optim.Adam(fused=True) and
dreamscene_b200.GaussianAdam on two parameter layouts, timed in one process with the variants alternating.

  object : one GaussianModel of 1.2 M Gaussians at M = 16 with the reference's seven groups (background without a
           gradient, as in training): 59 floats per Gaussian, 70.8 M elements per step.
  scene  : the scene of harness/room.py (walls + ceiling, floor, four objects; 2.63 M Gaussians, M = 4),
           one optimizer per GaussianModel as in the reference: six step() calls per training step.

Each variant owns a copy of the parameters, moments and (fixed, random) gradients.  One repetition times --steps
back-to-back steps between device events; the variants take turns, in alternating order, for --repeats rounds, so
load from other work on the GPU falls on all of them alike.  Reported per variant: the median ms per step over the
repetitions with the interquartile range and the extremes, the device time of the step's kernels (torch profiler,
separate pass), the host time of one step() call, and GB/s against the 28 B/element model of a single pass (read
p, g, m, v; write p, m, v).  After the run, GaussianAdam's parameters and moments are compared bitwise with the
default path's: both took the same steps with the same gradients.

  python benchmarks/optimizer.py [--layout object scene] [--steps 50] [--repeats 15]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch
from torch import nn

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from dreamscene_b200 import GaussianAdam  # noqa: E402
from harness.adam_ref import reference_adam  # noqa: E402

BYTES_PER_ELEMENT = 28
VARIANTS = ("torch_default", "torch_fused", "native")


def object_models(dev, P=1_200_000, M=16):
    return [dict(xyz=(P, 3), f_dc=(P, 1, 3), f_rest=(P, M - 1, 3), opacity=(P, 1), scaling=(P, 3), rotation=(P, 4),
                 background=(3, 1, 1))]


def scene_models(dev):
    from harness.room import build_scene
    shapes = [{k: tuple(v.shape) for k, v in g.items()} for g in build_scene(dev)]
    for s in shapes:
        s["background"] = (3, 1, 1)
    return shapes


def make_variant(name, shapes, seed, dev):
    """-> (optimizers, params): one optimizer per model, every parameter but the background with a gradient."""
    gen = torch.Generator(device=dev).manual_seed(seed)
    opts, params = [], []
    for shp in shapes:
        ps = {k: nn.Parameter(torch.randn(s, device=dev, generator=gen)) for k, s in shp.items()}
        for k, p in ps.items():
            p.grad = None if k == "background" else torch.randn(p.shape, device=dev, generator=gen) * 1e-3
        if name == "native":
            opts.append(reference_adam(ps, GaussianAdam))
        else:
            opts.append(reference_adam(ps, fused=True) if name == "torch_fused" else reference_adam(ps))
        params.append(ps)
    return opts, params


def step_all(opts):
    for o in opts:
        o.step()


def device_ms(opts, steps=5):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            step_all(opts)
        torch.cuda.synchronize()
    from torch.autograd import DeviceType
    evs = [e for e in prof.events() if e.device_type == DeviceType.CUDA]
    return sum(e.time_range.elapsed_us() for e in evs) / 1e3 / steps, len(evs) / steps


def host_us(opts, steps=20):
    """Host time of one training step's step() calls: the time to enqueue, with the device kept idle first."""
    out = []
    for _ in range(steps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        step_all(opts)
        out.append(time.perf_counter() - t0)
    torch.cuda.synchronize()
    return float(np.median(out)) * 1e6


def bench_layout(name, shapes, a, dev):
    elements = sum(int(np.prod(s)) for shp in shapes for k, s in shp.items() if k != "background")
    variants = {v: make_variant(v, shapes, seed=1, dev=dev) for v in VARIANTS}
    for v in VARIANTS:                                    # warm-up: state creation, module load
        for _ in range(a.warmup):
            step_all(variants[v][0])
    torch.cuda.synchronize()
    times = {v: [] for v in VARIANTS}
    for r in range(a.repeats):
        order = VARIANTS if r % 2 == 0 else VARIANTS[::-1]
        for v in order:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.steps):
                step_all(variants[v][0])
            e1.record()
            e1.synchronize()
            times[v].append(e0.elapsed_time(e1) / a.steps)
    dev_ms = {v: device_ms(variants[v][0]) for v in VARIANTS}
    host = {v: host_us(variants[v][0]) for v in VARIANTS}
    torch.cuda.synchronize()

    def same(x, y):
        for px, py, ox, oy in zip(variants[x][1], variants[y][1], variants[x][0], variants[y][0]):
            for k in px:
                if not torch.equal(px[k].detach().view(torch.int32), py[k].detach().view(torch.int32)):
                    return False
                sx, sy = ox.state.get(px[k], {}), oy.state.get(py[k], {})
                for key in ("exp_avg", "exp_avg_sq"):
                    if (key in sx) != (key in sy) or (key in sx and not torch.equal(sx[key].view(torch.int32),
                                                                                  sy[key].view(torch.int32))):
                        return False
        return True

    out = {"layout": name, "elements": elements, "optimizers": len(shapes), "steps": a.steps, "repeats": a.repeats,
           "bytes_model_per_step": BYTES_PER_ELEMENT * elements}
    for v in VARIANTS:
        t = np.array(times[v])
        ms = float(np.median(t))
        q1, q3 = (float(x) for x in np.percentile(t, [25, 75]))
        out[v] = {"ms_per_step": round(ms, 4), "ms_q1": round(q1, 4), "ms_q3": round(q3, 4),
                  "ms_min": round(float(t.min()), 4), "ms_max": round(float(t.max()), 4),
                  "host_us_per_step": round(host[v], 1),
                  "GBps_28B_model": round(BYTES_PER_ELEMENT * elements / ms / 1e6, 1),
                  "device_ms_per_step": round(dev_ms[v][0], 4), "kernels_per_step": dev_ms[v][1],
                  "GBps_28B_model_device": round(BYTES_PER_ELEMENT * elements / dev_ms[v][0] / 1e6, 1)}
    out["native_bitwise_equal_default"] = same("native", "torch_default")
    out["fused_bitwise_equal_default"] = same("torch_fused", "torch_default")
    del variants
    torch.cuda.empty_cache()
    return out


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else None
    except (OSError, subprocess.SubprocessError):
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layout", nargs="+", default=["object", "scene"], choices=["object", "scene"])
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--repeats", type=int, default=15)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("benchmarks/optimizer.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    info = {"gpu": gpu_info() or torch.cuda.get_device_name(dev), "torch": torch.__version__}
    for name in a.layout:
        shapes = object_models(dev) if name == "object" else scene_models(dev)
        print(json.dumps({**info, **bench_layout(name, shapes, a, dev)}), flush=True)


if __name__ == "__main__":
    main()
