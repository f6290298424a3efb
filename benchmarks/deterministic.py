#!/usr/bin/env python
"""Cost of deterministic mode: fwd+bwd of one bench.py workload, alternating the default mode and
torch.use_deterministic_algorithms(True) in one process, so both see the same card, clocks and neighbours.

  python benchmarks/deterministic.py [--workload cfg3_1M_1024] [--steps 50] [--warmup 20] [--rounds 3]

One step is the step bench.py times (GaussianRasterizer forward + backward with fixed incoming gradients).  While
deterministic mode is on, PyTorch's NaN fill of every torch.empty is switched off, so the numbers are the
rasterizer's own cost.  Prints one JSON line: ms/step (CUDA events) and mean kernel-stage times per mode and
round, the card's name and power limit, and whether two deterministic steps gave bitwise-equal gradients.
Writes nothing to disk.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402  (workloads and the seeded scene)
from dreamscene_b200 import GaussianRasterizationSettings, GaussianRasterizer, _lib  # noqa: E402

NAMES = ("means3D", "opacities", "shs", "scales", "rotations")


def card():
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=name,power.limit",
                              "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
        return out or torch.cuda.get_device_name()
    except Exception:
        return torch.cuda.get_device_name()


def set_mode(det):
    torch.use_deterministic_algorithms(det)
    torch.utils.deterministic.fill_uninitialized_memory = not det


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="cfg3_1M_1024", choices=sorted(bench.WORKLOADS))
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    wl = bench.WORKLOADS[args.workload]
    sc, cam, gc, gd = bench.make_scene(wl, 0)
    prm = {k: sc[k].to(dev).requires_grad_(True) for k in NAMES}
    gc, gd = gc.to(dev), gd.to(dev)
    m2d = torch.zeros(wl["P"], 3, device=dev, requires_grad=True)
    rast = GaussianRasterizer(GaussianRasterizationSettings(
        image_height=wl["H"], image_width=wl["W"], tanfovx=cam.tanfovx, tanfovy=cam.tanfovy,
        bg=torch.ones(3, device=dev), scale_modifier=1.0, viewmatrix=cam.world_view_transform.to(dev),
        projmatrix=cam.full_proj_transform.to(dev), sh_degree=3, campos=cam.camera_center.to(dev),
        prefiltered=False, score_flag=False))

    def step():
        for v in prm.values():
            v.grad = None
        m2d.grad = None
        color, _, da = rast(means3D=prm["means3D"], means2D=m2d, opacities=prm["opacities"], shs=prm["shs"],
                            scales=prm["scales"], rotations=prm["rotations"])
        torch.autograd.backward([color, da], [gc, gd])

    runs = []
    for r in range(args.rounds):
        for det in (False, True):
            set_mode(det)
            for _ in range(args.warmup):
                step()
            torch.cuda.synchronize()
            _lib.profile_enable(args.steps)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.steps):
                step()
            e1.record()
            torch.cuda.synchronize()
            stages = {k: float(np.mean(v)) for k, v in _lib.profile_collect().items() if v}
            _lib.profile_enable(0)
            runs.append({"round": r, "deterministic": det, "ms_per_step": e0.elapsed_time(e1) / args.steps,
                         "stages_ms": stages})

    set_mode(True)
    grads = []
    for _ in range(2):
        step()
        grads.append([t.grad.clone() for t in prm.values()] + [m2d.grad.clone()])
    repeatable = all(torch.equal(a, b) for a, b in zip(*grads))
    set_mode(False)
    print(json.dumps({"workload": args.workload, "card": card(), "steps": args.steps, "warmup": args.warmup,
                      "runs": runs, "deterministic_bitwise_repeatable": repeatable}), flush=True)


if __name__ == "__main__":
    main()
