#!/usr/bin/env python
"""One 3D Gaussian filtering event at object scale, timed two ways in one process:

  (a) the reference's flow restated (scene_gaussian.py:1046-1103): one GaussianRasterizer(score_flag=True) render per
      sphere camera with a grad-requiring means2D and score_render's disparity glue, scores summed in view order,
      calculate_v_imp_score with torch.sort, prune_gaussians' sorted percentile and a boolean-mask prune of every
      parameter, Adam moment and statistic;
  (b) dreamscene_b200.filtering.gaussian_filtering, in the default and the deterministic mode, at two views_per_pass.

  python benchmarks/filtering.py [--points 1200000] [--views 48] [--size 512] [--reps 3] [--warmup 1]

Scene: the ball scene of bench.py's workloads (exact 3-NN scales, SH degree 3, M = 16) as raw leaves; 48 sphere
cameras at radius 3.5, FoV 0.55.  Every repetition starts from the same parameters.  Prints one JSON line: ms per
event (CUDA events, median and all repetitions, alternating the variants), the stage times of the score passes and of
the reference's renders, the points kept by each, and the card's name and power limit.  Writes nothing to disk.
"""
import argparse
import json
import math
import os
import subprocess
import sys

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from dreamscene_b200 import GaussianRasterizationSettings, GaussianRasterizer, _lib  # noqa: E402
from dreamscene_b200 import filtering  # noqa: E402
from harness import cameras, synthetic  # noqa: E402

V_POW, PRUNE_DECAY, PRUNE_PERCENT = 0.1, 0.6, 0.5      # the object trainer's defaults


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


def reference_event(params, adam, stats, cams, settings):
    """(a): the reference's prune_list + calculate_v_imp_score + prune_gaussians + prune_points."""
    imp = None
    for cam, S in zip(cams, settings):
        xyz = params["xyz"]
        m2d = torch.zeros_like(xyz, dtype=xyz.dtype, requires_grad=True, device="cuda") + 0
        m2d.retain_grad()
        shs = torch.cat((params["f_dc"], params["f_rest"]), dim=1)
        score, _, _, depth_alpha = GaussianRasterizer(S)(
            means3D=xyz, means2D=m2d, shs=shs, colors_precomp=None, opacities=torch.sigmoid(params["opacity"]),
            scales=torch.exp(params["scaling"]), rotations=F.normalize(params["rotation"]), cov3D_precomp=None)
        depth, alpha = torch.chunk(depth_alpha, 2)
        focal = 1 / (2 * math.tan(cam.FoVx / 2))
        disp = focal / (depth + (alpha * 10) + 1e-5)
        try:
            min_d = disp[alpha <= 0.1].min()
        except Exception:
            min_d = disp.min()
        disp = torch.clamp((disp - min_d) / (disp.max() - min_d), 0.0, 1.0)
        imp = score if imp is None else imp + score.detach()
    volume = torch.prod(torch.exp(params["scaling"]), dim=1)
    sorted_volume, _ = torch.sort(volume, descending=True)
    v_list = torch.pow(volume / sorted_volume[int(len(volume) * 0.9)], V_POW) * imp
    sorted_t, _ = torch.sort(v_list, dim=0)
    thr = sorted_t[int((PRUNE_DECAY ** 1) * PRUNE_PERCENT * (sorted_t.shape[0] - 1))]
    keep = ~((v_list <= thr).squeeze())
    with torch.no_grad():
        new_p = {k: v[keep] for k, v in params.items()}
        new_a = {k: (m[keep], s[keep]) for k, (m, s) in adam.items()}
        new_s = {k: v[keep] for k, v in stats.items()}
    return new_p, new_a, new_s


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--points", type=int, default=1_200_000)
    ap.add_argument("--views", type=int, default=48)
    ap.add_argument("--size", type=int, default=512)
    ap.add_argument("--vpp", type=int, nargs=2, default=[16, 8])
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    sc = synthetic.ball_scene(args.points, radius=0.5, sh_degree_max=3, seed=0)
    params = {"xyz": sc["means3D"], "f_dc": sc["shs"][:, :1], "f_rest": sc["shs"][:, 1:],
              "opacity": torch.logit(sc["opacities"]), "scaling": torch.log(sc["scales"]), "rotation": sc["rotations"]}
    params = {k: v.contiguous().to(dev).requires_grad_(True) for k, v in params.items()}
    g = torch.Generator(device=dev).manual_seed(1)
    adam = {k: (torch.randn(v.shape, device=dev, generator=g), torch.rand(v.shape, device=dev, generator=g))
            for k, v in params.items()}
    stats = {"xyz_gradient_accum": torch.zeros(args.points, 1, device=dev), "denom": torch.zeros(args.points, 1, device=dev),
             "max_radii2D": torch.zeros(args.points, device=dev)}
    cams = cameras.sphere_cameras(args.views, H=args.size, W=args.size, generator=torch.Generator().manual_seed(0))
    settings = [GaussianRasterizationSettings(c.image_height, c.image_width, c.tanfovx, c.tanfovy, torch.ones(3, device=dev),
                                              1.0, c.world_view_transform.to(dev), c.full_proj_transform.to(dev), 3,
                                              c.camera_center.to(dev), False, True) for c in cams]
    variants = {"reference": (False, lambda: reference_event(params, adam, stats, cams, settings))}
    for det in (False, True):
        for vpp in args.vpp:
            variants[f"fused_{'det' if det else 'default'}_vpp{vpp}"] = (
                det, lambda vpp=vpp: filtering.gaussian_filtering(params, adam, stats, settings, V_POW, PRUNE_DECAY,
                                                                  PRUNE_PERCENT, views_per_pass=vpp))

    def timed(name):
        det, fn = variants[name]
        set_mode(det)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        out = fn()
        e1.record()
        torch.cuda.synchronize()
        set_mode(False)
        return e0.elapsed_time(e1), out

    kept = {}
    for name in variants:
        for _ in range(args.warmup):
            _, out = timed(name)
        kept[name] = int(out[0]["xyz"].shape[0])
    ms = {name: [] for name in variants}
    for _ in range(args.reps):
        for name in variants:
            ms[name].append(timed(name)[0])

    stages = {}
    for name in ["reference"] + [f"fused_default_vpp{v}" for v in args.vpp]:
        _lib.profile_enable(args.views)
        timed(name)
        st = _lib.profile_collect()
        _lib.profile_enable(0)
        calls = len(st["project_sh"])
        stages[name] = {"calls": calls, **{k: float(np.sum(v)) for k, v in st.items() if v}}
    fused_default = f"fused_default_vpp{args.vpp[0]}"
    med = {k: float(np.median(v)) for k, v in ms.items()}
    print(json.dumps({"card": card(), "points": args.points, "views": args.views, "size": args.size, "M": 16,
                      "reps": args.reps, "ms_median": med, "ms": ms,
                      "speedup_vs_reference": {k: med["reference"] / v for k, v in med.items() if k != "reference"},
                      "stage_ms_per_event": stages,
                      "stage_names": "score passes: project_sh = geometry-only projection, composite_fwd = score-only "
                                     "compositing; reference: the full score_flag forward of every view",
                      "kept": kept, "fused_default_kept_matches_reference": kept[fused_default] == kept["reference"]}),
          flush=True)


if __name__ == "__main__":
    main()
