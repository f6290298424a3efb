#!/usr/bin/env python
"""The video renders of a camera path, timed two ways in one process, alternating within each round:

  reference     : the reference's loop as written (training/scene_trainer.py scene_video_inference,
                  training/object_trainer.py video_inference): per frame, scene_render's eager assembly (torch.cat of
                  every group's leaves, the activations, a grad-requiring screen-space tensor, autograd on), the
                  GaussianRasterizer, its torch disparity expression with the boolean-mask min, then the two .cpu()
                  copies and the numpy quantisation of harness/video_ref.py;
  render_frames : dreamscene_b200.video.render_frames (stacked forward-only passes of 16 views, frames quantised on
                  the device, copied into pinned memory while the next pass renders).

Layouts (512 x 512): scene = harness/room.py::build_scene (cfg5: 2.63 M Gaussians in 6 groups, M = 4,
sh_degree 1; cameras inside the room); object = benchmarks/scene_render.py::object_layout (1.2 M Gaussians, M = 16,
sh_degree 3; orbit cameras).  Frame counts: 240 (one Circle(): 120 views around, 120 at 45 degrees) and 1440 (the
scene's inference cameras with K = 5 objects, 240 (K + 1)); the 240 are the first 240 of the 1440.

Per layout and frame count: wall ms per frame and per call (host clock around the whole call, which ends with the
frames on the host), median and range over --rounds rounds after one warm-up round.  Then, untimed: the frames of
render_frames against the reference loop over the project's per-view path (render_scene + disparity_from_depth_alpha,
harness/video_ref.native_render) at 1440 frames, asserted bit-equal; the bytes in which the as-written reference's
frames differ from render_frames' (its torch normalize of the rotations may differ by one ulp from the kernels'); the
pinned bytes render_frames allocates; and, in a torch.profiler run of its own, the device time per frame of both at
240 frames with render_frames' largest kernels.  Prints one JSON line per layout, with the card's name, power limit
and max SM clock.  Writes nothing to disk.

  python benchmarks/video_frames.py [--layouts scene,object] [--frames 240,1440] [--rounds 3]
"""
import argparse
import json
import math
import os
import subprocess
import sys
import time

import numpy as np
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
from dreamscene_b200 import GaussianRasterizationSettings, GaussianRasterizer  # noqa: E402
from dreamscene_b200.video import render_frames  # noqa: E402
from harness import cameras, room, video_ref  # noqa: E402
import scene_render  # noqa: E402


def card():
    try:
        return subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()),
                               "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        return torch.cuda.get_device_name()


def circle(n, dev, radius=2.5):
    """cam_utils Circle(): n / 2 views around at the default elevation, n / 2 at 45 degrees."""
    half = n // 2
    return [cameras.orbit_camera(radius=radius, theta_deg=60.0 if k < half else 45.0, phi_deg=360.0 * (k % half) / half,
                                 fovx=0.8, height=512, width=512, device=dev) for k in range(n)]


def layouts(dev, n):
    if "scene" in LAYOUTS:
        groups, _, deg = scene_render.scene_layout(dev)
        yield "scene", groups, [room.scene_camera(k, 512, dev) for k in range(n)], deg
    if "object" in LAYOUTS:
        groups, _, deg = scene_render.object_layout(dev)
        cams = [c for r in range(n // 240) for c in circle(240, dev, radius=2.5 + 0.25 * r)]
        yield "object", groups, cams, deg


def settings(cams, deg, bg):
    return [GaussianRasterizationSettings(
        image_height=c.image_height, image_width=c.image_width, tanfovx=c.tanfovx, tanfovy=c.tanfovy, bg=bg,
        scale_modifier=1.0, viewmatrix=c.world_view_transform, projmatrix=c.full_proj_transform, sh_degree=deg,
        campos=c.camera_center, prefiltered=False, score_flag=False) for c in cams]


def reference_render(groups):
    """scene_render(..., test=True) as written (scene_gaussian.py:753-893), without augmentation."""
    def render(s):
        xyz = torch.cat([g["_xyz"] for g in groups])
        opacity = torch.cat([torch.sigmoid(g["_opacity"]) for g in groups])
        scales = torch.cat([torch.exp(g["_scaling"]) for g in groups])
        rotations = torch.cat([F.normalize(g["_rotation"]) for g in groups])
        shs = torch.cat([torch.cat((g["_features_dc"], g["_features_rest"]), dim=1) for g in groups])
        screenspace_points = torch.zeros_like(xyz, dtype=xyz.dtype, requires_grad=True, device="cuda") + 0
        screenspace_points.retain_grad()
        image, radii, depth_alpha = GaussianRasterizer(s)(
            means3D=xyz, means2D=screenspace_points, shs=shs, colors_precomp=None, opacities=opacity, scales=scales,
            rotations=rotations, cov3D_precomp=None)
        depth, alpha = torch.chunk(depth_alpha, 2)
        focal = 1 / (2 * s.tanfovx)
        disp = focal / (depth + (alpha * 10) + 1e-5)
        try:
            min_d = disp[alpha <= 0.1].min()
        except Exception:
            min_d = disp.min()
        disp = torch.clamp((disp - min_d) / (disp.max() - min_d), 0.0, 1.0)
        return image, disp
    return render


def run_variant(name, groups, S):
    if name == "reference":
        img, dep = video_ref.frames(reference_render(groups), S)
        return img, dep
    return render_frames(groups, S)


def device_ms(fn):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    per = {}
    for e in prof.key_averages():
        if e.device_time_total > 0:
            name = e.key.replace("(anonymous namespace)::", "").replace("void ", "").split("<")[0].split("(")[0]
            per[name] = per.get(name, 0.0) + e.device_time_total / 1e3
    return sum(per.values()), dict(sorted(per.items(), key=lambda kv: -kv[1])[:8])


def main():
    global LAYOUTS
    ap = argparse.ArgumentParser()
    ap.add_argument("--layouts", default="scene,object")
    ap.add_argument("--frames", default="240,1440")
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    LAYOUTS = args.layouts.split(",")
    counts = [int(x) for x in args.frames.split(",")]
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    gpu = card()
    bg = torch.ones(3, device=dev)
    variants = ("reference", "render_frames")
    for name, groups, cams, deg in layouts(dev, max(counts)):
        for g in groups:
            for t in g.values():
                t.requires_grad_(True)
        S_all = settings(cams, deg, bg)
        P = sum(int(g["_xyz"].shape[0]) for g in groups)
        res = {"layout": name, "gaussians": P, "groups": len(groups), "size": 512, "gpu": gpu, "frames": {}}
        for n in counts:
            S = S_all[:n]
            wall = {v: [] for v in variants}
            for r in range(args.rounds + 1):                       # round 0 warms up
                for v in (variants if r % 2 == 0 else variants[::-1]):
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    out = run_variant(v, groups, S)
                    t1 = time.perf_counter()
                    del out
                    if r:
                        wall[v].append((t1 - t0) * 1e3)
            res["frames"][n] = {v: {"ms_per_frame": round(float(np.median(w)) / n, 3),
                                    "ms_per_frame_range": [round(min(w) / n, 3), round(max(w) / n, 3)],
                                    "ms_total": round(float(np.median(w)), 1),
                                    "ms_total_range": [round(min(w), 1), round(max(w), 1)]} for v, w in wall.items()}
            res["frames"][n]["speedup"] = round(float(np.median(wall["reference"]) / np.median(wall["render_frames"])), 2)
        # the frames at the largest timed size
        n = max(counts)
        rgb, depth = render_frames(groups, S_all[:n])
        res["pinned_bytes"] = rgb.numel() + depth.numel()
        with torch.no_grad():
            img, dep = video_ref.frames(video_ref.native_render(groups), S_all[:n])
        same = all(np.array_equal(rgb[v].numpy(), img[v]) and np.array_equal(depth[v].numpy(), dep[v]) for v in range(n))
        res["equal_to_per_view_path"] = same
        img, dep = video_ref.frames(reference_render(groups), S_all[:n])
        res["bytes_differing_from_as_written_reference"] = {
            "rgb": int(sum(int((rgb[v].numpy() != img[v]).sum()) for v in range(n))),
            "depth": int(sum(int((depth[v].numpy() != dep[v]).sum()) for v in range(n))), "of": int(rgb.numel() + depth.numel())}
        del img, dep, rgb, depth
        # device time per frame, profiler on, at the smallest size
        n = min(counts)
        ref_ms, _ = device_ms(lambda: video_ref.frames(reference_render(groups), S_all[:n]))
        rf_ms, rf_top = device_ms(lambda: render_frames(groups, S_all[:n]))
        res["device_ms_per_frame"] = {"reference": round(ref_ms / n, 3), "render_frames": round(rf_ms / n, 3),
                                      "frames": n, "render_frames_top_kernels_ms": {k: round(v, 2) for k, v in rf_top.items()}}
        print(json.dumps(res), flush=True)
        assert same, f"{name}: render_frames differs from the per-view path's frames"


if __name__ == "__main__":
    main()
