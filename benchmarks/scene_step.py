#!/usr/bin/env python
"""BASELINE.json config 5 re-enactment: the call pattern of DreamScene's scene_train_step
(/root/reference/training/scene_trainer.py:699-1080 -> scene_gaussian.py:673-893) with the SDS
guidance replaced by an L2 loss, on a synthetic indoor scene built with the reference's init
recipes (gs_renderer.py:218-248 walls, 279-296 floor; configs/scenes/sample_indoor.yaml box).
The reference modules cannot be imported on the GPU box (absent + missing deps), so the loop is
restated here: per view  torch.cat(env, floor, objects) -> SH/scale augmentation -> rasterizer ->
depth/alpha post-processing; 4 views per step (C_batch_size, config.py:163); one backward.

  python benchmarks/scene_step.py [--steps 10] [--views 4] [--size 512] [--optim none|torch|native]
                                  [--glue torch|fused|fused_rng|views|scene]
Prints a JSON line with the step time and the share spent inside the rasterizer.  --optim adds the optimizer step
after the backward, one Adam per GaussianModel as the reference builds it: torch.optim.Adam's default path or
dreamscene_b200.GaussianAdam (default none: no optimizer step, as before).
"""
import argparse
import json
import math
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from dreamscene_b200 import GaussianRasterizationSettings, GaussianRasterizer  # noqa: E402
from dreamscene_b200.multiview import rasterize_views  # noqa: E402
from dreamscene_b200.postprocess import disparity_from_depth_alpha  # noqa: E402
from dreamscene_b200.scene import assemble_scene, render_scene  # noqa: E402
from harness import cameras  # noqa: E402
from harness.scene_ref import reference_assemble  # noqa: E402

SH_C0 = 0.28209479177387814


def plane_points(n, origin, u, v, rng):
    a, b = rng.random_sample((n, 1)), rng.random_sample((n, 1))
    return origin[None] + a * u[None] + b * v[None]


def make_group(xyz, rng, M, dev, scale):
    P = xyz.shape[0]
    t = lambda a: torch.tensor(np.ascontiguousarray(a, dtype=np.float32), device=dev)
    return dict(
        xyz=t(xyz).requires_grad_(True),
        f_dc=t((rng.random_sample((P, 1, 3)) - 0.5) / SH_C0).requires_grad_(True),
        f_rest=t(rng.normal(0, 0.02, (P, M - 1, 3))).requires_grad_(True),
        scaling=t(np.log(np.full((P, 3), scale) * np.exp(rng.normal(0, 0.2, (P, 3))))).requires_grad_(True),
        rotation=t(np.tile([1.0, 0, 0, 0], (P, 1)) + rng.normal(0, 0.05, (P, 4))).requires_grad_(True),
        opacity=t(np.full((P, 1), math.log(0.1 / 0.9))).requires_grad_(True))


def build_scene(dev, M=4, n_wall=400_000, n_floor=300_000, n_obj=81_920, seed=0):
    rng = np.random.RandomState(seed)
    L, Wd, Hh = 6.0, 5.0, 2.8          # room box (m)
    o = np.array([-L / 2, -Wd / 2, 0.0])
    ex, ey, ez = np.array([L, 0, 0.0]), np.array([0, Wd, 0.0]), np.array([0, 0, Hh])
    walls = [plane_points(n_wall, o, ex, ez, rng), plane_points(n_wall, o + ey, ex, ez, rng),
             plane_points(n_wall, o, ey, ez, rng), plane_points(n_wall, o + ex, ey, ez, rng),
             plane_points(n_wall, o + ez, ex, ey, rng)]                     # 4 walls + ceiling
    env = make_group(np.concatenate(walls), rng, M, dev, scale=0.008)
    floor = make_group(plane_points(n_floor, o, ex, ey, rng), rng, M, dev, scale=0.008)
    objs = []
    for c in ([1.0, 0.8, 0.5], [-1.2, -0.6, 0.4], [0.3, -1.3, 0.45], [-0.5, 1.2, 0.6]):
        d = rng.normal(size=(n_obj, 3)); d /= np.linalg.norm(d, axis=1, keepdims=True)
        xyz = np.array(c)[None] + 0.35 * np.cbrt(rng.random_sample((n_obj, 1))) * d
        objs.append(make_group(xyz, rng, M, dev, scale=0.006))
    return [env, floor] + objs


def scene_camera(k, size, dev):
    # camera inside the room, looking roughly horizontally (Stage1_Indoor-like), FoV 0.96
    ang = 2 * math.pi * (k * 0.37 % 1.0)
    eye = np.array([0.8 * math.cos(ang * 1.7), 0.6 * math.sin(ang * 1.3), 1.4], np.float32)
    fwd = np.array([math.cos(ang), math.sin(ang), -0.1], np.float32); fwd /= np.linalg.norm(fwd)
    up = np.array([0, 0, 1], np.float32)
    right = np.cross(fwd, up); right /= np.linalg.norm(right)
    up = np.cross(right, fwd)
    pose = np.eye(4, dtype=np.float32)
    pose[:3, :3] = np.stack((-right, up, -fwd), axis=-1)    # same axes convention as cameras.orbit_pose
    pose[:3, 3] = eye
    return cameras.camera_from_pose(pose, 0.96, size, size, device=dev)


def render(groups, cam, dev, bg, aug=True, glue="torch"):
    """scene_gaussian.py:673-893 restated.  glue="torch": the reference's own PyTorch expressions
    (per-group activations, torch.cat, augmentation); glue="fused" / "fused_rng": dreamscene_b200.scene
    (one kernel each way; "fused_rng" also generates the noise in the kernel)."""
    S = GaussianRasterizationSettings(
        image_height=cam.image_height, image_width=cam.image_width, tanfovx=cam.tanfovx, tanfovy=cam.tanfovy,
        bg=bg, scale_modifier=1.0, viewmatrix=cam.world_view_transform, projmatrix=cam.full_proj_transform,
        sh_degree=1, campos=cam.camera_center, prefiltered=False, score_flag=False)
    named = [{"_xyz": g["xyz"], "_opacity": g["opacity"], "_scaling": g["scaling"], "_rotation": g["rotation"],
              "_features_dc": g["f_dc"], "_features_rest": g["f_rest"]} for g in groups]
    if glue == "torch":
        P = sum(g["xyz"].shape[0] for g in groups)
        M = 1 + groups[0]["f_rest"].shape[1]
        z_shs = torch.randn(P, M, 3, device=dev) if aug else None                   # :848-851
        z_sc = torch.randn(P, 3, device=dev) if aug else None                       # :853-856 (exact zeros)
        xyz, opacity, scales, rots, shs = reference_assemble(named, z_shs, z_sc)
    else:
        xyz, opacity, scales, rots, shs = assemble_scene(named, shs_aug=aug, scale_aug=aug,
                                                         noise="torch" if glue == "fused" else "fused")
    screenspace = torch.zeros_like(xyz, requires_grad=True) + 0
    screenspace.retain_grad()
    t0 = torch.cuda.Event(enable_timing=True); t1 = torch.cuda.Event(enable_timing=True)
    t0.record()
    image, radii, depth_alpha = GaussianRasterizer(S)(means3D=xyz, means2D=screenspace, shs=shs, colors_precomp=None,
                                                      opacities=opacity, scales=scales, rotations=rots,
                                                      cov3D_precomp=None)
    t1.record()
    focal = 1 / (2 * math.tan(cam.FoVx / 2))
    if glue == "torch":                                      # scene_gaussian.py:871-881 (one host sync per view)
        depth, alpha = torch.chunk(depth_alpha, 2)
        disp = focal / (depth + alpha * 10 + 1e-5)
        try:
            min_d = disp[alpha <= 0.1].min()
        except Exception:
            min_d = disp.min()
        disp = torch.clamp((disp - min_d) / (disp.max() - min_d), 0.0, 1.0)
    else:
        disp, alpha = disparity_from_depth_alpha(depth_alpha, focal)
    return dict(image=image, depth=disp, alpha=alpha, radii=radii, viewspace=screenspace, ev=(t0, t1))


def render_views(groups, cams, dev, bg, aug=True, scene=False):
    """All views of the step in one rasterizer pass (dreamscene_b200.multiview): per-view augmented shs / scales
    (in-kernel Philox noise), shared positions / opacities / rotations, batched fused disparity.  scene=True:
    dreamscene_b200.scene.render_scene renders them straight from the raw groups (the activations and the
    augmentation happen inside the projection kernels; the rasterizer time then includes them)."""
    named = [{"_xyz": g["xyz"], "_opacity": g["opacity"], "_scaling": g["scaling"], "_rotation": g["rotation"],
              "_features_dc": g["f_dc"], "_features_rest": g["f_rest"]} for g in groups]
    if not scene:
        xyz, opacity, scales_v, rots, shs_v = assemble_scene(named, shs_aug=aug, scale_aug=aug, noise="fused",
                                                             views=len(cams))
    S = [GaussianRasterizationSettings(
        image_height=c.image_height, image_width=c.image_width, tanfovx=c.tanfovx, tanfovy=c.tanfovy, bg=bg,
        scale_modifier=1.0, viewmatrix=c.world_view_transform, projmatrix=c.full_proj_transform, sh_degree=1,
        campos=c.camera_center, prefiltered=False, score_flag=False) for c in cams]
    P = sum(int(g["xyz"].shape[0]) for g in groups)
    screens = [torch.zeros(P, 3, device=dev, requires_grad=True) for _ in cams]
    t0 = torch.cuda.Event(enable_timing=True); t1 = torch.cuda.Event(enable_timing=True)
    t0.record()
    if scene:
        outs = render_scene(named, S, shs_aug=aug, scale_aug=aug, means2D=screens)
    else:
        outs = rasterize_views(S, xyz, opacity, shs=list(shs_v.unbind(0)), scales=list(scales_v.unbind(0)),
                               rotations=rots, means2D=screens)
    t1.record()
    da = torch.stack([o[2] for o in outs])                                  # [B,2,H,W]
    focals = [1 / (2 * math.tan(c.FoVx / 2)) for c in cams]
    disp, alpha = disparity_from_depth_alpha(da, focals)
    return [dict(image=o[0], depth=disp[v], alpha=alpha[v], radii=o[1], viewspace=screens[v], ev=(t0, t1) if v == 0 else None)
            for v, o in enumerate(outs)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--views", type=int, default=4)
    ap.add_argument("--size", type=int, default=512)
    ap.add_argument("--glue", default="torch", choices=["torch", "fused", "fused_rng", "views", "scene"])
    ap.add_argument("--optim", default="none", choices=["none", "torch", "native"])
    a = ap.parse_args()
    dev = torch.device("cuda", 0)
    torch.manual_seed(0)
    groups = build_scene(dev)
    opts = []
    if a.optim != "none":
        from dreamscene_b200 import GaussianAdam
        from harness.adam_ref import reference_adam
        opts = [reference_adam(g, GaussianAdam if a.optim == "native" else torch.optim.Adam) for g in groups]
    P = sum(g["xyz"].shape[0] for g in groups)
    params = [v for g in groups for v in g.values()]
    target = torch.rand(3, a.size, a.size, device=dev)
    bg = torch.ones(3, device=dev)
    times, ras_fwd, vis, pairs = [], [], [], []
    from dreamscene_b200 import rasterizer as R
    # cameras are built up front: constructing one costs three small synchronous host->device copies (pageable
    # memory), i.e. a hidden stream sync per view that has nothing to do with the render path
    all_cams = {it: [scene_camera(it * a.views + k, a.size, dev) for k in range(a.views)]
                for it in list(range(a.warmup + a.steps)) + [1000 + i for i in range(a.steps)] + [2000]}
    for it in range(a.warmup + a.steps):
        for p in params:
            p.grad = None
        torch.cuda.synchronize(); t0 = time.perf_counter()
        cams = all_cams[it]
        outs = render_views(groups, cams, dev, bg, scene=a.glue == "scene") if a.glue in ("views", "scene") else [render(groups, c, dev, bg, glue=a.glue) for c in cams]
        images = torch.stack([o["image"] for o in outs]); depths = torch.stack([o["depth"] for o in outs])
        loss = ((images - target) ** 2).mean() * 100 + depths.mean() * 0.1      # SDS -> L2 stub (+ depth path)
        loss.backward()
        for o in opts:
            o.step()
        torch.cuda.synchronize(); dt = time.perf_counter() - t0
        if it >= a.warmup:
            times.append(dt)
            ras_fwd.append(sum(o["ev"][0].elapsed_time(o["ev"][1]) for o in outs if o["ev"] is not None))
            vis.append(float(np.mean([(o["radii"] > 0).float().mean().item() for o in outs])))
            pairs.append(R.last_pair_count(dev))
    finite = all(torch.isfinite(p.grad).all().item() for p in params)

    def one_step(it):
        for p in params:
            p.grad = None
        cams = all_cams[it]
        outs = render_views(groups, cams, dev, bg, scene=a.glue == "scene") if a.glue in ("views", "scene") else [render(groups, c, dev, bg, glue=a.glue) for c in cams]
        images = torch.stack([o["image"] for o in outs]); depths = torch.stack([o["depth"] for o in outs])
        (((images - target) ** 2).mean() * 100 + depths.mean() * 0.1).backward()
        for o in opts:
            o.step()

    # (a) back-to-back steps without a host sync in between (the fused paths never force one; the reference glue
    #     syncs per view in its boolean-mask indexing): host and device overlap, time = max(host, device) per step
    torch.cuda.synchronize(); t0 = time.perf_counter()
    for it in range(a.steps):
        one_step(1000 + it)
    torch.cuda.synchronize()
    pipelined_ms = 1e3 * (time.perf_counter() - t0) / a.steps
    # (b) device-busy time of one step: sum of all kernel durations (torch profiler)
    gpu_ms = None
    try:
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            one_step(2000)
            torch.cuda.synchronize()
        gpu_ms = sum(e.device_time_total for e in prof.key_averages()) / 1e3
    except Exception:
        pass
    extra = {"optim": a.optim} if a.optim != "none" else {}
    print(json.dumps({"config": "cfg5_scene_step (re-enactment)", "glue": a.glue, **extra, "P": P, "views": a.views, "size": a.size,
                      "M": 4, "sh_degree": 1, "step_ms": 1e3 * float(np.median(times)),
                      "step_ms_no_sync_between_steps": pipelined_ms, "device_busy_ms_per_step": gpu_ms,
                      "rasterizer_fwd_ms_per_step": float(np.median(ras_fwd)),
                      "visible_fraction": float(np.mean(vis)), "tile_pairs_last_view": int(np.median(pairs)),
                      "grads_finite": finite}))


if __name__ == "__main__":
    main()
