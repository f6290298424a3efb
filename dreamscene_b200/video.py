"""8-bit video frames of a camera path, rendered in batched forward-only passes.

DreamScene's video loops (training/object_trainer.py video_inference, training/scene_trainer.py scene_video_inference
and scene_cams_record) render one view at a time through scene_render / object_render(test=True), then per frame

    depths = torch.clamp(depth / depth.max(), 0.0, 1.0).detach().cpu().permute(1, 2, 0).numpy()
    depths = (depths * 255).round().astype(np.uint8)
    image  = torch.clamp(rgb, 0.0, 1.0).detach().cpu().permute(1, 2, 0).numpy()
    image  = (image * 255).round().astype(np.uint8)

``render_frames(groups, settings_list)`` returns the same frames for all views at once: stacked passes of up to
views_per_pass views through b200gsr_forward_scene without backward state, each followed by b200gsr_frames, which
computes the disparity and quantises both images on the device, and an asynchronous copy into pinned host memory
while the next pass renders.
"""
from __future__ import annotations

import ctypes as C
from typing import Sequence, Tuple

import torch

from . import _lib
from . import rasterizer as R
from . import scene as S
from .filtering import view_chunks

_SETTLE_GROUP = 64          # passes whose pair counts are read together: bounds the notify slots one call holds


def _check_device(flat):
    if any(t.device.type != "cuda" for t in flat):
        raise RuntimeError("render_frames (b200gsr): parameters must be CUDA tensors; there is no CPU fallback")
    S._check_device(flat)


def render_frames(groups: Sequence, settings_list: Sequence[R.GaussianRasterizationSettings], *,
                  views_per_pass: int = 16) -> Tuple[torch.Tensor, torch.Tensor]:
    """The reference's video frames of every view of settings_list, rendered from the raw parameter groups.

    groups        : as render_scene (plain groups, or ReservedGroup.rows(); a ReservedGroup itself is refused).  For a
                    scene, the visible groups in the order the reference concatenates them.
    settings_list : N >= 0 GaussianRasterizationSettings of one image size H x W; camera, bg, sh_degree and
                    scale_modifier may differ per view; score_flag must be False.
    views_per_pass: 1..MAX_VIEWS views per stacked pass.  The frames do not depend on it.
    -> (rgb uint8 [N,H,W,3], depth uint8 [N,H,W,1]), pinned CPU tensors, complete when the call returns.

    View v's frames are those of the reference's loop (harness/video_ref.py) over render_scene(groups, [s_v],
    shs_aug=False, scale_aug=False) and disparity_from_depth_alpha with focal 1 / (2 tanfovx_v), bit for bit:
        rgb[v]   = round_half_even(float32(clamp(color_v, 0, 1)) * 255)
        depth[v] = round_half_even(clamp(disp_v / max(disp_v), 0, 1) * 255)
    There is no augmentation (the reference's test=True) and no autograd state.  Where numpy's cast of the reference
    is undefined the frames are fixed: a NaN colour value gives 0, and a view whose disparity is constant (its max
    equals its min, as in a view that sees nothing) gives an all-zero depth frame.

    The call waits for the pair counts of its passes (a pass that overflowed its pair capacity is rendered, quantised
    and copied again), so it cannot be captured into a CUDA graph.  Deterministic mode does not change the frames."""
    S._refuse_reserved(groups)
    views_per_pass = int(views_per_pass)
    if not 1 <= views_per_pass <= _lib.MAX_VIEWS:
        raise ValueError(f"render_frames: views_per_pass must be in 1..{_lib.MAX_VIEWS}, got {views_per_pass}")
    settings_list = list(settings_list)
    N = len(settings_list)
    H, W = (int(settings_list[0].image_height), int(settings_list[0].image_width)) if N else (0, 0)
    for s in settings_list:
        if int(s.image_height) != H or int(s.image_width) != W:
            raise ValueError("render_frames: all views must share the image size")
        if bool(s.score_flag):
            raise ValueError("render_frames: score_flag is not supported; use dreamscene_b200.filtering for the "
                             "important score")
    flat, M, P = S._scene_groups(groups)
    _check_device(flat)
    if torch.cuda.is_current_stream_capturing():
        raise RuntimeError("render_frames waits for the pair counts of its passes and cannot be captured into a "
                           "CUDA graph")
    dev = flat[0].device
    rgb = torch.empty(N, H, W, 3, dtype=torch.uint8, pin_memory=True)
    depth = torch.empty(N, H, W, 1, dtype=torch.uint8, pin_memory=True)
    if N == 0:
        return rgb, depth
    lib, ptr = _lib.load(), _lib.ptr
    num_groups, HW = len(groups), H * W
    with torch.no_grad(), torch.cuda.device(dev):
        raw = [[_lib.prepare(t.detach()) for t in flat[6 * k:6 * k + 6]] for k in range(num_groups)]
        table = S._group_table(raw)
        d = R._device_state(dev)
        d.resolve()                            # non-blocking overflow check of earlier forwards, as every forward does
        stream = _lib.stream(dev)
        main, side = torch.cuda.current_stream(dev), torch.cuda.Stream(dev)
        keep: list = []
        bg_all = torch.stack([R._const(s.bg, dev).reshape(3) for s in settings_list]).contiguous()
        params = [R._make_params(s, P, M, keep, dev, bg_all, v) for v, s in enumerate(settings_list)]
        focal = torch.tensor([1.0 / (2.0 * float(s.tanfovx)) for s in settings_list], dtype=torch.float32).to(dev)
        B_max = min(views_per_pass, N)
        no_noise = (C.c_float * B_max)()
        # one pass in flight on the main stream: the frames pass consumes color / depth_alpha before the next forward
        # overwrites them; only the staging slots are read by the other stream
        Hs_max = _lib.stacked_height(B_max, H, W)
        color = torch.empty(3 * Hs_max * W, dtype=torch.float32, device=dev)
        depth_alpha = torch.empty(2 * Hs_max * W, dtype=torch.float32, device=dev)
        radii = torch.empty(max(1, B_max * P), dtype=torch.int32, device=dev)
        stats = torch.empty(B_max * _lib.FRAMES_STATS_BYTES, dtype=torch.uint8, device=dev)
        stage = [(torch.empty(B_max * HW * 3, dtype=torch.uint8, device=dev),
                  torch.empty(B_max * HW, dtype=torch.uint8, device=dev)) for _ in range(2)]
        copied = [torch.cuda.Event(), torch.cuda.Event()]     # the copy out of each staging slot has finished
        rgb_flat, depth_flat = rgb.view(-1), depth.view(-1)
        turn = [0]

        def issue(b0, b1, cap):
            """Render views b0..b1 at pair capacity `cap`, quantise them into the next staging slot and copy that to
            the output on the side stream.  -> (slot, seq) of the forward's pair-count report."""
            B = b1 - b0
            Hs = _lib.stacked_height(B, H, W)
            prm = (_lib.Params * B)(*params[b0:b1])

            def launch(cap, flags, scratch, saved, notify_ptr, seq):
                return lib.b200gsr_forward_scene(B, prm, num_groups, table, no_noise, no_noise, 0, None, ptr(color),
                                                 ptr(depth_alpha), ptr(radii), ptr(scratch), scratch.numel(),
                                                 ptr(saved), saved.numel(), cap, flags, notify_ptr, seq, stream)

            _, slot, seq = R._issue_once(d, (B * P, Hs, W, False, False), _lib.FWD_NO_BACKWARD, cap, launch,
                                         stream.value, False, "b200gsr_forward_scene")
            k = turn[0]
            turn[0] ^= 1
            st_rgb, st_depth = stage[k]
            main.wait_event(copied[k])
            _lib.check(lib.b200gsr_frames(B, H, W, ptr(color), ptr(depth_alpha), C.c_void_p(focal.data_ptr() + 4 * b0),
                                          ptr(st_rgb), ptr(st_depth), ptr(stats), stream), "b200gsr_frames")
            side.wait_stream(main)
            with torch.cuda.stream(side):
                rgb_flat[b0 * HW * 3:b1 * HW * 3].copy_(st_rgb[:B * HW * 3], non_blocking=True)
                depth_flat[b0 * HW:b1 * HW].copy_(st_depth[:B * HW], non_blocking=True)
            copied[k].record(side)
            return slot, seq

        def settle(items):
            # A pass that overflowed is rendered, quantised and copied again; the side stream copies in issue order,
            # so the re-issued frames overwrite the invalid ones.
            for b0, b1, key, cap, slot, seq in items:
                d.settle(key, cap, slot, seq, lambda c, b0=b0, b1=b1: issue(b0, b1, c))

        pending = []
        for b0, b1 in view_chunks(N, views_per_pass):
            key = (b1 - b0, P, H, W)
            cap, known = d.capacity_for(key, (b1 - b0) * P, False)
            item = (b0, b1, key, cap) + issue(b0, b1, cap)
            if known:
                pending.append(item)
                if len(pending) >= _SETTLE_GROUP:
                    settle(pending)
                    pending = []
            else:
                settle([item])                      # a shape seen for the first time: learn its capacity now
        settle(pending)
        side.synchronize()
    return rgb, depth
