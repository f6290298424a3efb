"""The reference's video-frame loop restated over a render callable (training/object_trainer.py:91-103; the loops of
training/scene_trainer.py scene_video_inference and scene_cams_record are the same), with the same torch and numpy
operations in the same order.  The checker of dreamscene_b200.video.render_frames; not product code.

One rule is added where the reference's result is undefined: numpy's cast of a NaN to uint8 (a NaN colour value, or
the 0 / 0 of `depth / depth.max()` when a view's disparity is all zero) gives 0 here.
"""
import numpy as np
import torch


def _nan_to_zero(x: np.ndarray) -> np.ndarray:
    return np.where(np.isnan(x), np.float32(0.0), x)


def frames(render, views):
    """render(view) -> (rgb [3,H,W], depth [1,H,W] or None), the reference's out["image"], out["depth"].
    -> (img_frames, depth_frames): lists of uint8 [H,W,3] / [H,W,1] numpy arrays, as the reference hands to imageio."""
    img_frames = []
    depth_frames = []
    for viewpoint in views:
        rgb, depth = render(viewpoint)
        if depth is not None:
            depth_norm = depth / depth.max()
            depths = torch.clamp(depth_norm, 0.0, 1.0)
            depths = depths.detach().cpu().permute(1, 2, 0).numpy()
            depths = (_nan_to_zero(depths) * 255).round().astype(np.uint8)
            depth_frames.append(depths)
        image = torch.clamp(rgb, 0.0, 1.0)
        image = image.detach().cpu().permute(1, 2, 0).numpy()
        image = (_nan_to_zero(image) * 255).round().astype(np.uint8)
        img_frames.append(image)
    return img_frames, depth_frames


def native_render(groups):
    """The render callable of the project's per-view path: render_scene without augmentation and the native
    disparity, focal 1 / (2 tanfovx) as the reference computes it."""
    from dreamscene_b200.postprocess import disparity_from_depth_alpha
    from dreamscene_b200.scene import render_scene

    def render(s):
        color, _, depth_alpha = render_scene(groups, [s], shs_aug=False, scale_aug=False)[0]
        disp, _ = disparity_from_depth_alpha(depth_alpha, 1.0 / (2.0 * float(s.tanfovx)))
        return color, disp
    return render
