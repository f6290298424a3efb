/*
 * b200gsr_frames.h - 8-bit video frames of a stacked forward's views (additive to b200gsr.h and b200gsr_scene.h; same
 * conventions and the same library, libb200gsr.so; ABI version unchanged).
 *
 * DreamScene's video loops (training/object_trainer.py video_inference, training/scene_trainer.py
 * scene_video_inference / scene_cams_record) turn every rendered view into two uint8 frames:
 *     rgb   = (clamp(image, 0, 1) * 255).round().astype(uint8)                      permuted to [H,W,3]
 *     depth = (clamp(disp / disp.max(), 0, 1) * 255).round().astype(uint8)          permuted to [H,W,1]
 * with disp the normalised disparity of b200gsr_disparity_forward.  b200gsr_frames does both for B views on the device.
 *
 *   color, depth_alpha : the out_color [3,Hs,W] and out_depth_alpha [2,Hs,W] of a b200gsr_forward_views /
 *                        b200gsr_forward_scene of the same B views of H x W, as the forward writes them: for B > 1
 *                        Hs = b200gsr_views_geometry(B, H, W) and view v starts at row v * Hs / B; a single view is
 *                        written unpadded, Hs = H.  Read in place, no repacking.
 *   focal[B]           : device float32, the disparity's focal length per view, 1 / (2 tanfovx).
 *   rgb8               : [B,H,W,3] uint8, 4-byte aligned.   depth8 : [B,H,W,1] uint8, 4-byte aligned.
 *   stats              : device scratch of B * B200GSR_FRAMES_STATS_BYTES bytes (overwritten).
 *
 * The frames are bit for bit the reference's expressions above: float32 products by 255 rounded half to even, the
 * division by the maximum correctly rounded.  Where numpy's cast is undefined the result is fixed: a NaN colour value
 * gives 0, and a view whose disparity is constant (max == min, e.g. an empty view) gives an all-zero depth frame.
 * 1 <= B <= B200GSR_MAX_VIEWS, H, W >= 1 and B * H * W * 3 < 2^31, else B200GSR_ERR_BAD_ARG.  No host sync.
 */
#ifndef B200GSR_FRAMES_H
#define B200GSR_FRAMES_H

#include "b200gsr.h"

#define B200GSR_FRAMES_STATS_BYTES 32   /* per view */

#ifdef __cplusplus
extern "C" {
#endif

int b200gsr_frames(int32_t B, int32_t H, int32_t W, const float* color, const float* depth_alpha, const float* focal,
                   uint8_t* rgb8, uint8_t* depth8, void* stats, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B200GSR_FRAMES_H */
