/*
 * b200gsr_loss.h - the reconstruction loss of DreamScene's refine stages and its image gradient, and the guidance
 * stages' total-variation and scale regularisers (additive to b200gsr.h, same conventions and the same library,
 * libb200gsr.so; ABI version unchanged).
 *
 * B independent losses over N elements each; view v is image[v N .. (v + 1) N):
 *
 *   loss[v] = weight * mean((fp16(image_v) - target[idx[v]]) ** 2)
 *
 * which is the reference's `l2_loss(image.to(torch.float16), gt) * weight` with torch's dtype rules: a float16 target
 * keeps every intermediate in fp16; a float32 target makes the difference and the mean fp32.
 *
 *   image          : DEVICE float [B, N].
 *   target         : DEVICE [n_targets, N], float16 (target_is_half = 1) or float32 (0).
 *   target_index   : DEVICE int32 [B] (view v uses target target_index[v]) or NULL (view v uses target v, which needs
 *                    B <= n_targets).  Read on the device, so a captured graph may change it between replays; an
 *                    index outside [0, n_targets) gives that view a NaN loss and NaN gradients.
 *   weight         : the loss weight (100 in the reference).
 *   grad_out       : DEVICE [B] in the loss dtype (float16 if target_is_half, else float32): the incoming gradient of
 *                    each view's loss.  Needed only with d_image.
 *   loss_out       : DEVICE [B] in the loss dtype, or NULL for no loss.
 *   d_image        : DEVICE float [B, N], or NULL for no gradient.  Bit for bit torch's autograd gradient of the
 *                    expression with respect to the float32 image for the incoming gradient grad_out (DESIGN.md f9).
 *   scratch        : DEVICE, at least b200gsr_recon_l2_scratch_bytes(B, N) bytes, 8-byte aligned; needed only with
 *                    loss_out.  No initialisation needed: the loss is a fixed-order sum of per-block partials, so it is
 *                    bitwise reproducible.
 *
 * At least one of loss_out and d_image.  No memset, no allocation, no host sync.
 *
 * The guidance stages' regularisers (DESIGN.md f10), same conventions:
 *
 *   b200gsr_tv_loss     loss = 2 * (h_tv / (C (H-1) W) + w_tv / (C H (W-1))) / B over x [B,C,H,W], where h_tv / w_tv
 *                       are the sums of the squared differences of vertically / horizontally adjacent elements (the
 *                       reference's tv_loss).  H >= 2, W >= 2, at most 2^31 - 1 elements.
 *   b200gsr_scale_loss  loss = mean(mean(scales, -1)) over scales [rows, 3], at most 2^31 - 1 elements.
 *
 *   x / scales     : DEVICE float, contiguous.  Always required (the scale gradient does not read it).
 *   grad_out       : DEVICE float [1], the incoming gradient of the loss.  Needed only with d_x / d_scales.
 *   loss_out       : DEVICE float [1], or NULL for no loss.  A fixed-order double sum, bitwise reproducible.
 *   d_x / d_scales : DEVICE float of x's / scales' shape, or NULL for no gradient.  Bit for bit torch's CUDA
 *                    autograd gradient of the expression for grad_out (DESIGN.md f10).  With accumulate = 1 the
 *                    gradient g is added to what the buffer holds (d = d + g, one fp32 add per element), else it is
 *                    written.
 *   scratch        : DEVICE, at least *_scratch_bytes(...) bytes, 8-byte aligned; needed only with loss_out.
 *
 * At least one of loss_out and the gradient.  No memset, no allocation, no host sync.
 */
#ifndef B200GSR_LOSS_H
#define B200GSR_LOSS_H

#include "b200gsr.h"

#ifdef __cplusplus
extern "C" {
#endif

size_t b200gsr_recon_l2_scratch_bytes(int32_t B, int32_t N);
int b200gsr_recon_l2(int32_t B, int32_t N, const float* image, const void* target, int32_t target_is_half,
                     int32_t n_targets, const int32_t* target_index, float weight, const void* grad_out,
                     void* loss_out, float* d_image, void* scratch, size_t scratch_bytes, void* stream);
size_t b200gsr_tv_loss_scratch_bytes(int32_t B, int32_t C, int32_t H, int32_t W);
int b200gsr_tv_loss(int32_t B, int32_t C, int32_t H, int32_t W, const float* x, const float* grad_out, float* loss_out,
                    float* d_x, int32_t accumulate, void* scratch, size_t scratch_bytes, void* stream);
size_t b200gsr_scale_loss_scratch_bytes(int32_t rows);
int b200gsr_scale_loss(int32_t rows, const float* scales, const float* grad_out, float* loss_out, float* d_scales,
                       int32_t accumulate, void* scratch, size_t scratch_bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B200GSR_LOSS_H */
