/*
 * smirk_b200 — input-gradient entry points of the SmirkEncoder (frozen weights, eval-mode BN).
 *
 * Included at the end of smirk_b200.h, after smirk_b200_grad.h: C and C++ callers see one ABI (SMK_VERSION 100).
 * Conventions as there: status codes, caller-owned device buffers, no allocation and no synchronisation (CUDA-graph
 * capturable), an empty batch (B = 0) is a no-op.  The backward is deterministic: no atomics, fixed summation order.
 */
#ifndef SMIRK_B200_ENCODER_GRAD_H
#define SMIRK_B200_ENCODER_GRAD_H

#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

/* Grad-mode forward: the same launches and bitwise the same outputs as smk_encoder_forward at every precision, plus what
 * the backward needs (the output of every ReLU, fp32 NHWC, and the pre-clamp head outputs) written into `saved`
 * (caller-owned, >= smk_encoder_saved_bytes; one buffer per forward whose gradient will be taken).
 * ws / ws_bytes: the forward workspace (smk_encoder_workspace_bytes). */
size_t smk_encoder_saved_bytes(const SmkEncoder* h, int B);
int smk_encoder_forward_saved(const SmkEncoder* h, const float* img, int B, float* pose_cam, float* shape, float* expr,
                              float* saved, size_t saved_bytes, void* ws, size_t ws_bytes, void* stream);
/* Layout of tensor i of `saved`: its name (the reference's module path of the ReLU's BatchNorm, e.g.
 * "shape_encoder.encoder.bn1" for the stem, "shape_encoder.encoder.blocks.2.1.bn1" / ".bn2" for an inverted-residual
 * block's expand / depthwise output, or the head, "expression_encoder.expression_layers.0", for its pre-clamp output),
 * float offset, and dims [4] = B,H,W,C of the NHWC tensor (a head is 1 x 1 x n_out).  Forward order within each backbone,
 * backbones in slot order (pose, shape, expression).  Returns non-zero past the last tensor. */
int smk_encoder_saved_tensor(const SmkEncoder* h, int B, int i, const char** name, size_t* offset, int* dims);
/* Input gradient: upstream gradients of the raw outputs (pose_cam [B,6], shape [B,n_shape], expr [B,n_exp+5]; each may
 * be NULL, meaning zero, and then its backbone launches nothing) -> g_img [B,3,224,224] NCHW (written, not accumulated;
 * zero-filled when every upstream gradient is NULL).  ws >= smk_encoder_backward_workspace_bytes. */
size_t smk_encoder_backward_workspace_bytes(const SmkEncoder* h, int B);
int smk_encoder_backward(const SmkEncoder* h, int B, const float* saved, size_t saved_bytes, const float* g_pose_cam,
                         const float* g_shape, const float* g_expr, float* g_img, void* ws, size_t ws_bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* SMIRK_B200_ENCODER_GRAD_H */
