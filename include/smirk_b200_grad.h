/*
 * smirk_b200 — input-gradient entry points of the SmirkGenerator (frozen weights, eval-mode BN).
 *
 * Included at the end of smirk_b200.h: C and C++ callers see one ABI (SMK_VERSION 100).  Conventions as there:
 * status codes, caller-owned device buffers, no allocation and no synchronisation (CUDA-graph capturable), an empty
 * batch (B = 0) is a no-op.  The backward is deterministic: no atomics, fixed summation order.
 */
#ifndef SMIRK_B200_GRAD_H
#define SMIRK_B200_GRAD_H

#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

/* Grad-mode forward: the same launches and bitwise the same y as smk_generator_forward, plus the activations the backward
 * needs (the post-ReLU output of every block conv and every ResNet conv1, fp32 NHWC) written into `saved`
 * (caller-owned, >= smk_generator_saved_bytes; one buffer per forward whose gradient will be taken).
 * ws / ws_bytes: the forward workspace (smk_generator_workspace_bytes). */
size_t smk_generator_saved_bytes(const SmkGenerator* h, int B);
int smk_generator_forward_saved(const SmkGenerator* h, const float* x, int B, float* y, float* saved, size_t saved_bytes,
                                void* ws, size_t ws_bytes, void* stream);
/* Layout of tensor i of `saved`: its name (the reference's layer name, e.g. "enc1conv2", "res0conv1", "dec1conv2"),
 * float offset, and dims [4] = B,H,W,C of the NHWC tensor.  Returns non-zero past the last tensor. */
int smk_generator_saved_tensor(const SmkGenerator* h, int B, int i, const char** name, size_t* offset, int* dims);
/* Input gradient: y (the forward's output) and g_y [B,out_channels,224,224] NCHW -> g_x [B,in_channels,224,224] NCHW
 * (written, not accumulated).  ws >= smk_generator_backward_workspace_bytes. */
size_t smk_generator_backward_workspace_bytes(const SmkGenerator* h, int B);
int smk_generator_backward(const SmkGenerator* h, int B, const float* y, const float* saved, size_t saved_bytes,
                           const float* g_y, float* g_x, void* ws, size_t ws_bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* SMIRK_B200_GRAD_H */
