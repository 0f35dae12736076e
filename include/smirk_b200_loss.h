/*
 * smirk_b200 — C ABI of the trainer's losses: VGGPerceptualLoss (src/losses/VGGPerceptualLoss.py), forward and input
 * gradient.  The conventions of smirk_b200.h hold here: 0 = OK, <0 = argument error, >0 = cudaError_t, message via
 * smk_last_error(); create takes host tensors and uploads to the current device; forward / backward take device pointers,
 * never allocate or synchronise, and run in order on the caller's stream (CUDA-graph capturable).
 */
#ifndef SMIRK_B200_LOSS_H
#define SMIRK_B200_LOSS_H

#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ------------------------------------------------------------------------------------------------
 * VGGPerceptualLoss — replaces VGGPerceptualLoss.forward: sum over the taps relu1_2, relu2_2, relu3_3, relu4_3 of
 * torchvision VGG16 features[:23] of l1_loss(phi(x), phi(y)), x and y normalised as (v * 0.5 + 0.5 - mean) / std.
 * The weights are frozen; the input gradient goes to x, y or both.
 * ---------------------------------------------------------------------------------------------- */
typedef struct SmkVggLoss SmkVggLoss;

typedef struct {
    /* fp32 tensors of the module's state_dict in state_dict order: mean [1,3,1,1], std [1,3,1,1], then weight
     * [cout,cin,3,3] and bias [cout] of the ten convolutions (blocks.0.0 ... blocks.3.21).                     */
    const float* const* tensors;
    int n_tensors;             /* 22 */
    int precision;             /* 0 = fp32 CUDA-core implicit GEMM, 1 = TF32 wgmma implicit GEMM,
                                  3 = 1 with 3xTF32 error-compensated arithmetic (fp32-equivalent).  2 is not a precision. */
} SmkVggLossDesc;

int smk_vgg_loss_create(const SmkVggLossDesc* desc, SmkVggLoss** out);
void smk_vgg_loss_destroy(SmkVggLoss* h);
size_t smk_vgg_loss_workspace_bytes(const SmkVggLoss* h, int B);
/* x, y [B,3,224,224] NCHW -> loss, one fp32 device scalar (written).  x and y may be the same tensor.  Deterministic:
 * no atomics, fixed summation order.  An empty batch (B = 0) is an argument error: the loss of nothing is undefined. */
int smk_vgg_loss_forward(const SmkVggLoss* h, const float* x, const float* y, int B, float* loss,
                         void* ws, size_t ws_bytes, void* stream);
/* Grad-mode forward: the same launches and bitwise the same loss, plus what the backward needs in `saved` (caller-owned,
 * >= smk_vgg_loss_saved_bytes): the post-ReLU output of every convolution, fp32 NHWC, for each half whose gradient is
 * wanted, and per tap an int8 map of sign(phi(x) - phi(y)) (-1, 0, +1).  need: 1 = gradient to x, 2 = to y, 3 = both.
 * ws / ws_bytes: the forward workspace (smk_vgg_loss_workspace_bytes). */
size_t smk_vgg_loss_saved_bytes(const SmkVggLoss* h, int B, int need);
int smk_vgg_loss_forward_saved(const SmkVggLoss* h, const float* x, const float* y, int B, int need, float* loss,
                               float* saved, size_t saved_bytes, void* ws, size_t ws_bytes, void* stream);
/* Layout of tensor i of `saved`: its name ("relu1_1" ... "relu4_3": fp32, dims B' = B per saved half (x's first when both),
 * "sign1_2" ... "sign4_3": int8, dims B), offset in floats, and dims [4] = B,H,W,C of the NHWC tensor.  Returns non-zero
 * past the last tensor. */
int smk_vgg_loss_saved_tensor(const SmkVggLoss* h, int B, int need, int i, const char** name, size_t* offset, int* dims);
/* Input gradient of the loss times the device scalar g: g_x and g_y [B,3,224,224] NCHW (written, not accumulated; the one
 * `need` does not ask for may be null).  `need` and `saved` are those of the grad-mode forward.
 * ws >= smk_vgg_loss_backward_workspace_bytes. */
size_t smk_vgg_loss_backward_workspace_bytes(const SmkVggLoss* h, int B, int need);
int smk_vgg_loss_backward(const SmkVggLoss* h, int B, int need, const float* saved, size_t saved_bytes, const float* g,
                          float* g_x, float* g_y, void* ws, size_t ws_bytes, void* stream);

#ifdef __cplusplus
}
#endif

#endif /* SMIRK_B200_LOSS_H */
