/*
 * smirk_b200 — C ABI of the trainer's emotion loss: ExpressionLoss (src/losses/ExpressionLoss.py), EMOCA's ResNet-50
 * feature extractor on gen and tar and a per-face metric of the two features, forward and input gradient.  The
 * conventions of smirk_b200.h hold here: 0 = OK, <0 = argument error, >0 = cudaError_t, message via smk_last_error();
 * create takes host tensors and uploads to the current device; forward / backward take device pointers, never allocate
 * or synchronise, and run in order on the caller's stream (CUDA-graph capturable).
 */
#ifndef SMIRK_B200_EXPRESSION_H
#define SMIRK_B200_EXPRESSION_H

#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ------------------------------------------------------------------------------------------------
 * ExpressionLoss — replaces ExpressionLoss.forward(gen, tar, use_mean, metric): f = backbone(x).view(B, -1), the
 * eval-mode ResNet-50 (Bottleneck layers (3, 4, 6, 3), the stride of each layer's first block on its 3x3 conv) up to the
 * 7x7 average pool, on gen and tar [B,3,224,224] as they are; per face l2 = mean((f_gen - f_tar)^2), l1 = mean(|.|) or
 * cos = 1 - cosine_similarity (eps 1e-8); use_mean: their mean over the faces.  The weights are frozen; the input
 * gradient goes to gen, tar or both.
 * ---------------------------------------------------------------------------------------------- */
typedef struct SmkExpressionLoss SmkExpressionLoss;

typedef struct {
    /* fp32 tensors of backbone.* in state_dict order, num_batches_tracked and backbone.fc.* left out: conv1.weight,
     * bn1 (weight, bias, running_mean, running_var), then per Bottleneck conv1, conv2, bn1, bn2, conv3, bn3 and, in the
     * first block of each layer, downsample.0 and downsample.1.                                                    */
    const float* const* tensors;
    int n_tensors;             /* 265 */
    int precision;             /* 0 = fp32 CUDA-core GEMMs, 1 = TF32 wgmma, 3 = 1 with 3xTF32 error-compensated arithmetic
                                  (fp32-equivalent).  2 is not a precision. */
} SmkExpressionLossDesc;

int smk_expression_loss_create(const SmkExpressionLossDesc* desc, SmkExpressionLoss** out);
void smk_expression_loss_destroy(SmkExpressionLoss* h);
size_t smk_expression_loss_workspace_bytes(const SmkExpressionLoss* h, int B);
/* gen, tar [B,3,224,224] NCHW -> loss: [B] per-face values, or one scalar (their mean) when use_mean.  metric: 0 = l2,
 * 1 = l1, 2 = cos.  features (optional): [2B,2048], gen's then tar's.  Deterministic: no atomics, fixed summation
 * orders; face b's value does not depend on the other faces. */
int smk_expression_loss_forward(const SmkExpressionLoss* h, const float* gen, const float* tar, int B, int metric, int use_mean,
                                float* loss, float* features, void* ws, size_t ws_bytes, void* stream);
/* Grad-mode forward: the same launches and bitwise the same loss, plus what the backward needs in `saved` (caller-owned,
 * >= smk_expression_loss_saved_bytes): for each image whose gradient is wanted, the pool output and its int8 argmax tap,
 * and u1, u2 (the post-ReLU outputs of conv1 and conv2) and y of every block, fp32 NHWC; then both halves' features.
 * need: 1 = gradient to gen, 2 = to tar, 3 = both.  ws / ws_bytes: the forward workspace. */
size_t smk_expression_loss_saved_bytes(const SmkExpressionLoss* h, int B, int need);
int smk_expression_loss_forward_saved(const SmkExpressionLoss* h, const float* gen, const float* tar, int B, int metric, int use_mean,
                                      int need, float* loss, float* saved, size_t saved_bytes, void* ws, size_t ws_bytes, void* stream);
/* Layout of tensor i of `saved`: its name ("pool", "pool_argmax" (int8), "layer1.0.u1" ... "layer4.2.y", dims B' = B per
 * saved half, gen's first when both; last "features", dims [2B,1,1,2048]), offset in floats, and dims [4] = B,H,W,C of
 * the NHWC tensor.  Returns non-zero past the last tensor. */
int smk_expression_loss_saved_tensor(const SmkExpressionLoss* h, int B, int need, int i, const char** name, size_t* offset, int* dims);
/* Input gradient of the loss times g ([B], or one scalar when use_mean): g_gen and g_tar [B,3,224,224] NCHW (written,
 * not accumulated; the one `need` does not ask for may be null).  metric, use_mean, need and saved are those of the
 * grad-mode forward.  ws >= smk_expression_loss_backward_workspace_bytes. */
size_t smk_expression_loss_backward_workspace_bytes(const SmkExpressionLoss* h, int B, int need);
int smk_expression_loss_backward(const SmkExpressionLoss* h, int B, int metric, int use_mean, int need, const float* saved,
                                 size_t saved_bytes, const float* g, float* g_gen, float* g_tar, void* ws, size_t ws_bytes,
                                 void* stream);

#ifdef __cplusplus
}
#endif

#endif /* SMIRK_B200_EXPRESSION_H */
