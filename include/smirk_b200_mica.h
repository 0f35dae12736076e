/*
 * smirk_b200 — C ABI of MICA (src/models/MICA/mica.py): the frozen ArcFace iResNet-100 and shape regressor the pretraining
 * step's MICA shape loss runs, forward only, and that loss, mse_loss(shape_params, mica_shape), with its gradient to
 * shape_params.  The conventions of smirk_b200.h hold here: 0 = OK, <0 = argument error, >0 = cudaError_t, message via
 * smk_last_error(); create takes host tensors and uploads to the current device; the other entry points take device
 * pointers, never allocate or synchronise, and run in order on the caller's stream (CUDA-graph capturable).
 */
#ifndef SMIRK_B200_MICA_H
#define SMIRK_B200_MICA_H

#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct SmkMica SmkMica;

typedef struct {
    /* fp32 tensors of the module's state_dict in state_dict order, num_batches_tracked left out: arcface.* (conv1, bn1,
     * prelu, layer1.0 ... layer4.2, bn2, fc, features), then regressor.* (network.0 ... network.3, output).  781.    */
    const float* const* tensors;
    int n_tensors;
    int precision;             /* 0 = fp32 CUDA-core implicit GEMM, 1 = TF32 wgmma implicit GEMM,
                                  3 = 1 with 3xTF32 error-compensated arithmetic (fp32-equivalent).  2 is not a precision. */
} SmkMicaDesc;

int smk_mica_create(const SmkMicaDesc* desc, SmkMica** out);
void smk_mica_destroy(SmkMica* h);
size_t smk_mica_workspace_bytes(const SmkMica* h, int B);
/* images [B,3,112,112] NCHW (RGB in [0, 1]) -> shape_params [B,300]; features (optional, null: not written) [B,512]: the
 * ArcFace embedding before F.normalize.  Eval-mode BatchNorm throughout.  Deterministic and batch-independent. */
int smk_mica_forward(const SmkMica* h, const float* images, int B, float* shape_params, float* features,
                     void* ws, size_t ws_bytes, void* stream);
/* MICA shape loss over the first D columns: loss (one fp32 device scalar, written) = mean over b < B, d < D of
 * (shape_params[b*D + d] - mica_shape[b*ld + d])^2.  One CTA, fixed summation order, no atomics. */
int smk_mica_shape_loss_forward(const float* shape_params, const float* mica_shape, int B, int D, int ld, float* loss,
                                void* stream);
/* Its gradient times the device scalar g: grad [B,D] (written) = (2 / (B*D)) * (shape_params - mica_shape) * g. */
int smk_mica_shape_loss_backward(const float* shape_params, const float* mica_shape, int B, int D, int ld, const float* g,
                                 float* grad, void* stream);

#ifdef __cplusplus
}
#endif

#endif /* SMIRK_B200_MICA_H */
