/*
 * smirk_b200 — C ABI of SmirkEncoder in train mode: BatchNorm over batch statistics (the reference trainer's
 * encoder.train(), base_trainer.py:108-111) and the gradients of every parameter (src/smirk_trainer.py:34-73).
 *
 * Included at the end of smirk_b200.h and following its conventions.  It extends the encoder section there: the handle
 * type is SmkEncoder, destroyed by smk_encoder_destroy, and smk_encoder_saved_bytes / smk_encoder_saved_tensor describe a
 * train handle's saved buffer.
 */
#ifndef SMIRK_B200_TRAIN_H
#define SMIRK_B200_TRAIN_H

#include "smirk_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Train mode (BatchNorm over batch statistics, the reference trainer's encoder.train()) and the parameter gradients.
 * A train handle holds the topology only — the backbones in `backbones` (bit set: 1 pose, 2 shape, 4 expression), the head
 * widths and the precision (as SmkEncoderDesc's; precision 2 computes as 1, there is no fused train kernel) — and is
 * destroyed by smk_encoder_destroy.  Every call reads the parameters through the device pointers of SmkEncoderTrainArgs and
 * repacks the 1x1 weights into the workspace, so an optimizer step needs no new handle.  Calls never allocate or
 * synchronise, use no float atomics (bitwise reproducible) and are CUDA-graph capturable; the eval entry points above reject
 * a train handle.  BatchNorm couples the images of a batch: outputs are not independent of the other images. */
typedef struct {
    /* Per backbone, DEVICE pointers of its `encoder.*` tensors in the order of SmkEncoderDesc.tensors (per conv: weight,
     * BN weight, bias, running_mean, running_var); running_mean / running_var are updated in place.                   */
    float* const* tensors[3];
    int n_tensors[3];
    int64_t* const* num_batches_tracked[3];   /* one per BatchNorm, in the same order; each is incremented by one     */
    const float* head_w[3];
    const float* head_b[3];
    float momentum[3];         /* running-statistics factor; negative = None (cumulative average, 1 / num_batches_tracked) */
    float eps[3];
} SmkEncoderTrainArgs;
typedef struct {
    /* Gradient outputs (written, not accumulated), NULL = not wanted.  tensors[i][j] is the gradient of
     * SmkEncoderTrainArgs.tensors[i][j]; the running-statistics entries must be NULL.  tensors[i] itself may be NULL.  */
    float* const* tensors[3];
    float* head_w[3];
    float* head_b[3];
} SmkEncoderTrainGrads;
int smk_encoder_train_create(int backbones, int n_shape, int n_exp, int precision, SmkEncoder** out);
/* Workspace of both train calls.  smk_encoder_saved_bytes / smk_encoder_saved_tensor describe the train handle's saved
 * buffer: per BatchNorm the conv's pre-BN output (named after the conv, e.g. "shape_encoder.encoder.blocks.2.1.conv_pw"),
 * every ReLU output (named as in eval mode), every block output ("...blocks.2.1"), the pooled features
 * ("shape_encoder.pooled", [B,feat]) and the heads' pre-clamp outputs, followed by the batch statistics (not listed). */
size_t smk_encoder_train_workspace_bytes(const SmkEncoder* h, int B);
/* Train-mode forward: outputs as smk_encoder_forward; updates the running statistics and num_batches_tracked of every
 * BatchNorm.  saved (>= smk_encoder_saved_bytes) keeps the activations for smk_encoder_backward_train; with saved == NULL
 * they live in ws, which must then hold smk_encoder_saved_bytes more. */
int smk_encoder_forward_train(const SmkEncoder* h, const SmkEncoderTrainArgs* args, const float* img, int B, float* pose_cam,
                              float* shape, float* expr, float* saved, size_t saved_bytes, void* ws, size_t ws_bytes, void* stream);
/* Train-mode backward from the forward's saved buffer (args and img: those of the forward).  Upstream gradients may be
 * NULL: a backbone without one, or whose parameters want no gradient while g_img is NULL, launches nothing (and writes
 * none of its gradients).  g_img [B,3,224,224] (NULL: not wanted) is written. */
int smk_encoder_backward_train(const SmkEncoder* h, const SmkEncoderTrainArgs* args, const float* img, int B, const float* saved,
                               size_t saved_bytes, const float* g_pose_cam, const float* g_shape, const float* g_expr, float* g_img,
                               const SmkEncoderTrainGrads* grads, void* ws, size_t ws_bytes, void* stream);

#ifdef __cplusplus
}
#endif

#endif /* SMIRK_B200_TRAIN_H */
