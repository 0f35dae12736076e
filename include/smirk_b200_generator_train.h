/* smirk_b200 C ABI: SmirkGenerator in train mode.  Kept in a header of its own, next to include/smirk_b200.h (whose
 * generator section it extends and whose handle type it uses), so that each header's prototype list stays fixed. */
#pragma once
#include "smirk_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Train mode (BatchNorm over batch statistics, the reference trainer's generator.train(), base_trainer.py:108-111) and the
 * gradients of every parameter (src/smirk_trainer.py:94,295).
 * A train handle holds the topology only (the configuration and precision of SmkGeneratorDesc) and is destroyed by
 * smk_generator_destroy.  Every call reads the parameters through the device pointers of SmkGeneratorTrainArgs and repacks
 * the weights into the workspace, so an optimizer step needs no new handle.  Calls never allocate or synchronise, use no
 * float atomics (bitwise reproducible) and are CUDA-graph capturable; the eval entry points of smirk_b200.h reject a train handle.
 * BatchNorm couples the images of a batch: outputs are not independent of the other images. */
typedef struct {
    /* DEVICE pointers of the module's state_dict tensors in the order of SmkGeneratorDesc.tensors (num_batches_tracked
     * removed); running_mean / running_var are updated in place.                                                      */
    float* const* tensors;
    int n_tensors;
    int64_t* const* num_batches_tracked;   /* one per BatchNorm, in state_dict order; each is incremented by one */
    float momentum;            /* running-statistics factor of every BatchNorm; negative = None (1 / num_batches_tracked) */
    float eps;
} SmkGeneratorTrainArgs;
typedef struct {
    /* Gradient outputs (written, not accumulated), NULL = not wanted: tensors[j] is the gradient of
     * SmkGeneratorTrainArgs.tensors[j]; the running-statistics entries must be NULL.                                  */
    float* const* tensors;
} SmkGeneratorTrainGrads;
int smk_generator_train_create(int in_channels, int out_channels, int init_features, int res_blocks, int precision, SmkGenerator** out);
/* Workspace of both train calls.  smk_generator_saved_bytes / smk_generator_saved_tensor describe the train handle's saved
 * buffer: the NHWC input ("input", channels zero-padded), per conv its pre-BN output (named after the conv, e.g.
 * "enc1conv1", "res0conv2") and per BatchNorm its (+ residual) (+ ReLU) output (named after the BatchNorm, e.g.
 * "enc1norm1", "res0norm2"), each decoder's input ("dec1cat": torch.cat((upconv1 output, enc1norm2 output))) and each
 * pool's output ("pool1"), followed by the batch statistics (not listed). */
size_t smk_generator_train_workspace_bytes(const SmkGenerator* h, int B);
/* Train-mode forward: x [B,in_channels,224,224] -> y as smk_generator_forward; updates the running statistics and
 * num_batches_tracked of every BatchNorm.  saved (>= smk_generator_saved_bytes) keeps the activations for
 * smk_generator_backward_train; with saved == NULL they live in ws, which must then hold smk_generator_saved_bytes more. */
int smk_generator_forward_train(const SmkGenerator* h, const SmkGeneratorTrainArgs* args, const float* x, int B, float* y,
                                float* saved, size_t saved_bytes, void* ws, size_t ws_bytes, void* stream);
/* Train-mode backward from the forward's saved buffer and output y (args: those of the forward).  g_y [B,out_channels,
 * 224,224]; g_x [B,in_channels,224,224] (NULL: not wanted, and the first conv's dgrad does not run) is written. */
int smk_generator_backward_train(const SmkGenerator* h, const SmkGeneratorTrainArgs* args, int B, const float* y, const float* saved,
                                 size_t saved_bytes, const float* g_y, float* g_x, const SmkGeneratorTrainGrads* grads, void* ws,
                                 size_t ws_bytes, void* stream);

/* Test entry point of the train path's 3x3 weight gradient (tests/test_gpu_generator_train_kernels.py; not part of the
 * drop-in surface).  Device pointers; it calls the host helper the train backward uses.  g [B,H,W,cout] (the gradient
 * of the conv's output), a [B,H,W,lda] (the conv's input, its first cin channels) -> out [cout][cin][3][3] (torch's
 * layout), 3x3 stride 1 with zero padding 1 (reflect 0) or ReflectionPad2d(1) (reflect 1).  ws: kWgradPart floats
 * (16 MiB) of split-K partials. */
int smk_debug_train_conv3_wgrad(const float* g, const float* a, int lda, int B, int H, int W, int cin, int cout, int reflect, float* out,
                                void* ws, size_t ws_bytes, void* stream);

#ifdef __cplusplus
}
#endif
