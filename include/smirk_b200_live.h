/*
 * smirk_b200 — live eval handles of SmirkEncoder and SmirkGenerator: the eval path (folded BatchNorm, packed operands) over
 * weights that are refreshed on the device from the module's own tensors, for a frozen network whose weights and running
 * statistics another path keeps changing (the second path of the reference trainer's step).
 *
 * Conventions: those of smirk_b200.h, with two exceptions.
 *   - "handles are immutable afterwards" does not hold for a live handle: `*_refresh` rewrites its folded scales and biases
 *     and its packed operands in place.  A refresh is ordered only on the stream passed to it: work of the handle on other
 *     streams must be ordered against it by the caller.  A refresh never allocates or synchronises and is CUDA-graph
 *     capturable, so a graph that holds the refresh and the forward reads the weights of replay time.
 *   - a live handle is created without weights: its buffers are allocated but unset, and smk_encoder_forward /
 *     forward_saved / backward (smk_generator_* alike) fail with a message saying so until the first refresh.  The
 *     size and layout queries (workspace_bytes, saved_bytes, saved_tensor, backward_workspace_bytes) answer from creation.
 * Live handles are eval handles: every eval entry point of smirk_b200.h accepts one, the train entry points reject it, and
 * it is destroyed by smk_encoder_destroy / smk_generator_destroy.
 */
#ifndef SMIRK_B200_LIVE_H
#define SMIRK_B200_LIVE_H

#include "smirk_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* An eval encoder handle of the backbones in `backbones` (bit set: 1 pose, 2 shape, 4 expression) with the head widths and
 * precision (0-3) of SmkEncoderDesc: the topology, saved layout, fork sets, clamp codes, unit scales and zero biases that
 * smk_encoder_create builds at that precision, its weight, scale, bias and head buffers allocated but not filled. */
int smk_encoder_live_create(int backbones, int n_shape, int n_exp, int precision, SmkEncoder** out);
/* Sets the live handle's weights from the device tensors of args (SmkEncoderTrainArgs: per backbone the conv weights and
 * BatchNorm tensors in state_dict order, the heads, eps): folds every BatchNorm from its running statistics with
 * args->eps[i] (bit for bit smk_encoder_create's host fold) and repacks every operand the eval path reads, in place.
 * num_batches_tracked (may be NULL) and momentum are ignored.  Launches, at every precision: 1 fold launch per 160
 * BatchNorms, then 1 pack launch per 40 jobs (a forward and a dgrad operand per conv, each head) — 1 + 7 = 8 for the whole
 * encoder (126 BatchNorms, 258 jobs), 1 + 2 = 3 for the pose encoder alone (34, 70), 1 + 3 = 4 for the shape or the
 * expression encoder alone (46, 94). */
int smk_encoder_refresh(SmkEncoder* h, const SmkEncoderTrainArgs* args, void* stream);

/* The same for SmirkGenerator at precisions 0, 1 and 3 (the configuration of SmkGeneratorDesc). */
int smk_generator_live_create(int in_channels, int out_channels, int init_features, int res_blocks, int precision, SmkGenerator** out);
/* Folds every BatchNorm with args->eps and repacks the 3x3 convs (forward, and dgrad with the folded scale), the
 * up-convolutions (forward, dgrad and the bias repeated over the four sub-positions, unit scale) and the 1x1 head, in place;
 * num_batches_tracked and momentum are ignored.  Launches: 1 fold launch per 160 BatchNorms (18 + 2 res_blocks of them),
 * then 1 pack launch per 40 jobs (2 (18 + 2 res_blocks) + 3 * 4 + 2) — 1 + 2 = 3 with 5 ResNet blocks. */
int smk_generator_refresh(SmkGenerator* h, const SmkGeneratorTrainArgs* args, void* stream);

#ifdef __cplusplus
}
#endif

#endif /* SMIRK_B200_LIVE_H */
