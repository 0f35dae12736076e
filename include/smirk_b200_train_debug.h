/*
 * smirk_b200 — test entry points of the train-mode encoder kernels (csrc/encoder_train.cu).  Not part of the drop-in
 * surface: tests/ uses them to check each kernel on its own against torch.  Included at the end of smirk_b200_train.h.
 */
#ifndef SMIRK_B200_TRAIN_DEBUG_H
#define SMIRK_B200_TRAIN_DEBUG_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ------------------------------------------------------------------------------------------------
 * Train-kernel test entry points (used by tests/ to check the train-mode kernels one at a time against torch; not
 * part of the drop-in surface).  All pointers are device pointers; each calls the host helper the train calls use, so
 * the launches are theirs.  Activations are NHWC [M = B*H*W, C]; weights are in torch's layout.  ws / ws_bytes: scratch
 * for the partial sums, at least 512 * C * 16 bytes for bn_forward, that + 8 * C for bn_backward, and 16 MiB (4M
 * floats) for the weight gradients.
 *   bn_forward   : batch statistics of z -> mean, invstd; running_mean / running_var / num_batches_tracked updated as
 *                  the train forward does (momentum < 0: None); y = gamma * (z - mean) * invstd + beta (+ res) (ReLU when
 *                  relu) (TF32-rounded when round).  C % 4 == 0.
 *   bn_backward  : g (gradient of y; masked by [y > 0] when y is given) -> gz, which may alias g; g_gamma / g_beta
 *                  (either may be NULL).
 *   pw_wgrad     : out [Co][Ci] = sum over the M pixels of g[p][co] * a[p][ci].
 *   dw_*         : the 3x3 depthwise conv (TF-SAME, stride 1 or 2) of a [B,H,H,C] with w [C][1][3][3]; dgrad adds res
 *                  (may be NULL) to the input gradient [B,H,H,C].
 *   stem_*       : the stem conv of img [B,3,H,W] (3x3 stride 2 TF-SAME, 3 -> 16; H and W of one parity), z and its
 *                  gradient g [B,ceil(H/2),ceil(W/2),16]; out [16][3][3][3].
 *   head_backward: codes [n_out] (NULL: all 0) per output: 0 pass, 1 clamp [0, 1], 2 ReLU, 3 clamp [-0.2, 0.2], judged
 *                  on the pre-clamp output raw [B][n_out]; gp [B][n_out] (gradient of raw), g_feat [B,HW,C] (of the
 *                  features before the global pool), g_w [n_out][C] and g_b [n_out] (either may be NULL) from pooled [B][C].
 * ---------------------------------------------------------------------------------------------- */
int smk_debug_train_bn_forward(const float* z, int M, int C, float eps, float momentum, const float* gamma, const float* beta,
                               float* rmean, float* rvar, int64_t* nbt, const float* res, int relu, int round, float* mean,
                               float* invstd, float* y, void* ws, size_t ws_bytes, void* stream);
int smk_debug_train_bn_backward(const float* g, const float* y, const float* z, const float* mean, const float* invstd,
                                const float* gamma, int M, int C, int round, float* gz, float* g_gamma, float* g_beta, void* ws,
                                size_t ws_bytes, void* stream);
int smk_debug_train_pw_wgrad(const float* g, const float* a, int M, int Co, int Ci, float* out, void* ws, size_t ws_bytes, void* stream);
int smk_debug_train_dw_forward(const float* a, const float* w, int B, int H, int C, int stride, float* z, void* stream);
int smk_debug_train_dw_wgrad(const float* g, const float* a, int B, int H, int C, int stride, float* out, void* ws, size_t ws_bytes,
                             void* stream);
int smk_debug_train_dw_dgrad(const float* g, const float* w, const float* res, int B, int H, int C, int stride, float* out, void* stream);
int smk_debug_train_stem_forward(const float* img, const float* w, int B, int H, int W, float* z, void* stream);
int smk_debug_train_stem_wgrad(const float* g, const float* img, int B, int H, int W, float* out, void* ws, size_t ws_bytes, void* stream);
int smk_debug_train_head_backward(const float* g, const float* raw, const uint8_t* codes, const float* w, const float* pooled, int B,
                                  int n_out, int HW, int C, float* gp, float* g_feat, float* g_w, float* g_b, void* stream);

#ifdef __cplusplus
}
#endif

#endif /* SMIRK_B200_TRAIN_DEBUG_H */
