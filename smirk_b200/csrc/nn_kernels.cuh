// CUDA-core building blocks shared by the encoder and the generator (NHWC activations).
//
// The fp32 implicit-GEMM convolution `conv_gemm` (precision 0; declared with its descriptor in conv.cuh) with fused
// BN / ReLU / residual / pixel-shuffle epilogues, depthwise 3x3, the stem convolutions and the fused stem + first block,
// 2x2 max-pool, layout conversion, the final 1x1 + sigmoid and the fused global-average-pool + linear heads.
#pragma once
#include "conv.cuh"

namespace smk {

// Depthwise 3x3, TF-"SAME" padding (pad_beg = pad_total/2), stride 1 or 2, fused scale/bias/ReLU.
int dwconv3x3(const float* in, int B, int H, int W, int C, int stride, const float* w9c /*[9][C]*/,
              const float* scale, const float* bias, float* out, cudaStream_t st, bool round_out = false);
// Stems (NCHW fp32 image -> NHWC, 3x3 stride 2 TF-SAME, Cout = 16, fused scale/bias/ReLU) of n = 1 to 3 backbones.  Three
// run as one pass over the image (a CTA stages the input rows of one output row); fewer run a thread-per-pixel launch
// each, which is faster for one backbone than the one-pass kernel.
struct StemProblem { const float* w /*[27][16]*/; const float* scale; const float* bias; float* out; };
int stem_conv(const float* img_nchw, int B, int H, int W, const StemProblem* probs, int n, cudaStream_t st);
// Fused stem (3x3 s2, 3 -> 16, BN, ReLU) + depthwise-separable block 0 (dw 3x3 s{1,2} + BN + ReLU, 1x1 16 -> 16 + BN,
// + skip when stride 1) of one backbone: image NCHW fp32 -> [B, 112/stride, 112/stride, 16] NHWC.  pw_w is [ci][co] fp32.
struct StemDsProblem {
    const float* stem_w; const float* stem_s; const float* stem_b;      // [27][16], [16], [16]
    const float* dw_w; const float* dw_s; const float* dw_b;            // [9][16]
    const float* pw_w; const float* pw_s; const float* pw_b;            // [16 ci][16 co]
    float* out;
    float* s_out; float* d_out;          // optional, together: also store the stem output [B,112,112,16] and the depthwise output
    int stride;                          // of block 0's depthwise conv: 1 or 2
};
// n = 1 to 3 backbones in one launch, each with its own stride; the image is read once for all of them.
int stem_ds(const float* img_nchw, int B, int H, int W, const StemDsProblem* probs, int n, int round_out, cudaStream_t st);
int maxpool2x2(const float* in, int ld_in, int B, int H, int W, int C, float* out, cudaStream_t st);
// NCHW -> NHWC with the channel count zero-padded to Cp (a multiple of 4); round_out rounds to TF32 for a tensor-core consumer.
int nchw_to_nhwc_pad(const float* in, int B, int C, int H, int W, int Cp, float* out, cudaStream_t st, bool round_out = false);
// out[b, co, h, w] = sigmoid(bias[co] + sum_c in[b,h,w,c] * w[c][co])   (NHWC -> NCHW)
int conv1x1_sigmoid_nchw(const float* in, int B, int HW, int Cin, const float* w /*[Cin][Cout]*/, const float* bias,
                         int Cout, float* out, cudaStream_t st);
// Global average pool over HW pixels + Linear(C -> n_out) + clamp codes per output column (0 none, 1 clamp[0,1], 2 relu,
// 3 clamp[-0.2,0.2]) in one launch, for one or two backbones with the same feature shape [B, HW, C] (different head widths
// allowed).  w is [n_out][C]; codes (device) may be null.  raw (optional, for every problem or none): also store the
// pre-clamp values [B, n_out].
struct GapHeadProblem { const float* feat; const float* w; const float* bias; const uint8_t* codes; float* out; int n_out; float* raw; };
int gap_head(const GapHeadProblem* probs, int n, int B, int HW, int C, cudaStream_t st);

}  // namespace smk
