// fp32 CUDA-core building blocks shared by the encoder and the generator (NHWC activations).
//
// These are the exact-fp32 path (precision = 0): a tiled implicit-GEMM convolution with fused
// BN / ReLU / residual / pixel-shuffle epilogues, depthwise 3x3, stem conv, 2x2 max-pool, layout
// conversion, the final 1x1+sigmoid and the pooled linear heads.  The TF32 wgmma GEMM in
// gemm_tc.cu replaces `conv_gemm` for the tensor-bound layers when precision = 1.
#pragma once
#include "common.cuh"

namespace smk {

// One convolution / GEMM problem:  C[m, n] = epi( sum_k A(m, k) * W[k, n] )
//   m indexes output pixels (b, oh, ow) of an NHWC tensor, n output channels.
//   mode 0: 1x1 conv / plain GEMM: A(m,k) = in[m*ld_in + k]
//   mode 1: 3x3 stride-1 conv, zero padding 1:   k = (ky*3+kx)*Cin + c
//   mode 2: 3x3 stride-1 conv, reflection padding 1
struct ConvProblem {
    const float* in; int ld_in;          // pixel stride of the input (>= Cin; lets us read a channel slice)
    int B, H, W, Cin;                    // input spatial dims (= output dims: stride 1)
    const float* w;                      // [K][N], n fastest
    const float* scale; const float* bias;   // folded BN (or 1 / conv bias), per n
    int N, K, mode;
    int relu;
    const float* res; int ld_res;        // optional residual added after scale/bias (no ReLU afterwards)
    float* out; int ld_out;              // pixel stride of the output (>= N; lets us write a concat slice)
    int shuffle;                         // 1: n = (dy*2+dx)*Cout + co  ->  pixel (2h+dy, 2w+dx), channel co
    int round_out;                       // 1: round outputs to TF32 (they feed a tensor-core layer)
    const float* mask; int ld_mask;      // optional: zero output (m, n) where mask[m*ld_mask + n] <= 0 (ReLU backward)
    float* out2; int ld_out2;            // optional second store of the output at pixel m (no shuffle)
    const char* tag;                     // profiler tag (null: derived from the problem)
};

int conv_gemm(const ConvProblem& p, cudaStream_t st);

// Depthwise 3x3, TF-"SAME" padding (pad_beg = pad_total/2), stride 1 or 2, fused scale/bias/ReLU.
int dwconv3x3(const float* in, int B, int H, int W, int C, int stride, const float* w9c /*[9][C]*/,
              const float* scale, const float* bias, float* out, cudaStream_t st, bool round_out = false);
// Stem: NCHW fp32 image -> NHWC, 3x3 stride 2 TF-SAME, Cout = 16, fused scale/bias/ReLU.
int stem_conv(const float* img_nchw, int B, int H, int W, const float* w /*[27][16]*/, const float* scale,
              const float* bias, float* out, cudaStream_t st);
// Three 16-channel stems over the same image in one pass (the encoder's three backbones).
int stem_conv3(const float* img_nchw, int B, int H, int W, const float* const w[3], const float* const scale[3],
               const float* const bias[3], float* const out[3], cudaStream_t st);
// Fused stem (3x3 s2, 3 -> 16, BN, ReLU) + depthwise-separable block 0 (dw 3x3 s{1,2} + BN + ReLU, 1x1 16 -> 16 + BN,
// + skip when stride 1) of one backbone: image NCHW fp32 -> [B, 112/stride, 112/stride, 16] NHWC.  pw_w is [ci][co] fp32.
struct StemDsProblem {
    const float* stem_w; const float* stem_s; const float* stem_b;      // [27][16], [16], [16]
    const float* dw_w; const float* dw_s; const float* dw_b;            // [9][16]
    const float* pw_w; const float* pw_s; const float* pw_b;            // [16 ci][16 co]
    float* out;
};
// n = 1 or 2 backbones of the same block-0 stride in one launch (they read the same image).
int stem_ds(const float* img_nchw, int B, int H, int W, const StemDsProblem* probs, int n, int stride, int round_out, cudaStream_t st);
int stem_ds(const float* img_nchw, int B, int H, int W, const float* stem_w /*[27][16]*/, const float* stem_s, const float* stem_b,
            const float* dw_w /*[9][16]*/, const float* dw_s, const float* dw_b, const float* pw_w /*[16][16]*/, const float* pw_s,
            const float* pw_b, int stride, int round_out, float* out, cudaStream_t st);
int maxpool2x2(const float* in, int ld_in, int B, int H, int W, int C, float* out, cudaStream_t st);
// NCHW -> NHWC with the channel count zero-padded to Cp (a multiple of 4); round_out rounds to TF32 for a tensor-core consumer.
int nchw_to_nhwc_pad(const float* in, int B, int C, int H, int W, int Cp, float* out, cudaStream_t st, bool round_out = false);
// out[b, co, h, w] = sigmoid(bias[co] + sum_c in[b,h,w,c] * w[c][co])   (NHWC -> NCHW)
int conv1x1_sigmoid_nchw(const float* in, int B, int HW, int Cin, const float* w /*[Cin][Cout]*/, const float* bias,
                         int Cout, float* out, cudaStream_t st);
// Global average pool over HW pixels + Linear(C -> n_out); clamp codes per output column:
//   0 none, 1 clamp[0,1], 2 relu, 3 clamp[-0.2,0.2]
int gap_linear(const float* feat, int B, int HW, int C, const float* w /*[n_out][C]*/, const float* bias, int n_out,
               const uint8_t* clamp_codes /*device, may be null*/, float* pooled_scratch /*[B][C]*/, float* out, cudaStream_t st);

// The same in one launch, for one or two backbones with the same feature shape [B, HW, C] (different head widths allowed).
struct GapHeadProblem { const float* feat; const float* w; const float* bias; const uint8_t* codes; float* out; int n_out; };
int gap_head(const GapHeadProblem* probs, int n, int B, int HW, int C, cudaStream_t st);

}  // namespace smk
