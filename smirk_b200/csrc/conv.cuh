// One descriptor for the GEMM-shaped convolutions of the encoder and the generator, and the one place that picks
// their kernel: the fp32 CUDA-core `conv_gemm` (nn_kernels.cu) or the TF32 wgmma `tc_conv` (gemm_tc.cu).
#pragma once
#include "common.cuh"

namespace smk {

// One convolution / GEMM problem:  out[m, n] = epi( sum_k A(m, k) * W(k, n) )
//   m indexes the output pixels (b, h, w) of an NHWC tensor, n the output channels.  Stride 1: H x W are the output dims.
//   mode 0: 1x1 conv / plain GEMM: A(m, k) = in[m*ld_in + k]
//   mode 1: 3x3 conv, zero padding 1:  k = (ky*3 + kx)*Cin + c
//   mode 2: 3x3 conv, reflection padding 1.  conv_gemm reads an unpadded [B,H,W,*] input and reflects in its loader;
//           tc_conv reads a [B,H+2,W+2,*] buffer whose halo reflect_halo has filled.
struct Conv {
    const float* in; int ld_in;          // NHWC input, pixel stride ld_in (>= Cin; lets us read a channel slice)
    int B, H, W, Cin;
    int N, K, mode;
    const float* w;                      // fp32 weights [K][N], n fastest (conv_gemm)
    const float* wt;                     // TF32 weights [N][K], k fastest (tc_conv)
    const float* wt_lo;                  // optional: TF32 tails of the weights (wt holds the heads) -> 3xTF32 arithmetic
    const float* scale; const float* bias;   // folded BN (or 1 / conv bias), per n
    int relu;
    const float* res; int ld_res; int res_pad;   // optional residual, added before the ReLU; res_pad: read it from the
                                                 // interior of a padded buffer
    float* out; int ld_out;              // pixel stride of the output (>= N; lets us write a concat slice)
    int store;                           // 0 plain, 1 pixel shuffle: n = (dy*2+dx)*Cout + co -> pixel (2h+dy, 2w+dx), channel co,
                                         // 2 interior of a [B,H+2,W+2,*] padded buffer, 3 fused 1x1 head + sigmoid: out is
                                         // [B, head_c, H, W] NCHW, the activations are not stored
    const float* head_w; const float* head_b; int head_c;     // store 3: head weights [N][head_c], bias [head_c]
    int round_out;                       // 1: round stored activations to TF32 (RN) — they feed another tensor-core layer
    const float* mask; int ld_mask;      // optional (store 0): zero output (m, n) where mask[m*ld_mask + n] <= 0 (ReLU backward)
    float* out2; int ld_out2;            // optional (no pixel shuffle): the stored activations again, compact NHWC at pixel m
    const char* tag;                     // profiler tag (null: derived from the problem)
};

// fp32 CUDA cores: modes 0-2, stores 0 and 1; no TF32 weights, padded residual or paired problem.
int conv_gemm(const Conv& p, cudaStream_t st);
// TF32 tensor cores.  p2 (optional): a second problem of identical shape sharing the launch (tiles of both in one grid).
int tc_conv(const Conv& p, cudaStream_t st, const Conv* p2 = nullptr);

// TF32 weights (wt) run tc_conv, fp32 weights (w) conv_gemm.
inline int conv(const Conv& p, cudaStream_t st, const Conv* p2 = nullptr) {
    if (p.wt) return tc_conv(p, st, p2);
    SMK_REQUIRE(!p2, "conv: paired problems need TF32 weights");
    return conv_gemm(p, st);
}

}  // namespace smk
