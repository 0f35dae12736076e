// Fused expand-1x1 + depthwise-3x3 kernel (see xdw_tc.cu).
#pragma once
#include "common.cuh"

namespace smk {

struct XdwConv {
    const float* x;                       // [B,H,W,Cin] NHWC, contiguous
    int B, H, W, Cin;
    const float* w1t;                     // 1x1 expand weights [mid][Cin] (K-major, TF32-rounded)
    const float* w1t_lo;                  // non-null: TF32 tails of the weights (w1t holds the heads) -> 3xTF32 arithmetic
    const float* scale1; const float* bias1;     // folded BN after the 1x1 conv (ReLU follows)
    int mid;
    const float* wdw;                     // depthwise weights [9][mid]
    const float* scale2; const float* bias2;     // folded BN after the depthwise conv (ReLU follows)
    int stride;                           // 1 or 2, TF-"SAME" padding
    int round_out;                        // round d to TF32 (it feeds the projection GEMM)
    float* out;                           // d: [B,Ho,Wo,mid]
    float* e_out;                         // optional: also store e [B,H,W,mid] (the backward's ReLU mask)
};

// p2 (optional): a second problem of identical shape sharing the launch.
int xdw_conv(const XdwConv& p, cudaStream_t st, const XdwConv* p2 = nullptr);

}  // namespace smk
