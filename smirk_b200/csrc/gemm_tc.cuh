// TF32 wgmma implicit-GEMM convolution (see gemm_tc.cu).
#pragma once
#include "common.cuh"
#include <cuda.h>

namespace smk {

struct TcConv {
    const float* in; int ld_in;          // NHWC input, pixel stride ld_in (mode 2: buffer is [B,H+2,W+2,*], reflection padded)
    int B, H, W, Cin;                    // OUTPUT spatial dims H x W (stride-1 convs), input channels
    const float* wt;                     // [N][K], k fastest, k = (ky*3+kx)*Cin + c for 3x3
    const float* wt_lo;                  // non-null: TF32 tails of the weights (wt holds the heads) -> 3xTF32 arithmetic
    const float* scale; const float* bias;
    int N, K;
    int mode;                            // 0: 1x1 / plain GEMM, 1: 3x3 zero pad 1, 2: 3x3 over a pre-padded buffer
    int relu;
    const float* res; int ld_res; int res_pad;   // residual; res_pad: read it from the interior of a padded buffer
    float* out; int ld_out;
    int store;                           // 0 plain, 1 pixel-shuffle (N = 4*Cout), 2 interior of a (H+2)x(W+2) padded buffer,
                                         // 3 fused 1x1 head + sigmoid: out is [B, head_c, H, W] NCHW, the activations are not stored
    const float* head_w; const float* head_b; int head_c;     // store 3: head weights [N][head_c], bias [head_c]
    int round_out;                       // 1: round stored activations to TF32 (RN) — they feed another tensor-core layer
    const float* mask; int ld_mask;      // optional (store 0): zero output (m, n) where mask[m*ld_mask + n] <= 0 (ReLU backward)
    float* out2; int ld_out2;            // optional (store 0, 2, 3): the stored activations again, compact NHWC at pixel m
    const char* tag;                     // profiler tag (null: derived from the problem)
};

int tc_init();                                              // resolves the driver's tensor-map encoders

// TMA descriptors over fp32 tensors as the wgmma kernels read them: boxes of 32 elements (128 bytes) in the innermost
// dimension, SWIZZLE_128B, L2 promotion 128 B, zero fill out of bounds.  `what` names the operand in the error message.
// [rows][cols] matrix with a row stride of ld elements, boxes of box_rows x 32.
int encode_2d(CUtensorMap* map, const float* base, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows, const char* what);
// NHWC tensor [B][H][W][C] with a pixel stride of ld elements, boxes of box_h x box_w pixels x 32 channels of one image.
int encode_nhwc(CUtensorMap* map, const float* base, int B, int H, int W, int C, int ld, int box_w, int box_h, const char* what);
// The same tensor read as 3x3 windows with `pad` pixels of zero padding (im2col), boxes of 128 pixels x 32 channels.
int encode_im2col(CUtensorMap* map, const float* base, int B, int H, int W, int C, int ld, int pad, const char* what);

// p2 (optional): a second problem of identical shape sharing the launch (tiles of both in one grid).
int tc_conv(const TcConv& p, cudaStream_t st, const TcConv* p2 = nullptr);
int reflect_halo(float* buf, int B, int H, int W, int C, cudaStream_t st);
// Persistent windowed 3x3 kernel for the high-resolution narrow layers (conv3_win_tc.cu); tc_conv dispatches to it.
bool conv3_win_supported(const TcConv& p);
int conv3_win(const TcConv& p, cudaStream_t st);


}  // namespace smk
