// TF32 wgmma implicit-GEMM convolution (see gemm_tc.cu; `tc_conv` and its descriptor are declared in conv.cuh).
#pragma once
#include "conv.cuh"
#include <cuda.h>

namespace smk {

int tc_init();                                              // resolves the driver's tensor-map encoders

// TMA descriptors over fp32 tensors as the wgmma kernels read them: boxes of 32 elements (128 bytes) in the innermost
// dimension, SWIZZLE_128B, L2 promotion 128 B, zero fill out of bounds.  `what` names the operand in the error message.
// [rows][cols] matrix with a row stride of ld elements, boxes of box_rows x 32.
int encode_2d(CUtensorMap* map, const float* base, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows, const char* what);
// NHWC tensor [B][H][W][C] with a pixel stride of ld elements, boxes of box_h x box_w pixels x 32 channels of one image.
int encode_nhwc(CUtensorMap* map, const float* base, int B, int H, int W, int C, int ld, int box_w, int box_h, const char* what);
// The same tensor read as 3x3 windows with `pad` pixels of zero padding (im2col), boxes of 128 pixels x 32 channels.
int encode_im2col(CUtensorMap* map, const float* base, int B, int H, int W, int C, int ld, int pad, const char* what);

int reflect_halo(float* buf, int B, int H, int W, int C, cudaStream_t st);
// Persistent windowed 3x3 kernel for the high-resolution narrow layers (conv3_win_tc.cu); tc_conv dispatches to it.
bool conv3_win_supported(const Conv& p);
int conv3_win(const Conv& p, cudaStream_t st);

}  // namespace smk
