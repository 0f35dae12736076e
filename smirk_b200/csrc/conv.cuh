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
    int out2_rows;                       // out2 takes only the pixels m < out2_rows (0: every pixel), e.g. the first images
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

// Tensor-core weight v at index i: the TF32 head, and with x3 the TF32 tail of what the head leaves (v = head + tail up to
// 2^-22 |v|), the split encoder.cu packs for its 3xTF32 1x1 convs.
inline void pack_tc(std::vector<float>& hi, std::vector<float>& lo, size_t i, float v, bool x3) {
    hi[i] = round_tf32_host(v);
    if (x3) lo[i] = round_tf32_host(v - hi[i]);
}

// One 3x3 convolution's weights (PyTorch [cout][cin][3][3]) packed for smk::conv, forward and input gradient:
//   forward  w [9*cin_p][cout] (fp32) or wt [cout][9*cin_p] (TF32 heads, + wt_lo tails with x3), k = tap * cin_p + ci;
//   dgrad    W'[ci][8 - tap][co] = dscale[co] * W[co][ci][tap]: dw [9*cout][cin_p] (fp32) or [cin_p][9*cout] (TF32, + dw_lo),
//            the forward's GEMM kernels run it as a 3x3 conv of the output gradient.
// Input channels cin..cin_p-1 are zero.  dscale (null: 1) is multiplied in before the TF32 split.  Unused pointers are null.
struct Conv3Weights { float* w; float* wt; float* wt_lo; float* dw; float* dw_lo; };
inline cudaError_t pack_conv3(const float* w, const float* dscale, int cin, int cin_p, int cout, bool tc, bool x3,
                              DeviceArena& arena, Conv3Weights* out) {
    const size_t K = (size_t)9 * cin_p, Kd = (size_t)9 * cout;
    std::vector<float> W(K * cout, 0.f), D(Kd * cin_p, 0.f), Wlo, Dlo;
    if (x3) { Wlo.assign(W.size(), 0.f); Dlo.assign(D.size(), 0.f); }
    for (int o = 0; o < cout; ++o)
        for (int c = 0; c < cin; ++c)
            for (int k = 0; k < 9; ++k) {
                const float v = w[((size_t)o * cin + c) * 9 + k];
                if (tc) pack_tc(W, Wlo, (size_t)o * K + (size_t)k * cin_p + c, v, x3);   // [N][K], TF32 heads (+ tails)
                else W[((size_t)k * cin_p + c) * cout + o] = v;                // [K][N]
                const float vd = dscale ? v * dscale[o] : v;                   // split after the scale multiply
                const size_t kd = (size_t)(8 - k) * cout + o;                  // rotated tap
                if (tc) pack_tc(D, Dlo, (size_t)c * Kd + kd, vd, x3);
                else D[kd * cin_p + c] = vd;
            }
    *out = Conv3Weights{};
    cudaError_t e = arena.upload(W, tc ? &out->wt : &out->w);
    if (e == cudaSuccess && x3) e = arena.upload(Wlo, &out->wt_lo);
    if (e == cudaSuccess) e = arena.upload(D, &out->dw);
    if (e == cudaSuccess && x3) e = arena.upload(Dlo, &out->dw_lo);
    return e;
}

}  // namespace smk
