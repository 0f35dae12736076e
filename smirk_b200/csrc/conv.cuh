// One descriptor for the GEMM-shaped convolutions of the encoder, the generator and the VGG loss, the one place that picks
// their kernel: the fp32 CUDA-core `conv_gemm` (nn_kernels.cu) or the TF32 wgmma `tc_conv` (gemm_tc.cu), and the one
// packer of their weights.
#pragma once
#include "common.cuh"

namespace smk {

// The weight operand W(k, n) of a problem, in the layout of the kernel that reads it: exactly one of w / wt is set.
//   w      fp32 [K][N], n fastest (conv_gemm)
//   wt     TF32 [N][K], k fastest (tc_conv): the weights rounded to TF32, or with wt_lo their TF32 heads
//   wt_lo  optional: the TF32 tails, v - head rounded to TF32 (v = head + tail up to 2^-22 |v|) -> 3xTF32 arithmetic
// pack_gemm below packs one from the logical [N][K] matrix.
struct GemmW { const float* w; const float* wt; const float* wt_lo; };

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
    GemmW wgt;                           // the weights W(k, n)
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

// conv_gemm_kernel takes Conv by value: its parameter layout is pinned.
static_assert(offsetof(Conv, wgt) == 40 && offsetof(Conv, scale) == 64 && sizeof(Conv) == 184, "smk::Conv layout moved");

// fp32 CUDA cores: modes 0-2, stores 0 and 1; no TF32 weights, padded residual or paired problem.
int conv_gemm(const Conv& p, cudaStream_t st);
// TF32 tensor cores.  p2 (optional): a second problem of identical shape sharing the launch (tiles of both in one grid).
int tc_conv(const Conv& p, cudaStream_t st, const Conv* p2 = nullptr);

// TF32 weights (wt) run tc_conv, fp32 weights (w) conv_gemm.
inline int conv(const Conv& p, cudaStream_t st, const Conv* p2 = nullptr) {
    if (p.wgt.wt) return tc_conv(p, st, p2);
    SMK_REQUIRE(!p2, "conv: paired problems need TF32 weights");
    return conv_gemm(p, st);
}

// Packs the logical weight matrix W[n][k] = v(n, k), n < N, k < K, as smk::conv's operand: fp32 [K][N] (tc false), or
// TF32 [N][K] (tc), as heads plus tails when x3.  Where a matrix comes from a reordered or scaled tensor, v does that
// before the split.
template <typename V>
cudaError_t pack_gemm(DeviceArena& arena, int N, int K, bool tc, bool x3, V&& v, GemmW* out) {
    std::vector<float> hi((size_t)N * K), lo(tc && x3 ? hi.size() : 0);
    for (int n = 0; n < N; ++n)
        for (int k = 0; k < K; ++k) {
            const float x = v(n, k);
            if (!tc) { hi[(size_t)k * N + n] = x; continue; }
            const size_t i = (size_t)n * K + k;
            hi[i] = round_tf32_host(x);
            if (!lo.empty()) lo[i] = round_tf32_host(x - hi[i]);
        }
    float *d = nullptr, *d_lo = nullptr;
    cudaError_t e = arena.upload(hi, &d);
    if (e == cudaSuccess && !lo.empty()) e = arena.upload(lo, &d_lo);
    *out = tc ? GemmW{nullptr, d, d_lo} : GemmW{d, nullptr, nullptr};
    return e;
}
// The same from a dense [N][K] matrix.
inline cudaError_t pack_gemm(DeviceArena& arena, int N, int K, bool tc, bool x3, const float* nk, GemmW* out) {
    return pack_gemm(arena, N, K, tc, x3, [nk, K](int n, int k) { return nk[(size_t)n * K + k]; }, out);
}

// One 3x3 convolution's weights (PyTorch [cout][cin][3][3]) packed for smk::conv, forward and input gradient:
//   forward  N = cout, K = 9*cin_p:  W(k = tap * cin_p + ci, co) = W[co][ci][tap];
//   dgrad    N = cin_p, K = 9*cout:  W'(k = (8 - tap) * cout + co, ci) = dscale[co] * W[co][ci][tap], the rotated taps: the
//            forward's GEMM kernels run it as a 3x3 conv of the output gradient.
// Input channels cin..cin_p-1 are zero.  dscale (null: 1) is multiplied in before the TF32 split.
inline cudaError_t pack_conv3(const float* w, const float* dscale, int cin, int cin_p, int cout, bool tc, bool x3,
                              DeviceArena& arena, GemmW* fwd, GemmW* dgrad) {
    cudaError_t e = pack_gemm(arena, cout, 9 * cin_p, tc, x3, [&](int o, int k) {
        const int tap = k / cin_p, c = k % cin_p;
        return c < cin ? w[((size_t)o * cin + c) * 9 + tap] : 0.f;
    }, fwd);
    if (e == cudaSuccess) e = pack_gemm(arena, cin_p, 9 * cout, tc, x3, [&](int c, int k) {
        const int tap = 8 - k / cout, o = k % cout;
        if (c >= cin) return 0.f;
        const float v = w[((size_t)o * cin + c) * 9 + tap];
        return dscale ? v * dscale[o] : v;
    }, dgrad);
    return e;
}

}  // namespace smk
