// Host and device helpers shared by the trainer's frozen networks (vgg_loss.cu, mica.cu, expression_loss.cu): the create
// preamble and tail, the float64 BatchNorm fold, the precision -> profiler tag picker, the `need` checks of the two-image
// losses and the fixed-order block reduction.
#pragma once
#include "gemm_tc.cuh"
#include <array>
#include <cmath>
#include <vector>

namespace smk {

struct Affine { float* scale = nullptr; float* bias = nullptr; };

// The preamble of a frozen network's create: non-null arguments, a precision of 0, 1 or 3, n_expected non-null tensors
// (`what` says which, in the error) and, for the tensor-core precisions, the tensor-map set-up.
static int check_net_desc(const SmkNetDesc* desc, const void* out, const char* fn, int n_expected, const char* what) {
    SMK_REQUIRE(desc && out && desc->tensors, "%s: null argument", fn);
    SMK_REQUIRE(desc->precision == 0 || desc->precision == 1 || desc->precision == 3,
                "%s: precision must be 0, 1 or 3 (0 = fp32 CUDA cores, 1 = TF32 wgmma, 3 = 3xTF32 wgmma: fp32-equivalent)", fn);
    SMK_REQUIRE(desc->n_tensors == n_expected, "%s: expected %d tensors (%s), got %d", fn, n_expected, what, desc->n_tensors);
    for (int i = 0; i < desc->n_tensors; ++i) SMK_REQUIRE(desc->tensors[i], "%s: tensor %d is null", fn, i);
    return desc->precision != 0 ? tc_init() : 0;
}

// The tail of a create: hand the handle out, or record why an upload failed and free it.
template <typename H>
int finish_create(cudaError_t e, const char* fn, H* h, H** out) {
    if (e != cudaSuccess) {
        set_error("%s: upload failed: %s", fn, cudaGetErrorString(e));
        delete h; return (int)e;
    }
    *out = h;
    return 0;
}

// Eval-mode BatchNorm (weight, bias, running_mean, running_var; eps 1e-5) as y = scale * x + bias, folded in float64.
// Not smk::fold_bn, which folds in fp32: these networks' outputs are pinned to this arithmetic.
using Bn = std::array<const float*, 4>;

static Bn next_bn(TensorCursor& cur) { Bn t; for (auto& p : t) p = cur.next(); return t; }

static void bn_fold(const Bn& t, int C, std::vector<double>& s, std::vector<double>& b) {
    s.resize(C); b.resize(C);
    for (int c = 0; c < C; ++c) {
        s[c] = (double)t[0][c] / std::sqrt((double)t[3][c] + 1e-5);
        b[c] = (double)t[1][c] - (double)t[2][c] * s[c];
    }
}

static cudaError_t upload_bn(DeviceArena& arena, const std::vector<double>& s, const std::vector<double>& b, Affine* out) {
    std::vector<float> sf(s.begin(), s.end()), bf(b.begin(), b.end());
    cudaError_t e = arena.upload(sf, &out->scale);
    if (e == cudaSuccess) e = arena.upload(bf, &out->bias);
    return e;
}

static cudaError_t upload_bn(DeviceArena& arena, const Bn& t, int C, Affine* out) {
    std::vector<double> s, b;
    bn_fold(t, C, s, b);
    return upload_bn(arena, s, b, out);
}

// The profiler tag of a layer at the handle's precision (0 fp32, 1 TF32, 3 3xTF32).
static const char* tag_of(int precision, const char* f32, const char* tc, const char* tc3) {
    return precision == 0 ? f32 : precision == 1 ? tc : tc3;
}

// The two-image losses: need 1 = the gradient to the first input, 2 = to the second, 3 = both.  Their grad-mode forward
// and backward keep one half of the batch, or both.
static int halves(int need) { return need == 3 ? 2 : 1; }

// The `need` and saved-buffer checks of a grad-mode forward or backward; in1 / in2 name the inputs in the error.
static int check_need(const char* fn, const char* in1, const char* in2, int need, size_t saved_bytes, size_t saved_need) {
    SMK_REQUIRE(need >= 1 && need <= 3, "%s: need must be 1 (%s), 2 (%s) or 3 (both), got %d", fn, in1, in2, need);
    SMK_REQUIRE(saved_bytes >= saved_need, "%s: saved buffer too small", fn);
    return 0;
}

#ifdef __CUDACC__
// Sum over the 256 threads of a block in a fixed order (each warp's butterfly, then the eight warp sums in warp order); the
// result is valid in every thread.  The first barrier keeps a previous call's reads of wsum ahead of this call's writes.
static __device__ float block_sum(float v) {
    __shared__ float wsum[8];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) wsum[threadIdx.x >> 5] = v;
    __syncthreads();
    float t = 0.f;
    for (int w = 0; w < 8; ++w) t += wsum[w];
    return t;
}
#endif

}  // namespace smk
