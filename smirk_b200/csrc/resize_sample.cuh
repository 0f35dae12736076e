// The two resampling rules of the video demo without --crop (demo_video.py:130-136,154,205).
//
// cv2_resize3: cv2.resize(frame, (S, S)) of a uint8 3-channel image with the default INTER_LINEAR, bit for bit (OpenCV
// 4.x, whose SIMD vertical pass sets the rounding):
//   (H, W) == (S, S)      a copy
//   (H, W) == (2S, 2S)    cv2's INTER_AREA fast path: (a + b + c + d + 2) >> 2 over each 2x2 block
//   otherwise             per axis f = float((d + 0.5) * (double)src / dst - 0.5), s = floor(f), f -= s; weights
//                         rint((1 - f) * 2048), rint(f * 2048).  Horizontally s < 0 gives s = 0, f = 0 and s >= src - 1
//                         gives s = src - 1, f = 0; vertically only the two row indices are clamped, not the weights.
//                         h = x[s] a0 + x[min(s + 1, src - 1)] a1 exactly, then
//                         v = ((((h0 >> 4) b0) >> 16) + (((h1 >> 4) b1) >> 16) + 2) >> 2, saturated to uint8.
// Written once for the host and the device (warp.cu's resize_kernel).
//
// torch_bilinear: torch's upsample_bilinear2d (align_corners = False, no scale factor) of one channel, as its CUDA kernel
// computes it but without fused multiply-adds, so a float32 numpy restatement gives the same bits:
//   scale = (float)S / H, r = max(scale * (d + 0.5f) - 0.5f, 0), i0 = (int)r, i1 = i0 + (i0 < S - 1), l1 = r - i0,
//   l0 = 1 - l1;  v = h0l * (w0l * x00 + w1l * x01) + h1l * (w0l * x10 + w1l * x11)
#pragma once
#include <stdint.h>
#include <math.h>

#ifndef SMK_HD
#ifdef __CUDACC__
#define SMK_HD __host__ __device__ __forceinline__
#else
#define SMK_HD inline
#endif
#endif

namespace smk {
namespace resize {

// (d + 0.5) * scale - 0.5 in float64 with two roundings (the device compiler would fuse it otherwise)
SMK_HD double src_coord(int d, double scale) {
#ifdef __CUDA_ARCH__
    return __dsub_rn(__dmul_rn((double)d + 0.5, scale), 0.5);
#else
    return ((double)d + 0.5) * scale - 0.5;
#endif
}

struct Taps { int s, a0, a1; };

// cv2's fixed-point INTER_LINEAR taps of output index d along an axis of `src` samples resized to `dst`.
SMK_HD Taps linear_taps(int d, int src, int dst, bool clamp) {
    float f = (float)src_coord(d, (double)src / dst);
    const float fl = floorf(f);
    int s = (int)fl;
    f -= fl;
    if (clamp && s < 0) { s = 0; f = 0.0f; }
    if (clamp && s >= src - 1) { s = src - 1; f = 0.0f; }
    return Taps{s, (int)rintf((1.0f - f) * 2048.0f), (int)rintf(f * 2048.0f)};
}

// Output pixel (x, y) of cv2.resize(img, (S, S)), img uint8 [H,W,3] (pixel pitch 3): the three channel bytes.
SMK_HD void cv2_resize3(const uint8_t* img, int H, int W, int S, int x, int y, uint8_t v[3]) {
    const auto px = [img, W](int r, int c) { return img + ((size_t)r * W + c) * 3; };
    if (H == S && W == S) {
        for (int ch = 0; ch < 3; ++ch) v[ch] = px(y, x)[ch];
        return;
    }
    if (H == 2 * S && W == 2 * S) {
        for (int ch = 0; ch < 3; ++ch)
            v[ch] = (uint8_t)((px(2 * y, 2 * x)[ch] + px(2 * y, 2 * x + 1)[ch] + px(2 * y + 1, 2 * x)[ch] + px(2 * y + 1, 2 * x + 1)[ch] + 2) >> 2);
        return;
    }
    const Taps tx = linear_taps(x, W, S, true), ty = linear_taps(y, H, S, false);
    const int c0 = tx.s, c1 = tx.s + 1 < W - 1 ? tx.s + 1 : W - 1;
    const int r0 = ty.s < 0 ? 0 : ty.s > H - 1 ? H - 1 : ty.s;
    const int r1 = ty.s + 1 < 0 ? 0 : ty.s + 1 > H - 1 ? H - 1 : ty.s + 1;
    for (int ch = 0; ch < 3; ++ch) {
        const int h0 = px(r0, c0)[ch] * tx.a0 + px(r0, c1)[ch] * tx.a1;
        const int h1 = px(r1, c0)[ch] * tx.a0 + px(r1, c1)[ch] * tx.a1;
        const int s = ((((h0 >> 4) * ty.a0) >> 16) + (((h1 >> 4) * ty.a1) >> 16) + 2) >> 2;
        v[ch] = (uint8_t)(s < 0 ? 0 : s > 255 ? 255 : s);
    }
}

#ifdef __CUDACC__
// torch's area_pixel_compute_source_index (align_corners = False) of output index d, `src` samples resized to `dst`.
struct Lerp { int i0, i1; float l0, l1; };

__device__ __forceinline__ Lerp bilinear_index(int d, int src, int dst) {
    const float scale = __fdiv_rn((float)src, (float)dst);
    const float r = fmaxf(__fsub_rn(__fmul_rn(scale, __fadd_rn((float)d, 0.5f)), 0.5f), 0.0f);
    const int i0 = (int)r;
    const float l1 = __fsub_rn(r, (float)i0);
    return Lerp{i0, i0 + (i0 < src - 1), __fsub_rn(1.0f, l1), l1};
}

// One channel x [S,S] (row pitch S) sampled at the output pixel of taps (h, w).
template <class Load>
__device__ __forceinline__ float torch_bilinear(const Lerp& h, const Lerp& w, int S, Load load) {
    const float top = __fadd_rn(__fmul_rn(w.l0, load(h.i0 * S + w.i0)), __fmul_rn(w.l1, load(h.i0 * S + w.i1)));
    const float bot = __fadd_rn(__fmul_rn(w.l0, load(h.i1 * S + w.i0)), __fmul_rn(w.l1, load(h.i1 * S + w.i1)));
    return __fadd_rn(__fmul_rn(h.l0, top), __fmul_rn(h.l1, bot));
}
#endif

}  // namespace resize
}  // namespace smk
