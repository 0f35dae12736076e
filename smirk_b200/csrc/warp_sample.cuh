// skimage `_warp_fast` bilinear sample of one output pixel, all three channels (order = 1, mode = 'constant', cval = 0,
// clip = True, float64, then .astype(np.uint8)); see warp.cu for the arithmetic it restates.  Shared by the warp kernels
// (warp.cu) and the video grid composer (video.cu), which differ only in how they fetch a source texel.
#pragma once
#include <stdint.h>
#include <math.h>

namespace smk {

// tap(ch, row, col) -> the source texel as a double in [0, 255], for row in [0, Hs), col in [0, Ws).
// M: 3x3 row-major float64 map output (col, row, 1) -> source (col, row, 1); [lo, hi] = min / max of the whole source.
template <class Tap>
__device__ __forceinline__ void skimage_bilinear3(const double* __restrict__ m, int tfc, int tfr, int Hs, int Ws, double lo,
                                                  double hi, Tap tap, uint8_t res[3]) {
    // _transform_affine: c = M00 x + M01 y + M02 (left to right, no contraction)
    const double c = __dadd_rn(__dadd_rn(__dmul_rn(m[0], (double)tfc), __dmul_rn(m[1], (double)tfr)), m[2]);
    const double r = __dadd_rn(__dadd_rn(__dmul_rn(m[3], (double)tfc), __dmul_rn(m[4], (double)tfr)), m[5]);
    const double fr = floor(r), fc = floor(c);
    const long long minr = (long long)fr, minc = (long long)fc, maxr = (long long)ceil(r), maxc = (long long)ceil(c);
    const double dr = __dsub_rn(r, (double)minr), dc = __dsub_rn(c, (double)minc);
    const bool r0 = minr >= 0 && minr < Hs, r1 = maxr >= 0 && maxr < Hs, c0 = minc >= 0 && minc < Ws, c1 = maxc >= 0 && maxc < Ws;
    const bool keep_cval = !(lo <= 0.0 && 0.0 <= hi);              // cval = 0 outside the source's range: exact zeros survive the clip
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
        const double tl = (r0 && c0) ? tap(ch, (int)minr, (int)minc) : 0.0;
        const double tr = (r0 && c1) ? tap(ch, (int)minr, (int)maxc) : 0.0;
        const double bl = (r1 && c0) ? tap(ch, (int)maxr, (int)minc) : 0.0;
        const double br = (r1 && c1) ? tap(ch, (int)maxr, (int)maxc) : 0.0;
        const double omc = __dsub_rn(1.0, dc), omr = __dsub_rn(1.0, dr);
        const double top = __dadd_rn(__dmul_rn(omc, tl), __dmul_rn(dc, tr));
        const double bot = __dadd_rn(__dmul_rn(omc, bl), __dmul_rn(dc, br));
        double v = __dadd_rn(__dmul_rn(omr, top), __dmul_rn(dr, bot));
        if (!(keep_cval && v == 0.0)) v = fmin(fmax(v, lo), hi);
        res[ch] = (uint8_t)(int)v;
    }
}

// (x * 255.0f).astype(np.uint8) in float32, as numpy does it on a rendered image in [0, 1]: truncation.
__device__ __forceinline__ uint8_t unit_to_u8(float x) { return (uint8_t)(int)__fmul_rn(x, 255.0f); }

}  // namespace smk
