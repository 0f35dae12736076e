// Crop / warp front end and back end of the per-frame path (SURVEY.md §8f #2).
//
// Replaces, for frames that are already on the device,
//   demo.py:97 / demo_video.py:128   cropped = skimage.transform.warp(image, tform.inverse, output_shape=(224,224),
//                                              preserve_range=True).astype(np.uint8)
//   demo.py:103-105                  cv2.cvtColor(BGR2RGB) -> torch [1,3,224,224] float / 255
//   demo_video.py:148-149            rendered -> (x * 255).astype(uint8) -> warp(rendered, tform, output_shape=(H, W),
//                                              preserve_range=True).astype(np.uint8)
// The reference does this on the CPU per frame (skimage's Cython `_warp_fast`) between a D2H and an H2D copy; here
// it is one gather-bilinear pass per direction.  Without a crop (demo_video.py:130-136 without --crop) smk_crop_warp
// resizes the whole frame with cv2.resize's rule instead (resize_sample.cuh).
//
// Arithmetic follows skimage 0.2x `_warp_fast` / `bilinear_interpolation` / `_clip_warp_output` for order = 1,
// mode = 'constant', cval = 0, clip = True, evaluated in float64 like the reference (preserve_range=True converts
// the uint8 frame to float64):
//   (c, r) = M (tfc, tfr, 1)            M = 3x3 inverse map, row-major float64; affine rows only (M[2] = 0 0 1)
//   minr = floor(r), maxr = ceil(r), dr = r - minr (same for c); pixels outside the source read cval = 0
//   top = (1 - dc) tl + dc tr ; bottom = (1 - dc) bl + dc br ; v = (1 - dr) top + dr bottom
//   clip: v = clamp(v, min(src), max(src)) unless v == cval and cval lies outside [min(src), max(src)]
//   .astype(np.uint8): truncation towards zero
// skimage is not installed in this image, so this restatement is pinned only by the properties in tests/ (identity,
// integer shifts, scipy cross-check away from the border): "parity unpinned" for the border/clip rules.
// HBM traffic: the gather touches each source texel it needs once through L2; output 150 KB (crop) or H*W*3 (back).
#include "common.cuh"
#include "warp_sample.cuh"
#include "resize_sample.cuh"
#include <math.h>
#include <algorithm>

namespace {

struct MinMax { unsigned int mn, mx; };

// per-frame min / max of the uint8 source over all channels (skimage clips per warp() call = per whole image)
__global__ void __launch_bounds__(256)
u8_minmax_kernel(const uint8_t* __restrict__ src, size_t n_per_frame, MinMax* __restrict__ mm) {
    const int b = blockIdx.y;
    const uint8_t* s = src + (size_t)b * n_per_frame;
    unsigned int mn = 255u, mx = 0u;
    // 16 bytes per load where aligned
    const size_t n16 = (((uintptr_t)s & 15) == 0) ? n_per_frame / 16 : 0;
    const uint4* s16 = reinterpret_cast<const uint4*>(s);
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n16; i += (size_t)gridDim.x * blockDim.x) {
        const uint4 v = __ldg(s16 + i);
        const unsigned int w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int k = 0; k < 4; ++k)
#pragma unroll
            for (int j = 0; j < 4; ++j) { const unsigned int t = (w[k] >> (8 * j)) & 255u; mn = min(mn, t); mx = max(mx, t); }
    }
    for (size_t i = n16 * 16 + (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_per_frame; i += (size_t)gridDim.x * blockDim.x) {
        const unsigned int t = s[i]; mn = min(mn, t); mx = max(mx, t);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { mn = min(mn, __shfl_xor_sync(0xffffffffu, mn, o)); mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, o)); }
    if ((threadIdx.x & 31) == 0) { atomicMin(&mm[b].mn, mn); atomicMax(&mm[b].mx, mx); }
}

__global__ void minmax_init_kernel(MinMax* mm, int B) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < B) { mm[i].mn = 255u; mm[i].mx = 0u; }
}

// rendered float [B,3,S,S] -> uint8 [B,S,S,3]: (x * 255.0f).astype(uint8) in float32 like numpy (demo_video.py:148)
__global__ void __launch_bounds__(256)
f32chw_to_u8hwc_kernel(const float* __restrict__ in, int B, int S, uint8_t* __restrict__ out) {
    const size_t n = (size_t)B * S * S;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const size_t b = i / ((size_t)S * S), p = i - b * (size_t)S * S;
#pragma unroll
        for (int c = 0; c < 3; ++c) out[i * 3 + c] = smk::unit_to_u8(in[(b * 3 + c) * (size_t)S * S + p]);
    }
}

// One thread per output pixel, all three channels (the four source texels are adjacent 3-byte groups).
//   OUT_F32 = false: dst uint8 [B, Hd, Wd, 3], channel order kept.
//   OUT_F32 = true : dst float [B, 3, Hd, Wd] = uint8 result / 255, channels reversed when swap_rb (BGR frame -> RGB).
template <bool OUT_F32>
__global__ void __launch_bounds__(256)
warp_bilinear_kernel(const uint8_t* __restrict__ src, int Hs, int Ws, const double* __restrict__ M, const MinMax* __restrict__ mm,
                     int Hd, int Wd, int swap_rb, void* __restrict__ dst) {
    const int b = blockIdx.z;
    const int tfc = blockIdx.x * 32 + (threadIdx.x & 31), tfr = blockIdx.y * 8 + (threadIdx.x >> 5);
    if (tfc >= Wd || tfr >= Hd) return;
    const uint8_t* s = src + (size_t)b * Hs * Ws * 3;
    uint8_t res[3];
    smk::skimage_bilinear3(M + (size_t)b * 9, tfc, tfr, Hs, Ws, (double)mm[b].mn, (double)mm[b].mx,
                           [s, Ws](int ch, int row, int col) { return (double)s[((size_t)row * Ws + col) * 3 + ch]; }, res);
    if (OUT_F32) {
        float* o = reinterpret_cast<float*>(dst) + (size_t)b * 3 * Hd * Wd + (size_t)tfr * Wd + tfc;
#pragma unroll
        for (int ch = 0; ch < 3; ++ch) o[(size_t)(swap_rb ? 2 - ch : ch) * Hd * Wd] = __fdiv_rn((float)res[ch], 255.0f);
    } else {
        uint8_t* o = reinterpret_cast<uint8_t*>(dst) + (((size_t)b * Hd + tfr) * Wd + tfc) * 3;
        o[0] = res[0]; o[1] = res[1]; o[2] = res[2];
    }
}

// cv2.resize(frame, (S, S)) of whole frames (demo_video.py:134-136 without --crop): one thread per output pixel, float
// [B,3,S,S] = uint8 result / 255, channels reversed when swap_rb.
__global__ void __launch_bounds__(256)
resize_kernel(const uint8_t* __restrict__ src, int H, int W, int S, int swap_rb, float* __restrict__ dst) {
    const int b = blockIdx.z;
    const int x = blockIdx.x * 32 + (threadIdx.x & 31), y = blockIdx.y * 8 + (threadIdx.x >> 5);
    if (x >= S || y >= S) return;
    uint8_t res[3];
    smk::resize::cv2_resize3(src + (size_t)b * H * W * 3, H, W, S, x, y, res);
    float* o = dst + (size_t)b * 3 * S * S + (size_t)y * S + x;
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) o[(size_t)(swap_rb ? 2 - ch : ch) * S * S] = __fdiv_rn((float)res[ch], 255.0f);
}

int launch_warp(const uint8_t* src, int B, int Hs, int Ws, const double* M, int Hd, int Wd, bool out_f32, int swap_rb, void* dst,
                void* ws, size_t ws_bytes, cudaStream_t st) {
    SMK_REQUIRE(ws && ws_bytes >= (size_t)B * sizeof(MinMax), "warp: workspace too small");
    MinMax* mm = reinterpret_cast<MinMax*>(ws);
    SMK_TAG("warp_minmax", (double)B * Hs * Ws * 3, 0.0, st);
    SMK_LAUNCH(minmax_init_kernel, dim3(smk::cdiv(B, 64)), dim3(64), 0, st, mm, B);
    SMK_CHECK_LAUNCH();
    const size_t n = (size_t)Hs * Ws * 3;
    SMK_TAG("warp_minmax", 0.0, 0.0, st);
    SMK_LAUNCH(u8_minmax_kernel, dim3((unsigned)std::min<size_t>((n / 16 + 255) / 256 + 1, 2 * (size_t)smk::num_sms()), B), dim3(256), 0, st, src, n, mm);
    SMK_CHECK_LAUNCH();
    SMK_TAG("warp_bilinear", (double)B * Hd * Wd * (out_f32 ? 12.0 : 3.0) + (double)B * Hd * Wd * 12.0, 30.0 * B * Hd * Wd, st);
    dim3 grid(smk::cdiv(Wd, 32), smk::cdiv(Hd, 8), B);
    if (out_f32) SMK_LAUNCH((warp_bilinear_kernel<true>), grid, dim3(256), 0, st, src, Hs, Ws, M, (const MinMax*)mm, Hd, Wd, swap_rb, dst);
    else SMK_LAUNCH((warp_bilinear_kernel<false>), grid, dim3(256), 0, st, src, Hs, Ws, M, (const MinMax*)mm, Hd, Wd, swap_rb, dst);
    SMK_CHECK_LAUNCH();
    return 0;
}

}  // namespace

extern "C" size_t smk_warp_workspace_bytes(int B) { return smk::ws_round((size_t)(B > 0 ? B : 1) * sizeof(MinMax)); }

extern "C" int smk_crop_warp(const uint8_t* frames, int B, int H, int W, const double* minv, int S, int swap_rb, float* out,
                             void* ws, size_t ws_bytes, void* stream) {
    if (B == 0) return 0;
    SMK_REQUIRE(frames && out, "smk_crop_warp: null argument");
    SMK_REQUIRE(B > 0 && H > 0 && W > 0 && S > 0, "smk_crop_warp: bad sizes");
    if (!minv) {                                    // no crop transform: cv2.resize of the whole frame, no workspace
        SMK_REQUIRE(B <= 65535, "smk_crop_warp: too many frames");
        cudaStream_t st = (cudaStream_t)stream;
        // algorithmic bytes: the output, and the four 3-byte taps of each output pixel (at most the whole frame)
        SMK_TAG("resize", (double)B * S * S * 12.0 + (double)B * std::min((double)H * W * 3, (double)S * S * 12), 0.0, st);
        SMK_LAUNCH(resize_kernel, dim3(smk::cdiv(S, 32), smk::cdiv(S, 8), B), dim3(256), 0, st, frames, H, W, S, swap_rb ? 1 : 0, out);
        SMK_CHECK_LAUNCH();
        return 0;
    }
    return launch_warp(frames, B, H, W, minv, S, S, true, swap_rb ? 1 : 0, out, ws, ws_bytes, (cudaStream_t)stream);
}

extern "C" int smk_warp_u8(const uint8_t* src, int B, int Hs, int Ws, const double* m, int Hd, int Wd, uint8_t* dst,
                           void* ws, size_t ws_bytes, void* stream) {
    if (B == 0) return 0;
    SMK_REQUIRE(src && m && dst, "smk_warp_u8: null argument");
    SMK_REQUIRE(B > 0 && Hs > 0 && Ws > 0 && Hd > 0 && Wd > 0, "smk_warp_u8: bad sizes");
    return launch_warp(src, B, Hs, Ws, m, Hd, Wd, false, 0, dst, ws, ws_bytes, (cudaStream_t)stream);
}

extern "C" int smk_f32chw_to_u8hwc(const float* in, int B, int S, uint8_t* out, void* stream) {
    if (B == 0) return 0;
    SMK_REQUIRE(in && out && B > 0 && S > 0, "smk_f32chw_to_u8hwc: bad argument");
    cudaStream_t st = (cudaStream_t)stream;
    SMK_TAG("f32chw_to_u8hwc", 15.0 * B * S * S, 0.0, st);
    SMK_LAUNCH(f32chw_to_u8hwc_kernel, dim3((unsigned)std::min<size_t>(((size_t)B * S * S + 255) / 256, 8 * (size_t)smk::num_sms())), dim3(256), 0, st, in, B, S, out);
    SMK_CHECK_LAUNCH();
    return 0;
}
