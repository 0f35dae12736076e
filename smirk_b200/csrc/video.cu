// Output grid of the reference's video demo (demo_video.py:139-160,171,198-213), for a batch of frames on the device: one
// row per frame, the panels side by side, uint8 BGR — the bytes demo_video.py hands to cv2.VideoWriter.
//
//   panel 0        render_orig (1 or 2): the frame itself (its u8 -> RGB -> /255 -> *255 -> u8 -> BGR round trip is the
//                               identity)
//                  otherwise:   the 224x224 crop or resize, (crop * 255).astype(uint8) of the float image the encoder read
//                               (identity on u8 / 255 values), channels back to BGR
//   panel 1 (, 2)  the rendered (and reconstructed) image [3,S,S] in [0,1]:
//                  render_orig == 1 (--crop --render_orig):
//                               warp((x * 255).astype(uint8) HWC, tform, (H, W), preserve_range=True).astype(uint8)
//                               — skimage's bilinear sample of warp_sample.cuh, the float -> u8 conversion done per tap,
//                               clipped to the min / max of the converted panel (a small reduction launch first)
//                  render_orig == 2 (--render_orig without --crop):
//                               (F.interpolate(x, (H, W), mode='bilinear') * 255).astype(uint8) — torch's bilinear sample
//                               of resize_sample.cuh evaluated per output byte, so no resized float panel reaches HBM
//                  otherwise:   (x * 255).astype(uint8)
//                  channels RGB -> BGR.
// One launch writes the whole grid; no u8 intermediate of a panel reaches HBM.  Each thread owns one 16-byte-aligned
// segment of a grid row (plus one head segment per row up to the first 16-byte boundary, since the row pitch
// (n_panels + 1) * Wout * 3 need not be a multiple of 16) and writes it with one 16-byte store when it is whole.
#include "common.cuh"
#include "warp_sample.cuh"
#include "hull_mask.cuh"
#include "resize_sample.cuh"
#include <float.h>

namespace {

struct ComposeArgs {
    const uint8_t* frames;      // [B,H,W,3]
    const float* crop;          // [B,3,S,S] (panel 0 without render_orig)
    const float* p1;            // [B,3,S,S]
    const float* p2;            // [B,3,S,S] or null
    const double* m;            // [B,9] crop -> frame (tform.params), render_orig only
    const unsigned* mm;         // [B, n_panels, 2] min / max of the converted panels, render_orig only
    int H, W, S, n_panels, render_orig, Ho, Wo;
    long long pitch;            // bytes per grid row: (n_panels + 1) * Wo * 3
    uint8_t* grid;              // [B,Ho,(n_panels+1)*Wo,3]
};

// min / max over one converted panel: one CTA per (frame, panel).  The conversion is monotone, so min(u8(x)) = u8(min x).
__global__ void __launch_bounds__(512) panel_minmax_kernel(const float* __restrict__ p1, const float* __restrict__ p2, int S,
                                                           int n_panels, unsigned* __restrict__ mm) {
    const int b = blockIdx.x / n_panels, p = blockIdx.x - b * n_panels;
    const size_t n = (size_t)3 * S * S;
    const float* x = (p == 0 ? p1 : p2) + (size_t)b * n;
    float lo = FLT_MAX, hi = -FLT_MAX;
    for (size_t i = threadIdx.x; i < n; i += blockDim.x) { const float v = __ldg(x + i); lo = fminf(lo, v); hi = fmaxf(hi, v); }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { lo = fminf(lo, __shfl_xor_sync(0xffffffffu, lo, o)); hi = fmaxf(hi, __shfl_xor_sync(0xffffffffu, hi, o)); }
    __shared__ float slo[16], shi[16];
    const int w = threadIdx.x >> 5;
    if ((threadIdx.x & 31) == 0) { slo[w] = lo; shi[w] = hi; }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int k = 1; k < (int)(blockDim.x >> 5); ++k) { lo = fminf(lo, slo[k]); hi = fmaxf(hi, shi[k]); }
        mm[2 * blockIdx.x] = smk::unit_to_u8(lo);
        mm[2 * blockIdx.x + 1] = smk::unit_to_u8(hi);
    }
}

// The three BGR bytes of grid pixel (y, px) of frame b.  RESIZE: render_orig == 2 (the panels resized to the frame).
template <bool RESIZE>
__device__ __forceinline__ void grid_pixel(const ComposeArgs& a, int b, int y, int px, uint8_t v[3]) {
    const int p = px / a.Wo, x = px - p * a.Wo;
    const size_t SS = (size_t)a.S * a.S;
    if (p == 0 && a.render_orig) {
        const uint8_t* f = a.frames + (((size_t)b * a.H + y) * a.W + x) * 3;
        v[0] = __ldg(f); v[1] = __ldg(f + 1); v[2] = __ldg(f + 2);
        return;
    }
    const float* src = (p == 0 ? a.crop : p == 1 ? a.p1 : a.p2) + (size_t)b * 3 * SS;
    if (RESIZE) {
        const smk::resize::Lerp h = smk::resize::bilinear_index(y, a.S, a.Ho), w = smk::resize::bilinear_index(x, a.S, a.Wo);
#pragma unroll
        for (int ch = 0; ch < 3; ++ch) {
            const float* c = src + (2 - ch) * SS;
            v[ch] = smk::unit_to_u8(smk::resize::torch_bilinear(h, w, a.S, [c](int i) { return __ldg(c + i); }));
        }
        return;
    }
    if (p == 0 || !a.render_orig) {
#pragma unroll
        for (int ch = 0; ch < 3; ++ch) v[ch] = smk::unit_to_u8(__ldg(src + (2 - ch) * SS + (size_t)y * a.S + x));
        return;
    }
    const unsigned* mm = a.mm + 2 * (b * a.n_panels + p - 1);
    const int S = a.S;
    smk::skimage_bilinear3(a.m + (size_t)b * 9, x, y, S, S, (double)mm[0], (double)mm[1],
                           [src, S, SS](int ch, int row, int col) {
                               return (double)smk::unit_to_u8(__ldg(src + (2 - ch) * SS + (size_t)row * S + col));
                           }, v);
}

// RESIZE = false serves render_orig 0 and 1, RESIZE = true render_orig 2.
template <bool RESIZE>
__global__ void __launch_bounds__(256) video_compose_kernel(const ComposeArgs a) {
    const int y = blockIdx.y, b = blockIdx.z;
    uint8_t* row = a.grid + ((size_t)b * a.Ho + y) * a.pitch;
    const long long head = (long long)((16 - ((uintptr_t)row & 15)) & 15);
    const long long seg = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long o0 = seg == 0 ? 0 : head + 16 * (seg - 1);
    const long long o1 = min(seg == 0 ? head : o0 + 16, a.pitch);
    if (o0 >= o1) return;
    // the segment's bytes, packed little-endian into two 64-bit registers
    unsigned long long lo = 0, hi = 0;
    const int px0 = (int)(o0 / 3), px1 = (int)((o1 - 1) / 3);
    for (int px = px0; px <= px1; ++px) {
        uint8_t v[3];
        grid_pixel<RESIZE>(a, b, y, px, v);
#pragma unroll
        for (int ch = 0; ch < 3; ++ch) {
            const long long j = 3LL * px + ch - o0;
            if (j < 0 || j >= o1 - o0) continue;
            if (j < 8) lo |= (unsigned long long)v[ch] << (8 * j);
            else hi |= (unsigned long long)v[ch] << (8 * (j - 8));
        }
    }
    if (seg > 0 && o1 - o0 == 16) {
        *reinterpret_cast<uint4*>(row + o0) = make_uint4((unsigned)lo, (unsigned)(lo >> 32), (unsigned)hi, (unsigned)(hi >> 32));
    } else {
        for (long long j = 0; j < o1 - o0; ++j) row[o0 + j] = (uint8_t)((j < 8 ? lo >> (8 * j) : hi >> (8 * (j - 8))) & 255u);
    }
}

constexpr int kHullMaxPoints = 1024, kHullMaxSize = 256;

// create_mask(cropped_kpt, (S, S)) as float: one CTA per frame.  The points are sorted by (x, y) with a stable parallel
// rank sort, one thread builds the hull and walks the outline and the spans into shared memory (hull_mask.cuh), then
// the CTA writes the S x S mask (0 inside the hull, 1 outside).
__global__ void __launch_bounds__(256) hull_mask_kernel(const int* __restrict__ pts, int L, int S, float* __restrict__ mask) {
    __shared__ int px[kHullMaxPoints], py[kHullMaxPoints], ord[kHullMaxPoints], stack[kHullMaxPoints + 2], hull[kHullMaxPoints];
    __shared__ int vx[kHullMaxPoints], vy[kHullMaxPoints], xl[kHullMaxSize], xr[kHullMaxSize];
    __shared__ unsigned bits[kHullMaxSize * kHullMaxSize / 32];
    const int b = blockIdx.x;
    const int* p = pts + (size_t)b * L * 2;
    for (int i = threadIdx.x; i < L; i += blockDim.x) { px[i] = __ldg(p + 2 * i); py[i] = __ldg(p + 2 * i + 1); }
    for (int i = threadIdx.x; i < S; i += blockDim.x) { xl[i] = S; xr[i] = -1; }
    for (int i = threadIdx.x; i < (S * S + 31) / 32; i += blockDim.x) bits[i] = 0u;
    __syncthreads();
    for (int i = threadIdx.x; i < L; i += blockDim.x) {
        const int x = px[i], y = py[i];
        int rank = 0;
        for (int j = 0; j < L; ++j) rank += (px[j] < x || (px[j] == x && (py[j] < y || (py[j] == y && j < i))));
        ord[rank] = i;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        const int n = smk::hull::convex_hull(px, py, ord, L, stack, hull);
        for (int i = 0; i < n; ++i) { vx[i] = px[hull[i]]; vy[i] = py[hull[i]]; }
        smk::hull::fill_convex_poly(S, vx, vy, n, [&](int x, int y) { bits[(y * S + x) >> 5] |= 1u << ((y * S + x) & 31); },
                                    [&](int y, int x0, int x1) { xl[y] = x0; xr[y] = x1; });
    }
    __syncthreads();
    float* m = mask + (size_t)b * S * S;
    for (int i = threadIdx.x; i < S * S; i += blockDim.x) {
        const int y = i / S, x = i - y * S;
        m[i] = ((x >= xl[y] && x <= xr[y]) || ((bits[i >> 5] >> (i & 31)) & 1u)) ? 0.0f : 1.0f;
    }
}

}  // namespace

extern "C" int smk_hull_mask(const int32_t* pts, int B, int L, int S, float* mask, void* stream) {
    SMK_REQUIRE(B >= 0, "smk_hull_mask: negative batch");
    if (B == 0) return 0;
    SMK_REQUIRE(pts && mask, "smk_hull_mask: null argument");
    SMK_REQUIRE(L > 0 && L <= kHullMaxPoints && S > 0 && S <= kHullMaxSize, "smk_hull_mask: bad sizes (1 <= L <= 1024, 1 <= S <= 256)");
    cudaStream_t st = (cudaStream_t)stream;
    SMK_TAG("hull_mask", (double)B * L * 8 + (double)B * S * S * 4, 0.0, st);
    SMK_LAUNCH(hull_mask_kernel, dim3(B), dim3(256), 0, st, pts, L, S, mask);
    SMK_CHECK_LAUNCH();
    return 0;
}

extern "C" size_t smk_video_workspace_bytes(int B, int n_panels) {
    return smk::ws_round((size_t)(B > 0 ? B : 1) * (size_t)(n_panels > 0 ? n_panels : 1) * 2 * sizeof(unsigned));
}

extern "C" int smk_video_compose(const uint8_t* frames, int B, int H, int W, const float* crop, const float* const* panels,
                                 int n_panels, int S, const double* m, int render_orig, uint8_t* grid, void* ws,
                                 size_t ws_bytes, void* stream) {
    SMK_REQUIRE(B >= 0, "smk_video_compose: negative batch");
    if (B == 0) return 0;
    SMK_REQUIRE(panels && grid, "smk_video_compose: null argument");
    SMK_REQUIRE(H > 0 && W > 0 && S > 0 && (n_panels == 1 || n_panels == 2), "smk_video_compose: bad sizes");
    SMK_REQUIRE(panels[0] && (n_panels == 1 || panels[1]), "smk_video_compose: null panel");
    SMK_REQUIRE(render_orig >= 0 && render_orig <= 2, "smk_video_compose: render_orig must be 0, 1 or 2");
    const bool resize = render_orig == 2;
    if (resize) {
        SMK_REQUIRE(frames, "smk_video_compose: render_orig == 2 needs frames");
    } else {
        SMK_REQUIRE(render_orig ? (frames && m) : (crop != nullptr), "smk_video_compose: render_orig needs frames and m, "
                    "otherwise the crop is needed");
        SMK_REQUIRE(!render_orig || (ws && ws_bytes >= smk_video_workspace_bytes(B, n_panels)), "smk_video_compose: workspace too small");
    }
    cudaStream_t st = (cudaStream_t)stream;
    ComposeArgs a;
    a.frames = frames; a.crop = crop; a.p1 = panels[0]; a.p2 = n_panels > 1 ? panels[1] : nullptr; a.m = m;
    a.mm = reinterpret_cast<const unsigned*>(ws);
    a.H = H; a.W = W; a.S = S; a.n_panels = n_panels; a.render_orig = render_orig ? 1 : 0;
    a.Ho = render_orig ? H : S; a.Wo = render_orig ? W : S;
    a.pitch = (long long)(n_panels + 1) * a.Wo * 3;
    a.grid = grid;
    SMK_REQUIRE(a.Ho <= 65535 && B <= 65535, "smk_video_compose: too many rows or frames");
    const double panel_bytes = (double)B * n_panels * 3 * S * S * 4;
    if (render_orig == 1) {
        SMK_TAG("video_minmax", panel_bytes, 0.0, st);
        SMK_LAUNCH(panel_minmax_kernel, dim3(B * n_panels), dim3(512), 0, st, a.p1, a.p2, S, n_panels, reinterpret_cast<unsigned*>(ws));
        SMK_CHECK_LAUNCH();
    }
    // algorithmic bytes: the grid written once, the frame (or the crop) and each panel read once
    const double read = render_orig ? (double)B * H * W * 3 + panel_bytes : (double)B * 3 * S * S * 4 + panel_bytes;
    SMK_TAG("video_compose", (double)B * a.Ho * a.pitch + read, 0.0, st);
    const long long nseg = a.pitch / 16 + 2;
    const dim3 grid_dim(smk::cdiv(nseg, 256), a.Ho, B);
    if (resize) SMK_LAUNCH(video_compose_kernel<true>, grid_dim, dim3(256), 0, st, a);
    else SMK_LAUNCH(video_compose_kernel<false>, grid_dim, dim3(256), 0, st, a);
    SMK_CHECK_LAUNCH();
    return 0;
}
