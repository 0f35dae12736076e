// ExpressionLoss (src/losses/ExpressionLoss.py): EMOCA's ResNet-50 feature extractor, frozen and in eval mode, on gen and
// tar, and a per-face metric of the two 2048-d features (l2: mean of squares, l1: mean of absolute values, cos: 1 - cosine
// similarity), optionally averaged over the faces; forward and input gradient.
//
// Network at 224^2 (eval-mode BatchNorm, eps 1e-5, folded in float64 into the epilogue's scale / bias), NHWC fp32:
//   stem       7x7 s2 p3 conv 3 -> 64 + BN + ReLU: expr_im2col_kernel writes the dense [M, 148] patch matrix (147 columns,
//              one zero) straight from both NCHW inputs, then one plain GEMM                                        112^2
//   maxpool    3x3 s2 p1, torch's rule (-inf padding, the first maximum in row-major window order wins)           56^2
//   4 layers   (3, 4, 6, 3) Bottlenecks, planes (64, 128, 256, 512), expansion 4:
//              y = relu(bn3(conv3(relu(bn2(conv2(relu(bn1(conv1(x)))))))) + identity), identity = x or bn(conv1x1_s(x));
//              the first block of each layer has the downsample and (layers 2-4) its stride on the 3x3 conv2
//   head       7x7 average pool, the metric of each face, and the mean over the faces (expr_head_kernel,
//              expr_mean_kernel): fixed summation orders, no atomics
//
// gen and tar run as one batch of 2B images.  1x1 convs are smk::conv mode 0, 3x3 stride-1 convs mode 1; the stride-2
// layers (three 3x3 conv2, three 1x1 downsamples) gather their receptive fields (smk::gather_s2, shared with MICA) into a
// dense matrix that a plain GEMM reads.  Precision 0 = fp32 CUDA cores, 1 = TF32 wgmma, 3 = 3xTF32 wgmma.  Precision 1
// rounds every stored activation another tensor-core layer reads to TF32: the patch matrix, the stem output (hence the
// pool output), u1 = conv1's and u2 = conv2's outputs and the block outputs y, which are also the residual stream (one
// store per layer; the last y, which feeds only the head, stays fp32).  Precision 3 rounds nothing.
//
// Input gradient (frozen weights).  The grad-mode forward also keeps, for the images whose gradient is wanted (they come
// first in the batch, tar's first when only tar's is wanted), u1, u2 and y of every block and the pool output (the
// epilogue's second store; at precision 3 a copy after the layer), the pool's int8 argmax tap, and both halves' features.  The backward walks back over those
// images only: expr_head_bwd_kernel spreads the metric's gradient over the 7x7 map under the last ReLU mask; each block
// runs conv3, conv2 and conv1 as dgrad GEMMs with the BN scale folded into the weights and the saved ReLU masks in the
// epilogue, conv1's with the identity path's gradient as its residual; a stride-2 dgrad is a GEMM into the gathered
// layout and expr_col2im_s2_kernel, the gather's adjoint, which sums each input pixel's <= 4 taps in a fixed order.
// expr_pool_bwd_kernel routes the pool gradient to the saved argmax taps (the stem's ReLU mask at the argmax is
// pool_out > 0, already applied), and expr_stem_dgrad_kernel is the transposed 7x7 s2 conv into NCHW.  Precision 1
// TF32-rounds every gradient a TF32 dgrad reads.
#include "nn_kernels.cuh"
#include "frozen_net.cuh"
#include <string>

namespace {

constexpr int kBlocks = 16, kLayers = 4, kFeat = 2048, kStemK = 148, kTensors = 265;
constexpr int kLayerBlocks[kLayers] = {3, 4, 6, 3};
constexpr int kOnes = 9 * 512;                                // the widest dgrad: layer4.0's conv2, N = 9 * 512
constexpr int kImg = 224, kS = 112, kP = 56;                 // input, stem output and pool output sizes
constexpr size_t kPatch = (size_t)kS * kS * kStemK;          // floats per image of the stem's patch matrix
constexpr size_t kActMax = (size_t)kP * kP * 256;            // largest activation: layer1's y, the stem output (112^2 x 64)
constexpr size_t kU1Max = (size_t)kP * kP * 128;             // layer2.0's u1
constexpr size_t kU2Max = (size_t)kP * kP * 64;              // layer1's u2
constexpr size_t kGatherMax = (size_t)28 * 28 * 9 * 128;     // layer2.0's gathered conv2 input (also its dgrad)

// ---- kernels ---------------------------------------------------------------------------------------------------------

// The stem's patch matrix of the 2B-image batch: row m = (i, oh, ow), column k = (ky*7 + kx)*3 + c < 147 holds image i's
// channel c at (2oh + ky - 3, 2ow + kx - 3), 0 outside and in column 147.  Images [0, B) come from a, [B, 2B) from b.
__global__ void __launch_bounds__(256)
expr_im2col_kernel(const float* __restrict__ a, const float* __restrict__ b, int B, int round, float4* __restrict__ out) {
    constexpr int Q = kStemK / 4;
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= 2L * B * kS * kS * Q) return;
    const int q = (int)(i % Q); const long m = i / Q;
    const int ow = (int)(m % kS); const long t = m / kS; const int oh = (int)(t % kS); const int img = (int)(t / kS);
    const float* src = img < B ? a + (size_t)img * 3 * kImg * kImg : b + (size_t)(img - B) * 3 * kImg * kImg;
    float v[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const int k = 4 * q + j, tap = k / 3, c = k - 3 * tap;
        const int ih = 2 * oh + tap / 7 - 3, iw = 2 * ow + tap % 7 - 3;
        float x = 0.f;
        if (k < 147 && ih >= 0 && ih < kImg && iw >= 0 && iw < kImg) x = __ldg(src + ((size_t)c * kImg + ih) * kImg + iw);
        v[j] = round ? smk::round_tf32(x) : x;
    }
    out[i] = make_float4(v[0], v[1], v[2], v[3]);
}

// 3x3 s2 p1 max pool of in [Bi,H,W,C] -> out [Bi,Ho,Wo,C], Ho = (H+1)/2: -inf padding, the first maximum in row-major
// window order wins (v > max || isnan(v), torch's rule).  The first save_imgs images also go to out2 and their winning
// tap (ky*3 + kx) to arg as int8, NHWC like out.
__global__ void __launch_bounds__(256)
expr_maxpool_kernel(const float4* __restrict__ in, int Bi, int H, int W, int C, float4* __restrict__ out, int save_imgs,
                    float4* __restrict__ out2, char4* __restrict__ arg) {
    const int C4 = C >> 2, Ho = (H + 1) >> 1, Wo = (W + 1) >> 1;
    const long total = (long)Bi * Ho * Wo * C4;
    for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        const int c4 = (int)(i % C4); const long pix = i / C4;
        const int ow = (int)(pix % Wo); const long t = pix / Wo; const int oh = (int)(t % Ho); const int b = (int)(t / Ho);
        float mx[4] = {-INFINITY, -INFINITY, -INFINITY, -INFINITY};
        int am[4] = {-1, -1, -1, -1};
#pragma unroll
        for (int ky = 0; ky < 3; ++ky) {
            const int h = 2 * oh + ky - 1;
            if (h < 0 || h >= H) continue;
#pragma unroll
            for (int kx = 0; kx < 3; ++kx) {
                const int w = 2 * ow + kx - 1;
                if (w < 0 || w >= W) continue;
                const float4 q = __ldg(in + (((size_t)b * H + h) * W + w) * C4 + c4);
                const float v[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
                for (int j = 0; j < 4; ++j)
                    if (am[j] < 0 || v[j] > mx[j] || isnan(v[j])) { mx[j] = v[j]; am[j] = ky * 3 + kx; }
            }
        }
        const float4 o = make_float4(mx[0], mx[1], mx[2], mx[3]);
        out[i] = o;
        if (b < save_imgs) {
            out2[i] = o;
            arg[i] = make_char4((signed char)am[0], (signed char)am[1], (signed char)am[2], (signed char)am[3]);
        }
    }
}

// Max-pool backward: out [Bi,H,W,C] at input pixel (h, w) = sum of g [Bi,Ho,Wo,C] over the <= 4 windows (oh, ow ascending)
// whose saved argmax tap is that pixel.
__global__ void __launch_bounds__(256)
expr_pool_bwd_kernel(const float4* __restrict__ g, const char4* __restrict__ arg, int Bi, int H, int W, int C,
                     float4* __restrict__ out) {
    const int C4 = C >> 2, Ho = (H + 1) >> 1, Wo = (W + 1) >> 1;
    const long total = (long)Bi * H * W * C4;
    for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        const int c4 = (int)(i % C4); const long pix = i / C4;
        const int w = (int)(pix % W); const long t = pix / W; const int h = (int)(t % H); const int b = (int)(t / H);
        float s[4] = {0.f, 0.f, 0.f, 0.f};
        for (int oh = h / 2; oh <= (h + 1) / 2 && oh < Ho; ++oh) {        // 2oh - 1 <= h <= 2oh + 1
            if (2 * oh - 1 > h) continue;
            for (int ow = w / 2; ow <= (w + 1) / 2 && ow < Wo; ++ow) {
                if (2 * ow - 1 > w) continue;
                const int tap = (h - 2 * oh + 1) * 3 + (w - 2 * ow + 1);
                const size_t o = (((size_t)b * Ho + oh) * Wo + ow) * C4 + c4;
                const char4 a = arg[o];
                const float4 q = __ldg(g + o);
                if (a.x == tap) s[0] += q.x;
                if (a.y == tap) s[1] += q.y;
                if (a.z == tap) s[2] += q.z;
                if (a.w == tap) s[3] += q.w;
            }
        }
        out[i] = make_float4(s[0], s[1], s[2], s[3]);
    }
}

// Adjoint of smk::gather_s2: dg [Bi*Ho*Wo, taps*C] (the gradient of the gathered matrix) -> out [Bi,H,W,C], H = 2Ho.
//   taps 9: out[b,h,w,c] = sum over the (ky, kx) with h = 2ho + ky - 1, w = 2wo + kx - 1 (ky, then kx ascending) of
//           dg[(b,ho,wo), (ky*3 + kx)*C + c];
//   taps 1: out = dg[(b,h/2,w/2), c] at even (h, w), 0 elsewhere.
// mask (optional, [Bi,H,W,C]): zero where mask <= 0; round: TF32 for a TF32 consumer.
__global__ void __launch_bounds__(256)
expr_col2im_s2_kernel(const float4* __restrict__ dg, int Bi, int Ho, int C, int taps, const float4* __restrict__ mask, int round,
                      float4* __restrict__ out) {
    const int C4 = C >> 2, H = 2 * Ho;
    const long total = (long)Bi * H * H * C4;
    for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        const int c4 = (int)(i % C4); const long pix = i / C4;
        const int w = (int)(pix % H); const long t = pix / H; const int h = (int)(t % H); const int b = (int)(t / H);
        float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
        if (taps == 9) {
            for (int ky = 0; ky < 3; ++ky) {
                const int h2 = h + 1 - ky;
                if (h2 & 1) continue;
                const int ho = h2 >> 1;
                if (ho < 0 || ho >= Ho) continue;
                for (int kx = 0; kx < 3; ++kx) {
                    const int w2 = w + 1 - kx;
                    if (w2 & 1) continue;
                    const int wo = w2 >> 1;
                    if (wo < 0 || wo >= Ho) continue;
                    const float4 q = __ldg(dg + ((((size_t)b * Ho + ho) * Ho + wo) * 9 + ky * 3 + kx) * C4 + c4);
                    s.x += q.x; s.y += q.y; s.z += q.z; s.w += q.w;
                }
            }
        } else if (!(h & 1) && !(w & 1)) {
            s = __ldg(dg + (((size_t)b * Ho + (h >> 1)) * Ho + (w >> 1)) * C4 + c4);
        }
        if (mask) {
            const float4 k = __ldg(mask + i);
            if (!(k.x > 0.f)) s.x = 0.f;
            if (!(k.y > 0.f)) s.y = 0.f;
            if (!(k.z > 0.f)) s.z = 0.f;
            if (!(k.w > 0.f)) s.w = 0.f;
        }
        if (round) { s.x = smk::round_tf32(s.x); s.y = smk::round_tf32(s.y); s.z = smk::round_tf32(s.z); s.w = smk::round_tf32(s.w); }
        out[i] = s;
    }
}

// Transposed stem: g [Bi,112,112,64] (the gradient at the stem's conv output, masked) -> the image gradient, NCHW
// [3,224,224] per image: out[c, ih, iw] = sum over ky, kx (ascending; the taps with 2oh = ih + 3 - ky and 2ow = iw + 3 - kx
// inside the output) and co of wd[(ky*7 + kx)*3 + c][co] * g[oh, ow, co], wd = bn scale[co] * W[co][c][ky][kx].
// Images [0, B) go to out0, [B, Bi) to out1.  One thread per input pixel.
__global__ void __launch_bounds__(256)
expr_stem_dgrad_kernel(const float4* __restrict__ g, const float4* __restrict__ wd, int B, int Bi, float* __restrict__ out0,
                       float* __restrict__ out1) {
    __shared__ float4 sw[147 * 16];
    for (int j = threadIdx.x; j < 147 * 16; j += blockDim.x) sw[j] = wd[j];
    __syncthreads();
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long)Bi * kImg * kImg) return;
    const int iw = (int)(i % kImg); const long t = i / kImg; const int ih = (int)(t % kImg); const int b = (int)(t / kImg);
    float acc[3] = {0.f, 0.f, 0.f};
    for (int ky = (ih + 1) & 1; ky < 7; ky += 2) {              // ih + 3 - ky even
        const int oh = (ih + 3 - ky) >> 1;
        if (oh < 0 || oh >= kS) continue;
        for (int kx = (iw + 1) & 1; kx < 7; kx += 2) {
            const int ow = (iw + 3 - kx) >> 1;
            if (ow < 0 || ow >= kS) continue;
            const float4* gp = g + (((size_t)b * kS + oh) * kS + ow) * 16;
            const float4* wp = sw + (ky * 7 + kx) * 3 * 16;
#pragma unroll 4
            for (int q = 0; q < 16; ++q) {
                const float4 v = __ldg(gp + q);
#pragma unroll
                for (int c = 0; c < 3; ++c) {
                    const float4 k = wp[c * 16 + q];
                    acc[c] = fmaf(v.x, k.x, acc[c]); acc[c] = fmaf(v.y, k.y, acc[c]);
                    acc[c] = fmaf(v.z, k.z, acc[c]); acc[c] = fmaf(v.w, k.w, acc[c]);
                }
            }
        }
    }
    float* o = b < B ? out0 + (size_t)b * 3 * kImg * kImg : out1 + (size_t)(b - B) * 3 * kImg * kImg;
#pragma unroll
    for (int c = 0; c < 3; ++c) o[((size_t)c * kImg + ih) * kImg + iw] = acc[c];
}

__device__ __forceinline__ float sgnf(float d) { return (float)((d > 0.f) - (d < 0.f)); }
constexpr float kCosEps = 1e-8f;

// Thread tid's 8 channels of an image's features: float4 columns tid and tid + 256.
__device__ __forceinline__ void load_feat(const float* __restrict__ f, float (&v)[8]) {
    const float4 a = __ldg(reinterpret_cast<const float4*>(f) + threadIdx.x), b = __ldg(reinterpret_cast<const float4*>(f) + threadIdx.x + 256);
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}

// One CTA per face b: the 7x7 average pools of its gen and tar images in y [2B,49,2048] (gen's at image b, tar's at B + b;
// swapped when swap) -> features [2B,2048] (gen's then tar's), and the face's metric -> lossv[b]:
//   0 l2: mean of (g - t)^2;  1 l1: mean of |g - t|;  2 cos: 1 - sum (g / max(|g|, eps)) * (t / max(|t|, eps)), eps 1e-8.
__global__ void __launch_bounds__(256)
expr_head_kernel(const float* __restrict__ y, int B, int swap, int metric, float* __restrict__ feat, float* __restrict__ lossv) {
    const int b = blockIdx.x;
    float f[2][8];
#pragma unroll
    for (int half = 0; half < 2; ++half) {                      // 0 gen, 1 tar
        const int img = (half ^ swap) ? B + b : b;
        const float4* src = reinterpret_cast<const float4*>(y + (size_t)img * 49 * kFeat);
        float4 s0 = make_float4(0.f, 0.f, 0.f, 0.f), s1 = s0;
        for (int p = 0; p < 49; ++p) {
            const float4 a = __ldg(src + p * (kFeat / 4) + threadIdx.x), c = __ldg(src + p * (kFeat / 4) + threadIdx.x + 256);
            s0.x += a.x; s0.y += a.y; s0.z += a.z; s0.w += a.w; s1.x += c.x; s1.y += c.y; s1.z += c.z; s1.w += c.w;
        }
        const float v[8] = {s0.x, s0.y, s0.z, s0.w, s1.x, s1.y, s1.z, s1.w};
#pragma unroll
        for (int j = 0; j < 8; ++j) f[half][j] = __fdiv_rn(v[j], 49.f);
        float4* dst = reinterpret_cast<float4*>(feat + ((size_t)half * B + b) * kFeat);
        dst[threadIdx.x] = make_float4(f[half][0], f[half][1], f[half][2], f[half][3]);
        dst[threadIdx.x + 256] = make_float4(f[half][4], f[half][5], f[half][6], f[half][7]);
    }
    float r;
    if (metric == 2) {
        float gg = 0.f, tt = 0.f;
#pragma unroll
        for (int j = 0; j < 8; ++j) { gg = fmaf(f[0][j], f[0][j], gg); tt = fmaf(f[1][j], f[1][j], tt); }
        const float n1 = fmaxf(sqrtf(smk::block_sum(gg)), kCosEps), n2 = fmaxf(sqrtf(smk::block_sum(tt)), kCosEps);
        float s = 0.f;
#pragma unroll
        for (int j = 0; j < 8; ++j) s = fmaf(__fdiv_rn(f[0][j], n1), __fdiv_rn(f[1][j], n2), s);
        r = 1.f - smk::block_sum(s);
    } else {
        float s = 0.f;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const float d = f[0][j] - f[1][j];
            s = metric == 0 ? fmaf(d, d, s) : s + fabsf(d);
        }
        r = __fdiv_rn(smk::block_sum(s), (float)kFeat);
    }
    if (threadIdx.x == 0) lossv[b] = r;
}

// loss = (sum of lossv[0..B), in order) / B.  One thread.
__global__ void expr_mean_kernel(const float* __restrict__ lossv, int B, float* __restrict__ loss) {
    float s = 0.f;
    for (int b = 0; b < B; ++b) s += lossv[b];
    *loss = __fdiv_rn(s, (float)B);
}

// Head backward, one CTA per image i of the chain (Bc images: the first B are gen's, or tar's when swap, the next B tar's):
// the metric's gradient for that image's features (feat [2B,2048], gen's then tar's) times the face's upstream gradient
// (g[b], or g[0] / B when use_mean), / 49, at each of the 49 pixels, zero where the last block's output y [Bc,49,2048] <= 0.
__global__ void __launch_bounds__(256)
expr_head_bwd_kernel(const float* __restrict__ feat, const float* __restrict__ y, const float* __restrict__ g, int B, int swap,
                     int metric, int use_mean, int round, float* __restrict__ out) {
    const int i = blockIdx.x, b = i % B;
    const bool tar = swap || i >= B;
    float fg[8], ft[8], d[8];
    load_feat(feat + (size_t)b * kFeat, fg);
    load_feat(feat + ((size_t)B + b) * kFeat, ft);
    const float gb = use_mean ? __fdiv_rn(__ldg(g), (float)B) : __ldg(g + b);
    if (metric == 2) {
        float gg = 0.f, tt = 0.f;
#pragma unroll
        for (int j = 0; j < 8; ++j) { gg = fmaf(fg[j], fg[j], gg); tt = fmaf(ft[j], ft[j], tt); }
        const float ng = sqrtf(smk::block_sum(gg)), nt = sqrtf(smk::block_sum(tt));
        const float n1 = fmaxf(ng, kCosEps), n2 = fmaxf(nt, kCosEps);
        float s = 0.f;
#pragma unroll
        for (int j = 0; j < 8; ++j) s = fmaf(__fdiv_rn(fg[j], n1), __fdiv_rn(ft[j], n2), s);
        const float cs = smk::block_sum(s);
        // d(1 - cos)/dx = -(o / (n_x n_o) - cos * x / (n_x |x|)), x the image's features, o the other's
        const float nx = tar ? n2 : n1, no = tar ? n1 : n2, ax = tar ? nt : ng;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const float xj = tar ? ft[j] : fg[j], oj = tar ? fg[j] : ft[j];
            const float a = __fdiv_rn(__fdiv_rn(oj, no), nx);
            const float c = ax > 0.f ? __fdiv_rn(cs * xj, nx * ax) : 0.f;
            d[j] = -gb * (a - c);
        }
    } else {
        const float gm = __fdiv_rn(gb, (float)kFeat);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const float e = fg[j] - ft[j];
            const float v = metric == 0 ? gm * (2.f * e) : gm * sgnf(e);
            d[j] = tar ? -v : v;
        }
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) d[j] = __fdiv_rn(d[j], 49.f);
    const float4* yp = reinterpret_cast<const float4*>(y + (size_t)i * 49 * kFeat);
    float4* op = reinterpret_cast<float4*>(out + (size_t)i * 49 * kFeat);
    for (int p = 0; p < 49; ++p) {
#pragma unroll
        for (int hf = 0; hf < 2; ++hf) {
            const int q = p * (kFeat / 4) + threadIdx.x + 256 * hf;
            const float4 m = __ldg(yp + q);
            float4 v = make_float4(m.x > 0.f ? d[4 * hf] : 0.f, m.y > 0.f ? d[4 * hf + 1] : 0.f,
                                   m.z > 0.f ? d[4 * hf + 2] : 0.f, m.w > 0.f ? d[4 * hf + 3] : 0.f);
            if (round) { v.x = smk::round_tf32(v.x); v.y = smk::round_tf32(v.y); v.z = smk::round_tf32(v.z); v.w = smk::round_tf32(v.w); }
            op[q] = v;
        }
    }
}

// ---- host -----------------------------------------------------------------------------------------------------------
using smk::Affine;

struct ExprBlock {
    int cin, planes, H, stride;                // H: input size; conv2 and the downsample run at H / stride
    bool ds;
    Affine bn1, bn2, bn3, ds_bn;
    smk::GemmW conv1{}, conv2{}, conv3{}, dsw{};        // forward: conv2 of a stride-2 block reads the gathered matrix
    smk::GemmW dconv1{}, dconv2{}, dconv3{}, ddsw{};    // dgrad, the BN scale folded in
    int s_u1 = 0, s_u2 = 0, s_y = 0;                    // indices of u1, u2, y in the saved layout
};

}  // namespace

struct SmkExpressionLoss {
    int precision;
    smk::GemmW stem{};
    Affine stem_bn;
    float* stem_dw = nullptr;                  // [147][64] (k, co): bn scale[co] * W[co][c][ky][kx], k = (ky*7 + kx)*3 + c
    ExprBlock blk[kBlocks];
    float *ones = nullptr, *zeros = nullptr;   // [kOnes]: unit scale and zero bias of the dgrads
    smk::SavedLayout saved;                    // per wanted image: pool, pool argmax (int8, as floats), u1 / u2 / y per block
    int s_pool = 0, s_arg = 0;
    smk::DeviceArena arena;
};

namespace {

using smk::bn_fold;
using smk::upload_bn;

// A 1x1 conv's weight [cout][cin] and its BN scale s: forward (N = cout, K = cin) and dgrad (N = cin, K = cout,
// W'(k = co, n = ci) = s[co] * W[co][ci]).
cudaError_t pack1(smk::DeviceArena& A, const float* w, const std::vector<double>& s, int cin, int cout, bool tc, bool x3,
                  smk::GemmW* fwd, smk::GemmW* dgrad) {
    cudaError_t e = smk::pack_gemm(A, cout, cin, tc, x3, w, fwd);
    if (e == cudaSuccess) e = smk::pack_gemm(A, cin, cout, tc, x3, [&](int n, int k) { return (float)(s[k] * (double)w[(size_t)k * cin + n]); }, dgrad);
    return e;
}

}  // namespace

extern "C" int smk_expression_loss_create(const SmkNetDesc* desc, SmkExpressionLoss** out) {
    if (int rc = smk::check_net_desc(desc, out, "smk_expression_loss_create", kTensors,
                                     "backbone.* in state_dict order without num_batches_tracked and fc"))
        return rc;
    const bool tc = desc->precision != 0, x3 = desc->precision == 3;
    SmkExpressionLoss* h = new SmkExpressionLoss();
    h->precision = desc->precision;
    smk::TensorCursor cur{desc->tensors, desc->n_tensors};
    auto bn4 = [&]() { return smk::next_bn(cur); };
    smk::DeviceArena& A = h->arena;
    std::vector<double> s, b;
    cudaError_t e = cudaSuccess;
    {   // stem: W [64][3][7][7], k = (ky*7 + kx)*3 + c
        const float* w = cur.next();
        bn_fold(bn4(), 64, s, b);
        auto wk = [&](int co, int k) { return w[((size_t)co * 3 + k % 3) * 49 + k / 3]; };
        e = smk::pack_gemm(A, 64, kStemK, tc, x3, [&](int n, int k) { return k < 147 ? wk(n, k) : 0.f; }, &h->stem);
        if (e == cudaSuccess) e = upload_bn(A, s, b, &h->stem_bn);
        std::vector<float> dw((size_t)147 * 64);
        for (int k = 0; k < 147; ++k)
            for (int co = 0; co < 64; ++co) dw[(size_t)k * 64 + co] = (float)(s[co] * (double)wk(co, k));
        if (e == cudaSuccess) e = A.upload(dw, &h->stem_dw);
    }
    h->s_pool = h->saved.add("pool", kP, kP, 64);
    h->s_arg = h->saved.add("pool_argmax", kP, kP, 16);          // int8 [56,56,64] in 16 floats per pixel
    int l = 0, cin = 64, H = kP;
    for (int ly = 0; ly < kLayers; ++ly) {
        const int planes = 64 << ly;
        for (int j = 0; j < kLayerBlocks[ly] && e == cudaSuccess; ++j, ++l) {
            ExprBlock& k = h->blk[l];
            k.cin = cin; k.planes = planes; k.H = H; k.stride = j == 0 && ly > 0 ? 2 : 1; k.ds = j == 0;
            const int Ho = H / k.stride;
            // state_dict order: conv1, conv2, bn1, bn2, conv3, bn3[, downsample.0, downsample.1]
            const float* w1 = cur.next();
            const float* w2 = cur.next();
            std::vector<double> s1, b1, s2, b2;
            bn_fold(bn4(), planes, s1, b1);
            bn_fold(bn4(), planes, s2, b2);
            e = pack1(A, w1, s1, cin, planes, tc, x3, &k.conv1, &k.dconv1);
            if (e == cudaSuccess) e = upload_bn(A, s1, b1, &k.bn1);
            if (e == cudaSuccess) e = upload_bn(A, s2, b2, &k.bn2);
            if (e == cudaSuccess) {
                std::vector<float> s2f(s2.begin(), s2.end());
                if (k.stride == 1) {
                    e = smk::pack_conv3(w2, s2f.data(), planes, planes, planes, tc, x3, A, &k.conv2, &k.dconv2);
                } else {                   // the gathered layout: k = tap * planes + ci; dgrad W'(k = co, n = tap * planes + ci)
                    e = smk::pack_gemm(A, planes, 9 * planes, tc, x3, [&](int o, int kk) {
                        return w2[((size_t)o * planes + kk % planes) * 9 + kk / planes];
                    }, &k.conv2);
                    if (e == cudaSuccess) e = smk::pack_gemm(A, 9 * planes, planes, tc, x3, [&](int n, int o) {
                        return (float)(s2[o] * (double)w2[((size_t)o * planes + n % planes) * 9 + n / planes]);
                    }, &k.dconv2);
                }
            }
            const float* w3 = cur.next();
            bn_fold(bn4(), 4 * planes, s, b);
            if (e == cudaSuccess) e = pack1(A, w3, s, planes, 4 * planes, tc, x3, &k.conv3, &k.dconv3);
            if (e == cudaSuccess) e = upload_bn(A, s, b, &k.bn3);
            if (k.ds) {
                const float* wd = cur.next();
                bn_fold(bn4(), 4 * planes, s, b);
                if (e == cudaSuccess) e = pack1(A, wd, s, cin, 4 * planes, tc, x3, &k.dsw, &k.ddsw);
                if (e == cudaSuccess) e = upload_bn(A, s, b, &k.ds_bn);
            }
            const std::string pre = "layer" + std::to_string(ly + 1) + "." + std::to_string(j) + ".";
            k.s_u1 = h->saved.add(pre + "u1", H, H, planes);
            k.s_u2 = h->saved.add(pre + "u2", Ho, Ho, planes);
            k.s_y = h->saved.add(pre + "y", Ho, Ho, 4 * planes);
            cin = 4 * planes; H = Ho;
        }
    }
    const std::vector<float> one(kOnes, 1.f), zero(kOnes, 0.f);
    if (e == cudaSuccess) e = A.upload(one, &h->ones);
    if (e == cudaSuccess) e = A.upload(zero, &h->zeros);
    return smk::finish_create(e, "smk_expression_loss_create", h, out);
}

extern "C" void smk_expression_loss_destroy(SmkExpressionLoss* h) { delete h; }

namespace {

using smk::halves;
using smk::tag_of;

size_t feat_floats(int B) { return (size_t)2 * B * kFeat; }

// One smk::conv problem of the network: out = epi(in * W), scale / bias (null: 1 / 0), res, relu, mask, round, out2.
struct Prob {
    const float* in; int ld_in, B, H, W, Cin, N, K, mode; smk::GemmW wgt; const float* scale; const float* bias;
    const float* res; int ld_res, relu; const float* mask; float* out; int ld_out, round; float* out2; int out2_rows; const char* tag;
};

int run(const SmkExpressionLoss* h, const Prob& q, cudaStream_t st) {
    SMK_REQUIRE((q.scale && q.bias) || q.N <= kOnes, "expression loss: a dgrad of width %d exceeds the unit scale", q.N);
    smk::Conv p{};
    p.in = q.in; p.ld_in = q.ld_in; p.B = q.B; p.H = q.H; p.W = q.W; p.Cin = q.Cin; p.N = q.N; p.K = q.K; p.mode = q.mode;
    p.wgt = q.wgt; p.scale = q.scale ? q.scale : h->ones; p.bias = q.bias ? q.bias : h->zeros;
    p.res = q.res; p.ld_res = q.ld_res; p.relu = q.relu; p.mask = q.mask; p.ld_mask = q.N;
    p.out = q.out; p.ld_out = q.ld_out; p.round_out = q.round;
    p.out2 = q.out2; p.ld_out2 = q.N; p.out2_rows = q.out2_rows; p.tag = q.tag;
    return smk::conv(p, st);
}

int col2im(const float* dg, int Bi, int Ho, int C, int taps, const float* mask, bool round, float* out, cudaStream_t st) {
    const long total = (long)Bi * 4 * Ho * Ho * (C / 4);
    SMK_TAG(taps == 9 ? "expr_col2im3x3_s2" : "expr_col2im1x1_s2",
            4.0 * (double)Bi * Ho * Ho * taps * C + 4.0 * total * 4 * (mask ? 2 : 1), taps == 9 ? 9.0 * Bi * Ho * Ho * C : 0.0, st);
    SMK_LAUNCH(expr_col2im_s2_kernel, dim3(smk::grid_of(total)), dim3(256), 0, st, reinterpret_cast<const float4*>(dg), Bi, Ho, C, taps,
               reinterpret_cast<const float4*>(mask), round ? 1 : 0, reinterpret_cast<float4*>(out));
    SMK_CHECK_LAUNCH();
    return 0;
}

int maxpool(const float* in, int Bi, int H, int C, float* out, int save_imgs, float* out2, int8_t* arg, cudaStream_t st) {
    const int Ho = (H + 1) / 2;
    const long total = (long)Bi * Ho * Ho * (C / 4);
    SMK_TAG("expr_maxpool3x3_s2", 4.0 * Bi * ((double)H * H * C + Ho * Ho * C) + (double)save_imgs * Ho * Ho * C * 5, 9.0 * total * 4, st);
    SMK_LAUNCH(expr_maxpool_kernel, dim3(smk::grid_of(total)), dim3(256), 0, st, reinterpret_cast<const float4*>(in), Bi, H, H, C,
               reinterpret_cast<float4*>(out), save_imgs, reinterpret_cast<float4*>(out2), reinterpret_cast<char4*>(arg));
    SMK_CHECK_LAUNCH();
    return 0;
}

int pool_bwd(const float* g, const int8_t* arg, int Bi, int H, int C, float* out, cudaStream_t st) {
    const int Ho = (H + 1) / 2;
    const long total = (long)Bi * H * H * (C / 4);
    SMK_TAG("expr_maxpool_dgrad", 4.0 * Bi * ((double)H * H * C + Ho * Ho * C * 1.25), 0.0, st);
    SMK_LAUNCH(expr_pool_bwd_kernel, dim3(smk::grid_of(total)), dim3(256), 0, st, reinterpret_cast<const float4*>(g),
               reinterpret_cast<const char4*>(arg), Bi, H, H, C, reinterpret_cast<float4*>(out));
    SMK_CHECK_LAUNCH();
    return 0;
}

int stem_dgrad(const float* g, const float* wd, int B, int Bi, float* out0, float* out1, cudaStream_t st) {
    const long total = (long)Bi * kImg * kImg;
    SMK_TAG("expr_stem_dgrad", 4.0 * Bi * ((double)kS * kS * 64 + 3.0 * kImg * kImg), 2.0 * Bi * kS * kS * 64 * 147, st);
    SMK_LAUNCH(expr_stem_dgrad_kernel, dim3(smk::cdiv(total, 256)), dim3(256), 0, st, reinterpret_cast<const float4*>(g),
               reinterpret_cast<const float4*>(wd), B, Bi, out0, out1);
    SMK_CHECK_LAUNCH();
    return 0;
}

int head(const float* y, int B, int swap, int metric, int use_mean, float* feat, float* lossv, float* loss, cudaStream_t st) {
    SMK_TAG("expr_head", 4.0 * (2.0 * B * 49 * kFeat + 2.0 * B * kFeat + B), 2.0 * B * 49 * kFeat + 6.0 * B * kFeat, st);
    SMK_LAUNCH(expr_head_kernel, dim3(B), dim3(256), 0, st, y, B, swap, metric, feat, use_mean ? lossv : loss);
    SMK_CHECK_LAUNCH();
    if (use_mean) {
        SMK_TAG("expr_mean", 4.0 * (B + 1), (double)B, st);
        SMK_LAUNCH(expr_mean_kernel, dim3(1), dim3(1), 0, st, lossv, B, loss);
        SMK_CHECK_LAUNCH();
    }
    return 0;
}

int head_bwd(const float* feat, const float* y, const float* g, int B, int Bc, int swap, int metric, int use_mean, bool round,
             float* out, cudaStream_t st) {
    SMK_TAG("expr_head_dgrad", 4.0 * (2.0 * Bc * 49 * kFeat + 2.0 * Bc * kFeat), 3.0 * Bc * 49 * kFeat, st);
    SMK_LAUNCH(expr_head_bwd_kernel, dim3(Bc), dim3(256), 0, st, feat, y, g, B, swap, metric, use_mean, round ? 1 : 0, out);
    SMK_CHECK_LAUNCH();
    return 0;
}

// The forward.  need == 0: the forward-only path.  Otherwise the first halves(need) * B images of the batch (tar's first
// when need == 2) also store what the backward needs to `saved`, and the features go there.  The arithmetic is the same.
int expr_forward(const SmkExpressionLoss* h, const float* gen, const float* tar, int B, int metric, int use_mean, int need,
                 float* loss, float* features, float* saved, void* ws, size_t ws_bytes, cudaStream_t st) {
    const int P = h->precision, swap = need == 2 ? 1 : 0, B2 = 2 * B, nsv = need ? halves(need) * B : 0;
    const bool rnd = P == 1;
    smk::Workspace w(ws, ws_bytes);
    float* Pm = w.take<float>(kPatch * B2);
    float* X[2] = {w.take<float>(kActMax * B2), w.take<float>(kActMax * B2)};
    float* U1 = w.take<float>(kU1Max * B2);
    float* U2 = w.take<float>(kU2Max * B2);
    float* D = w.take<float>(kActMax * B2);
    float* G = w.take<float>(kGatherMax * B2);
    float* F = w.take<float>(feat_floats(B));
    float* Lv = w.take<float>(B);
    SMK_REQUIRE(Lv, "smk_expression_loss_forward: workspace carve-up failed");
    if (saved) F = saved + h->saved.total * nsv;
    else if (features) F = features;
    auto SV = [&](int i) { return saved ? saved + h->saved.off[i] * nsv : nullptr; };
    // The saved copies of u1, u2 and y: the epilogue's second store, or at precision 3 a copy of the first images' rows
    // after the layer (a second store moves tc_conv's plain 1x1 GEMMs from X3 = 2 to X3 = 3, and the grad-mode forward
    // must compute the forward's bits).
    const bool fused = P != 3;
    auto sv2 = [&](int i) { return fused ? SV(i) : nullptr; };
    auto copy_saved = [&](int i, const float* out, size_t floats_per_img) -> int {
        if (!fused && saved) SMK_CHECK_CUDA(cudaMemcpyAsync(SV(i), out, floats_per_img * nsv * sizeof(float), cudaMemcpyDeviceToDevice, st));
        return 0;
    };
    int rc;
    {
        const long total = (long)B2 * kS * kS * (kStemK / 4);
        SMK_TAG("expr_im2col", 4.0 * (B2 * 3.0 * kImg * kImg + (double)total * 4), 0.0, st);
        SMK_LAUNCH(expr_im2col_kernel, dim3(smk::cdiv(total, 256)), dim3(256), 0, st, swap ? tar : gen, swap ? gen : tar, B, rnd ? 1 : 0,
                   reinterpret_cast<float4*>(Pm));
        SMK_CHECK_LAUNCH();
    }
    if ((rc = run(h, Prob{Pm, kStemK, B2, kS, kS, kStemK, 64, kStemK, 0, h->stem, h->stem_bn.scale, h->stem_bn.bias, nullptr, 0, 1,
                          nullptr, X[1], 64, rnd, nullptr, 0, tag_of(P, "expr_stem_f32", "expr_stem_tc", "expr_stem_tc3x")}, st))) return rc;
    if ((rc = maxpool(X[1], B2, kS, 64, X[0], nsv, SV(h->s_pool), reinterpret_cast<int8_t*>(SV(h->s_arg)), st))) return rc;
    int x = 0;
    for (int l = 0; l < kBlocks; ++l) {
        const ExprBlock& k = h->blk[l];
        const int H = k.H, Ho = H / k.stride, p = k.planes, last = l == kBlocks - 1;
        if ((rc = run(h, Prob{X[x], k.cin, B2, H, H, k.cin, p, k.cin, 0, k.conv1, k.bn1.scale, k.bn1.bias, nullptr, 0, 1, nullptr, U1, p,
                              rnd, sv2(k.s_u1), nsv * H * H, tag_of(P, "expr_conv1_f32", "expr_conv1_tc", "expr_conv1_tc3x")}, st))) return rc;
        if ((rc = copy_saved(k.s_u1, U1, (size_t)H * H * p))) return rc;
        const float* res = X[x];
        if (k.ds) {
            const float* in = X[x];
            if (k.stride == 2) {
                if ((rc = smk::gather_s2(X[x], B2, H, k.cin, 1, rnd, G, "expr_gather1x1_s2", st))) return rc;
                in = G;
            }
            if ((rc = run(h, Prob{in, k.cin, B2, Ho, Ho, k.cin, 4 * p, k.cin, 0, k.dsw, k.ds_bn.scale, k.ds_bn.bias, nullptr, 0, 0, nullptr,
                                  D, 4 * p, 0, nullptr, 0, tag_of(P, "expr_downsample_f32", "expr_downsample_tc", "expr_downsample_tc3x")}, st)))
                return rc;
            res = D;
        }
        if (k.stride == 1) {
            if ((rc = run(h, Prob{U1, p, B2, H, H, p, p, 9 * p, 1, k.conv2, k.bn2.scale, k.bn2.bias, nullptr, 0, 1, nullptr, U2, p, rnd,
                                  sv2(k.s_u2), nsv * H * H, tag_of(P, "expr_conv2_f32", "expr_conv2_tc", "expr_conv2_tc3x")}, st))) return rc;
        } else {
            if ((rc = smk::gather_s2(U1, B2, H, p, 9, rnd, G, "expr_gather3x3_s2", st))) return rc;
            if ((rc = run(h, Prob{G, 9 * p, B2, Ho, Ho, 9 * p, p, 9 * p, 0, k.conv2, k.bn2.scale, k.bn2.bias, nullptr, 0, 1, nullptr, U2, p,
                                  rnd, sv2(k.s_u2), nsv * Ho * Ho, tag_of(P, "expr_conv2_s2_f32", "expr_conv2_s2_tc", "expr_conv2_s2_tc3x")}, st)))
                return rc;
        }
        if ((rc = copy_saved(k.s_u2, U2, (size_t)Ho * Ho * p))) return rc;
        if ((rc = run(h, Prob{U2, p, B2, Ho, Ho, p, 4 * p, p, 0, k.conv3, k.bn3.scale, k.bn3.bias, res, 4 * p, 1, nullptr, X[x ^ 1], 4 * p,
                              rnd && !last, sv2(k.s_y), nsv * Ho * Ho, tag_of(P, "expr_conv3_f32", "expr_conv3_tc", "expr_conv3_tc3x")}, st)))
            return rc;
        if ((rc = copy_saved(k.s_y, X[x ^ 1], (size_t)Ho * Ho * 4 * p))) return rc;
        x ^= 1;
    }
    return head(X[x], B, swap, metric, use_mean, F, Lv, loss, st);
}

bool metric_ok(int metric) { return metric >= 0 && metric <= 2; }

}  // namespace

extern "C" size_t smk_expression_loss_workspace_bytes(const SmkExpressionLoss* h, int B) {
    if (!h || B <= 0) return 0;
    const size_t B2 = 2 * (size_t)B, f = sizeof(float);
    return smk::ws_round(kPatch * B2 * f) + 3 * smk::ws_round(kActMax * B2 * f) + smk::ws_round(kU1Max * B2 * f) +
           smk::ws_round(kU2Max * B2 * f) + smk::ws_round(kGatherMax * B2 * f) + smk::ws_round(feat_floats(B) * f) +
           smk::ws_round((size_t)B * f) + 256;
}

extern "C" int smk_expression_loss_forward(const SmkExpressionLoss* h, const float* gen, const float* tar, int B, int metric, int use_mean,
                                           float* loss, float* features, void* ws, size_t ws_bytes, void* stream) {
    SMK_REQUIRE(h && gen && tar && loss, "smk_expression_loss_forward: null argument");
    SMK_REQUIRE(B > 0, "smk_expression_loss_forward: B must be positive (got %d)", B);
    SMK_REQUIRE(metric_ok(metric), "smk_expression_loss_forward: metric must be 0 (l2), 1 (l1) or 2 (cos), got %d", metric);
    SMK_REQUIRE(ws && ws_bytes >= smk_expression_loss_workspace_bytes(h, B), "smk_expression_loss_forward: workspace too small");
    return expr_forward(h, gen, tar, B, metric, use_mean, 0, loss, features, nullptr, ws, ws_bytes, (cudaStream_t)stream);
}

extern "C" size_t smk_expression_loss_saved_bytes(const SmkExpressionLoss* h, int B, int need) {
    if (!h || B <= 0 || need < 1 || need > 3) return 0;
    return (h->saved.total * halves(need) * (size_t)B + feat_floats(B)) * sizeof(float);
}

extern "C" int smk_expression_loss_forward_saved(const SmkExpressionLoss* h, const float* gen, const float* tar, int B, int metric,
                                                 int use_mean, int need, float* loss, float* saved, size_t saved_bytes, void* ws,
                                                 size_t ws_bytes, void* stream) {
    SMK_REQUIRE(h && gen && tar && loss && saved, "smk_expression_loss_forward_saved: null argument");
    SMK_REQUIRE(B > 0, "smk_expression_loss_forward_saved: B must be positive (got %d)", B);
    SMK_REQUIRE(metric_ok(metric), "smk_expression_loss_forward_saved: metric must be 0 (l2), 1 (l1) or 2 (cos), got %d", metric);
    if (int rc = smk::check_need("smk_expression_loss_forward_saved", "gen", "tar", need, saved_bytes,
                                 smk_expression_loss_saved_bytes(h, B, need)))
        return rc;
    SMK_REQUIRE(ws && ws_bytes >= smk_expression_loss_workspace_bytes(h, B), "smk_expression_loss_forward_saved: workspace too small");
    return expr_forward(h, gen, tar, B, metric, use_mean, need, loss, nullptr, saved, ws, ws_bytes, (cudaStream_t)stream);
}

extern "C" int smk_expression_loss_saved_tensor(const SmkExpressionLoss* h, int B, int need, int i, const char** name, size_t* offset,
                                                int* dims) {
    SMK_REQUIRE(h && name && offset && dims, "smk_expression_loss_saved_tensor: null argument");
    SMK_REQUIRE(B >= 0 && need >= 1 && need <= 3, "smk_expression_loss_saved_tensor: bad B (%d) or need (%d)", B, need);
    const int n = (int)h->saved.name.size();
    SMK_REQUIRE(i >= 0 && i <= n, "smk_expression_loss_saved_tensor: index %d out of range (%d tensors)", i, n + 1);
    const int nsv = halves(need) * B;
    if (i == n) {
        *name = "features"; *offset = h->saved.total * nsv;
        dims[0] = 2 * B; dims[1] = dims[2] = 1; dims[3] = kFeat;
        return 0;
    }
    if (int rc = smk::saved_tensor(&h->saved, "smk_expression_loss_saved_tensor", nsv, i, name, offset, dims)) return rc;
    if (i == h->s_arg) dims[3] = 64;                            // int8 elements
    return 0;
}

extern "C" size_t smk_expression_loss_backward_workspace_bytes(const SmkExpressionLoss* h, int B, int need) {
    if (!h || B <= 0 || need < 1 || need > 3) return 0;
    const size_t Bc = (size_t)halves(need) * B, f = sizeof(float);
    return 3 * smk::ws_round(kActMax * Bc * f) + smk::ws_round(kU1Max * Bc * f) + smk::ws_round(kU2Max * Bc * f) +
           smk::ws_round(kGatherMax * Bc * f) + 256;
}

extern "C" int smk_expression_loss_backward(const SmkExpressionLoss* h, int B, int metric, int use_mean, int need, const float* saved,
                                            size_t saved_bytes, const float* g, float* g_gen, float* g_tar, void* ws, size_t ws_bytes,
                                            void* stream) {
    SMK_REQUIRE(h && saved && g, "smk_expression_loss_backward: null argument");
    SMK_REQUIRE(B > 0, "smk_expression_loss_backward: B must be positive (got %d)", B);
    SMK_REQUIRE(metric_ok(metric), "smk_expression_loss_backward: metric must be 0 (l2), 1 (l1) or 2 (cos), got %d", metric);
    if (int rc = smk::check_need("smk_expression_loss_backward", "gen", "tar", need, saved_bytes, smk_expression_loss_saved_bytes(h, B, need)))
        return rc;
    SMK_REQUIRE((!(need & 1) || g_gen) && (!(need & 2) || g_tar), "smk_expression_loss_backward: a gradient `need` asks for is null");
    SMK_REQUIRE(ws && ws_bytes >= smk_expression_loss_backward_workspace_bytes(h, B, need), "smk_expression_loss_backward: workspace too small");
    cudaStream_t st = (cudaStream_t)stream;
    const int P = h->precision, swap = need == 2 ? 1 : 0, Bc = halves(need) * B;
    const bool rnd = P == 1;
    smk::Workspace w(ws, ws_bytes);
    float* cur = w.take<float>(kActMax * Bc);
    float* nxt = w.take<float>(kActMax * Bc);
    float* R = w.take<float>(kActMax * Bc);
    float* G1 = w.take<float>(kU1Max * Bc);
    float* G2 = w.take<float>(kU2Max * Bc);
    float* DG = w.take<float>(kGatherMax * Bc);
    SMK_REQUIRE(DG, "smk_expression_loss_backward: workspace carve-up failed");
    auto SV = [&](int i) { return saved + h->saved.off[i] * Bc; };
    int rc;
    if ((rc = head_bwd(saved + h->saved.total * Bc, SV(h->blk[kBlocks - 1].s_y), g, B, Bc, swap, metric, use_mean, rnd, cur, st))) return rc;
    for (int l = kBlocks - 1; l >= 0; --l) {
        const ExprBlock& k = h->blk[l];
        const int H = k.H, Ho = H / k.stride, p = k.planes;
        // conv3: gz [Bc,Ho,Ho,4p] -> the gradient at conv2's BN output, masked by u2
        if ((rc = run(h, Prob{cur, 4 * p, Bc, Ho, Ho, 4 * p, p, 4 * p, 0, k.dconv3, nullptr, nullptr, nullptr, 0, 0, SV(k.s_u2), G2, p, rnd,
                              nullptr, 0, tag_of(P, "expr_conv3_dgrad_f32", "expr_conv3_dgrad_tc", "expr_conv3_dgrad_tc3x")}, st))) return rc;
        // identity path -> R (or gz itself)
        const float* res = cur;
        if (k.ds) {
            if (k.stride == 1) {
                if ((rc = run(h, Prob{cur, 4 * p, Bc, H, H, 4 * p, k.cin, 4 * p, 0, k.ddsw, nullptr, nullptr, nullptr, 0, 0, nullptr, R, k.cin,
                                      0, nullptr, 0, tag_of(P, "expr_downsample_dgrad_f32", "expr_downsample_dgrad_tc", "expr_downsample_dgrad_tc3x")}, st)))
                    return rc;
            } else {
                if ((rc = run(h, Prob{cur, 4 * p, Bc, Ho, Ho, 4 * p, k.cin, 4 * p, 0, k.ddsw, nullptr, nullptr, nullptr, 0, 0, nullptr, DG, k.cin,
                                      0, nullptr, 0, tag_of(P, "expr_downsample_dgrad_f32", "expr_downsample_dgrad_tc", "expr_downsample_dgrad_tc3x")}, st)))
                    return rc;
                if ((rc = col2im(DG, Bc, Ho, k.cin, 1, nullptr, false, R, st))) return rc;
            }
            res = R;
        }
        // conv2 -> the gradient at conv1's BN output, masked by u1
        if (k.stride == 1) {
            if ((rc = run(h, Prob{G2, p, Bc, H, H, p, p, 9 * p, 1, k.dconv2, nullptr, nullptr, nullptr, 0, 0, SV(k.s_u1), G1, p, rnd,
                                  nullptr, 0, tag_of(P, "expr_conv2_dgrad_f32", "expr_conv2_dgrad_tc", "expr_conv2_dgrad_tc3x")}, st))) return rc;
        } else {
            if ((rc = run(h, Prob{G2, p, Bc, Ho, Ho, p, 9 * p, p, 0, k.dconv2, nullptr, nullptr, nullptr, 0, 0, nullptr, DG, 9 * p, 0,
                                  nullptr, 0, tag_of(P, "expr_conv2_s2_dgrad_f32", "expr_conv2_s2_dgrad_tc", "expr_conv2_s2_dgrad_tc3x")}, st)))
                return rc;
            if ((rc = col2im(DG, Bc, Ho, p, 9, SV(k.s_u1), rnd, G1, st))) return rc;
        }
        // conv1 + identity -> the gradient at the block input, masked by it (the previous y, or the pool output)
        const float* mask = l > 0 ? SV(h->blk[l - 1].s_y) : SV(h->s_pool);
        if ((rc = run(h, Prob{G1, p, Bc, H, H, p, k.cin, p, 0, k.dconv1, nullptr, nullptr, res, k.cin, 0, mask, nxt, k.cin, rnd && l > 0,
                              nullptr, 0, tag_of(P, "expr_conv1_dgrad_f32", "expr_conv1_dgrad_tc", "expr_conv1_dgrad_tc3x")}, st))) return rc;
        std::swap(cur, nxt);
    }
    if ((rc = pool_bwd(cur, reinterpret_cast<const int8_t*>(SV(h->s_arg)), Bc, kS, 64, R, st))) return rc;
    return stem_dgrad(R, h->stem_dw, B, Bc, swap ? g_tar : g_gen, g_tar, st);
}

// ---- kernel-test entry points (tests/test_gpu_expression_loss_layers.py) ---------------------------------------------
// Exported but not part of include/smirk_b200.h; the test declares their argument types itself.
//
// expr_im2col_kernel: a, b [B,3,224,224] -> out [2B*112*112, 148].
extern "C" int smk_debug_expression_im2col(const float* a, const float* b, int B, int round, float* out, void* stream) {
    SMK_REQUIRE(a && b && out && B > 0, "smk_debug_expression_im2col: bad arguments");
    const long total = 2L * B * kS * kS * (kStemK / 4);
    cudaStream_t st = (cudaStream_t)stream;
    SMK_TAG("expr_im2col", 0.0, 0.0, st);
    SMK_LAUNCH(expr_im2col_kernel, dim3(smk::cdiv(total, 256)), dim3(256), 0, st, a, b, B, round, reinterpret_cast<float4*>(out));
    SMK_CHECK_LAUNCH();
    return 0;
}
// expr_maxpool_kernel: in [Bi,H,H,C] -> out [Bi,Ho,Ho,C], Ho = (H+1)/2; out2 / arg (int8) for the first save_imgs images.
extern "C" int smk_debug_expression_maxpool(const float* in, int Bi, int H, int C, float* out, int save_imgs, float* out2, int8_t* arg,
                                            void* stream) {
    SMK_REQUIRE(in && out && Bi > 0 && H > 1 && C % 4 == 0 && save_imgs >= 0 && save_imgs <= Bi && (!save_imgs || (out2 && arg)),
                "smk_debug_expression_maxpool: bad arguments");
    return maxpool(in, Bi, H, C, out, save_imgs, out2, arg, (cudaStream_t)stream);
}
// expr_pool_bwd_kernel: g [Bi,Ho,Ho,C], arg (int8) -> out [Bi,H,H,C].
extern "C" int smk_debug_expression_maxpool_bwd(const float* g, const int8_t* arg, int Bi, int H, int C, float* out, void* stream) {
    SMK_REQUIRE(g && arg && out && Bi > 0 && H > 1 && C % 4 == 0, "smk_debug_expression_maxpool_bwd: bad arguments");
    return pool_bwd(g, arg, Bi, H, C, out, (cudaStream_t)stream);
}
// expr_col2im_s2_kernel: dg [Bi*Ho*Ho, taps*C] -> out [Bi,2Ho,2Ho,C], mask optional.
extern "C" int smk_debug_expression_col2im(const float* dg, int Bi, int Ho, int C, int taps, const float* mask, int round, float* out,
                                           void* stream) {
    SMK_REQUIRE(dg && out && Bi > 0 && Ho > 0 && C % 4 == 0 && (taps == 1 || taps == 9), "smk_debug_expression_col2im: bad arguments");
    return col2im(dg, Bi, Ho, C, taps, mask, round != 0, out, (cudaStream_t)stream);
}
// expr_stem_dgrad_kernel: g [Bi,112,112,64], wd [147][64] -> out0 (images < B), out1 [.,3,224,224].
extern "C" int smk_debug_expression_stem_dgrad(const float* g, const float* wd, int B, int Bi, float* out0, float* out1, void* stream) {
    SMK_REQUIRE(g && wd && out0 && Bi > 0 && B > 0 && B <= Bi && (B == Bi || out1), "smk_debug_expression_stem_dgrad: bad arguments");
    return stem_dgrad(g, wd, B, Bi, out0, out1, (cudaStream_t)stream);
}
// The head: y [2B,7,7,2048] -> feat [2B,2048] and loss ([B], or the mean with use_mean; lossv [B] scratch).
extern "C" int smk_debug_expression_head(const float* y, int B, int swap, int metric, int use_mean, float* feat, float* lossv, float* loss,
                                         void* stream) {
    SMK_REQUIRE(y && feat && lossv && loss && B > 0 && metric_ok(metric), "smk_debug_expression_head: bad arguments");
    return head(y, B, swap, metric, use_mean, feat, lossv, loss, (cudaStream_t)stream);
}
// The head backward: feat [2B,2048], y [Bc,7,7,2048] (the mask), g ([B] or a scalar) -> out [Bc,7,7,2048].
extern "C" int smk_debug_expression_head_bwd(const float* feat, const float* y, const float* g, int B, int Bc, int swap, int metric,
                                             int use_mean, int round, float* out, void* stream) {
    SMK_REQUIRE(feat && y && g && out && B > 0 && (Bc == B || (Bc == 2 * B && !swap)) && metric_ok(metric),
                "smk_debug_expression_head_bwd: bad arguments");
    return head_bwd(feat, y, g, B, Bc, swap, metric, use_mean, round != 0, out, (cudaStream_t)stream);
}
