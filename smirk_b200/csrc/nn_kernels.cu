// fp32 CUDA-core kernels for the encoder / generator (see nn_kernels.cuh).
#include "nn_kernels.cuh"

namespace smk {
namespace {

constexpr int BK = 16;
constexpr int NT = 256;

// ---------------------------------------------------------------------------------------------------
// Implicit-GEMM convolution, BMxBN tile, BK = 16, 256 threads as a 16x16 grid of (BM/16)x(BN/16)
// register tiles; global->register prefetch of the next k-slab overlaps the FMAs of the current one.
// AFF: the epilogue also applies p.prelu and writes out2 through p.scale2 / p.bias2 (smk::conv_aff problems only).
template <int BM, int BN, bool AFF = false>
__global__ void __launch_bounds__(NT)
conv_gemm_kernel(Conv p, int M) {
    constexpr int TM = BM / 16, TN = BN / 16;
    constexpr int A_LD = BM + 4, B_LD = BN + 4;
    constexpr int A_PER = BM / 64;                 // float4 loads of A per thread per slab (BM*BK/4/NT)
    constexpr int B_PER = (BN * BK / 4 + NT - 1) / NT;
    __shared__ __align__(16) float As[BK][A_LD];
    __shared__ __align__(16) float Bs[BK][B_LD];
    const int tid = threadIdx.x, tx = tid % 16, ty = tid / 16;
    const int m0 = blockIdx.x * BM, n0 = blockIdx.y * BN;
    const int HW = p.H * p.W;

    // per-thread A rows: r = tid/4 + 64*j, k-quad kq = tid%4
    const int kq = tid & 3;
    int a_b[A_PER], a_h[A_PER], a_w[A_PER];
    bool a_ok[A_PER];
#pragma unroll
    for (int j = 0; j < A_PER; ++j) {
        int m = m0 + (tid >> 2) + 64 * j;
        a_ok[j] = m < M;
        int mm = a_ok[j] ? m : 0;
        a_b[j] = mm / HW; int r = mm - a_b[j] * HW; a_h[j] = r / p.W; a_w[j] = r - a_h[j] * p.W;
    }
    float4 a_reg[A_PER], b_reg[B_PER];

    auto load_slab = [&](int k0) {
        const int k = k0 + kq * 4;
#pragma unroll
        for (int j = 0; j < A_PER; ++j) {
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (a_ok[j] && k < p.K) {
                if (p.mode == 0) {
                    v = *reinterpret_cast<const float4*>(p.in + ((size_t)(a_b[j] * HW + a_h[j] * p.W + a_w[j])) * p.ld_in + k);
                } else {
                    int tap = k / p.Cin, c = k - tap * p.Cin;
                    int ky = tap / 3, kx = tap - ky * 3;
                    int hh = a_h[j] + ky - 1, ww = a_w[j] + kx - 1;
                    bool inside = hh >= 0 && hh < p.H && ww >= 0 && ww < p.W;
                    if (p.mode == 2) {                                  // ReflectionPad2d(1)
                        hh = hh < 0 ? 1 : (hh >= p.H ? p.H - 2 : hh);
                        ww = ww < 0 ? 1 : (ww >= p.W ? p.W - 2 : ww);
                        inside = true;
                    }
                    if (inside)
                        v = *reinterpret_cast<const float4*>(p.in + ((size_t)(a_b[j] * p.H + hh) * p.W + ww) * p.ld_in + c);
                }
            }
            a_reg[j] = v;
        }
#pragma unroll
        for (int j = 0; j < B_PER; ++j) {
            int idx = tid + j * NT;                     // float4 index within the BK x BN slab
            int kk = idx / (BN / 4), nq = idx - kk * (BN / 4);
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (kk < BK && k0 + kk < p.K && n0 + nq * 4 < p.N)
                v = *reinterpret_cast<const float4*>(p.wgt.w + (size_t)(k0 + kk) * p.N + n0 + nq * 4);
            b_reg[j] = v;
        }
    };
    auto store_slab = [&]() {
#pragma unroll
        for (int j = 0; j < A_PER; ++j) {
            int r = (tid >> 2) + 64 * j;
            As[kq * 4 + 0][r] = a_reg[j].x; As[kq * 4 + 1][r] = a_reg[j].y;
            As[kq * 4 + 2][r] = a_reg[j].z; As[kq * 4 + 3][r] = a_reg[j].w;
        }
#pragma unroll
        for (int j = 0; j < B_PER; ++j) {
            int idx = tid + j * NT;
            int kk = idx / (BN / 4), nq = idx - kk * (BN / 4);
            if (kk < BK) *reinterpret_cast<float4*>(&Bs[kk][nq * 4]) = b_reg[j];
        }
    };

    float acc[TM][TN];
#pragma unroll
    for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

    load_slab(0);
    for (int k0 = 0; k0 < p.K; k0 += BK) {
        __syncthreads();
        store_slab();
        __syncthreads();
        if (k0 + BK < p.K) load_slab(k0 + BK);
#pragma unroll
        for (int kk = 0; kk < BK; ++kk) {
            float a[TM], b[TN];
#pragma unroll
            for (int i = 0; i < TM; ++i) a[i] = As[kk][ty * TM + i];
#pragma unroll
            for (int j = 0; j < TN; ++j) b[j] = Bs[kk][tx * TN + j];
#pragma unroll
            for (int i = 0; i < TM; ++i)
#pragma unroll
                for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
        }
    }
    // epilogue
#pragma unroll
    for (int i = 0; i < TM; ++i) {
        int m = m0 + ty * TM + i;
        if (m >= M) continue;
        size_t opix = m;
        int nbase = n0 + tx * TN;
#pragma unroll
        for (int j = 0; j < TN; ++j) {
            int n = nbase + j;
            if (n >= p.N) continue;
            float v = fmaf(acc[i][j], p.scale[n], p.bias[n]);
            if (p.res) v += p.res[(size_t)m * p.ld_res + n];
            if (p.relu) v = fmaxf(v, 0.f);
            if constexpr (AFF) { if (p.prelu && v < 0.f) v *= p.prelu[n]; }
            if (p.mask && !(p.mask[(size_t)m * p.ld_mask + n] > 0.f)) v = 0.f;
            float v2 = 0.f;
            if constexpr (AFF) {
                if (p.scale2) { v2 = fmaf(v, p.scale2[n], p.bias2[n]); if (p.round_out2) v2 = round_tf32(v2); }
            }
            if (p.round_out) v = round_tf32(v);
            if constexpr (AFF) {
                if (p.out2 && (p.out2_rows <= 0 || m < p.out2_rows)) p.out2[(size_t)m * p.ld_out2 + n] = p.scale2 ? v2 : v;
            } else {
                if (p.out2 && (p.out2_rows <= 0 || m < p.out2_rows)) p.out2[(size_t)m * p.ld_out2 + n] = v;
            }
            if (p.store == 1) {
                int cout = p.N >> 2, q = n / cout, co = n - q * cout;
                int b = m / HW, r = m - b * HW, h = r / p.W, w = r - h * p.W;
                size_t dp = ((size_t)b * (2 * p.H) + 2 * h + (q >> 1)) * (2 * p.W) + 2 * w + (q & 1);
                p.out[dp * p.ld_out + co] = v;
            } else {
                p.out[opix * p.ld_out + n] = v;
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------------
// Depthwise 3x3, 4 output pixels along W x 4 channels per thread: the 3 x (3 + 3*STRIDE) input window is
// loaded once (float4 per pixel) and reused by the 4 outputs; weights stay in registers.
template <int STRIDE>
__global__ void __launch_bounds__(256)
dwconv3x3_px4_kernel(const float* __restrict__ in, int B, int H, int W, int C, int pad, int Ho, int Wo,
                     const float* __restrict__ w9c, const float* __restrict__ scale, const float* __restrict__ bias,
                     float* __restrict__ out, int round_out) {
    constexpr int PX = 4, NC = 3 + (PX - 1) * STRIDE;
    const int C4 = C >> 2, WG = (Wo + PX - 1) / PX;
    const long total = (long)B * Ho * WG * C4;
    for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        int c4 = (int)(i % C4); long t = i / C4;
        int wg = (int)(t % WG); t /= WG; int oh = (int)(t % Ho); int b = (int)(t / Ho);
        const int ow0 = wg * PX, iw0 = ow0 * STRIDE - pad;
        float4 k[9];
#pragma unroll
        for (int q = 0; q < 9; ++q) k[q] = __ldg(reinterpret_cast<const float4*>(w9c + (size_t)q * C) + c4);
        float4 acc[PX];
#pragma unroll
        for (int p = 0; p < PX; ++p) acc[p] = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int ky = 0; ky < 3; ++ky) {
            int ih = oh * STRIDE + ky - pad;
            if (ih < 0 || ih >= H) continue;
            const float4* row = reinterpret_cast<const float4*>(in + ((size_t)b * H + ih) * W * C) + c4;
            float4 x[NC];
#pragma unroll
            for (int j = 0; j < NC; ++j) {
                int iw = iw0 + j;
                x[j] = (iw >= 0 && iw < W) ? __ldg(row + (size_t)iw * C4) : make_float4(0.f, 0.f, 0.f, 0.f);
            }
#pragma unroll
            for (int p = 0; p < PX; ++p)
#pragma unroll
                for (int kx = 0; kx < 3; ++kx) {
                    const float4 xv = x[p * STRIDE + kx], kv = k[ky * 3 + kx];
                    acc[p].x = fmaf(xv.x, kv.x, acc[p].x); acc[p].y = fmaf(xv.y, kv.y, acc[p].y);
                    acc[p].z = fmaf(xv.z, kv.z, acc[p].z); acc[p].w = fmaf(xv.w, kv.w, acc[p].w);
                }
        }
        const float4 s = __ldg(reinterpret_cast<const float4*>(scale) + c4), bb = __ldg(reinterpret_cast<const float4*>(bias) + c4);
        float4* orow = reinterpret_cast<float4*>(out + (((size_t)b * Ho + oh) * Wo) * C) + c4;
#pragma unroll
        for (int p = 0; p < PX; ++p) {
            if (ow0 + p >= Wo) break;
            float4 o;
            o.x = fmaxf(fmaf(acc[p].x, s.x, bb.x), 0.f); o.y = fmaxf(fmaf(acc[p].y, s.y, bb.y), 0.f);
            o.z = fmaxf(fmaf(acc[p].z, s.z, bb.z), 0.f); o.w = fmaxf(fmaf(acc[p].w, s.w, bb.w), 0.f);
            if (round_out) { o.x = round_tf32(o.x); o.y = round_tf32(o.y); o.z = round_tf32(o.z); o.w = round_tf32(o.w); }
            orow[(size_t)(ow0 + p) * C4] = o;
        }
    }
}

// Global average pool + linear head + clamps in ONE launch for one or two backbones (blockIdx.z): every CTA pools its
// image's feature map into shared memory (the map is L2-resident: 188 KB at 7x7x960) and computes 32 head outputs, one
// warp per output (smirk_encoder.py:34-45,66-73,95-110).
// SAVE: also store the pre-clamp head values (raw) for the backward's clamp masks.
struct GapHead { const float* feat[2]; const float* w[2]; const float* bias[2]; const uint8_t* codes[2]; float* out[2]; int n_out[2]; float* raw[2]; };
template <bool SAVE>
__global__ void __launch_bounds__(256)
gap_head_kernel(const __grid_constant__ GapHead g, int HW, int C) {
    extern __shared__ float pooled[];                 // [C]
    const int q = blockIdx.z, b = blockIdx.x;
    const int n_out = g.n_out[q];
    if ((int)blockIdx.y * 32 >= n_out) return;
    const float* f = g.feat[q] + (size_t)b * HW * C;
    const float inv = 1.f / (float)HW;
    for (int c = threadIdx.x; c < C; c += 256) {
        float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
        int p = 0;
        for (; p + 4 <= HW; p += 4) {
            s0 += f[(size_t)p * C + c]; s1 += f[(size_t)(p + 1) * C + c]; s2 += f[(size_t)(p + 2) * C + c]; s3 += f[(size_t)(p + 3) * C + c];
        }
        for (; p < HW; ++p) s0 += f[(size_t)p * C + c];
        pooled[c] = ((s0 + s1) + (s2 + s3)) * inv;
    }
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const float* w = g.w[q]; const float* bias = g.bias[q]; const uint8_t* codes = g.codes[q];
#pragma unroll 1
    for (int j = 0; j < 4; ++j) {
        const int o = blockIdx.y * 32 + warp * 4 + j;
        if (o >= n_out) break;
        const float* wr = w + (size_t)o * C;
        float acc = 0.f;
        for (int c = lane; c < C; c += 32) acc = fmaf(pooled[c], __ldg(wr + c), acc);
#pragma unroll
        for (int s = 16; s > 0; s >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, s);
        if (lane == 0) {
            float v = acc + bias[o];
            if (SAVE) g.raw[q][(size_t)b * n_out + o] = v;
            const int code = codes ? codes[o] : 0;
            if (code == 1) v = fminf(fmaxf(v, 0.f), 1.f);
            else if (code == 2) v = fmaxf(v, 0.f);
            else if (code == 3) v = fminf(fmaxf(v, -0.2f), 0.2f);
            g.out[q][(size_t)b * n_out + o] = v;
        }
    }
}

__global__ void __launch_bounds__(128)
stem_conv_kernel(const float* __restrict__ img, int B, int H, int W, int Ho, int Wo, int pad,
                 const float* __restrict__ w /*[27][16]*/, const float* __restrict__ scale,
                 const float* __restrict__ bias, float* __restrict__ out) {
    __shared__ float sw[27 * 16];
    __shared__ float ss[16], sb[16];
    for (int i = threadIdx.x; i < 27 * 16; i += blockDim.x) sw[i] = w[i];
    if (threadIdx.x < 16) { ss[threadIdx.x] = scale[threadIdx.x]; sb[threadIdx.x] = bias[threadIdx.x]; }
    __syncthreads();
    long pix = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (pix >= (long)B * Ho * Wo) return;
    int ow = (int)(pix % Wo); long t = pix / Wo; int oh = (int)(t % Ho); int b = (int)(t / Ho);
    float acc[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) acc[i] = 0.f;
#pragma unroll
    for (int c = 0; c < 3; ++c)
#pragma unroll
        for (int ky = 0; ky < 3; ++ky) {
            int ih = oh * 2 + ky - pad;
#pragma unroll
            for (int kx = 0; kx < 3; ++kx) {
                int iw = ow * 2 + kx - pad;
                float x = (ih >= 0 && ih < H && iw >= 0 && iw < W) ? img[(((size_t)b * 3 + c) * H + ih) * W + iw] : 0.f;
                const float* wk = sw + ((c * 3 + ky) * 3 + kx) * 16;
#pragma unroll
                for (int i = 0; i < 16; ++i) acc[i] = fmaf(x, wk[i], acc[i]);
            }
        }
    float4* o = reinterpret_cast<float4*>(out + (size_t)pix * 16);
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        float4 v;
        v.x = fmaxf(fmaf(acc[q * 4 + 0], ss[q * 4 + 0], sb[q * 4 + 0]), 0.f);
        v.y = fmaxf(fmaf(acc[q * 4 + 1], ss[q * 4 + 1], sb[q * 4 + 1]), 0.f);
        v.z = fmaxf(fmaf(acc[q * 4 + 2], ss[q * 4 + 2], sb[q * 4 + 2]), 0.f);
        v.w = fmaxf(fmaf(acc[q * 4 + 3], ss[q * 4 + 3], sb[q * 4 + 3]), 0.f);
        o[q] = v;
    }
}

// The three backbones' stems read the same image: one pass over the pixels produces all 3 x 16 channels.
struct Stem3 { const float* w[3]; const float* scale[3]; const float* bias[3]; float* out[3]; };

// CTA = one output row (b, oh): the 3 channels x 3 input rows it needs are staged in shared memory with
// coalesced 16-byte loads (instead of 27 strided 4-byte loads per thread); thread = output pixel, 48 accumulators.
constexpr int STEM_MAXW = 512;                     // staged row length (floats), >= W + 2
__global__ void __launch_bounds__(128)
stem_conv3_kernel(const float* __restrict__ img, int B, int H, int W, int Ho, int Wo, int pad, Stem3 p) {
    __shared__ float sw[27 * 48];                  // [tap][group*16 + co]
    __shared__ float ss[48], sb[48];
    __shared__ __align__(16) float sin_[9][STEM_MAXW];   // [c*3+ky][1 + iw]  (column 0 = left padding)
    const int oh = blockIdx.x % Ho, b = blockIdx.x / Ho;
    for (int i = threadIdx.x; i < 27 * 48; i += blockDim.x) { int tap = i / 48, gc = i % 48; sw[i] = p.w[gc / 16][tap * 16 + gc % 16]; }
    if (threadIdx.x < 48) { ss[threadIdx.x] = p.scale[threadIdx.x / 16][threadIdx.x % 16]; sb[threadIdx.x] = p.bias[threadIdx.x / 16][threadIdx.x % 16]; }
    {   // stage rows: element iw of row (c,ky) lands at sin_[c*3+ky][4 + iw] so 16-byte stores stay aligned; halo columns zeroed
        const int W4 = W >> 2;
        for (int i = threadIdx.x; i < 9 * W4; i += blockDim.x) {
            const int r = i / W4, q = i - r * W4, c = r / 3, ky = r - c * 3;
            const int ih = oh * 2 + ky - pad;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (ih >= 0 && ih < H) v = __ldg(reinterpret_cast<const float4*>(img + (((size_t)b * 3 + c) * H + ih) * W) + q);
            *reinterpret_cast<float4*>(&sin_[r][4 + 4 * q]) = v;
        }
        if (threadIdx.x < 9) { sin_[threadIdx.x][3] = 0.f; sin_[threadIdx.x][4 + W] = 0.f; sin_[threadIdx.x][5 + W] = 0.f; }
    }
    __syncthreads();
    for (int ow = threadIdx.x; ow < Wo; ow += blockDim.x) {
    const long pix = ((long)b * Ho + oh) * Wo + ow;
    float acc[48];
#pragma unroll
    for (int i = 0; i < 48; ++i) acc[i] = 0.f;
#pragma unroll
    for (int c = 0; c < 3; ++c)
#pragma unroll
        for (int ky = 0; ky < 3; ++ky) {
#pragma unroll
            for (int kx = 0; kx < 3; ++kx) {
                const float x = sin_[c * 3 + ky][4 + ow * 2 + kx - pad];
                const float* wk = sw + ((c * 3 + ky) * 3 + kx) * 48;
#pragma unroll
                for (int i = 0; i < 48; ++i) acc[i] = fmaf(x, wk[i], acc[i]);
            }
        }
#pragma unroll
    for (int g = 0; g < 3; ++g) {
        float4* o = reinterpret_cast<float4*>(p.out[g] + (size_t)pix * 16);
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const int i = g * 16 + q * 4;
            float4 v;
            v.x = fmaxf(fmaf(acc[i + 0], ss[i + 0], sb[i + 0]), 0.f); v.y = fmaxf(fmaf(acc[i + 1], ss[i + 1], sb[i + 1]), 0.f);
            v.z = fmaxf(fmaf(acc[i + 2], ss[i + 2], sb[i + 2]), 0.f); v.w = fmaxf(fmaf(acc[i + 3], ss[i + 3], sb[i + 3]), 0.f);
            o[q] = v;
        }
    }
    }   // ow
}

__global__ void __launch_bounds__(256)
maxpool2x2_kernel(const float* __restrict__ in, int ld_in, int B, int H, int W, int C, float* __restrict__ out) {
    const int Ho = H >> 1, Wo = W >> 1, C4 = C >> 2;
    const long total = (long)B * Ho * Wo * C4;
    for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        int c4 = (int)(i % C4); long pix = i / C4;
        int ow = (int)(pix % Wo); long t = pix / Wo; int oh = (int)(t % Ho); int b = (int)(t / Ho);
        const float* p00 = in + (((size_t)b * H + 2 * oh) * W + 2 * ow) * ld_in + c4 * 4;
        float4 a = *reinterpret_cast<const float4*>(p00), bq = *reinterpret_cast<const float4*>(p00 + ld_in);
        float4 c = *reinterpret_cast<const float4*>(p00 + (size_t)W * ld_in), d = *reinterpret_cast<const float4*>(p00 + (size_t)W * ld_in + ld_in);
        float4 o;
        o.x = fmaxf(fmaxf(a.x, bq.x), fmaxf(c.x, d.x)); o.y = fmaxf(fmaxf(a.y, bq.y), fmaxf(c.y, d.y));
        o.z = fmaxf(fmaxf(a.z, bq.z), fmaxf(c.z, d.z)); o.w = fmaxf(fmaxf(a.w, bq.w), fmaxf(c.w, d.w));
        *reinterpret_cast<float4*>(out + (size_t)pix * C + c4 * 4) = o;
    }
}

__global__ void __launch_bounds__(256)
nchw_to_nhwc_pad_kernel(const float* __restrict__ in, int B, int C, int HW, int Cp, int round, float* __restrict__ out) {
    // thread = (pixel, channel quad), quads of a pixel in adjacent lanes: every warp stores 512 contiguous bytes
    const int Q = Cp >> 2;
    long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long)B * HW * Q) return;
    const int q = (int)(i % Q); const long pix = i / Q;
    const int b = (int)(pix / HW); const int r = (int)(pix - (long)b * HW);
    float v[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const int c = q * 4 + k;
        v[k] = c < C ? __ldg(in + ((size_t)b * C + c) * HW + r) : 0.f;
        if (round) v[k] = round_tf32(v[k]);
    }
    reinterpret_cast<float4*>(out)[i] = make_float4(v[0], v[1], v[2], v[3]);
}

__global__ void __launch_bounds__(256)
conv1x1_sigmoid_kernel(const float* __restrict__ in, int B, int HW, int Cin, const float* __restrict__ w,
                       const float* __restrict__ bias, int Cout, float* __restrict__ out) {
    extern __shared__ float sw[];                 // [Cin][Cout] + [Cout]
    for (int i = threadIdx.x; i < Cin * Cout; i += blockDim.x) sw[i] = w[i];
    for (int i = threadIdx.x; i < Cout; i += blockDim.x) sw[Cin * Cout + i] = bias[i];
    __syncthreads();
    long pix = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (pix >= (long)B * HW) return;
    int b = (int)(pix / HW); int r = (int)(pix - (long)b * HW);
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    const float4* x4 = reinterpret_cast<const float4*>(in + (size_t)pix * Cin);
    for (int c4 = 0; c4 < Cin / 4; ++c4) {
        float4 x = x4[c4];
        float xs[4] = {x.x, x.y, x.z, x.w};
#pragma unroll
        for (int q = 0; q < 4; ++q)
            for (int co = 0; co < Cout; ++co) acc[co] = fmaf(xs[q], sw[(c4 * 4 + q) * Cout + co], acc[co]);
    }
    for (int co = 0; co < Cout; ++co) {
        float v = acc[co] + sw[Cin * Cout + co];
        out[((size_t)b * Cout + co) * HW + r] = 1.f / (1.f + expf(-v));
    }
}

}  // namespace

int conv_gemm(const Conv& p, cudaStream_t st) {
    const int M = p.B * p.H * p.W;
    SMK_REQUIRE(!p.wgt.wt && !p.wgt.wt_lo, "conv_gemm: TF32 weights need tc_conv");
    SMK_REQUIRE(!p.res_pad && (p.store == 0 || p.store == 1), "conv_gemm: padded residuals and stores 2 / 3 need tc_conv");
    SMK_REQUIRE(p.K % 4 == 0 && p.N % 4 == 0 && p.ld_in % 4 == 0, "conv_gemm: K, N, ld_in must be multiples of 4");
    SMK_REQUIRE(p.mode == 0 || p.Cin % 4 == 0, "conv_gemm: Cin must be a multiple of 4");
    SMK_REQUIRE(!p.out2 || p.store != 1, "conv_gemm: the second store does not support the pixel-shuffle layout");
    SMK_REQUIRE(!conv_aff(p) || (p.store == 0 && p.N > 32 && (!p.scale2 || (p.bias2 && p.out2))),
                "conv_gemm: PReLU / second-store affine need store 0, N > 32, and scale2 with bias2 and out2");
    {
        const double cin_eff = p.mode == 0 ? p.K : p.Cin;       // unique input bytes (not im2col-expanded)
        const char* tag = p.tag ? p.tag : p.mode == 0 ? (p.store == 1 ? "upconv_gemm_f32" : "pw_gemm_f32") : "conv3x3_gemm_f32";
        if (g_prof_detail) tag = prof_shape_tag(tag, M, p.K, p.N);
        SMK_TAG(tag,
                4.0 * ((double)M * cin_eff + (double)p.K * p.N + (double)M * p.N * (1 + !!p.res + !!p.mask + !!p.out2) + 2.0 * p.N),
                2.0 * (double)M * p.N * p.K, st);
    }
    if (p.N <= 32) {
        dim3 grid(cdiv(M, 128), cdiv(p.N, 32));
        SMK_LAUNCH((conv_gemm_kernel<128, 32>), dim3(grid), dim3(NT), 0, st, p, M);
    } else {
        dim3 grid(cdiv(M, 64), cdiv(p.N, 64));
        if (conv_aff(p)) SMK_LAUNCH((conv_gemm_kernel<64, 64, true>), dim3(grid), dim3(NT), 0, st, p, M);
        else SMK_LAUNCH((conv_gemm_kernel<64, 64>), dim3(grid), dim3(NT), 0, st, p, M);
    }
    SMK_CHECK_LAUNCH();
    return 0;
}

int dwconv3x3(const float* in, int B, int H, int W, int C, int stride, const float* w9c, const float* scale,
              const float* bias, float* out, cudaStream_t st, bool round_out) {
    SMK_REQUIRE(C % 4 == 0, "dwconv3x3: C must be a multiple of 4");
    int Ho = (H + stride - 1) / stride, Wo = (W + stride - 1) / stride;
    SMK_REQUIRE(stride == 1 || stride == 2, "dwconv3x3: stride must be 1 or 2");
    long total = (long)B * Ho * ((Wo + 3) / 4) * (C / 4);
    int blocks = (int)std::min<long>((total + 255) / 256, 148L * 32);
    SMK_TAG(g_prof_detail ? prof_shape_tag("dwconv3x3", (long)B * Ho * Wo, stride, C) : "dwconv3x3", 4.0 * ((double)B * H * W * C + (double)B * Ho * Wo * C + 11.0 * C), 18.0 * B * Ho * Wo * C, st);
    if (stride == 1)
        SMK_LAUNCH((dwconv3x3_px4_kernel<1>), dim3(blocks), dim3(256), 0, st, in, B, H, W, C, same_pad_begin(H, 1), Ho, Wo, w9c, scale, bias, out, round_out ? 1 : 0);
    else
        SMK_LAUNCH((dwconv3x3_px4_kernel<2>), dim3(blocks), dim3(256), 0, st, in, B, H, W, C, same_pad_begin(H, 2), Ho, Wo, w9c, scale, bias, out, round_out ? 1 : 0);
    SMK_CHECK_LAUNCH();
    return 0;
}

int stem_conv(const float* img, int B, int H, int W, const StemProblem* probs, int n, cudaStream_t st) {
    SMK_REQUIRE(n >= 1 && n <= 3, "stem_conv: one to three backbones");
    const int Ho = (H + 1) / 2, Wo = (W + 1) / 2, pad = same_pad_begin(H, 2);
    if (n == 3) {
        Stem3 p;
        for (int g = 0; g < 3; ++g) { p.w[g] = probs[g].w; p.scale[g] = probs[g].scale; p.bias[g] = probs[g].bias; p.out[g] = probs[g].out; }
        SMK_TAG("stem_conv3", 4.0 * ((double)B * 3 * H * W + (double)B * Ho * Wo * 48 + 27 * 48 + 96), 2.0 * 27 * 48 * (double)B * Ho * Wo, st);
        SMK_REQUIRE(W % 4 == 0 && W + 8 <= STEM_MAXW && pad <= 1, "stem_conv: unsupported image width %d", W);
        SMK_LAUNCH(stem_conv3_kernel, dim3(B * Ho), dim3(128), 0, st, img, B, H, W, Ho, Wo, pad, p);
        SMK_CHECK_LAUNCH();
        return 0;
    }
    for (int g = 0; g < n; ++g) {
        const StemProblem& q = probs[g];
        SMK_TAG("stem_conv", 4.0 * ((double)B * 3 * H * W + (double)B * Ho * Wo * 16 + 27 * 16 + 32), 2.0 * 27 * 16 * (double)B * Ho * Wo, st);
        SMK_LAUNCH(stem_conv_kernel, dim3(cdiv((long)B * Ho * Wo, 128)), dim3(128), 0, st, img, B, H, W, Ho, Wo, pad, q.w, q.scale, q.bias, q.out);
        SMK_CHECK_LAUNCH();
    }
    return 0;
}

// ---- fused stem + first block --------------------------------------------------------------------------
// conv_stem 3x3 s2 (3 -> 16) + BN + ReLU  ->  block 0 of tf_mobilenetv3_*_minimal_100, a depthwise-separable
// block (depthwise 3x3 s{1,2} + BN + ReLU -> 1x1 16 -> 16 + BN, + skip when stride 1); reference
// src/smirk_encoder.py:7-12 -> timm MobileNetV3.conv_stem/bn1 + DepthwiseSeparableConv.  These are the three
// largest activations of a backbone (112 x 112 x 16).  One launch runs every backbone the handle holds (up to three,
// each with its own block-0 stride) from one pass over the image.  Persistent CTAs walk 16 x 16 tiles of the stem
// output; a tile's stem region carries a one-pixel halo on every side (18 x 18, stem rows / columns 16 t - 1 ...
// 16 t + 16), which covers the depthwise window of both strides (TF-SAME pads 1 before at stride 1, 0 at stride 2).
//   1. the 37 x 37 x 3 image patch of the NEXT tile is fetched by 4-byte cp.async into the other half of a double
//      buffer, rows and columns de-interleaved by parity (zero-filled outside the image), while this tile computes;
//   2. stem convs: thread = (backbone, 4 stem pixels (sy, sx) + {0, 9} x {0, 9}) x 16 channels, 81 threads per
//      backbone, BN + ReLU, zero outside the 112 x 112 map (= the depthwise conv's zero padding) -> S (one per backbone);
//   3. per backbone: depthwise 3x3 over S: thread = (pixel, channel quad), taps in registers, BN + ReLU -> D (aliases
//      the consumed patch);
//   4. 1x1 conv on D: thread = (pixel, output-channel quad), BN, + S (skip), optional TF32 rounding, one coalesced
//      16-byte store per thread.
// All arithmetic is fp32 FMA in the reference's tap order; the image is the only HBM read, the block outputs the only
// writes.
namespace {
constexpr int SD_T = 16, SD_ST = SD_T + 2;                 // stem-resolution tile edge, with halo
constexpr int SD_PR = 2 * SD_ST + 1;                       // image patch rows / cols (37)
// Patch word of (channel c, row r, column x): [c][r & 1][r >> 1][x & 1][x >> 1], column-parity pitch SD_PC, row pitch
// SD_PU.  SD_PU = 9 (mod 32): the quarter-grid pixel j = 9 sy + sx of a stem thread reads word SD_PU sy + sx + const,
// so a warp's 32 threads of one backbone hit 32 consecutive banks on every tap.
constexpr int SD_PC = 20, SD_PU = 41, SD_PH = (SD_PR + 1) / 2;
constexpr int SD_PATCH = (3 * 2 * SD_PH * SD_PU + 3) / 4 * 4;  // floats per patch buffer (16-byte multiple: D is float4)
constexpr int SD_STILE = SD_ST * SD_ST * 16;               // floats of one backbone's stem tile
constexpr int SD_WK = 9 * 16 + 16 * 16;                    // depthwise taps + 1x1 weights of one backbone
constexpr int SD_Q = SD_ST / 2;                            // stem threads per backbone: SD_Q x SD_Q, 4 pixels each
constexpr int SD_SMEM = 4 * (2 * SD_PATCH + 3 * (SD_STILE + 27 * 16 + SD_WK + 6 * 16));
static_assert(2 * (SD_SMEM + 1024) <= 228 * 1024, "stem_ds: shared memory of two resident CTAs");
static_assert(SD_PC >= SD_PH && SD_PU >= SD_PC + SD_PH && SD_PU % 32 == SD_Q, "stem_ds: patch layout");
static_assert(16 * 16 * 16 <= SD_PATCH && 3 * SD_Q * SD_Q <= 256, "stem_ds: D fits a patch buffer; one stem pass");

struct StemDs { StemDsProblem q[3]; int n, round_out; };

__device__ __forceinline__ int sd_patch_idx(int c, int r, int x) {
    return ((c * 2 + (r & 1)) * SD_PH + (r >> 1)) * SD_PU + (x & 1) * SD_PC + (x >> 1);
}
__device__ __forceinline__ void cp_async4(float* dst, const float* src, int src_bytes) {   // src_bytes 0: zero fill
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;\n" ::"r"((unsigned)__cvta_generic_to_shared(dst)), "l"(src),
                 "r"(src_bytes) : "memory");
}

// Steps 3 and 4 for one backbone.  S: its stem tile, K / Bv: its taps, weights, scales and biases, D: scratch.
template <int STRIDE, bool SAVE>
__device__ __forceinline__ void sd_block(const StemDsProblem& p, const float* S, const float* K, const float* Bv, float* D,
                                         int b, int ty, int tx, int Hs, int Ws, int round_out) {
    constexpr int TO = SD_T / STRIDE, NJ = TO * TO / 64;  // output tile edge, pixels per thread
    constexpr int O = STRIDE - 1;                         // local stem row / column of the depthwise window's first tap
    const int tid = threadIdx.x, q = tid & 3;
    const int Ho = Hs / STRIDE, Wo = Ws / STRIDE;
    __syncthreads();                                      // S complete; D's previous readers done
    {
        float4 k[9];
#pragma unroll
        for (int t = 0; t < 9; ++t) k[t] = *reinterpret_cast<const float4*>(K + t * 16 + 4 * q);
        const float4 sc = *reinterpret_cast<const float4*>(Bv + 32 + 4 * q), bi = *reinterpret_cast<const float4*>(Bv + 48 + 4 * q);
#pragma unroll
        for (int j = 0; j < NJ; ++j) {
            const int px = (tid >> 2) + 64 * j, oy = px / TO, ox = px - oy * TO;
            const float* s = S + ((oy * STRIDE + O) * SD_ST + ox * STRIDE + O) * 16 + 4 * q;
            float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
            for (int ky = 0; ky < 3; ++ky)
#pragma unroll
                for (int kx = 0; kx < 3; ++kx)
                    fma4_acc(acc, *reinterpret_cast<const float4*>(s + (ky * SD_ST + kx) * 16), k[ky * 3 + kx]);
            float4 o = fma4(acc, sc, bi);
            o.x = fmaxf(o.x, 0.f); o.y = fmaxf(o.y, 0.f); o.z = fmaxf(o.z, 0.f); o.w = fmaxf(o.w, 0.f);
            *reinterpret_cast<float4*>(D + px * 16 + 4 * q) = o;
            if (SAVE)
                *reinterpret_cast<float4*>(p.d_out + (((size_t)b * Ho + ty * TO + oy) * Wo + tx * TO + ox) * 16 + 4 * q) = o;
        }
    }
    __syncthreads();
    {
        const float4 sc = *reinterpret_cast<const float4*>(Bv + 64 + 4 * q), bi = *reinterpret_cast<const float4*>(Bv + 80 + 4 * q);
        float4 accs[NJ];
#pragma unroll
        for (int j = 0; j < NJ; ++j) accs[j] = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int g = 0; g < 4; ++g) {                      // four input channels at a time: their weights serve all NJ pixels
            float4 w[4];
#pragma unroll
            for (int ci = 0; ci < 4; ++ci) w[ci] = *reinterpret_cast<const float4*>(K + 9 * 16 + (4 * g + ci) * 16 + 4 * q);
#pragma unroll
            for (int j = 0; j < NJ; ++j) {
                const float4 d = *reinterpret_cast<const float4*>(D + ((tid >> 2) + 64 * j) * 16 + 4 * g);
                fma4_s(accs[j], d.x, w[0]); fma4_s(accs[j], d.y, w[1]); fma4_s(accs[j], d.z, w[2]); fma4_s(accs[j], d.w, w[3]);
            }
        }
#pragma unroll
        for (int j = 0; j < NJ; ++j) {
            const int px = (tid >> 2) + 64 * j, oy = px / TO, ox = px - oy * TO;
            float4 o = fma4(accs[j], sc, bi);
            if (STRIDE == 1) {                             // skip connection: block input = stem output at the same pixel
                const float4 r = *reinterpret_cast<const float4*>(S + ((oy + 1) * SD_ST + ox + 1) * 16 + 4 * q);
                o.x += r.x; o.y += r.y; o.z += r.z; o.w += r.w;
            }
            if (round_out) { o.x = round_tf32(o.x); o.y = round_tf32(o.y); o.z = round_tf32(o.z); o.w = round_tf32(o.w); }
            *reinterpret_cast<float4*>(p.out + (((size_t)b * Ho + ty * TO + oy) * Wo + tx * TO + ox) * 16 + 4 * q) = o;
        }
    }
}

// SAVE: also store the stem output of the tile's own 16 x 16 pixels (s_out) and the depthwise output (d_out), the ReLU
// outputs the backward masks with.
template <bool SAVE>
__global__ void __launch_bounds__(256, 2)
stem_ds_kernel(const float* __restrict__ img, int H, int W, int Hs, int Ws, int pad, int n_tiles, const __grid_constant__ StemDs pp) {
    extern __shared__ __align__(16) float sd_smem[];
    float* sP = sd_smem;                                   // [2][SD_PATCH] image patches; the consumed one is D
    float* sS = sP + 2 * SD_PATCH;                         // [3][SD_ST * SD_ST][16] stem tiles
    float* sW = sS + 3 * SD_STILE;                         // [3][27][16] stem weights
    float* sK = sW + 3 * 27 * 16;                          // [3][SD_WK] depthwise taps, 1x1 weights [ci][co]
    float* sB = sK + 3 * SD_WK;                            // [3][6][16] stem / dw / pw scale, bias
    const int tid = threadIdx.x, n = pp.n;
    for (int g = 0; g < n; ++g) {
        const StemDsProblem& p = pp.q[g];
        for (int i = tid; i < 27 * 16; i += 256) sW[g * 27 * 16 + i] = p.stem_w[i];
        for (int i = tid; i < 9 * 16; i += 256) sK[g * SD_WK + i] = p.dw_w[i];
        sK[g * SD_WK + 9 * 16 + tid] = p.pw_w[tid];
        if (tid < 16) {
            float* B6 = sB + g * 96;
            B6[tid] = p.stem_s[tid]; B6[16 + tid] = p.stem_b[tid]; B6[32 + tid] = p.dw_s[tid]; B6[48 + tid] = p.dw_b[tid];
            B6[64 + tid] = p.pw_s[tid]; B6[80 + tid] = p.pw_b[tid];
        }
    }
    const int tiles_x = Ws / SD_T, tiles_img = (Hs / SD_T) * tiles_x;
    auto stage = [&](int t, float* dst) {                  // issue the patch of tile t (one cp.async group)
        const int b = t / tiles_img, r = t - b * tiles_img, ty = r / tiles_x, tx = r - ty * tiles_x;
        const int iy0 = 2 * (ty * SD_T - 1) - pad, ix0 = 2 * (tx * SD_T - 1) - pad;
        for (int i = tid; i < 3 * SD_PR * SD_PR; i += 256) {
            const int row = i / SD_PR, x = i - row * SD_PR, c = row / SD_PR, y = row - c * SD_PR;
            const int iy = iy0 + y, ix = ix0 + x;
            const bool in = iy >= 0 && iy < H && ix >= 0 && ix < W;
            cp_async4(dst + sd_patch_idx(c, y, x), in ? img + (((size_t)b * 3 + c) * H + iy) * W + ix : img, in ? 4 : 0);
        }
        asm volatile("cp.async.commit_group;\n" ::: "memory");
    };
    int buf = 0;
    if ((int)blockIdx.x < n_tiles) stage(blockIdx.x, sP);
    for (int t = blockIdx.x; t < n_tiles; t += gridDim.x, buf ^= 1) {
        const int b = t / tiles_img, r = t - b * tiles_img, ty = r / tiles_x, tx = r - ty * tiles_x;
        const int sy0 = ty * SD_T - 1, sx0 = tx * SD_T - 1;          // stem-tile origin
        float* P = sP + buf * SD_PATCH;
        asm volatile("cp.async.wait_group 0;\n" ::: "memory");
        __syncthreads();                                   // this tile's patch landed; the previous tile is done with S / D
        if (t + (int)gridDim.x < n_tiles) stage(t + gridDim.x, sP + (buf ^ 1) * SD_PATCH);
        // -- 2. stem convs
        if (tid < n * SD_Q * SD_Q) {
            const int g = tid / (SD_Q * SD_Q), j = tid - g * (SD_Q * SD_Q), sy = j / SD_Q, sx = j - sy * SD_Q;
            const float* Wg = sW + g * 27 * 16;
            float4 a[4][4];                                // [pixel (dy, dx) = (a >> 1, a & 1) * SD_Q][channel quad]
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int qq = 0; qq < 4; ++qq) a[i][qq] = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
            for (int c = 0; c < 3; ++c)
#pragma unroll
                for (int ky = 0; ky < 3; ++ky)
#pragma unroll
                    for (int kx = 0; kx < 3; ++kx) {
                        const float* x0 = P + sd_patch_idx(c, 2 * sy + ky, 2 * sx + kx);
                        float x[4];
#pragma unroll
                        for (int i = 0; i < 4; ++i) x[i] = x0[(i >> 1) * SD_Q * SD_PU + (i & 1) * SD_Q];
                        const float4* wk = reinterpret_cast<const float4*>(Wg + ((c * 3 + ky) * 3 + kx) * 16);
#pragma unroll
                        for (int qq = 0; qq < 4; ++qq) {
                            const float4 w4 = wk[qq];
#pragma unroll
                            for (int i = 0; i < 4; ++i) fma4_s(a[i][qq], x[i], w4);
                        }
                    }
            const float* Bg = sB + g * 96;
            float* Sg = sS + g * SD_STILE;
            float* s_out = SAVE ? pp.q[g].s_out : nullptr;
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int ly = sy + (i >> 1) * SD_Q, lx = sx + (i & 1) * SD_Q;           // local stem pixel
                const int gy = sy0 + ly, gx = sx0 + lx;
                const bool v = gy >= 0 && gy < Hs && gx >= 0 && gx < Ws;
                const bool own = ly >= 1 && ly <= SD_T && lx >= 1 && lx <= SD_T;
#pragma unroll
                for (int qq = 0; qq < 4; ++qq) {
                    const float4 sc = *reinterpret_cast<const float4*>(Bg + 4 * qq), bi = *reinterpret_cast<const float4*>(Bg + 16 + 4 * qq);
                    float4 o = fma4(a[i][qq], sc, bi);
                    o.x = v ? fmaxf(o.x, 0.f) : 0.f; o.y = v ? fmaxf(o.y, 0.f) : 0.f; o.z = v ? fmaxf(o.z, 0.f) : 0.f; o.w = v ? fmaxf(o.w, 0.f) : 0.f;
                    reinterpret_cast<float4*>(Sg + (ly * SD_ST + lx) * 16)[qq] = o;
                    if (SAVE && own) reinterpret_cast<float4*>(s_out + (((size_t)b * Hs + gy) * Ws + gx) * 16)[qq] = o;
                }
            }
        }
        // -- 3, 4. depthwise + 1x1 per backbone
        for (int g = 0; g < n; ++g) {
            if (pp.q[g].stride == 1)
                sd_block<1, SAVE>(pp.q[g], sS + g * SD_STILE, sK + g * SD_WK, sB + g * 96, P, b, ty, tx, Hs, Ws, pp.round_out);
            else
                sd_block<2, SAVE>(pp.q[g], sS + g * SD_STILE, sK + g * SD_WK, sB + g * 96, P, b, ty, tx, Hs, Ws, pp.round_out);
        }
    }
}
}  // namespace

int stem_ds(const float* img, int B, int H, int W, const StemDsProblem* probs, int n, int round_out, cudaStream_t st) {
    const int Hs = (H + 1) / 2, Ws = (W + 1) / 2;
    SMK_REQUIRE(n >= 1 && n <= 3, "stem_ds: one to three backbones per launch");
    SMK_REQUIRE(H % 2 == 0 && W % 2 == 0 && Hs % SD_T == 0 && Ws % SD_T == 0, "stem_ds: image size %dx%d must be a multiple of 32", H, W);
    const bool save = probs[0].s_out != nullptr;
    StemDs p{};
    double bytes = 4.0 * B * 3 * H * W, flops = 0;
    for (int k = 0; k < n; ++k) {
        const StemDsProblem& q = probs[k];
        SMK_REQUIRE(q.stride == 1 || q.stride == 2, "stem_ds: stride must be 1 or 2");
        SMK_REQUIRE(!q.s_out == !save && !q.d_out == !save, "stem_ds: s_out and d_out are given together, for every problem or none");
        p.q[k] = q;
        const double px_o = (double)B * (Hs / q.stride) * (Ws / q.stride);
        bytes += 4.0 * (px_o * 16 + 27 * 16 + 9 * 16 + 256 + 96);
        flops += 2.0 * ((double)B * Hs * Ws * 16 * 27 + px_o * 16 * (9 + 16));
    }
    p.n = n; p.round_out = round_out;
    const int n_tiles = B * (Hs / SD_T) * (Ws / SD_T);
    SMK_CHECK_CUDA(set_max_dynamic_smem<stem_ds_kernel<true>>(SD_SMEM));
    SMK_CHECK_CUDA(set_max_dynamic_smem<stem_ds_kernel<false>>(SD_SMEM));
    SMK_TAG("stem_ds_fused", bytes, flops, st);
    const dim3 grid((unsigned)std::min(n_tiles, 2 * num_sms()));
    if (save) SMK_LAUNCH(stem_ds_kernel<true>, grid, dim3(256), SD_SMEM, st, img, H, W, Hs, Ws, same_pad_begin(H, 2), n_tiles, p);
    else SMK_LAUNCH(stem_ds_kernel<false>, grid, dim3(256), SD_SMEM, st, img, H, W, Hs, Ws, same_pad_begin(H, 2), n_tiles, p);
    SMK_CHECK_LAUNCH();
    return 0;
}

int maxpool2x2(const float* in, int ld_in, int B, int H, int W, int C, float* out, cudaStream_t st) {
    long total = (long)B * (H / 2) * (W / 2) * (C / 4);
    int blocks = (int)std::min<long>((total + 255) / 256, 148L * 16);
    SMK_TAG("maxpool2x2", 4.0 * 1.25 * (double)B * H * W * C, 0.0, st);
    SMK_LAUNCH(maxpool2x2_kernel, dim3(blocks), dim3(256), 0, st, in, ld_in, B, H, W, C, out);
    SMK_CHECK_LAUNCH();
    return 0;
}

int nchw_to_nhwc_pad(const float* in, int B, int C, int H, int W, int Cp, float* out, cudaStream_t st, bool round_out) {
    SMK_REQUIRE(Cp % 4 == 0 && Cp >= C, "nchw_to_nhwc_pad: padded channel count must be a multiple of 4 and >= C");
    SMK_TAG("nchw_to_nhwc", 4.0 * (double)B * H * W * (C + Cp), 0.0, st);
    SMK_LAUNCH(nchw_to_nhwc_pad_kernel, dim3(cdiv((long)B * H * W * (Cp / 4), 256)), dim3(256), 0, st, in, B, C, H * W, Cp, round_out ? 1 : 0, out);
    SMK_CHECK_LAUNCH();
    return 0;
}

int conv1x1_sigmoid_nchw(const float* in, int B, int HW, int Cin, const float* w, const float* bias, int Cout, float* out,
                         cudaStream_t st) {
    SMK_REQUIRE(Cout <= 4 && Cin % 4 == 0, "conv1x1_sigmoid_nchw: Cout <= 4 and Cin %% 4 == 0 required");
    size_t smem = (size_t)(Cin * Cout + Cout) * 4;
    SMK_TAG("conv1x1_sigmoid", 4.0 * (double)B * HW * (Cin + Cout), 2.0 * (double)B * HW * Cin * Cout, st);
    SMK_LAUNCH(conv1x1_sigmoid_kernel, dim3(cdiv((long)B * HW, 256)), dim3(256), smem, st, in, B, HW, Cin, w, bias, Cout, out);
    SMK_CHECK_LAUNCH();
    return 0;
}

int gap_head(const GapHeadProblem* probs, int n, int B, int HW, int C, cudaStream_t st) {
    SMK_REQUIRE(n == 1 || n == 2, "gap_head: one or two backbones per launch");
    SMK_REQUIRE((size_t)C * 4 <= 48 * 1024, "gap_head: feature width too large for the shared-memory pool");
    GapHead g{};
    int max_out = 0;
    const bool save = probs[0].raw != nullptr;
    SMK_REQUIRE(!probs[n - 1].raw == !save, "gap_head: raw is given for every problem or none");
    for (int k = 0; k < 2; ++k) {
        const GapHeadProblem& q = probs[k < n ? k : n - 1];
        g.feat[k] = q.feat; g.w[k] = q.w; g.bias[k] = q.bias; g.codes[k] = q.codes; g.out[k] = q.out; g.n_out[k] = q.n_out; g.raw[k] = q.raw;
        max_out = std::max(max_out, q.n_out);
    }
    double by = 0, fl = 0;
    for (int k = 0; k < n; ++k) { by += 4.0 * ((double)B * HW * C + (double)probs[k].n_out * C + (double)B * probs[k].n_out); fl += (double)B * C * HW + 2.0 * B * C * probs[k].n_out; }
    SMK_TAG("gap_head", by, fl, st);
    if (save) SMK_LAUNCH(gap_head_kernel<true>, dim3(B, cdiv(max_out, 32), n), dim3(256), (size_t)C * 4, st, g, HW, C);
    else SMK_LAUNCH(gap_head_kernel<false>, dim3(B, cdiv(max_out, 32), n), dim3(256), (size_t)C * 4, st, g, HW, C);
    SMK_CHECK_LAUNCH();
    return 0;
}

}  // namespace smk

extern "C" int smk_debug_conv_f32(const float* in, int ld_in, int B, int H, int W, int Cin, const float* w_kn, const float* scale,
                                  const float* bias, int N, int K, int mode, int relu, const float* res, int ld_res,
                                  float* out, int ld_out, int shuffle, void* stream) {
    smk::Conv p{};
    p.in = in; p.ld_in = ld_in; p.B = B; p.H = H; p.W = W; p.Cin = Cin; p.wgt = smk::GemmW{w_kn, nullptr, nullptr}; p.scale = scale; p.bias = bias; p.N = N; p.K = K;
    p.mode = mode; p.relu = relu; p.res = res; p.ld_res = ld_res; p.out = out; p.ld_out = ld_out; p.store = shuffle;
    return smk::conv_gemm(p, (cudaStream_t)stream);
}

extern "C" int smk_debug_stem_ds(const float* img, int B, int H, int W, const float* stem_w, const float* stem_s, const float* stem_b,
                                 const float* dw_w, const float* dw_s, const float* dw_b, const float* pw_w, const float* pw_s,
                                 const float* pw_b, int stride, int round_out, float* out, void* stream) {
    if (B == 0) return 0;
    SMK_REQUIRE(img && stem_w && stem_s && stem_b && dw_w && dw_s && dw_b && pw_w && pw_s && pw_b && out, "smk_debug_stem_ds: null argument");
    const smk::StemDsProblem q{stem_w, stem_s, stem_b, dw_w, dw_s, dw_b, pw_w, pw_s, pw_b, out, nullptr, nullptr, stride};
    return smk::stem_ds(img, B, H, W, &q, 1, round_out, (cudaStream_t)stream);
}
