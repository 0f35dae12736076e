// SmirkEncoder in train mode: BatchNorm over batch statistics (with the running-statistics update) and the weight, BN and
// head gradients, for the reference trainer's encoder steps (src/smirk_trainer.py:34-73 with base_trainer.py:108-111's
// .train()).
//
// A train handle holds the topology only; every call reads the module's current parameters through device pointers
// (SmkEncoderTrainArgs) and repacks the 1x1 weights into the workspace, so an optimizer step needs no new handle.  The
// forward runs the unfused layer sequence (BN cannot be folded): per conv the pre-BN output z, then per BatchNorm a
// per-channel reduction over fixed pixel chunks (fp64 partial sums), a one-CTA finalise (mean, invstd, running stats,
// num_batches_tracked), and an apply step (gamma * xhat + beta, + skip, ReLU).  The backward walks each backbone in
// reverse: BN backward (fixed-order fp64 sums of g and g * xhat, then g_z), 1x1 dgrads through smk::conv over W^T, a
// depthwise transposed conv, and weight gradients as split-K reductions over fixed pixel chunks with a fixed-order
// reduce.  No atomics: results are bitwise reproducible, and every call is CUDA-graph capturable.
#include "encoder.cuh"
#include "nn_kernels.cuh"
#include "gemm_tc.cuh"
#include <string>

namespace {

using namespace enc;
using smk::cdiv;
using smk::grid_of;
using smk::same_pad_begin;

constexpr int kMaxChunks = 512;            // BN reductions: at most this many pixel chunks per layer
constexpr size_t kWgradPart = 1u << 22;    // floats of split-K partials of one weight gradient (see wgrad_chunks)

// Pixel chunks of a per-channel reduction over M pixels: a function of M only, so the summation order is fixed.
int bn_chunks(long M) { return (int)std::min<long>(cdiv(M, 256), kMaxChunks); }

// ---- forward layers (raw weights in torch layout, no BN) -------------------------------------------------------------

// Stem conv 3x3 stride 2 TF-SAME, 3 -> 16: img NCHW -> z [B,Ho,Wo,16].  w: torch [16][3][3][3].  Thread = output pixel.
__global__ void __launch_bounds__(128)
stem_fwd_kernel(const float* __restrict__ img, const float* __restrict__ w, int B, int H, int W, int Ho, int Wo, int pad, float* __restrict__ z) {
    __shared__ float sw[27][16];
    for (int i = threadIdx.x; i < 27 * 16; i += blockDim.x) sw[i % 27][i / 27] = w[i];
    __syncthreads();
    const long pix = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (pix >= (long)B * Ho * Wo) return;
    const int ow = (int)(pix % Wo); const long t = pix / Wo; const int oh = (int)(t % Ho); const int b = (int)(t / Ho);
    float acc[16];
#pragma unroll
    for (int o = 0; o < 16; ++o) acc[o] = 0.f;
#pragma unroll
    for (int c = 0; c < 3; ++c)
#pragma unroll
        for (int ky = 0; ky < 3; ++ky)
#pragma unroll
            for (int kx = 0; kx < 3; ++kx) {           // out-of-image taps read as zero (fmaf(0, w, acc) == acc)
                const int iy = oh * 2 + ky - pad, ix = ow * 2 + kx - pad;
                const bool in = iy >= 0 && iy < H && ix >= 0 && ix < W;
                const float v = in ? __ldg(img + (((size_t)b * 3 + c) * H + iy) * W + ix) : 0.f;
                const float* wk = sw[(c * 3 + ky) * 3 + kx];
#pragma unroll
                for (int o = 0; o < 16; ++o) acc[o] = fmaf(v, wk[o], acc[o]);
            }
    float4* out = reinterpret_cast<float4*>(z + pix * 16);
#pragma unroll
    for (int v = 0; v < 4; ++v) out[v] = make_float4(acc[4 * v], acc[4 * v + 1], acc[4 * v + 2], acc[4 * v + 3]);
}

// Depthwise 3x3 TF-SAME: a [B,H,W,C] -> z [B,Ho,Wo,C].  w: torch [C][1][3][3].  Thread = output element.
template <int S>
__global__ void __launch_bounds__(256)
dw_fwd_kernel(const float* __restrict__ a, const float* __restrict__ w, int B, int H, int W, int C, int Ho, int Wo, int pad, float* __restrict__ z) {
    const long total = (long)B * Ho * Wo * C;
    for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        const int c = (int)(i % C); const long pix = i / C;
        const int ow = (int)(pix % Wo); const long t = pix / Wo; const int oh = (int)(t % Ho); const int b = (int)(t / Ho);
        const float* wc = w + (size_t)c * 9;
        float acc = 0.f;
#pragma unroll
        for (int ky = 0; ky < 3; ++ky) {
            const int iy = oh * S + ky - pad;
            if (iy < 0 || iy >= H) continue;
#pragma unroll
            for (int kx = 0; kx < 3; ++kx) {
                const int ix = ow * S + kx - pad;
                if (ix < 0 || ix >= W) continue;
                acc = fmaf(__ldg(a + (((size_t)b * H + iy) * W + ix) * C + c), __ldg(wc + ky * 3 + kx), acc);
            }
        }
        z[i] = acc;
    }
}

// ---- BatchNorm ---------------------------------------------------------------------------------------------------------

// Per-channel partial sums over the pixel chunk blockIdx.y of [M, C] tensors, CTA = (32 channels, 8 pixel rows):
//   BWD = 0: (sum z, sum z^2);  BWD = 1: (sum g', sum g' * xhat), g' = g * [y > 0] (y null: no ReLU), xhat = (z - mean) * invstd.
// The 8 rows are summed in fixed order; part[chunk][c].
template <int BWD>
__global__ void __launch_bounds__(256)
bn_reduce_kernel(const float* __restrict__ z, const float* __restrict__ g, const float* __restrict__ y, const float* __restrict__ mean,
                 const float* __restrict__ invstd, long M, int C, long chunk, double2* __restrict__ part) {
    __shared__ double2 red[8][32];
    const int c = blockIdx.x * 32 + threadIdx.x;
    const long p0 = blockIdx.y * chunk, p1 = min(M, p0 + chunk);
    double s0 = 0.0, s1 = 0.0;
    if (c < C) {
        const float mu = BWD ? mean[c] : 0.f, is = BWD ? invstd[c] : 0.f;
        for (long p = p0 + threadIdx.y; p < p1; p += 8) {
            const size_t i = (size_t)p * C + c;
            const float v = __ldg(z + i);
            if (BWD) {
                float gv = __ldg(g + i);
                if (y && !(__ldg(y + i) > 0.f)) gv = 0.f;
                const float xh = (v - mu) * is;
                s0 += gv; s1 += (double)gv * xh;
            } else {
                s0 += v; s1 += (double)v * v;
            }
        }
    }
    red[threadIdx.y][threadIdx.x] = make_double2(s0, s1);
    __syncthreads();
    if (threadIdx.y == 0 && c < C) {
        double2 r = red[0][threadIdx.x];
        for (int k = 1; k < 8; ++k) { r.x += red[k][threadIdx.x].x; r.y += red[k][threadIdx.x].y; }
        part[(size_t)blockIdx.y * C + c] = r;
    }
}

// Forward finalise, one CTA: batch mean and biased variance -> mean, invstd; running_mean / running_var (unbiased) with
// factor momentum, or 1 / num_batches_tracked when momentum < 0 (torch's momentum=None); num_batches_tracked += 1.
__global__ void __launch_bounds__(256)
bn_finalize_fwd_kernel(const double2* __restrict__ part, int n_chunks, long M, int C, float eps, float momentum,
                       float* __restrict__ rmean, float* __restrict__ rvar, long long* __restrict__ nbt, float* __restrict__ mean, float* __restrict__ invstd) {
    __shared__ long long count;
    if (threadIdx.x == 0) count = *nbt + 1;
    __syncthreads();
    const float f = momentum < 0.f ? (float)(1.0 / (double)count) : momentum;
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
        double s = 0.0, ss = 0.0;
        for (int k = 0; k < n_chunks; ++k) { const double2 v = part[(size_t)k * C + c]; s += v.x; ss += v.y; }
        const double mu = s / (double)M;
        const double var = fmax(ss / (double)M - mu * mu, 0.0);
        mean[c] = (float)mu;
        invstd[c] = (float)(1.0 / sqrt(var + (double)eps));
        const float unbiased = (float)(M > 1 ? var * (double)M / (double)(M - 1) : var);
        rmean[c] = (1.f - f) * rmean[c] + f * (float)mu;
        rvar[c] = (1.f - f) * rvar[c] + f * unbiased;
    }
    __syncthreads();
    if (threadIdx.x == 0) *nbt = count;
}

// y = gamma * (z - mean) * invstd + beta (+ res) (ReLU) (TF32 rounding for a tensor-core consumer), [M, C], C % 4 == 0.
__global__ void __launch_bounds__(256)
bn_apply_kernel(const float* __restrict__ z, const float* __restrict__ mean, const float* __restrict__ invstd, const float* __restrict__ gamma,
                const float* __restrict__ beta, const float* __restrict__ res, long M, int C, int relu, int round, float* __restrict__ y) {
    const int C4 = C >> 2;
    const long total = M * C4;
    for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        const int c = (int)(i % C4) * 4;
        const float4 v = __ldg(reinterpret_cast<const float4*>(z) + i);
        float o[4] = {v.x, v.y, v.z, v.w};
        float4 r = res ? __ldg(reinterpret_cast<const float4*>(res) + i) : make_float4(0.f, 0.f, 0.f, 0.f);
        const float rr[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            float t = (o[k] - mean[c + k]) * invstd[c + k] * gamma[c + k] + beta[c + k];
            if (res) t += rr[k];
            if (relu) t = fmaxf(t, 0.f);
            o[k] = round ? smk::round_tf32(t) : t;
        }
        reinterpret_cast<float4*>(y)[i] = make_float4(o[0], o[1], o[2], o[3]);
    }
}

// Backward finalise, one CTA: g_beta = sum g', g_gamma = sum g' * xhat (fixed order over the chunks) into gb[0..C) and
// gb[C..2C), and into the caller's gradients when given.
__global__ void __launch_bounds__(256)
bn_finalize_bwd_kernel(const double2* __restrict__ part, int n_chunks, int C, float* __restrict__ gb, float* __restrict__ g_gamma, float* __restrict__ g_beta) {
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
        double s = 0.0, sx = 0.0;
        for (int k = 0; k < n_chunks; ++k) { const double2 v = part[(size_t)k * C + c]; s += v.x; sx += v.y; }
        gb[c] = (float)s; gb[C + c] = (float)sx;
        if (g_beta) g_beta[c] = (float)s;
        if (g_gamma) g_gamma[c] = (float)sx;
    }
}

// g_z = gamma * invstd * (g' - g_beta / M - xhat * g_gamma / M), g' = g * [y > 0] (y null: no ReLU).  g_z may alias g.
__global__ void __launch_bounds__(256)
bn_bwd_apply_kernel(const float* g, const float* __restrict__ y, const float* __restrict__ z, const float* __restrict__ mean,
                    const float* __restrict__ invstd, const float* __restrict__ gamma, const float* __restrict__ gb, long M, int C, int round, float* gz) {
    const long total = M * C;
    const float inv_m = 1.f / (float)M;
    for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        const int c = (int)(i % C);
        float gv = g[i];
        if (y && !(__ldg(y + i) > 0.f)) gv = 0.f;
        const float xh = (__ldg(z + i) - mean[c]) * invstd[c];
        const float t = gamma[c] * invstd[c] * (gv - gb[c] * inv_m - xh * (gb[C + c] * inv_m));
        gz[i] = round ? smk::round_tf32(t) : t;
    }
}

// ---- weight gradients -------------------------------------------------------------------------------------------------

// 1x1 weight gradient, split K: part[chunk][co][ci] = sum over the chunk's pixels p of g[p][co] * a[p][ci].
// 64 x 64 output tile per CTA, 16 pixels per step, 4 x 4 outputs per thread (fp32 CUDA cores).
__global__ void __launch_bounds__(256)
pw_wgrad_kernel(const float* __restrict__ g, const float* __restrict__ a, long M, int Co, int Ci, long chunk, float* __restrict__ part) {
    __shared__ float gs[16][64], as[16][64];
    const int ci0 = blockIdx.x * 64, co0 = blockIdx.y * 64, tid = threadIdx.x;
    const int tx = tid % 16, ty = tid / 16;
    const long p0 = blockIdx.z * chunk, p1 = min(M, p0 + chunk);
    float acc[4][4] = {};
    for (long pb = p0; pb < p1; pb += 16) {
#pragma unroll
        for (int r = 0; r < 4; ++r) {
            const int e = tid + 256 * r, row = e / 64, col = e % 64;
            const long p = pb + row;
            const bool ok = p < p1;
            gs[row][col] = ok && co0 + col < Co ? __ldg(g + (size_t)p * Co + co0 + col) : 0.f;
            as[row][col] = ok && ci0 + col < Ci ? __ldg(a + (size_t)p * Ci + ci0 + col) : 0.f;
        }
        __syncthreads();
#pragma unroll
        for (int k = 0; k < 16; ++k) {
            float gv[4], av[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) { gv[j] = gs[k][ty * 4 + j]; av[j] = as[k][tx * 4 + j]; }
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(gv[i], av[j], acc[i][j]);
        }
        __syncthreads();
    }
    float* out = part + (size_t)blockIdx.z * Co * Ci;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int co = co0 + ty * 4 + i;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int ci = ci0 + tx * 4 + j;
            if (co < Co && ci < Ci) out[(size_t)co * Ci + ci] = acc[i][j];
        }
    }
}

// Depthwise weight gradient: part[chunk][c][tap] = sum over the chunk's output pixels of g[p][c] * a[input of tap][c].
// CTA = (32 channels, 8 pixel rows); the rows are summed in fixed order.
template <int S>
__global__ void __launch_bounds__(256)
dw_wgrad_kernel(const float* __restrict__ g, const float* __restrict__ a, int B, int H, int W, int C, int Ho, int Wo, int pad, long chunk,
                float* __restrict__ part) {
    __shared__ float red[8][32][9];
    const int c = blockIdx.x * 32 + threadIdx.x;
    const long M = (long)B * Ho * Wo, p0 = blockIdx.y * chunk, p1 = min(M, p0 + chunk);
    float acc[9] = {};
    if (c < C) {
        for (long p = p0 + threadIdx.y; p < p1; p += 8) {
            const int ow = (int)(p % Wo); const long t = p / Wo; const int oh = (int)(t % Ho); const int b = (int)(t / Ho);
            const float gv = __ldg(g + (size_t)p * C + c);
#pragma unroll
            for (int ky = 0; ky < 3; ++ky) {
                const int iy = oh * S + ky - pad;
                if (iy < 0 || iy >= H) continue;
#pragma unroll
                for (int kx = 0; kx < 3; ++kx) {
                    const int ix = ow * S + kx - pad;
                    if (ix < 0 || ix >= W) continue;
                    acc[ky * 3 + kx] = fmaf(gv, __ldg(a + (((size_t)b * H + iy) * W + ix) * C + c), acc[ky * 3 + kx]);
                }
            }
        }
    }
#pragma unroll
    for (int k = 0; k < 9; ++k) red[threadIdx.y][threadIdx.x][k] = acc[k];
    __syncthreads();
    if (threadIdx.y == 0 && c < C) {
        for (int k = 0; k < 9; ++k) {
            float s = red[0][threadIdx.x][k];
            for (int r = 1; r < 8; ++r) s += red[r][threadIdx.x][k];
            part[((size_t)blockIdx.y * C + c) * 9 + k] = s;
        }
    }
}

// Stem weight gradient: part[chunk][o][k] (k = (c*3 + ky)*3 + kx, torch's [16][3][3][3]) = sum over the chunk's output
// pixels of g[p][o] * img[b, c, iy, ix].  32 pixels per step staged in shared memory; thread = one of the 432 weights.
__global__ void __launch_bounds__(448)
stem_wgrad_kernel(const float* __restrict__ g, const float* __restrict__ img, int B, int H, int W, int Ho, int Wo, int pad, long chunk,
                  float* __restrict__ part) {
    __shared__ float gs[32][16], xs[32][27];
    const int t = threadIdx.x, o = t / 27, k = t % 27;
    const long M = (long)B * Ho * Wo, p0 = blockIdx.x * chunk, p1 = min(M, p0 + chunk);
    float acc = 0.f;
    for (long pb = p0; pb < p1; pb += 32) {
        for (int e = t; e < 32 * 16; e += blockDim.x) {
            const long p = pb + e / 16;
            gs[e / 16][e % 16] = p < p1 ? __ldg(g + (size_t)p * 16 + e % 16) : 0.f;
        }
        for (int e = t; e < 32 * 27; e += blockDim.x) {
            const long p = pb + e / 27;
            const int kk = e % 27, c = kk / 9, ky = kk / 3 % 3, kx = kk % 3;
            float v = 0.f;
            if (p < p1) {
                const int ow = (int)(p % Wo); const long q = p / Wo; const int oh = (int)(q % Ho); const int b = (int)(q / Ho);
                const int iy = oh * 2 + ky - pad, ix = ow * 2 + kx - pad;
                if (iy >= 0 && iy < H && ix >= 0 && ix < W) v = __ldg(img + (((size_t)b * 3 + c) * H + iy) * W + ix);
            }
            xs[e / 27][kk] = v;
        }
        __syncthreads();
        if (t < 432)
#pragma unroll 8
            for (int j = 0; j < 32; ++j) acc = fmaf(gs[j][o], xs[j][k], acc);
        __syncthreads();
    }
    if (t < 432) part[(size_t)blockIdx.x * 432 + t] = acc;
}

// out[i] = sum_j part[j][i] over n chunks in fixed order (fp64).
__global__ void __launch_bounds__(256)
sum_chunks_kernel(const float* __restrict__ part, int n, long len, float* __restrict__ out) {
    for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < len; i += (long)gridDim.x * blockDim.x) {
        double s = 0.0;
        for (int j = 0; j < n; ++j) s += part[(size_t)j * len + i];
        out[i] = (float)s;
    }
}

// Depthwise dgrad (transposed depthwise conv with the raw weights): out[b,ih,iw,c] = sum_taps w[c][tap] * g[b,oh,ow,c]
// (+ res).  g: [B,Ho,Wo,C], out: [B,H,W,C].
template <int S>
__global__ void __launch_bounds__(256)
dw_dgrad_raw_kernel(const float* __restrict__ g, const float* __restrict__ w, const float* __restrict__ res, int B, int H, int W, int C,
                    int Ho, int Wo, int pad, float* __restrict__ out) {
    const long total = (long)B * H * W * C;
    for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        const int c = (int)(i % C); const long pix = i / C;
        const int iw = (int)(pix % W); const long t = pix / W; const int ih = (int)(t % H); const int b = (int)(t / H);
        const float* wc = w + (size_t)c * 9;
        float acc = 0.f;
#pragma unroll
        for (int ky = 0; ky < 3; ++ky) {
            const int ny = ih + pad - ky;
            if (ny < 0 || ny % S) continue;
            const int oh = ny / S;
            if (oh >= Ho) continue;
#pragma unroll
            for (int kx = 0; kx < 3; ++kx) {
                const int nx = iw + pad - kx;
                if (nx < 0 || nx % S) continue;
                const int ow = nx / S;
                if (ow >= Wo) continue;
                acc = fmaf(__ldg(wc + ky * 3 + kx), __ldg(g + (((size_t)b * Ho + oh) * Wo + ow) * C + c), acc);
            }
        }
        if (res) acc += __ldg(res + i);
        out[i] = acc;
    }
}

// ---- head ---------------------------------------------------------------------------------------------------------------

// pooled[b][c] = mean over the HW pixels of feat[b, :, c].
__global__ void __launch_bounds__(256)
pool_kernel(const float* __restrict__ feat, int B, int HW, int C, float* __restrict__ pooled) {
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long)B * C) return;
    const int c = (int)(i % C), b = (int)(i / C);
    float s = 0.f;
    for (int p = 0; p < HW; ++p) s += __ldg(feat + ((size_t)b * HW + p) * C + c);
    pooled[i] = s / (float)HW;
}

// Head backward, CTA = (image b, 256 channels): gp = g_out * [the clamp / ReLU passes] (torch's rules, on the saved
// pre-clamp output raw), stored to gp_out [B][n_out] by the y = 0 CTAs; g_feat = W^T gp / HW broadcast over the HW
// pixels of the cn output -> gy [B, HW, C].
__global__ void __launch_bounds__(256)
head_bwd_train_kernel(const float* __restrict__ g, const float* __restrict__ raw, const uint8_t* __restrict__ codes, const float* __restrict__ w,
                      int n_out, int HW, int C, float* __restrict__ gp_out, float* __restrict__ gy) {
    extern __shared__ float gp[];
    const int b = blockIdx.x;
    for (int o = threadIdx.x; o < n_out; o += blockDim.x) {
        const float v = raw[(size_t)b * n_out + o];
        const int code = codes ? codes[o] : 0;
        const bool pass = code == 1 ? (v >= 0.f && v <= 1.f) : code == 2 ? v > 0.f : code == 3 ? (v >= -0.2f && v <= 0.2f) : true;
        gp[o] = pass ? g[(size_t)b * n_out + o] : 0.f;
        if (blockIdx.y == 0) gp_out[(size_t)b * n_out + o] = gp[o];
    }
    __syncthreads();
    const int c = blockIdx.y * blockDim.x + threadIdx.x;
    if (c >= C) return;
    float acc = 0.f;
    for (int o = 0; o < n_out; ++o) acc = fmaf(__ldg(w + (size_t)o * C + c), gp[o], acc);
    const float gf = acc / (float)HW;
    for (int p = 0; p < HW; ++p) gy[((size_t)b * HW + p) * C + c] = gf;
}

// g_W[o][c] = sum_b gp[b][o] * pooled[b][c] (c < C), g_b[o] = sum_b gp[b][o] (column C); either may be null.
__global__ void __launch_bounds__(256)
head_wgrad_kernel(const float* __restrict__ gp, const float* __restrict__ pooled, int B, int n_out, int C, float* __restrict__ gw, float* __restrict__ gbias) {
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long)n_out * (C + 1)) return;
    const int o = (int)(i / (C + 1)), c = (int)(i % (C + 1));
    float s = 0.f;
    if (c < C) {
        if (!gw) return;
        for (int b = 0; b < B; ++b) s = fmaf(gp[(size_t)b * n_out + o], pooled[(size_t)b * C + c], s);
        gw[(size_t)o * C + c] = s;
    } else {
        if (!gbias) return;
        for (int b = 0; b < B; ++b) s += gp[(size_t)b * n_out + o];
        gbias[o] = s;
    }
}

// ---- per-call weight packing ------------------------------------------------------------------------------------------

// One job per 1x1 weight (or the stem): src [rows][cols] -> hi (and lo), transposed when `transpose`; split: hi = tf32(v),
// lo = tf32(v - hi) (lo null: hi only); otherwise hi = v.
struct PackJob { const float* src; float* hi; float* lo; int rows, cols, transpose, split; };
constexpr int kMaxPackJobs = 40;
struct PackJobs { PackJob j[kMaxPackJobs]; };
__global__ void __launch_bounds__(256)
pack_kernel(const __grid_constant__ PackJobs p) {
    const PackJob& q = p.j[blockIdx.y];
    const int n = q.rows * q.cols;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const int r = i / q.cols, c = i % q.cols;
        const float v = __ldg(q.src + i);
        const int d = q.transpose ? c * q.rows + r : i;
        const float hi = q.split ? smk::round_tf32(v) : v;
        q.hi[d] = hi;
        if (q.lo) q.lo[d] = smk::round_tf32(v - hi);
    }
}

// ---- host side ----------------------------------------------------------------------------------------------------------

// Tensors of backbone i in tensor_list() order: 5 per conv (weight, gamma, beta, running_mean, running_var).
struct BnRef { float *w, *gamma, *beta, *rmean, *rvar; long long* nbt; float *gw, *ggamma, *gbeta; };
struct View {
    const SmkEncoder* h; const SmkEncoderTrainArgs* a; const SmkEncoderTrainGrads* gr; int i;
    BnRef bn(int k) const {      // k-th conv + BN of the backbone
        BnRef r;
        float* const* t = a->tensors[i];
        r.w = t[5 * k]; r.gamma = t[5 * k + 1]; r.beta = t[5 * k + 2]; r.rmean = t[5 * k + 3]; r.rvar = t[5 * k + 4];
        r.nbt = (long long*)a->num_batches_tracked[i][k];
        float* const* g = gr && gr->tensors[i] ? gr->tensors[i] : nullptr;
        r.gw = g ? g[5 * k] : nullptr; r.ggamma = g ? g[5 * k + 1] : nullptr; r.gbeta = g ? g[5 * k + 2] : nullptr;
        return r;
    }
};

int n_bn(const Backbone& bb) {
    int n = 1;
    for (const Block& b : bb.blocks) n += b.kind == IR ? 3 : b.kind == DS ? 2 : 1;
    return n;
}
// floats of one copy of a backbone's 1x1 weights
size_t pw_floats(const Backbone& bb) {
    size_t n = 0;
    for (const Block& b : bb.blocks) n += b.kind == IR ? (size_t)b.cin * b.mid + (size_t)b.mid * b.cout : (size_t)b.cin * b.cout;
    return n;
}
int max_channels(const Backbone& bb) {
    int c = 16;
    for (const Block& b : bb.blocks) c = std::max(c, std::max(b.mid, b.cout));
    return c;
}

// Workspace of one backbone: packed 1x1 weights (2 copies when x3) + the stem's [27][16] dgrad weights, BN partials,
// BN backward sums, weight-gradient partials, head gradient, and 3 activation-gradient buffers.
struct BackboneWs { float* pw; float* stem_t; double2* part; float* gb; float* wpart; float* gp; float* buf[3]; };
size_t backbone_ws_bytes(const SmkEncoder* h, const Backbone& bb, int B) {
    const size_t C = max_channels(bb);
    return smk::ws_round(pw_floats(bb) * (h->x3 ? 2 : 1) * 4) + smk::ws_round(27 * 16 * 4) + smk::ws_round((size_t)kMaxChunks * C * 16) +
           smk::ws_round(2 * C * 4) + smk::ws_round(kWgradPart * 4) + smk::ws_round((size_t)B * bb.n_out * 4) +
           3 * smk::ws_round((size_t)B * bb.max_act * 4);
}
bool carve(smk::Workspace& w, const SmkEncoder* h, const Backbone& bb, int B, BackboneWs* o) {
    o->pw = w.take<float>(pw_floats(bb) * (h->x3 ? 2 : 1));
    o->stem_t = w.take<float>(27 * 16);
    o->part = w.take<double2>((size_t)kMaxChunks * max_channels(bb));
    o->gb = w.take<float>(2 * (size_t)max_channels(bb));
    o->wpart = w.take<float>(kWgradPart);
    o->gp = w.take<float>((size_t)B * bb.n_out);
    for (int j = 0; j < 3; ++j) o->buf[j] = w.take<float>((size_t)B * bb.max_act);
    return o->buf[2] != nullptr;
}

// Forward and dgrad copies of a 1x1 weight W [cout][cin] in the packed buffer: conv_gemm reads [K][N], tc_conv [N][K]
// (+ tails).  fwd: K = cin, N = cout; dgrad: K = cout, N = cin.
struct PwPack { const float* w; const float* wt; const float* wt_lo; };

// Packs the backbone's 1x1 weights for the forward (dgrad = false) or the dgrad (true), and the stem's dgrad weights, in
// one launch.  packed[k]: where the k-th 1x1 conv's copy went.
int pack_weights(const SmkEncoder* h, const View& v, const BackboneWs& ws, bool dgrad, std::vector<PwPack>& packed, cudaStream_t st) {
    const Backbone& bb = h->bb[v.i];
    const bool tc = h->precision >= 1;
    PackJobs jobs{};
    int nj = 0, max_n = 432;
    float* dst = ws.pw;
    int bn = 1;
    packed.clear();
    auto add = [&](const float* w, int cin, int cout) {
        const size_t n = (size_t)cin * cout;
        max_n = std::max(max_n, (int)n);
        if (!tc && dgrad) { packed.push_back(PwPack{w, nullptr, nullptr}); return; }   // torch's [cout][cin] is the dgrad's [K][N]
        PackJob& j = jobs.j[nj++];
        j.src = w; j.rows = cout; j.cols = cin; j.hi = dst; j.lo = tc && h->x3 ? dst + n : nullptr;
        // fp32 forward: [cin][cout]; tensor-core forward: torch's own layout, split; tensor-core dgrad: [cin][cout], split
        j.transpose = !tc || dgrad; j.split = tc;
        packed.push_back(tc ? PwPack{nullptr, j.hi, j.lo} : PwPack{j.hi, nullptr, nullptr});
        dst += n * (j.lo ? 2 : 1);
    };
    for (const Block& b : bb.blocks) {
        if (b.kind == DS) { add(v.bn(bn + 1).w, b.cin, b.cout); bn += 2; }
        else if (b.kind == IR) { add(v.bn(bn).w, b.cin, b.mid); add(v.bn(bn + 2).w, b.mid, b.cout); bn += 3; }
        else { add(v.bn(bn).w, b.cin, b.cout); bn += 1; }
    }
    if (dgrad) {                                          // stem [16][27] -> [27][16], the layout of stem_dgrad
        PackJob& j = jobs.j[nj++];
        j.src = v.bn(0).w; j.rows = 16; j.cols = 27; j.hi = ws.stem_t; j.lo = nullptr; j.transpose = 1; j.split = 0;
    }
    if (nj == 0) return 0;
    SMK_TAG("train_pack", 8.0 * pw_floats(bb) * (h->x3 ? 1.5 : 1.0), 0.0, st);
    SMK_LAUNCH(pack_kernel, dim3(cdiv(max_n, 256), nj), dim3(256), 0, st, jobs);
    SMK_CHECK_LAUNCH();
    return 0;
}

// One 1x1 conv through smk::conv: out[m, :N] = in[m, :K] . W (+ res), unit scale and zero bias.
int conv1x1(const SmkEncoder* h, const PwPack& w, const float* in, int K, int N, int B, int H, const float* res, float* out, bool round, const char* tag,
            cudaStream_t st) {
    smk::Conv q{};
    q.in = in; q.ld_in = K; q.B = B; q.H = H; q.W = H; q.Cin = K; q.N = N; q.K = K; q.mode = 0;
    q.w = w.w; q.wt = w.wt; q.wt_lo = w.wt_lo; q.scale = h->ones; q.bias = h->zeros;
    q.res = res; q.ld_res = N; q.out = out; q.ld_out = N; q.round_out = round ? 1 : 0; q.tag = tag;
    return smk::conv(q, st);
}

// Train-mode BatchNorm of z [M, C]: statistics (+ running-stat update), then y = BN(z) (+ res) (ReLU).
int bn_forward(const BnRef& r, const float* z, long M, int C, float eps, float momentum, float* mean, float* invstd, const float* res, bool relu,
               bool round, float* y, double2* part, cudaStream_t st) {
    const int nch = bn_chunks(M);
    const long chunk = cdiv(M, nch);
    SMK_TAG("bn_stats", 4.0 * M * C + 16.0 * nch * C, 3.0 * M * C, st);
    SMK_LAUNCH(bn_reduce_kernel<0>, dim3(cdiv(C, 32), nch), dim3(32, 8), 0, st, z, nullptr, nullptr, nullptr, nullptr, M, C, chunk, part);
    SMK_CHECK_LAUNCH();
    SMK_TAG("bn_finalize", 16.0 * nch * C + 24.0 * C, 0.0, st);
    SMK_LAUNCH(bn_finalize_fwd_kernel, dim3(1), dim3(256), 0, st, part, nch, M, C, eps, momentum, r.rmean, r.rvar, r.nbt, mean, invstd);
    SMK_CHECK_LAUNCH();
    SMK_TAG("bn_apply", 4.0 * M * C * (res ? 3 : 2), 4.0 * M * C, st);
    SMK_LAUNCH(bn_apply_kernel, dim3(grid_of(M * C / 4)), dim3(256), 0, st, z, mean, invstd, r.gamma, r.beta, res, M, C, relu ? 1 : 0, round ? 1 : 0, y);
    SMK_CHECK_LAUNCH();
    return 0;
}

// Train-mode BatchNorm backward: g (gradient of y, masked by [y > 0] when y is given) -> gz (may alias g); g_gamma / g_beta.
int bn_backward(const BnRef& r, const float* g, const float* y, const float* z, const float* mean, const float* invstd, long M, int C, bool round,
                float* gz, double2* part, float* gb, cudaStream_t st) {
    const int nch = bn_chunks(M);
    const long chunk = cdiv(M, nch);
    SMK_TAG("bn_bwd_reduce", 4.0 * M * C * (y ? 3 : 2), 5.0 * M * C, st);
    SMK_LAUNCH(bn_reduce_kernel<1>, dim3(cdiv(C, 32), nch), dim3(32, 8), 0, st, z, g, y, mean, invstd, M, C, chunk, part);
    SMK_CHECK_LAUNCH();
    SMK_TAG("bn_bwd_finalize", 16.0 * nch * C, 0.0, st);
    SMK_LAUNCH(bn_finalize_bwd_kernel, dim3(1), dim3(256), 0, st, part, nch, C, gb, r.ggamma, r.gbeta);
    SMK_CHECK_LAUNCH();
    SMK_TAG("bn_bwd_apply", 4.0 * M * C * (y ? 4 : 3), 8.0 * M * C, st);
    SMK_LAUNCH(bn_bwd_apply_kernel, dim3(grid_of(M * C)), dim3(256), 0, st, g, y, z, mean, invstd, r.gamma, gb, M, C, round ? 1 : 0, gz);
    SMK_CHECK_LAUNCH();
    return 0;
}

// Split-K chunks of a weight gradient with `tiles` output tiles of `tile_floats` each over M pixels: a function of the
// shape only (fixed summation order), with at most kWgradPart floats of partials.
int wgrad_chunks(long M, long tiles, long tile_floats, long per_chunk_min) {
    const long cap = std::max(1L, (long)kWgradPart / (tiles * tile_floats));
    return (int)std::max(1L, std::min({(long)cdiv(M, per_chunk_min), 1024L / tiles + 1, cap}));
}

int sum_chunks(const float* part, int n, long len, float* out, cudaStream_t st) {
    SMK_TAG("wgrad_reduce", 4.0 * len * (n + 1), (double)len * n, st);
    SMK_LAUNCH(sum_chunks_kernel, dim3(grid_of(len)), dim3(256), 0, st, part, n, len, out);
    SMK_CHECK_LAUNCH();
    return 0;
}

int pw_wgrad(const float* g, const float* a, long M, int Co, int Ci, float* part, float* out, cudaStream_t st) {
    const long tiles = (long)cdiv(Ci, 64) * cdiv(Co, 64);
    const int nch = wgrad_chunks(M, tiles, 64 * 64, 512);
    const long chunk = cdiv(M, nch);
    SMK_TAG("pw_wgrad", 4.0 * M * (Co + Ci) + 4.0 * nch * Co * Ci, 2.0 * M * Co * Ci, st);
    SMK_LAUNCH(pw_wgrad_kernel, dim3(cdiv(Ci, 64), cdiv(Co, 64), nch), dim3(256), 0, st, g, a, M, Co, Ci, chunk, part);
    SMK_CHECK_LAUNCH();
    return sum_chunks(part, nch, (long)Co * Ci, out, st);
}

int dw_wgrad(const float* g, const float* a, int B, int H, int C, int S, float* part, float* out, cudaStream_t st) {
    const int Ho = (H + S - 1) / S;
    const long M = (long)B * Ho * Ho;
    const int tiles = cdiv(C, 32);
    const int nch = std::min(wgrad_chunks(M, tiles, 32 * 9, 256), 256);
    const long chunk = cdiv(M, nch);
    SMK_TAG("dw_wgrad", 4.0 * ((double)M * C + (double)B * H * H * C), 18.0 * M * C, st);
    if (S == 1) SMK_LAUNCH(dw_wgrad_kernel<1>, dim3(tiles, nch), dim3(32, 8), 0, st, g, a, B, H, H, C, Ho, Ho, same_pad_begin(H, 1), chunk, part);
    else SMK_LAUNCH(dw_wgrad_kernel<2>, dim3(tiles, nch), dim3(32, 8), 0, st, g, a, B, H, H, C, Ho, Ho, same_pad_begin(H, 2), chunk, part);
    SMK_CHECK_LAUNCH();
    return sum_chunks(part, nch, (long)C * 9, out, st);
}

int dw_forward(const float* a, const float* w, int B, int H, int C, int S, float* z, cudaStream_t st) {
    const int Ho = (H + S - 1) / S;
    const long total = (long)B * Ho * Ho * C;
    SMK_TAG("dw_fwd", 4.0 * ((double)B * H * H * C + total), 18.0 * total, st);
    if (S == 1) SMK_LAUNCH(dw_fwd_kernel<1>, dim3(grid_of(total)), dim3(256), 0, st, a, w, B, H, H, C, Ho, Ho, same_pad_begin(H, 1), z);
    else SMK_LAUNCH(dw_fwd_kernel<2>, dim3(grid_of(total)), dim3(256), 0, st, a, w, B, H, H, C, Ho, Ho, same_pad_begin(H, 2), z);
    SMK_CHECK_LAUNCH();
    return 0;
}

int dw_dgrad(const float* g, const float* w, const float* res, int B, int H, int C, int S, float* out, cudaStream_t st) {
    const int Ho = (H + S - 1) / S;
    const long total = (long)B * H * H * C;
    SMK_TAG("dw_dgrad_train", 4.0 * ((double)B * Ho * Ho * C + total * (res ? 2 : 1)), 18.0 * B * Ho * Ho * C, st);
    if (S == 1) SMK_LAUNCH(dw_dgrad_raw_kernel<1>, dim3(grid_of(total)), dim3(256), 0, st, g, w, res, B, H, H, C, Ho, Ho, same_pad_begin(H, 1), out);
    else SMK_LAUNCH(dw_dgrad_raw_kernel<2>, dim3(grid_of(total)), dim3(256), 0, st, g, w, res, B, H, H, C, Ho, Ho, same_pad_begin(H, 2), out);
    SMK_CHECK_LAUNCH();
    return 0;
}

// Topology of a train handle: the layer list, activation sizes and the saved layout (names: the reference's module paths
// — a conv's pre-BN output under the conv, a ReLU output under its BatchNorm as in the eval layout, a block's output
// under the block, the pooled features under `<encoder>.pooled`, a head's pre-clamp output under the head).
void build_topology(SmkEncoder* h) {
    for (int i = 0; i < 3; ++i) {
        if (!h->present[i]) continue;
        Backbone& bb = h->bb[i];
        const BlockDef* defs = i == 0 ? kSmall : kLarge;
        const int nb = i == 0 ? (int)(sizeof(kSmall) / sizeof(BlockDef)) : (int)(sizeof(kLarge) / sizeof(BlockDef));
        const int* stages = i == 0 ? kStageSmall : kStageLarge;
        const std::string enc = std::string(kEncName[i]) + ".encoder.";
        auto add = [h](const std::string& name, int H, int C) { return h->saved.add(name, H, H, C); };
        bb.sv_zstem = add(enc + "conv_stem", 112, 16);
        bb.sv_stem = add(enc + "bn1", 112, 16);
        int cin = 16, res = 112, stage = 0, in_stage = 0, bn = 1;
        size_t max_act = (size_t)112 * 112 * 16;
        for (int k = 0; k < nb; ++k) {
            Block b{};
            b.kind = defs[k].kind; b.stride = defs[k].stride; b.cin = cin; b.cout = defs[k].cout;
            b.skip = b.kind != CN && b.stride == 1 && b.cin == b.cout;
            b.mid = b.kind == IR ? make_divisible((double)cin * defs[k].exp) : cin;
            b.bn0 = bn;
            const int ro = (res + b.stride - 1) / b.stride;
            const std::string pre = enc + "blocks." + std::to_string(stage) + "." + std::to_string(in_stage);
            if (b.kind == DS) {
                b.sv_z[0] = add(pre + ".conv_dw", ro, cin); b.sv_a = add(pre + ".bn1", ro, cin);
                b.sv_z[1] = add(pre + ".conv_pw", ro, b.cout); b.sv_out = add(pre, ro, b.cout);
                bn += 2;
            } else if (b.kind == IR) {
                b.sv_z[0] = add(pre + ".conv_pw", res, b.mid); b.sv_a = add(pre + ".bn1", res, b.mid);
                b.sv_z[1] = add(pre + ".conv_dw", ro, b.mid); b.sv_b = add(pre + ".bn2", ro, b.mid);
                b.sv_z[2] = add(pre + ".conv_pwl", ro, b.cout); b.sv_out = add(pre, ro, b.cout);
                bn += 3;
            } else {
                b.sv_z[0] = add(pre + ".conv", ro, b.cout); b.sv_a = add(pre + ".bn1", ro, b.cout);
                bn += 1;
            }
            max_act = std::max(max_act, (size_t)res * res * b.mid);
            max_act = std::max(max_act, (size_t)ro * ro * std::max(b.mid, b.cout));
            res = ro; cin = b.cout;
            if (++in_stage == stages[stage]) { ++stage; in_stage = 0; }
            bb.blocks.push_back(b);
        }
        bb.feat = cin;
        bb.n_out = i == 0 ? 6 : i == 1 ? h->n_shape : h->n_exp + 5;
        bb.max_act = max_act;
        h->max_act = std::max(h->max_act, max_act);
        bb.sv_pool = h->saved.add(std::string(kEncName[i]) + ".pooled", 1, 1, bb.feat);
        bb.sv_head = h->saved.add(std::string(kEncName[i]) + "." + kHeadName[i], 1, 1, bb.n_out);
    }
    // BatchNorm statistics after the saved tensors: per backbone, per BN, mean[C] then invstd[C]
    for (int i = 0; i < 3; ++i) {
        if (!h->present[i]) continue;
        const Backbone& bb = h->bb[i];
        size_t n = 2 * 16;
        for (const Block& b : bb.blocks) n += b.kind == IR ? 2 * (2 * (size_t)b.mid + b.cout) : b.kind == DS ? 2 * ((size_t)b.cin + b.cout) : 2 * (size_t)b.cout;
        h->stats_floats += n;
    }
}

}  // namespace

extern "C" int smk_encoder_train_create(int backbones, int n_shape, int n_exp, int precision, SmkEncoder** out) {
    SMK_REQUIRE(out, "smk_encoder_train_create: null argument");
    SMK_REQUIRE(backbones > 0 && backbones < 8, "smk_encoder_train_create: backbones is a non-empty bit set of {1 pose, 2 shape, 4 expression}");
    SMK_REQUIRE(precision >= 0 && precision <= 3, "smk_encoder_train_create: precision must be 0, 1, 2 or 3");
    SMK_REQUIRE(n_shape > 0 && n_exp >= 0 && n_shape <= 4096 && n_exp <= 4096, "smk_encoder_train_create: bad head widths");
    if (precision >= 1) { if (int rc = smk::tc_init()) return rc; }
    SmkEncoder* h = new SmkEncoder();
    h->train = true;
    h->n_shape = n_shape; h->n_exp = n_exp; h->precision = precision >= 1 ? 1 : 0; h->x3 = precision == 3;
    for (int i = 0; i < 3; ++i) h->present[i] = (backbones >> i) & 1;
    build_topology(h);
    cudaError_t e = cudaSuccess;
    if (h->present[2]) {                                  // smirk_encoder.py:105-108
        std::vector<uint8_t> codes(h->bb[2].n_out, 0);
        codes[n_exp] = codes[n_exp + 1] = 1; codes[n_exp + 2] = 2; codes[n_exp + 3] = codes[n_exp + 4] = 3;
        e = h->arena.upload(codes, &h->bb[2].codes);
    }
    std::vector<float> ones(1024, 1.f), zeros(1024, 0.f);
    if (e == cudaSuccess) e = h->arena.upload(ones, &h->ones);
    if (e == cudaSuccess) e = h->arena.upload(zeros, &h->zeros);
    if (e == cudaSuccess) e = create_forks(h);
    if (e != cudaSuccess) { smk::set_error("smk_encoder_train_create: %s", cudaGetErrorString(e)); delete h; return (int)e; }
    *out = h;
    return 0;
}

extern "C" size_t smk_encoder_train_workspace_bytes(const SmkEncoder* h, int B) {
    if (!h || !h->train || B <= 0) return 0;
    size_t n = 0;
    for (int i = 0; i < 3; ++i) if (h->present[i]) n += backbone_ws_bytes(h, h->bb[i], B);
    return n;
}

namespace {

// Statistics offset (floats, from the start of the stats area) of backbone i's first BN.
size_t stats_base(const SmkEncoder* h, int i) {
    size_t o = 0;
    for (int j = 0; j < i; ++j) {
        if (!h->present[j]) continue;
        o += 2 * 16;
        for (const Block& b : h->bb[j].blocks) o += b.kind == IR ? 2 * (2 * (size_t)b.mid + b.cout) : b.kind == DS ? 2 * ((size_t)b.cin + b.cout) : 2 * (size_t)b.cout;
    }
    return o;
}

int check_args(const SmkEncoder* h, const SmkEncoderTrainArgs* a, const char* fn) {
    SMK_REQUIRE(h && h->train, "%s: not a train-mode handle (smk_encoder_train_create)", fn);
    SMK_REQUIRE(a, "%s: null args", fn);
    for (int i = 0; i < 3; ++i) {
        if (!h->present[i]) continue;
        const int nbn = n_bn(h->bb[i]);
        SMK_REQUIRE(a->tensors[i] && a->n_tensors[i] == 5 * nbn, "%s: backbone %d expects %d tensors (conv weight + 4 BN tensors per conv), got %d",
                    fn, i, 5 * nbn, a->n_tensors[i]);
        SMK_REQUIRE(a->num_batches_tracked[i] && a->head_w[i] && a->head_b[i], "%s: backbone %d: null num_batches_tracked or head", fn, i);
        for (int k = 0; k < 5 * nbn; ++k) SMK_REQUIRE(a->tensors[i][k], "%s: backbone %d: null tensor %d", fn, i, k);
        for (int k = 0; k < nbn; ++k) SMK_REQUIRE(a->num_batches_tracked[i][k], "%s: backbone %d: null num_batches_tracked %d", fn, i, k);
        SMK_REQUIRE(a->momentum[i] <= 1.f && a->eps[i] > 0.f, "%s: backbone %d: momentum must be in [0, 1] (or negative for None) and eps > 0", fn, i);
    }
    return 0;
}

}  // namespace

extern "C" int smk_encoder_forward_train(const SmkEncoder* h, const SmkEncoderTrainArgs* args, const float* img, int B, float* pose_cam,
                                         float* shape, float* expr, float* saved, size_t saved_bytes, void* ws, size_t ws_bytes, void* stream) {
    const char* fn = "smk_encoder_forward_train";
    if (int rc = check_args(h, args, fn)) return rc;
    SMK_REQUIRE(B >= 0, "%s: negative batch", fn);
    if (B == 0) return 0;
    SMK_REQUIRE(img, "%s: null image", fn);
    SMK_REQUIRE((pose_cam || !h->present[0]) && (shape || !h->present[1]) && (expr || !h->present[2]), "%s: null output for a backbone this handle holds", fn);
    const size_t sv_bytes = smk_encoder_saved_bytes(h, B), need = smk_encoder_train_workspace_bytes(h, B);
    SMK_REQUIRE(!saved || saved_bytes >= sv_bytes, "%s: saved buffer too small", fn);
    SMK_REQUIRE(ws && ws_bytes >= need + (saved ? 0 : sv_bytes), "%s: workspace too small (without `saved` it also holds the activations)", fn);
    smk::Workspace w(ws, ws_bytes);
    BackboneWs bw[3];
    for (int i = 0; i < 3; ++i) if (h->present[i]) SMK_REQUIRE(carve(w, h, h->bb[i], B, &bw[i]), "%s: workspace carve-up failed", fn);
    float* sv = saved ? saved : w.take<float>(sv_bytes / 4);
    SMK_REQUIRE(sv, "%s: workspace carve-up failed", fn);
    float* stats = sv + (size_t)B * h->saved.total;
    float* outs[3] = {pose_cam, shape, expr};
    const bool rnd = h->precision >= 1 && !h->x3;           // TF32 (precision 1-2): activations that feed a GEMM are rounded
    auto SV = [&](int k) { return sv + (size_t)B * h->saved.off[k]; };
    return for_each_unit(h, h->present, (cudaStream_t)stream, fn, [&](const Unit& unit) -> int {
        const int i = unit.idx[0];
        cudaStream_t st = unit.st;
        const Backbone& bb = h->bb[i];
        const View v{h, args, nullptr, i};
        const BackboneWs& W = bw[i];
        const float eps = args->eps[i], mom = args->momentum[i];
        float* st_i = stats + stats_base(h, i);
        std::vector<PwPack> pk;
        if (int rc = pack_weights(h, v, W, false, pk, st)) return rc;
        // the stem
        {
            const long M = (long)B * 112 * 112;
            SMK_TAG("stem_fwd", 4.0 * ((double)B * 3 * 224 * 224 + M * 16), 2.0 * 27 * 16 * M, st);
            SMK_LAUNCH(stem_fwd_kernel, dim3(cdiv(M, 128)), dim3(128), 0, st, img, v.bn(0).w, B, 224, 224, 112, 112, same_pad_begin(224, 2), SV(bb.sv_zstem));
            SMK_CHECK_LAUNCH();
            if (int rc = bn_forward(v.bn(0), SV(bb.sv_zstem), M, 16, eps, mom, st_i, st_i + 16, nullptr, true, false, SV(bb.sv_stem), W.part, st)) return rc;
            st_i += 32;
        }
        const float* x = SV(bb.sv_stem);
        int res = 112, p = 0;
        for (const Block& b : bb.blocks) {
            const int ro = (res + b.stride - 1) / b.stride;
            const long Mi = (long)B * res * res, Mo = (long)B * ro * ro;
            auto bnf = [&](int j, const float* z, long M, int C, const float* skip, bool relu, float* y) {
                const int rc = bn_forward(v.bn(b.bn0 + j), z, M, C, eps, mom, st_i, st_i + C, skip, relu, rnd, y, W.part, st);
                st_i += 2 * C;
                return rc;
            };
            int rc = 0;
            if (b.kind == DS) {
                rc = dw_forward(x, v.bn(b.bn0).w, B, res, b.cin, b.stride, SV(b.sv_z[0]), st);
                if (!rc) rc = bnf(0, SV(b.sv_z[0]), Mo, b.cin, nullptr, true, SV(b.sv_a));
                if (!rc) rc = conv1x1(h, pk[p++], SV(b.sv_a), b.cin, b.cout, B, ro, nullptr, SV(b.sv_z[1]), false, "train_pw", st);
                if (!rc) rc = bnf(1, SV(b.sv_z[1]), Mo, b.cout, b.skip ? x : nullptr, false, SV(b.sv_out));
                x = SV(b.sv_out);
            } else if (b.kind == IR) {
                rc = conv1x1(h, pk[p++], x, b.cin, b.mid, B, res, nullptr, SV(b.sv_z[0]), false, "train_pw", st);
                if (!rc) rc = bnf(0, SV(b.sv_z[0]), Mi, b.mid, nullptr, true, SV(b.sv_a));
                if (!rc) rc = dw_forward(SV(b.sv_a), v.bn(b.bn0 + 1).w, B, res, b.mid, b.stride, SV(b.sv_z[1]), st);
                if (!rc) rc = bnf(1, SV(b.sv_z[1]), Mo, b.mid, nullptr, true, SV(b.sv_b));
                if (!rc) rc = conv1x1(h, pk[p++], SV(b.sv_b), b.mid, b.cout, B, ro, nullptr, SV(b.sv_z[2]), false, "train_pw", st);
                if (!rc) rc = bnf(2, SV(b.sv_z[2]), Mo, b.cout, b.skip ? x : nullptr, false, SV(b.sv_out));
                x = SV(b.sv_out);
            } else {
                rc = conv1x1(h, pk[p++], x, b.cin, b.cout, B, res, nullptr, SV(b.sv_z[0]), false, "train_pw", st);
                if (!rc) rc = bnf(0, SV(b.sv_z[0]), Mo, b.cout, nullptr, true, SV(b.sv_a));
                x = SV(b.sv_a);
            }
            if (rc) return rc;
            res = ro;
        }
        // global average pool, then the head on the pooled features (HW = 1)
        SMK_TAG("train_pool", 4.0 * B * bb.feat * (res * res + 1), (double)B * bb.feat * res * res, st);
        SMK_LAUNCH(pool_kernel, dim3(cdiv((long)B * bb.feat, 256)), dim3(256), 0, st, x, B, res * res, bb.feat, SV(bb.sv_pool));
        SMK_CHECK_LAUNCH();
        smk::GapHeadProblem gp{SV(bb.sv_pool), args->head_w[i], args->head_b[i], bb.codes, outs[i], bb.n_out, SV(bb.sv_head)};
        return smk::gap_head(&gp, 1, B, 1, bb.feat, st);
    });
}

extern "C" int smk_encoder_backward_train(const SmkEncoder* h, const SmkEncoderTrainArgs* args, const float* img, int B, const float* saved,
                                          size_t saved_bytes, const float* g_pose_cam, const float* g_shape, const float* g_expr, float* g_img,
                                          const SmkEncoderTrainGrads* grads, void* ws, size_t ws_bytes, void* stream) {
    const char* fn = "smk_encoder_backward_train";
    if (int rc = check_args(h, args, fn)) return rc;
    SMK_REQUIRE(B >= 0, "%s: negative batch", fn);
    if (B == 0) return 0;
    SMK_REQUIRE(img && saved, "%s: null image or saved buffer", fn);
    SMK_REQUIRE(saved_bytes >= smk_encoder_saved_bytes(h, B), "%s: saved buffer too small", fn);
    SMK_REQUIRE(ws && ws_bytes >= smk_encoder_train_workspace_bytes(h, B), "%s: workspace too small", fn);
    const float* g_out[3] = {g_pose_cam, g_shape, g_expr};
    bool active[3];
    for (int i = 0; i < 3; ++i) {                 // a backbone runs when its output has a gradient and something needs one
        bool want = g_img != nullptr;
        if (h->present[i] && grads) {
            want = want || grads->head_w[i] || grads->head_b[i];
            for (int k = 0; grads->tensors[i] && k < args->n_tensors[i] && !want; ++k) want = grads->tensors[i][k] != nullptr;
        }
        active[i] = h->present[i] && g_out[i] && want;
    }
    for (int i = 0; i < 3; ++i)
        for (int k = 0; h->present[i] && grads && grads->tensors[i] && k < args->n_tensors[i]; ++k)
            SMK_REQUIRE(k % 5 < 3 || !grads->tensors[i][k], "%s: running statistics have no gradient (backbone %d, tensor %d)", fn, i, k);
    smk::Workspace w(ws, ws_bytes);
    BackboneWs bw[3];
    for (int i = 0; i < 3; ++i) if (h->present[i]) SMK_REQUIRE(carve(w, h, h->bb[i], B, &bw[i]), "%s: workspace carve-up failed", fn);
    const float* stats = saved + (size_t)B * h->saved.total;
    const bool rnd = h->precision >= 1 && !h->x3;            // gradients that feed a TF32 GEMM are rounded
    auto SV = [&](int k) { return saved + (size_t)B * h->saved.off[k]; };
    const float* g_stem[3] = {nullptr, nullptr, nullptr};
    const float* w_stem[3] = {nullptr, nullptr, nullptr};
    cudaStream_t main_st = (cudaStream_t)stream;
    int rc = for_each_unit(h, active, main_st, fn, [&](const Unit& unit) -> int {
        const int i = unit.idx[0];
        cudaStream_t st = unit.st;
        const Backbone& bb = h->bb[i];
        const View v{h, args, grads, i};
        const BackboneWs& W = bw[i];
        std::vector<PwPack> pk;
        if (int rc = pack_weights(h, v, W, true, pk, st)) return rc;
        // statistics of each BN, in forward order
        std::vector<const float*> mean;
        std::vector<int> chans;
        {
            const float* s = stats + stats_base(h, i);
            auto push = [&](int C) { mean.push_back(s); chans.push_back(C); s += 2 * C; };
            push(16);
            for (const Block& b : bb.blocks) {
                if (b.kind == DS) { push(b.cin); push(b.cout); }
                else if (b.kind == IR) { push(b.mid); push(b.mid); push(b.cout); }
                else push(b.cout);
            }
        }
        auto bnb = [&](int k, const float* g, const float* y, const float* z, long M, float* gz) {
            return bn_backward(v.bn(k), g, y, z, mean[k], mean[k] + chans[k], M, chans[k], rnd, gz, W.part, W.gb, st);
        };
        float *gy = W.buf[0], *t1 = W.buf[1], *t2 = W.buf[2];
        int res = 7;
        {   // head -> gradient of the cn output (t1); head weight gradients
            const int C = bb.feat;
            SMK_TAG("train_head_bwd", 4.0 * ((double)B * res * res * C + (double)bb.n_out * C + 3.0 * B * bb.n_out), 2.0 * B * C * bb.n_out, st);
            SMK_LAUNCH(head_bwd_train_kernel, dim3(B, cdiv(C, 256)), dim3(256), (size_t)bb.n_out * 4, st, g_out[i], SV(bb.sv_head), bb.codes,
                       args->head_w[i], bb.n_out, res * res, C, W.gp, t1);
            SMK_CHECK_LAUNCH();
            float* gw = grads ? grads->head_w[i] : nullptr;
            float* gb = grads ? grads->head_b[i] : nullptr;
            if (gw || gb) {
                SMK_TAG("train_head_wgrad", 4.0 * ((double)B * (bb.n_out + C) + (double)bb.n_out * C), 2.0 * B * C * bb.n_out, st);
                SMK_LAUNCH(head_wgrad_kernel, dim3(cdiv((long)bb.n_out * (C + 1), 256)), dim3(256), 0, st, W.gp, SV(bb.sv_pool), B, bb.n_out, C, gw, gb);
                SMK_CHECK_LAUNCH();
            }
        }
        int p = (int)pk.size();
        for (int bi = (int)bb.blocks.size() - 1; bi >= 0; --bi) {
            const Block& b = bb.blocks[bi];
            const int ro = res, ri = bi == 0 ? 112 : ro * b.stride;
            const long Mi = (long)B * ri * ri, Mo = (long)B * ro * ro;
            const float* x = bi == 0 ? SV(bb.sv_stem) : SV(bb.blocks[bi - 1].sv_out);     // the block input
            int rc = 0;
            if (b.kind == CN) {                      // t1: gradient of the cn output -> gy: of the block input
                const BnRef r = v.bn(b.bn0);
                rc = bnb(b.bn0, t1, SV(b.sv_a), SV(b.sv_z[0]), Mo, t1);
                if (!rc && r.gw) rc = pw_wgrad(t1, x, Mo, b.cout, b.cin, W.wpart, r.gw, st);
                if (!rc) rc = conv1x1(h, pk[--p], t1, b.cout, b.cin, B, ro, nullptr, gy, false, "train_pw_dgrad", st);
            } else if (b.kind == IR) {               // gy: gradient of the block output -> gy: of the block input
                const BnRef rp = v.bn(b.bn0), rd = v.bn(b.bn0 + 1), rl = v.bn(b.bn0 + 2);
                const PwPack& wl = pk[--p];
                const PwPack& we = pk[--p];
                rc = bnb(b.bn0 + 2, gy, nullptr, SV(b.sv_z[2]), Mo, t1);
                if (!rc && rl.gw) rc = pw_wgrad(t1, SV(b.sv_b), Mo, b.cout, b.mid, W.wpart, rl.gw, st);
                if (!rc) rc = conv1x1(h, wl, t1, b.cout, b.mid, B, ro, nullptr, t2, false, "train_pw_dgrad", st);
                if (!rc) rc = bnb(b.bn0 + 1, t2, SV(b.sv_b), SV(b.sv_z[1]), Mo, t2);
                if (!rc && rd.gw) rc = dw_wgrad(t2, SV(b.sv_a), B, ri, b.mid, b.stride, W.wpart, rd.gw, st);
                if (!rc) rc = dw_dgrad(t2, rd.w, nullptr, B, ri, b.mid, b.stride, t1, st);
                if (!rc) rc = bnb(b.bn0, t1, SV(b.sv_a), SV(b.sv_z[0]), Mi, t1);
                if (!rc && rp.gw) rc = pw_wgrad(t1, x, Mi, b.mid, b.cin, W.wpart, rp.gw, st);
                if (!rc) rc = conv1x1(h, we, t1, b.mid, b.cin, B, ri, b.skip ? gy : nullptr, t2, false, "train_pw_dgrad", st);
                std::swap(gy, t2);
            } else {                                 // DS block 0: gy -> t1: gradient of the stem output
                const BnRef rd = v.bn(b.bn0), rp = v.bn(b.bn0 + 1);
                rc = bnb(b.bn0 + 1, gy, nullptr, SV(b.sv_z[1]), Mo, t1);
                if (!rc && rp.gw) rc = pw_wgrad(t1, SV(b.sv_a), Mo, b.cout, b.cin, W.wpart, rp.gw, st);
                if (!rc) rc = conv1x1(h, pk[--p], t1, b.cout, b.cin, B, ro, nullptr, t2, false, "train_pw_dgrad", st);
                if (!rc) rc = bnb(b.bn0, t2, SV(b.sv_a), SV(b.sv_z[0]), Mo, t2);
                if (!rc && rd.gw) rc = dw_wgrad(t2, x, B, ri, b.cin, b.stride, W.wpart, rd.gw, st);
                if (!rc) rc = dw_dgrad(t2, rd.w, b.skip ? gy : nullptr, B, ri, b.cin, b.stride, t1, st);
            }
            if (rc) return rc;
            res = ri;
        }
        // the stem: t1 -> gradient of its pre-BN output (t1); its weight gradient; the image gradient after the join
        const BnRef r0 = v.bn(0);
        const long M = (long)B * 112 * 112;
        if (int rc = bnb(0, t1, SV(bb.sv_stem), SV(bb.sv_zstem), M, t1)) return rc;
        if (r0.gw) {
            const int nch = (int)std::min<long>(cdiv(M, 1024), 512);
            SMK_TAG("stem_wgrad", 4.0 * ((double)M * 16 + (double)B * 3 * 224 * 224), 2.0 * 432 * M, st);
            SMK_LAUNCH(stem_wgrad_kernel, dim3(nch), dim3(448), 0, st, t1, img, B, 224, 224, 112, 112, same_pad_begin(224, 2), cdiv(M, nch), W.wpart);
            SMK_CHECK_LAUNCH();
            if (int rc = sum_chunks(W.wpart, nch, 432, r0.gw, st)) return rc;
        }
        g_stem[i] = t1; w_stem[i] = W.stem_t;
        return 0;
    });
    if (rc || !g_img) return rc;
    return enc::stem_dgrad(g_stem, w_stem, B, g_img, main_st);
}
