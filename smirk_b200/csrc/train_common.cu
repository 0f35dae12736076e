// Train-mode BatchNorm, split-K weight-gradient reductions and per-call weight packing (see train_common.cuh).
#include "train_common.cuh"

namespace trn {

using smk::cdiv;
using smk::grid_of;

namespace {

// Pixel chunks of a per-channel reduction over M pixels: a function of M only, so the summation order is fixed.
int bn_chunks(long M) { return (int)std::min<long>(cdiv(M, 256), kMaxChunks); }

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

// y = gamma * (z - mean) * invstd + beta (+ res) (ReLU) (TF32 rounding for a tensor-core consumer), z / res [M, C], C % 4 == 0.
// y has a pixel stride of ld_y; ypad (optional) takes the same values in the interior of a [B, H+2, W+2, C] buffer.
__global__ void __launch_bounds__(256)
bn_apply_kernel(const float* __restrict__ z, const float* __restrict__ mean, const float* __restrict__ invstd, const float* __restrict__ gamma,
                const float* __restrict__ beta, const float* __restrict__ res, long M, int C, int relu, int round, float* __restrict__ y, int ld_y,
                float* __restrict__ ypad, int H, int W) {
    const int C4 = C >> 2;
    const long total = M * C4;
    for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        const int c = (int)(i % C4) * 4;
        const long pix = i / C4;
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
        const float4 ov = make_float4(o[0], o[1], o[2], o[3]);
        *reinterpret_cast<float4*>(y + (size_t)pix * ld_y + c) = ov;
        if (ypad) {
            const int w = (int)(pix % W); const long t = pix / W; const int h = (int)(t % H); const long b = t / H;
            *reinterpret_cast<float4*>(ypad + (((size_t)b * (H + 2) + h + 1) * (W + 2) + w + 1) * C + c) = ov;
        }
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

// out[i] = sum_j part[j][i] over n chunks in fixed order (fp64).
__global__ void __launch_bounds__(256)
sum_chunks_kernel(const float* __restrict__ part, int n, long len, float* __restrict__ out) {
    for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < len; i += (long)gridDim.x * blockDim.x) {
        double s = 0.0;
        for (int j = 0; j < n; ++j) s += part[(size_t)j * len + i];
        out[i] = (float)s;
    }
}

// ---- per-call weight packing ------------------------------------------------------------------------------------------

constexpr int kMaxPackJobs = 40;           // jobs per launch (the kernel takes them by value)
struct PackJobs { PackJob j[kMaxPackJobs]; };

__host__ __device__ inline void pack_dims(const PackJob& q, int* N, int* K) {
    switch (q.kind) {
        case CONV3_FWD: *N = q.cout; *K = 9 * q.cin_p; break;
        case CONV3_DGRAD: *N = q.cin_p; *K = 9 * q.cout; break;
        case UP_FWD: *N = 4 * q.cout; *K = q.cin; break;
        case UP_DGRAD: *N = q.cin; *K = 4 * q.cout; break;
        case UP_BIAS: *N = 4 * q.cout; *K = 1; break;
        default: *N = q.rows; *K = q.cols; break;
    }
}

// W[n][k] of a non-MAT job (see PackKind).
__device__ inline float pack_value(const PackJob& q, int n, int k) {
    switch (q.kind) {
        case CONV3_FWD: { const int tap = k / q.cin_p, ci = k % q.cin_p; return ci < q.cin ? __ldg(q.src + ((size_t)n * q.cin + ci) * 9 + tap) : 0.f; }
        case CONV3_DGRAD: { const int tap = 8 - k / q.cout, co = k % q.cout; return n < q.cin ? __ldg(q.src + ((size_t)co * q.cin + n) * 9 + tap) : 0.f; }
        case UP_FWD: return __ldg(q.src + ((size_t)k * q.cout + n % q.cout) * 4 + n / q.cout);
        case UP_DGRAD: return __ldg(q.src + ((size_t)n * q.cout + k % q.cout) * 4 + k / q.cout);
        default: return __ldg(q.src + n % q.cout);                 // UP_BIAS
    }
}

__global__ void __launch_bounds__(256)
pack_kernel(const __grid_constant__ PackJobs p) {
    const PackJob& q = p.j[blockIdx.y];
    if (q.kind == MAT) {
        const int n = q.rows * q.cols;
        for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
            const int r = i / q.cols, c = i % q.cols;
            const float v = __ldg(q.src + i);
            const int d = q.transpose ? c * q.rows + r : i;
            const float hi = q.split ? smk::round_tf32(v) : v;
            q.hi[d] = hi;
            if (q.lo) q.lo[d] = smk::round_tf32(v - hi);
        }
        return;
    }
    int N, K;
    pack_dims(q, &N, &K);
    const int n_all = N * K;
    for (int d = blockIdx.x * blockDim.x + threadIdx.x; d < n_all; d += gridDim.x * blockDim.x) {
        const int n = q.split ? d / K : d % N, k = q.split ? d % K : d / N;    // TF32 [N][K] or fp32 [K][N]
        const float v = pack_value(q, n, k);
        const float hi = q.split ? smk::round_tf32(v) : v;
        q.hi[d] = hi;
        if (q.lo) q.lo[d] = smk::round_tf32(v - hi);
    }
}

}  // namespace

int bn_forward(const BnRef& r, const float* z, long M, int C, float eps, float momentum, float* mean, float* invstd, const float* res, bool relu,
               bool round, const BnOut& out, double2* part, cudaStream_t st) {
    const int nch = bn_chunks(M);
    const long chunk = cdiv(M, nch);
    SMK_TAG("bn_stats", 4.0 * M * C + 16.0 * nch * C, 3.0 * M * C, st);
    SMK_LAUNCH(bn_reduce_kernel<0>, dim3(cdiv(C, 32), nch), dim3(32, 8), 0, st, z, nullptr, nullptr, nullptr, nullptr, M, C, chunk, part);
    SMK_CHECK_LAUNCH();
    SMK_TAG("bn_finalize", 16.0 * nch * C + 24.0 * C, 0.0, st);
    SMK_LAUNCH(bn_finalize_fwd_kernel, dim3(1), dim3(256), 0, st, part, nch, M, C, eps, momentum, r.rmean, r.rvar, r.nbt, mean, invstd);
    SMK_CHECK_LAUNCH();
    SMK_TAG("bn_apply", 4.0 * M * C * ((res ? 3 : 2) + (out.pad ? 1 : 0)), 4.0 * M * C, st);
    SMK_LAUNCH(bn_apply_kernel, dim3(grid_of(M * C / 4)), dim3(256), 0, st, z, mean, invstd, r.gamma, r.beta, res, M, C, relu ? 1 : 0, round ? 1 : 0,
               out.y, out.ld, out.pad, out.H, out.W);
    SMK_CHECK_LAUNCH();
    return 0;
}

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

int channel_sum(const float* x, long M, int C, float* out, double2* part, float* gb, cudaStream_t st) {
    const int nch = bn_chunks(M);
    const long chunk = cdiv(M, nch);
    SMK_TAG("channel_sum", 4.0 * M * C + 16.0 * nch * C, (double)M * C, st);
    SMK_LAUNCH(bn_reduce_kernel<0>, dim3(cdiv(C, 32), nch), dim3(32, 8), 0, st, x, nullptr, nullptr, nullptr, nullptr, M, C, chunk, part);
    SMK_CHECK_LAUNCH();
    SMK_TAG("channel_sum_finalize", 16.0 * nch * C, 0.0, st);
    SMK_LAUNCH(bn_finalize_bwd_kernel, dim3(1), dim3(256), 0, st, part, nch, C, gb, nullptr, out);
    SMK_CHECK_LAUNCH();
    return 0;
}

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
    SMK_REQUIRE((size_t)nch * Co * Ci <= kWgradPart, "pw_wgrad: %d x %d weight gradient exceeds the split-K partials", Co, Ci);
    SMK_TAG("pw_wgrad", 4.0 * M * (Co + Ci) + 4.0 * nch * Co * Ci, 2.0 * M * Co * Ci, st);
    SMK_LAUNCH(pw_wgrad_kernel, dim3(cdiv(Ci, 64), cdiv(Co, 64), nch), dim3(256), 0, st, g, a, M, Co, Ci, chunk, part);
    SMK_CHECK_LAUNCH();
    return sum_chunks(part, nch, (long)Co * Ci, out, st);
}

size_t pack_floats(const PackJob& j) {
    int N, K;
    pack_dims(j, &N, &K);
    return (size_t)N * K;
}

int pack(const std::vector<PackJob>& jobs, double bytes, cudaStream_t st) {
    for (size_t j0 = 0; j0 < jobs.size(); j0 += kMaxPackJobs) {
        const int nj = (int)std::min<size_t>(kMaxPackJobs, jobs.size() - j0);
        PackJobs p{};
        size_t max_n = 432;
        for (int j = 0; j < nj; ++j) { p.j[j] = jobs[j0 + j]; max_n = std::max(max_n, pack_floats(p.j[j])); }
        SMK_TAG("train_pack", j0 == 0 ? bytes : 0.0, 0.0, st);
        SMK_LAUNCH(pack_kernel, dim3(std::min(cdiv((long)max_n, 256), 4096), nj), dim3(256), 0, st, p);
        SMK_CHECK_LAUNCH();
    }
    return 0;
}

}  // namespace trn
