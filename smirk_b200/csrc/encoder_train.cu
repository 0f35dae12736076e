// SmirkEncoder in train mode: BatchNorm over batch statistics (with the running-statistics update) and the weight, BN and
// head gradients, for the reference trainer's encoder steps (src/smirk_trainer.py:34-73 with base_trainer.py:108-111's
// .train()).
//
// A train handle holds the topology only: per backbone a flat list of conv + BatchNorm layers (enc::Layer, built from the
// blocks of enc::build_backbone), which the forward walks front to back and the backward back to front.  Every call reads
// the module's current parameters through device pointers (SmkEncoderTrainArgs) and repacks the 1x1 weights into the
// workspace, so an optimizer step needs no new handle.  The forward runs the unfused layer sequence (BN cannot be
// folded): per conv the pre-BN output z, then per BatchNorm a per-channel reduction over fixed pixel chunks (fp64 partial
// sums), a one-CTA finalise (mean, invstd, running stats, num_batches_tracked), and an apply step (gamma * xhat + beta,
// + skip, ReLU).  The backward runs per layer the BN backward (fixed-order fp64 sums of g and g * xhat, then g_z), the
// weight gradient as a split-K reduction over fixed pixel chunks with a fixed-order reduce, and the dgrad: a 1x1 through
// smk::conv over W^T, or a depthwise transposed conv.  No atomics: results are bitwise reproducible, and every call is
// CUDA-graph capturable.
#include "encoder.cuh"
#include "nn_kernels.cuh"
#include "gemm_tc.cuh"
#include "train_common.cuh"

namespace {

using namespace enc;
using namespace trn;
using smk::cdiv;
using smk::grid_of;
using smk::same_pad_begin;


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

// ---- weight gradients -------------------------------------------------------------------------------------------------

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

// ---- host side ----------------------------------------------------------------------------------------------------------

// Tensors of backbone i in tensor_list() order: 5 per conv (weight, gamma, beta, running_mean, running_var).
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

// floats of one copy of a backbone's 1x1 weights
size_t pw_floats(const Backbone& bb) {
    size_t n = 0;
    for (const Layer& L : bb.layers) if (L.op == PW) n += (size_t)L.cin * L.cout;
    return n;
}
int max_channels(const Backbone& bb) {
    int c = 0;
    for (const Layer& L : bb.layers) c = std::max(c, L.cout);
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

// Packs the backbone's 1x1 weights for the forward (dgrad = false: N = cout, K = cin) or the dgrad (true: N = cin,
// K = cout), and the stem's dgrad weights, in one launch.  packed[Layer::pw]: that 1x1 conv's operand.
int pack_weights(const SmkEncoder* h, const View& v, const BackboneWs& ws, bool dgrad, std::vector<smk::GemmW>& packed, cudaStream_t st) {
    const Backbone& bb = h->bb[v.i];
    const bool tc = h->precision >= 1;
    std::vector<PackJob> jobs;
    float* dst = ws.pw;
    packed.clear();
    auto add = [&](const float* w, int cin, int cout) {
        const size_t n = (size_t)cin * cout;
        // The layout rule of smk::pack_gemm: fp32 [K][N], or TF32 [N][K] split into heads (+ tails).  Torch's [cout][cin] is
        // the forward's [N][K] and the dgrad's [K][N], so it is transposed exactly when that is not the layout wanted.
        const bool torch_nk = !dgrad;
        if (!tc && !torch_nk) { packed.push_back(smk::GemmW{w, nullptr, nullptr}); return; }   // the fp32 dgrad reads it as is
        PackJob j{};
        j.src = w; j.rows = cout; j.cols = cin; j.hi = dst; j.lo = tc && h->x3 ? dst + n : nullptr;
        j.transpose = torch_nk != tc; j.split = tc;
        jobs.push_back(j);
        packed.push_back(tc ? smk::GemmW{nullptr, j.hi, j.lo} : smk::GemmW{j.hi, nullptr, nullptr});
        dst += n * (j.lo ? 2 : 1);
    };
    for (size_t k = 0; k < bb.layers.size(); ++k)
        if (bb.layers[k].op == PW) add(v.bn((int)k).w, bb.layers[k].cin, bb.layers[k].cout);
    if (dgrad) {                                          // stem [16][27] -> [27][16], the layout of stem_dgrad
        PackJob j{};
        j.src = v.bn(0).w; j.rows = 16; j.cols = 27; j.hi = ws.stem_t; j.lo = nullptr; j.transpose = 1; j.split = 0;
        jobs.push_back(j);
    }
    return trn::pack(jobs, 8.0 * pw_floats(bb) * (h->x3 ? 1.5 : 1.0), st);
}

// One 1x1 conv through smk::conv: out[m, :N] = in[m, :K] . W (+ res), unit scale and zero bias.
int conv1x1(const SmkEncoder* h, const smk::GemmW& w, const float* in, int K, int N, int B, int H, const float* res, float* out, bool round, const char* tag,
            cudaStream_t st) {
    smk::Conv q{};
    q.in = in; q.ld_in = K; q.B = B; q.H = H; q.W = H; q.Cin = K; q.N = N; q.K = K; q.mode = 0;
    q.wgt = w; q.scale = h->ones; q.bias = h->zeros;
    q.res = res; q.ld_res = N; q.out = out; q.ld_out = N; q.round_out = round ? 1 : 0; q.tag = tag;
    return smk::conv(q, st);
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

// The stem conv (3x3 stride 2 TF-SAME, one padding for both axes): img [B,3,H,W] -> z [B,Ho,Wo,16].
int stem_forward(const float* img, const float* w, int B, int H, int W, float* z, cudaStream_t st) {
    const int Ho = (H + 1) / 2, Wo = (W + 1) / 2;
    const long M = (long)B * Ho * Wo;
    SMK_TAG("stem_fwd", 4.0 * ((double)B * 3 * H * W + M * 16), 2.0 * 27 * 16 * M, st);
    SMK_LAUNCH(stem_fwd_kernel, dim3(cdiv(M, 128)), dim3(128), 0, st, img, w, B, H, W, Ho, Wo, same_pad_begin(H, 2), z);
    SMK_CHECK_LAUNCH();
    return 0;
}

// The stem's weight gradient from g [B,Ho,Wo,16] (gradient of z): split K over at most 512 chunks of >= 1024 pixels.
int stem_wgrad(const float* g, const float* img, int B, int H, int W, float* part, float* out, cudaStream_t st) {
    const int Ho = (H + 1) / 2, Wo = (W + 1) / 2;
    const long M = (long)B * Ho * Wo;
    const int nch = (int)std::min<long>(cdiv(M, 1024), 512);
    SMK_TAG("stem_wgrad", 4.0 * ((double)M * 16 + (double)B * 3 * H * W), 2.0 * 432 * M, st);
    SMK_LAUNCH(stem_wgrad_kernel, dim3(nch), dim3(448), 0, st, g, img, B, H, W, Ho, Wo, same_pad_begin(H, 2), cdiv(M, nch), part);
    SMK_CHECK_LAUNCH();
    return sum_chunks(part, nch, 432, out, st);
}

// The head's backward: g [B][n_out] (gradient of the clamped output) -> gp (gradient of the pre-clamp output), gy
// [B,HW,C] (of the features before the pool), and the head's weight gradients gw [n_out][C] / gbias [n_out] (either may
// be null) from the pooled features [B][C].
int head_backward(const float* g, const float* raw, const uint8_t* codes, const float* w, const float* pooled, int B, int n_out, int HW, int C,
                  float* gp, float* gy, float* gw, float* gbias, cudaStream_t st) {
    SMK_TAG("train_head_bwd", 4.0 * ((double)B * HW * C + (double)n_out * C + 3.0 * B * n_out), 2.0 * B * C * n_out, st);
    SMK_LAUNCH(head_bwd_train_kernel, dim3(B, cdiv(C, 256)), dim3(256), (size_t)n_out * 4, st, g, raw, codes, w, n_out, HW, C, gp, gy);
    SMK_CHECK_LAUNCH();
    if (gw || gbias) {
        SMK_TAG("train_head_wgrad", 4.0 * ((double)B * (n_out + C) + (double)n_out * C), 2.0 * B * C * n_out, st);
        SMK_LAUNCH(head_wgrad_kernel, dim3(cdiv((long)n_out * (C + 1), 256)), dim3(256), 0, st, gp, pooled, B, n_out, C, gw, gbias);
        SMK_CHECK_LAUNCH();
    }
    return 0;
}

// Backbone i of a train handle: the layer list, and with it the saved layout (names: the reference's module paths — a
// conv's pre-BN output under the conv, a ReLU output under its BatchNorm as in the eval layout, a block's output under the
// block, the pooled features under `<encoder>.pooled`, a head's pre-clamp output under the head) and the BatchNorm
// statistics after the saved tensors (backbones in slot order; per BatchNorm mean[C], then invstd[C]).
void build_layers(SmkEncoder* h, int i) {
    build_backbone(h, i);
    Backbone& bb = h->bb[i];
    const std::string enc = std::string(kEncName[i]) + ".";
    int n_pw = 0;
    // One conv (cin -> cout at resolution hin) + BatchNorm, fed by the previous layer; y: the name of the BatchNorm's output.
    auto add = [&](Op op, int cin, int cout, int stride, int hin, const std::string& conv, const std::string& y, bool relu) {
        Layer L{};
        L.op = op; L.cin = cin; L.cout = cout; L.stride = stride; L.hin = hin; L.hout = (hin + stride - 1) / stride;
        L.sv_in = bb.layers.empty() ? -1 : bb.layers.back().sv_y;
        L.sv_z = h->saved.add(conv, L.hout, L.hout, cout);
        L.sv_y = h->saved.add(y, L.hout, L.hout, cout);
        L.relu = relu; L.skip = -1;
        L.stats = h->stats_floats; h->stats_floats += 2 * (size_t)cout;
        L.pw = op == PW ? n_pw++ : -1;
        bb.layers.push_back(L);
    };
    add(STEM, 3, 16, 2, 224, enc + "encoder.conv_stem", enc + "encoder.bn1", true);
    for (const Block& b : bb.blocks) {
        const size_t first = bb.layers.size();
        const int block_in = bb.layers.back().sv_y;
        if (b.kind == IR) add(PW, b.cin, b.mid, 1, b.hin, b.path + ".conv_pw", b.path + ".bn1", true);
        if (b.kind != CN) add(DW, b.mid, b.mid, b.stride, b.hin, b.path + ".conv_dw", b.path + (b.kind == IR ? ".bn2" : ".bn1"), true);
        if (b.kind == CN) add(PW, b.cin, b.cout, 1, b.hout, b.path + ".conv", b.path + ".bn1", true);
        else add(PW, b.mid, b.cout, 1, b.hout, b.path + (b.kind == IR ? ".conv_pwl" : ".conv_pw"), b.path, false);
        bb.layers[first].first = true;
        if (b.skip) bb.layers.back().skip = block_in;
    }
    bb.sv_pool = h->saved.add(enc + "pooled", 1, 1, bb.feat);
    bb.sv_head = h->saved.add(enc + kHeadName[i], 1, 1, bb.n_out);
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
    for (int i = 0; i < 3; ++i) {
        h->present[i] = (backbones >> i) & 1;
        if (h->present[i]) build_layers(h, i);
    }
    const cudaError_t e = finish_create(h);
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

int check_args(const SmkEncoder* h, const SmkEncoderTrainArgs* a, const char* fn) {
    SMK_REQUIRE(h && h->train, "%s: not a train-mode handle (smk_encoder_train_create)", fn);
    SMK_REQUIRE(a, "%s: null args", fn);
    for (int i = 0; i < 3; ++i) {
        if (!h->present[i]) continue;
        const int nbn = (int)h->bb[i].layers.size();
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
        std::vector<smk::GemmW> pk;
        if (int rc = pack_weights(h, v, W, false, pk, st)) return rc;
        for (size_t k = 0; k < bb.layers.size(); ++k) {
            const Layer& L = bb.layers[k];
            const BnRef r = v.bn((int)k);
            int rc;
            if (L.op == STEM) rc = stem_forward(img, r.w, B, L.hin, L.hin, SV(L.sv_z), st);
            else if (L.op == PW) rc = conv1x1(h, pk[L.pw], SV(L.sv_in), L.cin, L.cout, B, L.hin, nullptr, SV(L.sv_z), false, "train_pw", st);
            else rc = dw_forward(SV(L.sv_in), r.w, B, L.hin, L.cin, L.stride, SV(L.sv_z), st);
            if (rc) return rc;
            // At precisions 1-2 every BatchNorm output inside a block is TF32-rounded, also one that feeds the depthwise conv,
            // while the stem's never is, and no 1x1 conv rounds its own output: results stay bitwise what they have been.
            float* mean = stats + L.stats;
            rc = bn_forward(r, SV(L.sv_z), (long)B * L.hout * L.hout, L.cout, eps, mom, mean, mean + L.cout, L.skip >= 0 ? SV(L.skip) : nullptr,
                            L.relu, rnd && L.op != STEM, BnOut{SV(L.sv_y), L.cout}, W.part, st);
            if (rc) return rc;
        }
        const float* x = SV(bb.layers.back().sv_y);
        const int res = bb.layers.back().hout;
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
        std::vector<smk::GemmW> pk;
        if (int rc = pack_weights(h, v, W, true, pk, st)) return rc;
        // g: the gradient of the current layer's output; out: where its dgrad goes; held: the gradient of a block's output, kept
        // from the block's last layer to its first, where the skip connection adds it to the gradient of the block's input
        float *g = W.buf[0], *out = W.buf[1], *spare = W.buf[2], *held = nullptr;
        const Layer& top = bb.layers.back();
        if (int rc = head_backward(g_out[i], SV(bb.sv_head), bb.codes, args->head_w[i], SV(bb.sv_pool), B, bb.n_out, top.hout * top.hout, bb.feat, W.gp, g,
                                   grads ? grads->head_w[i] : nullptr, grads ? grads->head_b[i] : nullptr, st))
            return rc;
        for (int k = (int)bb.layers.size() - 1; k >= 0; --k) {
            const Layer& L = bb.layers[k];
            const BnRef r = v.bn(k);
            const long M = (long)B * L.hout * L.hout;
            const float* mean = stats + L.stats;
            float* gz = L.skip >= 0 ? out : g;        // in place, unless g is to be held
            // Every BatchNorm backward rounds its result at precisions 1-2, whatever consumes it, and no 1x1 dgrad rounds
            // its own: results stay bitwise what they have been.
            int rc = bn_backward(r, g, L.relu ? SV(L.sv_y) : nullptr, SV(L.sv_z), mean, mean + L.cout, M, L.cout, rnd, gz, W.part, W.gb, st);
            if (rc) return rc;
            if (L.skip >= 0) { held = g; g = out; out = spare; }
            if (r.gw) {
                if (L.op == STEM) rc = stem_wgrad(g, img, B, L.hin, L.hin, W.wpart, r.gw, st);
                else if (L.op == PW) rc = pw_wgrad(g, SV(L.sv_in), M, L.cout, L.cin, W.wpart, r.gw, st);
                else rc = dw_wgrad(g, SV(L.sv_in), B, L.hin, L.cin, L.stride, W.wpart, r.gw, st);
                if (rc) return rc;
            }
            if (L.op == STEM) break;                  // g: the gradient of the stem's pre-BN output; its dgrad runs after the join
            const float* res = L.first ? held : nullptr;
            if (L.op == PW) rc = conv1x1(h, pk[L.pw], g, L.cout, L.cin, B, L.hin, res, out, false, "train_pw_dgrad", st);
            else rc = dw_dgrad(g, r.w, res, B, L.hin, L.cin, L.stride, out, st);
            if (rc) return rc;
            std::swap(g, out);
            if (res) { spare = held; held = nullptr; }
        }
        g_stem[i] = g; w_stem[i] = W.stem_t;
        return 0;
    });
    if (rc || !g_img) return rc;
    return enc::stem_dgrad(g_stem, w_stem, B, g_img, main_st);
}

// ---- test entry points (smk_debug_train_*): each runs the host helper of the train path ------------------------------

namespace {

BnRef debug_bn(const float* gamma, const float* beta, float* rmean, float* rvar, int64_t* nbt, float* g_gamma, float* g_beta) {
    BnRef r{};
    r.gamma = const_cast<float*>(gamma); r.beta = const_cast<float*>(beta); r.rmean = rmean; r.rvar = rvar; r.nbt = (long long*)nbt;
    r.ggamma = g_gamma; r.gbeta = g_beta;
    return r;
}

int check_dw(const char* fn, int B, int H, int C, int stride) {
    SMK_REQUIRE(B > 0 && H > 0 && C > 0, "%s: B, H and C must be positive", fn);
    SMK_REQUIRE(stride == 1 || stride == 2, "%s: stride must be 1 or 2", fn);
    return 0;
}

}  // namespace

extern "C" int smk_debug_train_bn_forward(const float* z, int M, int C, float eps, float momentum, const float* gamma, const float* beta,
                                          float* rmean, float* rvar, int64_t* nbt, const float* res, int relu, int round, float* mean,
                                          float* invstd, float* y, void* ws, size_t ws_bytes, void* stream) {
    const char* fn = "smk_debug_train_bn_forward";
    SMK_REQUIRE(z && gamma && beta && rmean && rvar && nbt && mean && invstd && y && ws, "%s: null argument", fn);
    SMK_REQUIRE(M > 0 && C > 0 && C % 4 == 0, "%s: M > 0 and C > 0 with C %% 4 == 0 (the apply reads float4)", fn);
    SMK_REQUIRE(momentum <= 1.f && eps > 0.f, "%s: momentum must be in [0, 1] (or negative for None) and eps > 0", fn);
    smk::Workspace w(ws, ws_bytes);
    double2* part = w.take<double2>((size_t)kMaxChunks * C);
    SMK_REQUIRE(part, "%s: workspace too small", fn);
    return bn_forward(debug_bn(gamma, beta, rmean, rvar, nbt, nullptr, nullptr), z, M, C, eps, momentum, mean, invstd, res, relu != 0, round != 0,
                      BnOut{y, C}, part, (cudaStream_t)stream);
}

extern "C" int smk_debug_train_bn_backward(const float* g, const float* y, const float* z, const float* mean, const float* invstd,
                                           const float* gamma, int M, int C, int round, float* gz, float* g_gamma, float* g_beta, void* ws,
                                           size_t ws_bytes, void* stream) {
    const char* fn = "smk_debug_train_bn_backward";
    SMK_REQUIRE(g && z && mean && invstd && gamma && gz && ws, "%s: null argument", fn);
    SMK_REQUIRE(M > 0 && C > 0, "%s: M and C must be positive", fn);
    smk::Workspace w(ws, ws_bytes);
    double2* part = w.take<double2>((size_t)kMaxChunks * C);
    float* gb = w.take<float>(2 * (size_t)C);
    SMK_REQUIRE(part && gb, "%s: workspace too small", fn);
    return bn_backward(debug_bn(gamma, nullptr, nullptr, nullptr, nullptr, g_gamma, g_beta), g, y, z, mean, invstd, M, C, round != 0, gz, part, gb,
                       (cudaStream_t)stream);
}

extern "C" int smk_debug_train_pw_wgrad(const float* g, const float* a, int M, int Co, int Ci, float* out, void* ws, size_t ws_bytes, void* stream) {
    const char* fn = "smk_debug_train_pw_wgrad";
    SMK_REQUIRE(g && a && out && ws, "%s: null argument", fn);
    SMK_REQUIRE(M > 0 && Co > 0 && Ci > 0, "%s: M, Co and Ci must be positive", fn);
    smk::Workspace w(ws, ws_bytes);
    float* part = w.take<float>(kWgradPart);
    SMK_REQUIRE(part, "%s: workspace too small", fn);
    return pw_wgrad(g, a, M, Co, Ci, part, out, (cudaStream_t)stream);
}

extern "C" int smk_debug_train_dw_forward(const float* a, const float* w, int B, int H, int C, int stride, float* z, void* stream) {
    const char* fn = "smk_debug_train_dw_forward";
    SMK_REQUIRE(a && w && z, "%s: null argument", fn);
    if (int rc = check_dw(fn, B, H, C, stride)) return rc;
    return dw_forward(a, w, B, H, C, stride, z, (cudaStream_t)stream);
}

extern "C" int smk_debug_train_dw_wgrad(const float* g, const float* a, int B, int H, int C, int stride, float* out, void* ws, size_t ws_bytes,
                                        void* stream) {
    const char* fn = "smk_debug_train_dw_wgrad";
    SMK_REQUIRE(g && a && out && ws, "%s: null argument", fn);
    if (int rc = check_dw(fn, B, H, C, stride)) return rc;
    smk::Workspace w(ws, ws_bytes);
    float* part = w.take<float>(kWgradPart);
    SMK_REQUIRE(part, "%s: workspace too small", fn);
    return dw_wgrad(g, a, B, H, C, stride, part, out, (cudaStream_t)stream);
}

extern "C" int smk_debug_train_dw_dgrad(const float* g, const float* w, const float* res, int B, int H, int C, int stride, float* out, void* stream) {
    const char* fn = "smk_debug_train_dw_dgrad";
    SMK_REQUIRE(g && w && out, "%s: null argument", fn);
    if (int rc = check_dw(fn, B, H, C, stride)) return rc;
    return dw_dgrad(g, w, res, B, H, C, stride, out, (cudaStream_t)stream);
}

extern "C" int smk_debug_train_stem_forward(const float* img, const float* w, int B, int H, int W, float* z, void* stream) {
    const char* fn = "smk_debug_train_stem_forward";
    SMK_REQUIRE(img && w && z, "%s: null argument", fn);
    SMK_REQUIRE(B > 0 && H > 0 && W > 0, "%s: B, H and W must be positive", fn);
    SMK_REQUIRE(same_pad_begin(H, 2) == same_pad_begin(W, 2), "%s: H and W must have the same parity (one TF-SAME padding)", fn);
    return stem_forward(img, w, B, H, W, z, (cudaStream_t)stream);
}

extern "C" int smk_debug_train_stem_wgrad(const float* g, const float* img, int B, int H, int W, float* out, void* ws, size_t ws_bytes, void* stream) {
    const char* fn = "smk_debug_train_stem_wgrad";
    SMK_REQUIRE(g && img && out && ws, "%s: null argument", fn);
    SMK_REQUIRE(B > 0 && H > 0 && W > 0, "%s: B, H and W must be positive", fn);
    SMK_REQUIRE(same_pad_begin(H, 2) == same_pad_begin(W, 2), "%s: H and W must have the same parity (one TF-SAME padding)", fn);
    smk::Workspace w(ws, ws_bytes);
    float* part = w.take<float>(kWgradPart);
    SMK_REQUIRE(part, "%s: workspace too small", fn);
    return stem_wgrad(g, img, B, H, W, part, out, (cudaStream_t)stream);
}

extern "C" int smk_debug_train_head_backward(const float* g, const float* raw, const uint8_t* codes, const float* w, const float* pooled, int B,
                                             int n_out, int HW, int C, float* gp, float* g_feat, float* g_w, float* g_b, void* stream) {
    const char* fn = "smk_debug_train_head_backward";
    SMK_REQUIRE(g && raw && w && pooled && gp && g_feat, "%s: null argument", fn);
    SMK_REQUIRE(B > 0 && n_out > 0 && n_out <= 4096 && HW > 0 && C > 0, "%s: B, HW and C must be positive and n_out in [1, 4096]", fn);
    return head_backward(g, raw, codes, w, pooled, B, n_out, HW, C, gp, g_feat, g_w, g_b, (cudaStream_t)stream);
}
