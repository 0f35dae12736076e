// VGGPerceptualLoss forward and input gradient (src/losses/VGGPerceptualLoss.py): torchvision VGG16 features[:23], frozen,
// on x and y normalised as (v * 0.5 + 0.5 - mean) / std; loss = sum over the taps relu1_2, relu2_2, relu3_3, relu4_3 of
// l1_loss(phi(x), phi(y)), in that order.  The resize to 224^2 the reference applies is the identity at 224^2, the only size
// accepted here.
//
// x and y run as one batch of 2B images (NHWC fp32), so each layer is one launch: vgg_prep_kernel normalises and converts
// both inputs, the ten 3x3 convs (bias, ReLU) run through smk::conv on the same kernels and precisions as SmirkGenerator's
// (0 = fp32 CUDA cores, 1 = TF32 wgmma with TF32-rounded activations, 3 = 3xTF32 wgmma), the pools through
// smk::maxpool2x2.  At each tap vgg_l1_kernel sums |phi(x) - phi(y)| per fixed chunk into one partial per CTA, and
// vgg_l1_finalize_kernel adds each tap's partials in a fixed order and the four means as ((l0 + l1) + l2) + l3: no atomics,
// the same bits on every run.
//
// Input gradient (frozen weights): the grad-mode forward also keeps the post-ReLU output of every conv for the half (x, y)
// or halves whose gradient is wanted (the conv epilogue's second store, limited to those images: they come first in the
// batch, y before x when only y's gradient is wanted) and, per tap, sign(phi(x) - phi(y)) as int8.  The backward then runs
// only over those images: at each tap vgg_pool_l1_bwd_kernel adds sign * g / N (negated for y) to the max-pool backward of
// the deeper gradient and applies the tap's ReLU mask; every conv's dgrad is a 3x3 conv with the rotated, transposed
// weights (smk::pack_conv3, as the generator's) whose epilogue applies the ReLU mask of its input; vgg_input_bwd_kernel
// undoes the normalisation into NCHW.
#include "nn_kernels.cuh"
#include "gemm_tc.cuh"
#include "../../include/smirk_b200_loss.h"
#include <string>

namespace {

constexpr int kConvs = 10, kTaps = 4;
constexpr int kStage[kConvs] = {0, 0, 1, 1, 2, 2, 2, 3, 3, 3};      // stage s runs at 224 >> s, with 64 << s channels
constexpr int kTapConv[kTaps] = {1, 3, 6, 9};                       // the last conv of each stage
const char* const kActName[kConvs] = {"relu1_1", "relu1_2", "relu2_1", "relu2_2", "relu3_1", "relu3_2", "relu3_3",
                                      "relu4_1", "relu4_2", "relu4_3"};
const char* const kSignName[kTaps] = {"sign1_2", "sign2_2", "sign3_3", "sign4_3"};
constexpr size_t kActMax = (size_t)224 * 224 * 64;                  // floats per image of the largest activation
constexpr int kChunk4 = 4096;                                       // float4s per vgg_l1_kernel CTA (16384 elements)

struct Norm { float mean[3], std[3]; };

struct VggConv { smk::Conv3Weights pk; float* bias; int cin, cin_p, cout, S; };

int tap_S(int t) { return 224 >> t; }
int tap_C(int t) { return 64 << t; }
size_t tap_elems(int t) { return (size_t)tap_S(t) * tap_S(t) * tap_C(t); }          // per image
int n_partials(int B, int t) { return smk::cdiv((long)(B * tap_elems(t) / 4), kChunk4); }

// ---- kernels ---------------------------------------------------------------------------------------------------------
__device__ __forceinline__ float pick3(const float (&v)[3], int c) { return c == 0 ? v[0] : c == 1 ? v[1] : v[2]; }   // no local copy

// NCHW x (images [0, B)) and y (images [B, 2B)) -> NHWC [2B, HW, Cp], ((v * 0.5) + 0.5 - mean[c]) / std[c] with the
// reference's separate fp32 operations (no contraction), channels 3..Cp-1 zero; round: TF32 for a TF32 consumer.
__global__ void __launch_bounds__(256)
vgg_prep_kernel(const float* __restrict__ x, const float* __restrict__ y, int B, int HW, int Cp, Norm nm, int round, float* __restrict__ out) {
    const int Q = Cp >> 2;
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= 2L * B * HW * Q) return;
    const int q = (int)(i % Q); const long pix = i / Q;
    const int b = (int)(pix / HW), r = (int)(pix - (long)b * HW);
    const float* src = b < B ? x + (size_t)b * 3 * HW : y + (size_t)(b - B) * 3 * HW;
    float v[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const int c = q * 4 + k;
        float t = 0.f;
        if (c < 3) {
            t = __fadd_rn(__fmul_rn(__ldg(src + (size_t)c * HW + r), 0.5f), 0.5f);
            t = __fdiv_rn(__fsub_rn(t, pick3(nm.mean, c)), pick3(nm.std, c));
            if (round) t = smk::round_tf32(t);
        }
        v[k] = t;
    }
    reinterpret_cast<float4*>(out)[i] = make_float4(v[0], v[1], v[2], v[3]);
}

// Sum over the 256 threads of a block in a fixed order; the result is valid in thread 0.
__device__ float block_sum(float v) {
    __shared__ float wsum[8];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) wsum[threadIdx.x >> 5] = v;
    __syncthreads();
    float t = 0.f;
    if (threadIdx.x == 0)
        for (int w = 0; w < 8; ++w) t += wsum[w];
    __syncthreads();
    return t;
}

__device__ __forceinline__ signed char sgn(float d) { return (signed char)((d > 0.f) - (d < 0.f)); }

// One tap: partial[cta] = sum of |d| over the CTA's chunk of kChunk4 float4s, d = phi(x) - phi(y); a holds the batch's first
// B images, b the next B (swap: a is y's).  sign (optional): int8 sign(d), NHWC like the activations.
__global__ void __launch_bounds__(256)
vgg_l1_kernel(const float4* __restrict__ a, const float4* __restrict__ b, long n4, int swap, char4* __restrict__ sign,
              float* __restrict__ partial) {
    const long base = (long)blockIdx.x * kChunk4;
    float s = 0.f;
    for (int j = threadIdx.x; j < kChunk4; j += 256) {
        const long i = base + j;
        if (i >= n4) break;
        const float4 u = __ldg(a + i), v = __ldg(b + i);
        const float4 d = swap ? make_float4(v.x - u.x, v.y - u.y, v.z - u.z, v.w - u.w)
                              : make_float4(u.x - v.x, u.y - v.y, u.z - v.z, u.w - v.w);
        s += fabsf(d.x); s += fabsf(d.y); s += fabsf(d.z); s += fabsf(d.w);
        if (sign) sign[i] = make_char4(sgn(d.x), sgn(d.y), sgn(d.z), sgn(d.w));
    }
    s = block_sum(s);
    if (threadIdx.x == 0) partial[blockIdx.x] = s;
}

struct TapSums { int count[kTaps]; float numel[kTaps]; };

// loss = ((l0 + l1) + l2) + l3, l_t = (sum of tap t's partials, fixed order) / numel_t.  One block.
__global__ void __launch_bounds__(256)
vgg_l1_finalize_kernel(const float* __restrict__ partial, TapSums ts, float* __restrict__ loss) {
    float total = 0.f;
    for (int t = 0; t < kTaps; ++t) {
        float s = 0.f;
        for (int i = threadIdx.x; i < ts.count[t]; i += 256) s += partial[i];
        s = block_sum(s);
        if (threadIdx.x == 0) total = t == 0 ? s / ts.numel[t] : total + s / ts.numel[t];
        partial += ts.count[t];
    }
    if (threadIdx.x == 0) *loss = total;
}

// Gradient at a tap's ReLU output e [Bc,S,S,C] (the chain's images: the first B are x's unless swap, the next B y's), with
// respect to the conv output before the ReLU:  (pool backward of gp [Bc,S/2,S/2,C] (first maximum of each window in
// row-major order; gp null: none) + sign * (g / numel) (negated for y)) * [e > 0].
__global__ void __launch_bounds__(256)
vgg_pool_l1_bwd_kernel(const float* __restrict__ e, const char4* __restrict__ sign, const float* __restrict__ gp,
                       const float* __restrict__ g, float numel, int B, int Bc, int swap, int S, int C, int round,
                       float* __restrict__ out) {
    const int Ho = S >> 1, C4 = C >> 2;
    const long total = (long)Bc * Ho * Ho * C4;
    const float gn = __fdiv_rn(__ldg(g), numel);
    for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        const int c4 = (int)(i % C4); const long pix = i / C4;
        const int ow = (int)(pix % Ho); const long t = pix / Ho; const int oh = (int)(t % Ho); const int b = (int)(t / Ho);
        const float gs = b < B && !swap ? gn : -gn;                   // y takes -sign
        const size_t p00 = ((size_t)b * S + 2 * oh) * S + 2 * ow;
        const size_t px[4] = {p00, p00 + 1, p00 + S, p00 + S + 1};
        const size_t shift = b >= B ? (size_t)B * S * S : 0;           // the sign maps hold one image per face
        float v[4][4], r[4][4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const float4 a = __ldg(reinterpret_cast<const float4*>(e + px[k] * C) + c4);
            const char4 s = sign[(px[k] - shift) * C4 + c4];
            v[k][0] = a.x; v[k][1] = a.y; v[k][2] = a.z; v[k][3] = a.w;
            r[k][0] = s.x > 0 ? gs : s.x < 0 ? -gs : 0.f; r[k][1] = s.y > 0 ? gs : s.y < 0 ? -gs : 0.f;
            r[k][2] = s.z > 0 ? gs : s.z < 0 ? -gs : 0.f; r[k][3] = s.w > 0 ? gs : s.w < 0 ? -gs : 0.f;
        }
        if (gp) {
            const float4 q = __ldg(reinterpret_cast<const float4*>(gp + (size_t)pix * C) + c4);
            const float gv[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
            for (int ch = 0; ch < 4; ++ch) {
                const float mx = fmaxf(fmaxf(v[0][ch], v[1][ch]), fmaxf(v[2][ch], v[3][ch]));
                const int arg = v[0][ch] == mx ? 0 : v[1][ch] == mx ? 1 : v[2][ch] == mx ? 2 : 3;
#pragma unroll
                for (int k = 0; k < 4; ++k)
                    if (k == arg) r[k][ch] += gv[ch];
            }
        }
#pragma unroll
        for (int k = 0; k < 4; ++k) {
#pragma unroll
            for (int ch = 0; ch < 4; ++ch) {
                const float m = v[k][ch] > 0.f ? r[k][ch] : 0.f;
                r[k][ch] = round ? smk::round_tf32(m) : m;
            }
            reinterpret_cast<float4*>(out + px[k] * C)[c4] = make_float4(r[k][0], r[k][1], r[k][2], r[k][3]);
        }
    }
}

// conv1_1's input gradient [Bc,HW,Cp] NHWC -> NCHW, first 3 channels, (g / std[c]) * 0.5 (the order autograd applies the
// normalisation's backward in); images [0, B) to out0, [B, Bc) to out1.
__global__ void __launch_bounds__(256)
vgg_input_bwd_kernel(const float* __restrict__ g, int B, int Bc, int HW, int Cp, Norm nm, float* __restrict__ out0,
                     float* __restrict__ out1) {
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long)Bc * 3 * HW) return;
    const int r = (int)(i % HW); const long t = i / HW; const int c = (int)(t % 3); const int b = (int)(t / 3);
    const float v = __fmul_rn(__fdiv_rn(__ldg(g + ((size_t)b * HW + r) * Cp + c), pick3(nm.std, c)), 0.5f);
    if (b < B) out0[i] = v;
    else out1[i - 3L * B * HW] = v;
}

}  // namespace

struct SmkVggLoss {
    int precision;
    VggConv conv[kConvs];
    Norm norm;
    float *ones = nullptr, *zeros = nullptr;      // unit scale of every epilogue, zero bias of the dgrads
    size_t act_off[kConvs], act_total = 0;        // per-image float offsets of the saved activations
    size_t sign_off[kTaps], sign_total = 0;       // per-face float offsets of the int8 sign maps
    smk::DeviceArena arena;
};

extern "C" int smk_vgg_loss_create(const SmkVggLossDesc* desc, SmkVggLoss** out) {
    SMK_REQUIRE(desc && out && desc->tensors, "smk_vgg_loss_create: null argument");
    SMK_REQUIRE(desc->precision == 0 || desc->precision == 1 || desc->precision == 3,
                "smk_vgg_loss_create: precision must be 0, 1 or 3 (0 = fp32 CUDA cores, 1 = TF32 wgmma, 3 = 3xTF32 wgmma: fp32-equivalent)");
    SMK_REQUIRE(desc->n_tensors == 2 + 2 * kConvs,
                "smk_vgg_loss_create: expected %d tensors (mean, std, then weight and bias of 10 convs), got %d", 2 + 2 * kConvs, desc->n_tensors);
    for (int i = 0; i < desc->n_tensors; ++i) SMK_REQUIRE(desc->tensors[i], "smk_vgg_loss_create: tensor %d is null", i);
    const bool tc = desc->precision != 0, x3 = desc->precision == 3;
    if (tc) { if (int rc = smk::tc_init()) return rc; }
    SmkVggLoss* h = new SmkVggLoss();
    h->precision = desc->precision;
    for (int c = 0; c < 3; ++c) { h->norm.mean[c] = desc->tensors[0][c]; h->norm.std[c] = desc->tensors[1][c]; }
    cudaError_t e = cudaSuccess;
    for (int l = 0; l < kConvs && e == cudaSuccess; ++l) {
        VggConv& c = h->conv[l];
        c.S = 224 >> kStage[l]; c.cout = 64 << kStage[l];
        c.cin = l == 0 ? 3 : h->conv[l - 1].cout;
        c.cin_p = l > 0 ? c.cin : tc ? 32 : 8;         // the tensor-core path reads 128-byte pixel rows
        e = smk::pack_conv3(desc->tensors[2 + 2 * l], nullptr, c.cin, c.cin_p, c.cout, tc, x3, h->arena, &c.pk);
        if (e == cudaSuccess) e = h->arena.upload(desc->tensors[3 + 2 * l], (size_t)c.cout, &c.bias);
    }
    const std::vector<float> one(512, 1.f), zero(512, 0.f);
    if (e == cudaSuccess) e = h->arena.upload(one, &h->ones);
    if (e == cudaSuccess) e = h->arena.upload(zero, &h->zeros);
    if (e != cudaSuccess) {
        smk::set_error("smk_vgg_loss_create: upload failed: %s", cudaGetErrorString(e));
        delete h; return (int)e;
    }
    for (int l = 0; l < kConvs; ++l) {               // every size is a multiple of 64 floats
        h->act_off[l] = h->act_total;
        h->act_total += (size_t)h->conv[l].S * h->conv[l].S * h->conv[l].cout;
    }
    for (int t = 0; t < kTaps; ++t) { h->sign_off[t] = h->sign_total; h->sign_total += tap_elems(t) / 4; }
    *out = h;
    return 0;
}

extern "C" void smk_vgg_loss_destroy(SmkVggLoss* h) { delete h; }

namespace {

int halves(int need) { return need == 3 ? 2 : 1; }

size_t total_partials(int B) {
    size_t n = 0;
    for (int t = 0; t < kTaps; ++t) n += n_partials(B, t);
    return n;
}

// One 3x3 conv + bias + ReLU over the 2B-image batch; out2: the saved copy of the first out2_imgs images.
int conv_fwd(const SmkVggLoss* h, const VggConv& c, const float* in, int B2, float* out, float* out2, int out2_imgs, bool round,
             cudaStream_t st) {
    smk::Conv p{};
    p.in = in; p.ld_in = c.cin_p; p.B = B2; p.H = c.S; p.W = c.S; p.Cin = c.cin_p;
    p.w = c.pk.w; p.wt = c.pk.wt; p.wt_lo = c.pk.wt_lo; p.scale = h->ones; p.bias = c.bias;
    p.N = c.cout; p.K = 9 * c.cin_p; p.mode = 1; p.relu = 1; p.out = out; p.ld_out = c.cout;
    p.round_out = round ? 1 : 0;
    p.out2 = out2; p.ld_out2 = c.cout; p.out2_rows = out2_imgs * c.S * c.S;
    return smk::conv(p, st);
}

// dgrad of conv c over Bc images: g_in = conv3x3(g, W') * [mask > 0] (mask: the saved input activation, or null).
int conv_dgrad(const SmkVggLoss* h, const VggConv& c, const float* g, int Bc, const float* mask, float* out, bool round, cudaStream_t st) {
    const bool tc = h->precision != 0;
    smk::Conv p{};
    p.in = g; p.ld_in = c.cout; p.B = Bc; p.H = c.S; p.W = c.S; p.Cin = c.cout;
    p.w = tc ? nullptr : c.pk.dw; p.wt = tc ? c.pk.dw : nullptr; p.wt_lo = c.pk.dw_lo;
    p.scale = h->ones; p.bias = h->zeros;
    p.N = c.cin_p; p.K = 9 * c.cout; p.mode = 1; p.out = out; p.ld_out = c.cin_p; p.round_out = round ? 1 : 0;
    p.mask = mask; p.ld_mask = c.cin_p;
    p.tag = c.pk.dw_lo ? "vgg_conv_dgrad_tc3x" : tc ? "vgg_conv_dgrad_tc" : "vgg_conv_dgrad_f32";
    return smk::conv(p, st);
}

// The forward.  need == 0: the forward-only path.  Otherwise the activations of the first halves(need) * B images (y's
// first when need == 2) are also stored to `saved`, and the sign maps.  The arithmetic is the same.
int vgg_forward(const SmkVggLoss* h, const float* x, const float* y, int B, int need, float* loss, float* saved, void* ws,
                size_t ws_bytes, cudaStream_t st) {
    const bool swap = need == 2;
    const int B2 = 2 * B, nsv = need ? halves(need) * B : 0;
    smk::Workspace w(ws, ws_bytes);
    float* A = w.take<float>(kActMax * B2);
    float* Bf = w.take<float>(kActMax * B2);
    float* part = w.take<float>(total_partials(B));
    SMK_REQUIRE(part, "smk_vgg_loss_forward: workspace carve-up failed");
    int8_t* signs = saved ? reinterpret_cast<int8_t*>(saved + h->act_total * nsv) : nullptr;
    const int cin_p = h->conv[0].cin_p;
    {
        const long total = (long)B2 * 224 * 224 * (cin_p / 4);
        SMK_TAG("vgg_prep", 4.0 * B2 * 224.0 * 224.0 * (3 + cin_p), 0.0, st);
        SMK_LAUNCH(vgg_prep_kernel, dim3(smk::cdiv(total, 256)), dim3(256), 0, st, swap ? y : x, swap ? x : y, B, 224 * 224, cin_p,
                   h->norm, h->precision == 1 ? 1 : 0, Bf);
        SMK_CHECK_LAUNCH();
    }
    const float* in = Bf;
    float* o = A;
    float* pp = part;
    TapSums ts{};
    int rc, t = 0;
    for (int l = 0; l < kConvs; ++l) {
        const VggConv& c = h->conv[l];
        if (l > 0 && c.S != h->conv[l - 1].S) {
            const VggConv& q = h->conv[l - 1];
            if ((rc = smk::maxpool2x2(in, q.cout, B2, q.S, q.S, q.cout, o, st))) return rc;
            in = o; o = o == A ? Bf : A;
        }
        float* sv = saved ? saved + h->act_off[l] * nsv : nullptr;
        if ((rc = conv_fwd(h, c, in, B2, o, sv, nsv, h->precision == 1 && l < kConvs - 1, st))) return rc;
        in = o; o = o == A ? Bf : A;
        if (l == kTapConv[t]) {
            const long n4 = (long)(B * tap_elems(t) / 4);
            ts.count[t] = n_partials(B, t); ts.numel[t] = (float)(B * tap_elems(t));
            SMK_TAG("vgg_l1", 4.0 * 2 * n4 * 4 + (signs ? n4 * 4.0 : 0.0), 3.0 * n4 * 4, st);
            SMK_LAUNCH(vgg_l1_kernel, dim3(ts.count[t]), dim3(256), 0, st, reinterpret_cast<const float4*>(in),
                       reinterpret_cast<const float4*>(in + (size_t)B * tap_elems(t)), n4, swap ? 1 : 0,
                       signs ? reinterpret_cast<char4*>(signs + 4 * h->sign_off[t] * B) : nullptr, pp);
            SMK_CHECK_LAUNCH();
            pp += ts.count[t];
            ++t;
        }
    }
    SMK_TAG("vgg_l1_finalize", 4.0 * total_partials(B), 0.0, st);
    SMK_LAUNCH(vgg_l1_finalize_kernel, dim3(1), dim3(256), 0, st, part, ts, loss);
    SMK_CHECK_LAUNCH();
    return 0;
}

}  // namespace

extern "C" size_t smk_vgg_loss_workspace_bytes(const SmkVggLoss* h, int B) {
    if (!h || B <= 0) return 0;
    return 2 * smk::ws_round(kActMax * 2 * B * sizeof(float)) + smk::ws_round(total_partials(B) * sizeof(float)) + 256;
}

extern "C" int smk_vgg_loss_forward(const SmkVggLoss* h, const float* x, const float* y, int B, float* loss, void* ws, size_t ws_bytes,
                                    void* stream) {
    SMK_REQUIRE(h && x && y && loss, "smk_vgg_loss_forward: null argument");
    SMK_REQUIRE(B > 0, "smk_vgg_loss_forward: B must be positive (got %d)", B);
    SMK_REQUIRE(ws && ws_bytes >= smk_vgg_loss_workspace_bytes(h, B), "smk_vgg_loss_forward: workspace too small");
    return vgg_forward(h, x, y, B, 0, loss, nullptr, ws, ws_bytes, (cudaStream_t)stream);
}

extern "C" size_t smk_vgg_loss_saved_bytes(const SmkVggLoss* h, int B, int need) {
    if (!h || B <= 0 || need < 1 || need > 3) return 0;
    return (h->act_total * halves(need) + h->sign_total) * (size_t)B * sizeof(float);
}

extern "C" int smk_vgg_loss_forward_saved(const SmkVggLoss* h, const float* x, const float* y, int B, int need, float* loss,
                                          float* saved, size_t saved_bytes, void* ws, size_t ws_bytes, void* stream) {
    SMK_REQUIRE(h && x && y && loss && saved, "smk_vgg_loss_forward_saved: null argument");
    SMK_REQUIRE(B > 0, "smk_vgg_loss_forward_saved: B must be positive (got %d)", B);
    SMK_REQUIRE(need >= 1 && need <= 3, "smk_vgg_loss_forward_saved: need must be 1 (x), 2 (y) or 3 (both), got %d", need);
    SMK_REQUIRE(saved_bytes >= smk_vgg_loss_saved_bytes(h, B, need), "smk_vgg_loss_forward_saved: saved buffer too small");
    SMK_REQUIRE(ws && ws_bytes >= smk_vgg_loss_workspace_bytes(h, B), "smk_vgg_loss_forward_saved: workspace too small");
    return vgg_forward(h, x, y, B, need, loss, saved, ws, ws_bytes, (cudaStream_t)stream);
}

extern "C" int smk_vgg_loss_saved_tensor(const SmkVggLoss* h, int B, int need, int i, const char** name, size_t* offset, int* dims) {
    SMK_REQUIRE(h && name && offset && dims, "smk_vgg_loss_saved_tensor: null argument");
    SMK_REQUIRE(B >= 0 && need >= 1 && need <= 3, "smk_vgg_loss_saved_tensor: bad B (%d) or need (%d)", B, need);
    SMK_REQUIRE(i >= 0 && i < kConvs + kTaps, "smk_vgg_loss_saved_tensor: index %d out of range (%d tensors)", i, kConvs + kTaps);
    const size_t nsv = (size_t)halves(need) * B;
    if (i < kConvs) {
        *name = kActName[i]; *offset = h->act_off[i] * nsv;
        dims[0] = (int)nsv; dims[1] = dims[2] = h->conv[i].S; dims[3] = h->conv[i].cout;
    } else {
        const int t = i - kConvs;
        *name = kSignName[t]; *offset = h->act_total * nsv + h->sign_off[t] * B;
        dims[0] = B; dims[1] = dims[2] = tap_S(t); dims[3] = tap_C(t);
    }
    return 0;
}

extern "C" size_t smk_vgg_loss_backward_workspace_bytes(const SmkVggLoss* h, int B, int need) {
    if (!h || B <= 0 || need < 1 || need > 3) return 0;
    return 2 * smk::ws_round(kActMax * halves(need) * B * sizeof(float)) + 256;
}

extern "C" int smk_vgg_loss_backward(const SmkVggLoss* h, int B, int need, const float* saved, size_t saved_bytes, const float* g,
                                     float* g_x, float* g_y, void* ws, size_t ws_bytes, void* stream) {
    SMK_REQUIRE(h && saved && g, "smk_vgg_loss_backward: null argument");
    SMK_REQUIRE(B > 0, "smk_vgg_loss_backward: B must be positive (got %d)", B);
    SMK_REQUIRE(need >= 1 && need <= 3, "smk_vgg_loss_backward: need must be 1 (x), 2 (y) or 3 (both), got %d", need);
    SMK_REQUIRE((!(need & 1) || g_x) && (!(need & 2) || g_y), "smk_vgg_loss_backward: a gradient `need` asks for is null");
    SMK_REQUIRE(saved_bytes >= smk_vgg_loss_saved_bytes(h, B, need), "smk_vgg_loss_backward: saved buffer too small");
    SMK_REQUIRE(ws && ws_bytes >= smk_vgg_loss_backward_workspace_bytes(h, B, need), "smk_vgg_loss_backward: workspace too small");
    cudaStream_t st = (cudaStream_t)stream;
    const bool swap = need == 2, rnd = h->precision == 1;     // TF32 rounding of every gradient a TF32 dgrad reads
    const int Bc = halves(need) * B;
    smk::Workspace w(ws, ws_bytes);
    float* cur = w.take<float>(kActMax * Bc);
    float* oth = w.take<float>(kActMax * Bc);
    SMK_REQUIRE(oth, "smk_vgg_loss_backward: workspace carve-up failed");
    auto SV = [&](int l) { return saved + h->act_off[l] * Bc; };
    auto SIGN = [&](int t) { return reinterpret_cast<const char4*>(reinterpret_cast<const int8_t*>(saved + h->act_total * Bc) + 4 * h->sign_off[t] * B); };
    auto pool_l1 = [&](int t, const float* gp, float* out) -> int {
        const int S = tap_S(t), C = tap_C(t);
        const long total = (long)Bc * (S / 2) * (S / 2) * (C / 4);
        SMK_TAG("vgg_pool_l1_dgrad", 4.0 * Bc * ((double)S * S * C * 2 + (gp ? (S / 2.0) * (S / 2.0) * C : 0.0)) + (double)B * S * S * C, 0.0, st);
        SMK_LAUNCH(vgg_pool_l1_bwd_kernel, dim3(smk::grid_of(total)), dim3(256), 0, st, SV(kTapConv[t]), SIGN(t), gp, g,
                   (float)(B * tap_elems(t)), B, Bc, swap ? 1 : 0, S, C, rnd ? 1 : 0, out);
        SMK_CHECK_LAUNCH();
        return 0;
    };
    int rc;
    if ((rc = pool_l1(kTaps - 1, nullptr, cur))) return rc;             // relu4_3: the L1 term alone
    for (int l = kConvs - 1; l >= 0; --l) {
        const VggConv& c = h->conv[l];
        const bool first = l == 0 || h->conv[l - 1].S != c.S;         // its input is a pool output or the image: no ReLU
        if ((rc = conv_dgrad(h, c, cur, Bc, first ? nullptr : SV(l - 1), oth, rnd && l > 0, st))) return rc;
        std::swap(cur, oth);
        if (l > 0 && first) {
            if ((rc = pool_l1(kStage[l] - 1, cur, oth))) return rc;
            std::swap(cur, oth);
        }
    }
    const long total = (long)Bc * 3 * 224 * 224;
    SMK_TAG("vgg_input_dgrad", 4.0 * (double)Bc * 224 * 224 * (3 + h->conv[0].cin_p), 0.0, st);
    SMK_LAUNCH(vgg_input_bwd_kernel, dim3(smk::cdiv(total, 256)), dim3(256), 0, st, cur, B, Bc, 224 * 224, h->conv[0].cin_p, h->norm,
               swap ? g_y : g_x, g_y);
    SMK_CHECK_LAUNCH();
    return 0;
}
