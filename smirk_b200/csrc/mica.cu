// MICA (src/models/MICA/mica.py): the frozen ArcFace iResNet-100 on 112^2 crops, F.normalize and the shape regressor,
// forward only, and the trainer's MICA shape loss mse_loss(shape_params, mica_shape) with its gradient to shape_params.
//
// Network (eval-mode BatchNorm, eps 1e-5), NHWC fp32 activations:
//   prep       2 * (x - 0.5) as the reference's (x - 0.5) / 0.5, channels flipped to BGR, padded to the stem's Cin
//   stem       3x3 conv 3 -> 64 + BN + PReLU                                                                    112^2
//   4 stages   (64, 128, 256, 512) planes, (3, 13, 30, 3) IBasicBlocks, the first of each with stride 2    -> 56 .. 7
//              y = bn3(conv2_s(prelu(bn2(conv1(bn1(x)))))) + identity, identity = x or bn(conv1x1_s(x)), no ReLU
//   head       bn2, NCHW flatten, fc 25088 -> 512, BatchNorm1d: folded on the host (float64) into one GEMM whose
//              columns are permuted to the NHWC flatten order
//   regressor  F.normalize, 4 x (Linear + leaky_relu(0.2)), Linear 300 -> 300: mica_map_kernel, one CTA per image
//
// Every convolution runs through smk::conv at the handle's precision (0 = fp32 CUDA cores, 1 = TF32 wgmma, 3 = 3xTF32
// wgmma), with its BatchNorm as the epilogue's scale / bias.  bn1 of a block cannot be folded into conv1 (conv1 zero-pads
// bn1(x), not x), so the epilogue that writes a block's output y also writes bn1_next(y), the next conv1's input, as its
// second store with its own affine (smk::Conv::scale2 / bias2); the stem and every conv1 apply their PReLU there too
// (smk::Conv::prelu).  The stride-2 layers (four 3x3 and four 1x1, 3.8 % of the MACs) gather their receptive fields into a
// dense [M, 9 Cin] (or [M, Cin]) matrix that a plain GEMM then reads (smk::gather_s2): one simple kernel serves the
// fp32 and tensor-core paths alike, at the cost of one extra pass over those eight layers' inputs.
//
// Precision 1 rounds every stored activation that another tensor-core layer reads to TF32 (conv1's output, bn1(y), the
// gathered matrices, the last block's output); the residual stream y itself stays fp32.  Precision 3 rounds nothing, and
// its deep problems (every 3x3 conv, the gathered stride-2 convs, the fc) sum each 32-deep k-block apart (gemm_tc X3 = 3).
#include "nn_kernels.cuh"
#include "frozen_net.cuh"

namespace {

constexpr int kStages = 4, kBlocks = 49, kFeat = 512, kHid = 300, kOut = 300, kMapLayers = 5;
constexpr int kStageBlocks[kStages] = {3, 13, 30, 3};
constexpr int kTensors = 6 + kBlocks * 15 + kStages * 5 + 10 + 2 * kMapLayers;    // 781
constexpr size_t kActMax = (size_t)112 * 112 * 64;        // floats per image of the largest activation
constexpr size_t kDsMax = (size_t)56 * 56 * 64;           // largest downsample output
constexpr size_t kGatherMax = (size_t)56 * 56 * 9 * 64;   // largest gathered stride-2 matrix (layer1.0.conv2)

// ---- kernels ---------------------------------------------------------------------------------------------------------

// images NCHW [B,3,112,112] -> NHWC [B,112,112,Cp]: channel c takes input channel 2 - c (BGR), (v - 0.5) / 0.5 as two
// fp32 operations; channels 3..Cp-1 zero; round: TF32 for a TF32 consumer.
__global__ void __launch_bounds__(256)
mica_prep_kernel(const float* __restrict__ x, int B, int HW, int Cp, int round, float* __restrict__ out) {
    const int Q = Cp >> 2;
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long)B * HW * Q) return;
    const int q = (int)(i % Q); const long pix = i / Q;
    const int b = (int)(pix / HW), r = (int)(pix - (long)b * HW);
    float v[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const int c = q * 4 + k;
        float t = 0.f;
        if (c < 3) {
            t = __fdiv_rn(__fsub_rn(__ldg(x + ((size_t)b * 3 + (2 - c)) * HW + r), 0.5f), 0.5f);
            if (round) t = smk::round_tf32(t);
        }
        v[k] = t;
    }
    reinterpret_cast<float4*>(out)[i] = make_float4(v[0], v[1], v[2], v[3]);
}

struct MapW { const float* w[kMapLayers]; const float* b[kMapLayers]; };   // w: [K][N] (n fastest), b: [N]

// One image per CTA: z = f / max(|f|_2, 1e-12), then the regressor's five Linears (leaky_relu 0.2 after the first four).
__global__ void __launch_bounds__(256)
mica_map_kernel(const float* __restrict__ feat, MapW mw, float* __restrict__ out) {
    __shared__ float h[2][kFeat];
    const int b = blockIdx.x, tid = threadIdx.x;
    const float* f = feat + (size_t)b * kFeat;
    float ss = 0.f;
    for (int k = tid; k < kFeat; k += 256) { const float v = f[k]; ss = fmaf(v, v, ss); }
    const float den = fmaxf(sqrtf(smk::block_sum(ss)), 1e-12f);
    for (int k = tid; k < kFeat; k += 256) h[0][k] = __fdiv_rn(f[k], den);
    __syncthreads();
    int cur = 0, K = kFeat;
    for (int l = 0; l < kMapLayers; ++l) {
        const int N = l == kMapLayers - 1 ? kOut : kHid;
        for (int n = tid; n < N; n += 256) {
            float acc = 0.f;
            for (int k = 0; k < K; ++k) acc = fmaf(h[cur][k], __ldg(mw.w[l] + (size_t)k * N + n), acc);
            acc += __ldg(mw.b[l] + n);
            if (l < kMapLayers - 1) acc = acc < 0.f ? acc * 0.2f : acc;
            if (l == kMapLayers - 1) out[(size_t)b * kOut + n] = acc;
            else h[cur ^ 1][n] = acc;
        }
        __syncthreads();
        cur ^= 1; K = N;
    }
}

// loss = sum over (b, d < D) of (s[b, d] - m[b*ld + d])^2 / (B*D): one CTA, fixed order.
__global__ void __launch_bounds__(256)
mica_mse_kernel(const float* __restrict__ s, const float* __restrict__ m, int B, int D, int ld, float* __restrict__ loss) {
    float acc = 0.f;
    const long n = (long)B * D;
    for (long i = threadIdx.x; i < n; i += 256) {
        const int b = (int)(i / D), d = (int)(i - (long)b * D);
        const float e = s[i] - m[(size_t)b * ld + d];
        acc = fmaf(e, e, acc);
    }
    acc = smk::block_sum(acc);
    if (threadIdx.x == 0) *loss = __fdiv_rn(acc, (float)n);
}

// grad[b, d] = (2 / (B*D)) * (s - m) * g, as autograd's mse_loss backward orders it.
__global__ void __launch_bounds__(256)
mica_mse_bwd_kernel(const float* __restrict__ s, const float* __restrict__ m, int B, int D, int ld, float norm,
                    const float* __restrict__ g, float* __restrict__ grad) {
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long)B * D) return;
    const int b = (int)(i / D), d = (int)(i - (long)b * D);
    grad[i] = norm * (s[i] - m[(size_t)b * ld + d]) * __ldg(g);
}

// ---- host -----------------------------------------------------------------------------------------------------------
using smk::Affine;

struct MicaBlock {
    int cin, cout, H, stride;                  // H: input size; conv2 (and the downsample) output H / stride
    Affine bn1, bn2, bn3, ds_bn;
    float* prelu = nullptr;
    smk::GemmW conv1{}, conv2{}, ds{};         // conv2 of a stride-2 block and ds: plain GEMMs over the gathered matrix
};

}  // namespace

struct SmkMica {
    int precision;
    int cin_p;                                 // the stem's padded input channels
    smk::GemmW stem{};
    Affine stem_bn;
    float* stem_prelu = nullptr;
    MicaBlock blk[kBlocks];
    smk::GemmW fc{};                           // bn2, fc and features folded, K in NHWC flatten order
    float* fc_bias = nullptr;
    float* ones = nullptr;
    MapW map{};
    smk::DeviceArena arena;
};

namespace {

using smk::bn_fold;
using smk::upload_bn;

// A 3x3 conv's PyTorch weight [cout][cin][3][3] as the GEMM operand, k = tap * cin_p + c (modes 1 and the gathered matrix).
cudaError_t pack3(smk::DeviceArena& arena, const float* w, int cin, int cin_p, int cout, bool tc, bool x3, smk::GemmW* out) {
    return smk::pack_gemm(arena, cout, 9 * cin_p, tc, x3, [&](int o, int k) {
        const int tap = k / cin_p, c = k % cin_p;
        return c < cin ? w[((size_t)o * cin + c) * 9 + tap] : 0.f;
    }, out);
}

}  // namespace

extern "C" int smk_mica_create(const SmkNetDesc* desc, SmkMica** out) {
    if (int rc = smk::check_net_desc(desc, out, "smk_mica_create", kTensors, "the state_dict without num_batches_tracked")) return rc;
    const bool tc = desc->precision != 0, x3 = desc->precision == 3;
    SmkMica* h = new SmkMica();
    h->precision = desc->precision;
    h->cin_p = tc ? 32 : 4;                   // the tensor-core path reads 128-byte pixel rows
    smk::TensorCursor cur{desc->tensors, desc->n_tensors};
    auto bn4 = [&]() { return smk::next_bn(cur); };
    smk::DeviceArena& A = h->arena;
    cudaError_t e = pack3(A, cur.next(), 3, h->cin_p, 64, tc, x3, &h->stem);
    if (e == cudaSuccess) e = upload_bn(A, bn4(), 64, &h->stem_bn);
    if (e == cudaSuccess) e = A.upload(cur.next(), 64, &h->stem_prelu);
    int l = 0, cin = 64, H = 112;
    for (int s = 0; s < kStages; ++s) {
        const int planes = 64 << s;
        for (int j = 0; j < kStageBlocks[s] && e == cudaSuccess; ++j, ++l) {
            MicaBlock& k = h->blk[l];
            k.cin = cin; k.cout = planes; k.H = H; k.stride = j == 0 ? 2 : 1;
            e = upload_bn(A, bn4(), cin, &k.bn1);
            if (e == cudaSuccess) e = pack3(A, cur.next(), cin, cin, planes, tc, x3, &k.conv1);
            if (e == cudaSuccess) e = upload_bn(A, bn4(), planes, &k.bn2);
            if (e == cudaSuccess) e = A.upload(cur.next(), (size_t)planes, &k.prelu);
            if (e == cudaSuccess) e = pack3(A, cur.next(), planes, planes, planes, tc, x3, &k.conv2);
            if (e == cudaSuccess) e = upload_bn(A, bn4(), planes, &k.bn3);
            if (j == 0) {
                if (e == cudaSuccess) e = smk::pack_gemm(A, planes, cin, tc, x3, cur.next(), &k.ds);
                if (e == cudaSuccess) e = upload_bn(A, bn4(), planes, &k.ds_bn);
                H /= 2;
            }
            cin = planes;
        }
    }
    if (e == cudaSuccess) {                   // head: features(fc(flatten_nchw(bn2(x)))), folded in float64
        std::vector<double> s2, t2, sf, tf;
        bn_fold(bn4(), kFeat, s2, t2);
        const float* W = cur.next();
        const float* b = cur.next();
        bn_fold(bn4(), kFeat, sf, tf);
        constexpr int HW = 49, K = kFeat * HW;
        std::vector<float> bias(kFeat);
        for (int n = 0; n < kFeat; ++n) {
            double acc = b[n];
            for (int k = 0; k < K; ++k) acc += (double)W[(size_t)n * K + k] * t2[k / HW];
            bias[n] = (float)(sf[n] * acc + tf[n]);
        }
        e = smk::pack_gemm(A, kFeat, K, tc, x3, [&](int n, int k) {     // k = pixel * 512 + c  <-  c * 49 + pixel
            const int c = k % kFeat, px = k / kFeat;
            return (float)(sf[n] * (double)W[(size_t)n * K + c * HW + px] * s2[c]);
        }, &h->fc);
        if (e == cudaSuccess) e = A.upload(bias, &h->fc_bias);
    }
    for (int i = 0, K = kFeat; i < kMapLayers && e == cudaSuccess; ++i) {   // Linear [N][K] -> [K][N]
        const int N = i == kMapLayers - 1 ? kOut : kHid;
        const float* w = cur.next();
        std::vector<float> wt((size_t)K * N);
        for (int n = 0; n < N; ++n)
            for (int k = 0; k < K; ++k) wt[(size_t)k * N + n] = w[(size_t)n * K + k];
        float *dw = nullptr, *db = nullptr;
        e = A.upload(wt, &dw);
        if (e == cudaSuccess) e = A.upload(cur.next(), (size_t)N, &db);
        h->map.w[i] = dw; h->map.b[i] = db;
        K = N;
    }
    const std::vector<float> one(kFeat, 1.f);
    if (e == cudaSuccess) e = A.upload(one, &h->ones);
    return smk::finish_create(e, "smk_mica_create", h, out);
}

extern "C" void smk_mica_destroy(SmkMica* h) { delete h; }

extern "C" size_t smk_mica_workspace_bytes(const SmkMica* h, int B) {
    if (!h || B <= 0) return 0;
    return 4 * smk::ws_round(kActMax * B * sizeof(float)) + smk::ws_round(kDsMax * B * sizeof(float)) +
           smk::ws_round(kGatherMax * B * sizeof(float)) + smk::ws_round((size_t)kFeat * B * sizeof(float)) + 256;
}

namespace {

using smk::tag_of;

int gather_s2(const float* in, int B, int H, int C, int taps, bool round, float* out, cudaStream_t st) {
    return smk::gather_s2(in, B, H, C, taps, round, out, taps == 9 ? "mica_gather3x3_s2" : "mica_gather1x1_s2", st);
}

}  // namespace

extern "C" int smk_mica_forward(const SmkMica* h, const float* images, int B, float* shape_params, float* features,
                                void* ws, size_t ws_bytes, void* stream) {
    SMK_REQUIRE(h && images && shape_params, "smk_mica_forward: null argument");
    SMK_REQUIRE(B > 0, "smk_mica_forward: B must be positive (got %d)", B);
    SMK_REQUIRE(ws && ws_bytes >= smk_mica_workspace_bytes(h, B), "smk_mica_forward: workspace too small");
    cudaStream_t st = (cudaStream_t)stream;
    const int P = h->precision;
    const bool rnd = P == 1;
    smk::Workspace w(ws, ws_bytes);
    float* X[2] = {w.take<float>(kActMax * B), w.take<float>(kActMax * B)};   // the residual stream y, ping-pong
    float* T = w.take<float>(kActMax * B);                                     // bn1(y): the next conv1's input
    float* U = w.take<float>(kActMax * B);                                     // prelu(bn2(conv1(.))), the prep output first
    float* D = w.take<float>(kDsMax * B);                                      // downsample output
    float* G = w.take<float>(kGatherMax * B);                                  // gathered stride-2 matrix
    float* F = w.take<float>((size_t)kFeat * B);
    SMK_REQUIRE(F, "smk_mica_forward: workspace carve-up failed");
    if (features) F = features;
    {
        const long total = (long)B * 112 * 112 * (h->cin_p / 4);
        SMK_TAG("mica_prep", 4.0 * B * 112.0 * 112.0 * (3 + h->cin_p), 0.0, st);
        SMK_LAUNCH(mica_prep_kernel, dim3(smk::cdiv(total, 256)), dim3(256), 0, st, images, B, 112 * 112, h->cin_p, rnd ? 1 : 0, U);
        SMK_CHECK_LAUNCH();
    }
    int rc, x = 0;
    {   // stem: y = prelu(bn(conv(img))), and bn1 of the first block as the second store
        smk::Conv p{};
        p.in = U; p.ld_in = h->cin_p; p.B = B; p.H = 112; p.W = 112; p.Cin = h->cin_p;
        p.N = 64; p.K = 9 * h->cin_p; p.mode = 1; p.wgt = h->stem; p.scale = h->stem_bn.scale; p.bias = h->stem_bn.bias;
        p.prelu = h->stem_prelu; p.out = X[x]; p.ld_out = 64;
        p.out2 = T; p.ld_out2 = 64; p.scale2 = h->blk[0].bn1.scale; p.bias2 = h->blk[0].bn1.bias; p.round_out2 = rnd;
        p.tag = tag_of(P, "mica_stem_f32", "mica_stem_tc", "mica_stem_tc3x");
        if ((rc = smk::conv(p, st))) return rc;
    }
    for (int l = 0; l < kBlocks; ++l) {
        const MicaBlock& k = h->blk[l];
        const int Ho = k.H / k.stride;
        {   // conv1 (stride 1) + bn2 + PReLU
            smk::Conv p{};
            p.in = T; p.ld_in = k.cin; p.B = B; p.H = k.H; p.W = k.H; p.Cin = k.cin;
            p.N = k.cout; p.K = 9 * k.cin; p.mode = 1; p.wgt = k.conv1; p.scale = k.bn2.scale; p.bias = k.bn2.bias;
            p.prelu = k.prelu; p.out = U; p.ld_out = k.cout; p.round_out = rnd;
            p.tag = tag_of(P, "mica_conv1_f32", "mica_conv1_tc", "mica_conv1_tc3x");
            if ((rc = smk::conv(p, st))) return rc;
        }
        const float* res = X[x];
        if (k.stride == 2) {      // identity = bn(conv1x1_s2(x)), from the raw x
            if ((rc = gather_s2(X[x], B, k.H, k.cin, 1, rnd, G, st))) return rc;
            smk::Conv p{};
            p.in = G; p.ld_in = k.cin; p.B = B; p.H = Ho; p.W = Ho; p.Cin = k.cin;
            p.N = k.cout; p.K = k.cin; p.mode = 0; p.wgt = k.ds; p.scale = k.ds_bn.scale; p.bias = k.ds_bn.bias;
            p.out = D; p.ld_out = k.cout;
            p.tag = tag_of(P, "mica_downsample_f32", "mica_downsample_tc", "mica_downsample_tc3x");
            if ((rc = smk::conv(p, st))) return rc;
            if ((rc = gather_s2(U, B, k.H, k.cout, 9, rnd, G, st))) return rc;
            res = D;
        }
        {   // conv2 + bn3 + identity -> y; bn1 of the next block -> its conv1's input
            const bool last = l == kBlocks - 1;
            smk::Conv p{};
            p.B = B; p.H = Ho; p.W = Ho; p.N = k.cout; p.K = 9 * k.cout; p.wgt = k.conv2;
            if (k.stride == 2) { p.in = G; p.ld_in = 9 * k.cout; p.Cin = 9 * k.cout; p.mode = 0; }
            else { p.in = U; p.ld_in = k.cout; p.Cin = k.cout; p.mode = 1; }
            p.scale = k.bn3.scale; p.bias = k.bn3.bias; p.res = res; p.ld_res = k.cout;
            p.out = X[x ^ 1]; p.ld_out = k.cout; p.round_out = rnd && last;      // the last y feeds only the fc
            if (!last) {
                p.out2 = T; p.ld_out2 = k.cout; p.scale2 = h->blk[l + 1].bn1.scale; p.bias2 = h->blk[l + 1].bn1.bias; p.round_out2 = rnd;
            }
            p.tag = k.stride == 2 ? tag_of(P, "mica_conv2_s2_f32", "mica_conv2_s2_tc", "mica_conv2_s2_tc3x")
                                  : tag_of(P, "mica_conv2_f32", "mica_conv2_tc", "mica_conv2_tc3x");
            if ((rc = smk::conv(p, st))) return rc;
            x ^= 1;
        }
    }
    {   // head: one K = 25088 GEMM over the NHWC-flattened y
        smk::Conv p{};
        p.in = X[x]; p.ld_in = kFeat * 49; p.B = 1; p.H = 1; p.W = B; p.Cin = kFeat * 49;
        p.N = kFeat; p.K = kFeat * 49; p.mode = 0; p.wgt = h->fc; p.scale = h->ones; p.bias = h->fc_bias;
        p.out = F; p.ld_out = kFeat;
        p.tag = tag_of(P, "mica_fc_f32", "mica_fc_tc", "mica_fc_tc3x");
        if ((rc = smk::conv(p, st))) return rc;
    }
    SMK_TAG("mica_map", 4.0 * B * (kFeat + kOut) + 4.0 * (kFeat * kHid + 3 * kHid * kHid + kHid * kOut),
            2.0 * B * (kFeat * kHid + 3 * kHid * kHid + kHid * kOut), st);
    SMK_LAUNCH(mica_map_kernel, dim3(B), dim3(256), 0, st, F, h->map, shape_params);
    SMK_CHECK_LAUNCH();
    return 0;
}

extern "C" int smk_mica_shape_loss_forward(const float* shape_params, const float* mica_shape, int B, int D, int ld, float* loss,
                                           void* stream) {
    SMK_REQUIRE(shape_params && mica_shape && loss, "smk_mica_shape_loss_forward: null argument");
    SMK_REQUIRE(B > 0 && D > 0 && ld >= D, "smk_mica_shape_loss_forward: need B > 0, D > 0 and ld >= D (got %d, %d, %d)", B, D, ld);
    cudaStream_t st = (cudaStream_t)stream;
    SMK_TAG("mica_mse", 4.0 * (2.0 * B * D + 1), 3.0 * B * D, st);
    SMK_LAUNCH(mica_mse_kernel, dim3(1), dim3(256), 0, st, shape_params, mica_shape, B, D, ld, loss);
    SMK_CHECK_LAUNCH();
    return 0;
}

extern "C" int smk_mica_shape_loss_backward(const float* shape_params, const float* mica_shape, int B, int D, int ld, const float* g,
                                            float* grad, void* stream) {
    SMK_REQUIRE(shape_params && mica_shape && g && grad, "smk_mica_shape_loss_backward: null argument");
    SMK_REQUIRE(B > 0 && D > 0 && ld >= D, "smk_mica_shape_loss_backward: need B > 0, D > 0 and ld >= D (got %d, %d, %d)", B, D, ld);
    cudaStream_t st = (cudaStream_t)stream;
    const long n = (long)B * D;
    SMK_TAG("mica_mse_dgrad", 4.0 * (3.0 * n + 1), 3.0 * n, st);
    SMK_LAUNCH(mica_mse_bwd_kernel, dim3(smk::cdiv(n, 256)), dim3(256), 0, st, shape_params, mica_shape, B, D, ld,
               (float)(2.0 / (double)n), g, grad);
    SMK_CHECK_LAUNCH();
    return 0;
}

// ---- kernel-test entry points (tests/test_gpu_mica_layers.py) ---------------------------------------------------------
// Exported but not part of include/smirk_b200.h; the test declares their argument types itself.
//
// One smk::conv problem with MICA's epilogue options: w_kn fp32 [K][N] (conv_gemm), or wt_hi [N][K] TF32 (tc_conv) with
// optional tails wt_lo (3xTF32); res / prelu / out2 / scale2 null: not used.
extern "C" int smk_debug_mica_conv(const float* in, int ld_in, int B, int H, int W, int Cin, const float* w_kn, const float* wt_hi,
                                   const float* wt_lo, const float* scale, const float* bias, int N, int K, int mode, const float* res,
                                   int ld_res, const float* prelu, float* out, int ld_out, int round_out, float* out2, int ld_out2,
                                   const float* scale2, const float* bias2, int round_out2, void* stream) {
    SMK_REQUIRE(!w_kn != !wt_hi, "smk_debug_mica_conv: exactly one of w_kn and wt_hi");
    smk::Conv p{};
    p.in = in; p.ld_in = ld_in; p.B = B; p.H = H; p.W = W; p.Cin = Cin; p.wgt = smk::GemmW{w_kn, wt_hi, wt_lo};
    p.scale = scale; p.bias = bias; p.N = N; p.K = K; p.mode = mode; p.res = res; p.ld_res = ld_res; p.prelu = prelu;
    p.out = out; p.ld_out = ld_out; p.round_out = round_out; p.out2 = out2; p.ld_out2 = ld_out2;
    p.scale2 = scale2; p.bias2 = bias2; p.round_out2 = round_out2;
    return smk::conv(p, (cudaStream_t)stream);
}
// smk::gather_s2: in [B,H,H,C] -> out [B*(H/2)^2, taps*C], taps 9 (3x3, zero padding 1) or 1.
extern "C" int smk_debug_mica_gather_s2(const float* in, int B, int H, int C, int taps, int round, float* out, void* stream) {
    SMK_REQUIRE(in && out && B > 0 && H % 2 == 0 && C % 4 == 0 && (taps == 1 || taps == 9), "smk_debug_mica_gather_s2: bad arguments");
    return gather_s2(in, B, H, C, taps, round != 0, out, (cudaStream_t)stream);
}
